"""GPU: range queries in the MVCC stage (fabgpu_validate_mvcc) over an ordered index of the public keys (fabgpu_state_versions_indexed,
fabgpu_state_index_info) -- every range case through validate_block and validate_envelopes in both validator modes, generated block
sequences submitted three slots deep, and the index's growth, fold, byte bound, refusals, replace and removal through the library."""
import os

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from util import pkg
import mvcc_oracle as mo
import range_oracle as ro
import rangecases
import rangeutil

pytestmark = pytest.mark.gpu

CC = rangecases.CC
POLICIES = {CC: 0, "othercc": 0}
SIG_FAULTS = ("bad_creator_sig", "bad_endorsement_sig", "dup_endorser", "unknown_endorser", "dup_txid", "bad_proposal_hash")


@pytest.fixture(scope="module")
def net():
    return blockgen.Network()


@pytest.fixture(scope="module")
def ctx(net):
    c = pkg().binding.Context(max_batch=8192)
    _configure(c, net, pkg().binding.CAP_V2_0)
    yield c
    c.close()


def _ids(net):
    return [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]


def _configure(c, net, cap):
    c.msp_configure(_ids(net), net.policy_n_of(3), net.principals, net.channel, policies=POLICIES)
    c.namespace_versions({CC: "1.0"})
    c.channel_capability(cap)


def _block(net, txs, seed, faults=None):
    """a signed block whose transaction t carries txs[t]'s read/write set; None: a config-update transaction (no results reached)"""
    faults = dict(faults or {})
    faults.update({t: "config_update_type" for t, tx in enumerate(txs) if tx is None})
    hook = lambda t, part, b: ro.encode(txs[t]) if part == "TxReadWriteSet" and txs[t] is not None else b
    return blockgen.build_block(net, len(txs), 3, faults, seed=seed, mutate=hook)


def _entries(state):
    return [(k, v) for k, v in sorted(state.items()) if v != mo.UNKNOWN]


def _public(state):
    return sum(1 for k in state if k[1] == "")


@pytest.mark.parametrize("entry", ["block", "envelopes"])
@pytest.mark.parametrize("mode", ["v20", "v13"])
def test_cases_on_the_device(ctx, net, entry, mode):
    """Every case: with the case's validator flags the device gives the codes written out; with the device's own flags it gives what the
    oracle gives for them; the table's and the index's counts follow the oracle's state."""
    B = pkg().binding
    _configure(ctx, net, B.CAP_V1_3 if mode == "v13" else B.CAP_V2_0)
    try:
        for name, state0, steps in rangecases.cases():
            for own in (False, True):
                ctx.state_versions_indexed(_entries(state0), 1)
                state, height = dict(state0), 1
                for step in steps:
                    if step[0] == "update":
                        ctx.state_versions_update(step[1], height)
                        for k, v in step[1]:
                            if v == mo.REMOVE:
                                state.pop(k, None)
                            else:
                                state[k] = v
                        continue
                    txs, tv, codes = step
                    blk, info = _block(net, txs, seed=40 + height)
                    dev_tv = ctx.validate_block(blk) if entry == "block" else ctx.validate_envelopes(info["env_blob"], info["env_off"])
                    use = dev_tv.tolist() if own else tv
                    got = ctx.validate_mvcc(0, height, use).tolist()
                    exp, state, is_open = ro.validate(state, height, txs, use)
                    assert got == exp, (name, own, height)
                    if not own:
                        assert got == codes, (name, height)
                    if is_open:
                        ctx.state_versions_update([], height + 1)
                    height += 1
                    held, _, _, unknown = ctx.state_versions_info()
                    assert (held, unknown) == mo.info(state), (name, own, height)
                live, entries, nbytes = ctx.state_index_info()
                assert live == _public(state) and entries >= live and nbytes > 0, (name, own)
    finally:
        _configure(ctx, net, B.CAP_V2_0)
        ctx.state_versions([], 0)


@pytest.mark.parametrize("settled", [False, True], ids=["device_flags", "settled_flags"])
def test_three_slots_deep_over_hot_ranges(ctx, net, settled):
    """About 30 generated blocks with range queries over hot keys, submitted three slots deep: each block's flags equal the oracle's for
    the validator flags given (the device's own, or with the 254s settled by the validator oracle); open blocks are closed and unknown
    keys re-read every five blocks, as a peer would."""
    rng = np.random.default_rng(23 if settled else 24)
    pool = ["hot%d" % i for i in range(10)]
    state = {(CC, "", ("hot%d" % i).encode()): (0, i % 3) for i in range(6)}
    ctx.state_versions_indexed(_entries(state), 1, capacity=64)
    ids = _ids(net)
    S = pkg().binding.SLOTS
    n_blocks = 30
    seq = {}

    def make(b):
        n = int(rng.integers(8, 24))
        txs = [rangeutil.random_range_tx(rng, pool, state) for _ in range(n)]
        faults = {t: SIG_FAULTS[int(rng.integers(len(SIG_FAULTS)))] for t in range(n) if txs[t] is not None and rng.random() < 0.1}
        blk, _ = _block(net, txs, seed=700 + b, faults=faults)
        seq[b] = (txs, blk)
        ctx.validate_block_async(b % S, blk)
    try:
        for b in range(min(S, n_blocks)):
            make(b)
        decided = {0: 0, 11: 0}
        for b in range(n_blocks):
            txs, blk = seq.pop(b)
            tv = ctx.validate_wait(b % S, len(txs) + 16)
            if settled:
                ref = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=[i[0] for i in ids])
                tv = np.where(tv == 254, ref, tv).astype(np.uint8)
            got = ctx.validate_mvcc(b % S, 1 + b, tv).tolist()
            exp, state, is_open = ro.validate(state, 1 + b, txs, tv.tolist())
            assert got == exp, b
            for t, x in zip(txs, exp):
                if t is not None and t[0].get("ranges") and x in decided:
                    decided[x] += 1
            if is_open:
                ctx.state_versions_update([], 2 + b)
            if b % 5 == 4:
                fix = [(key, (1 + b, 0)) for key, v in state.items() if v == mo.UNKNOWN]
                ctx.state_versions_update(fix, 2 + b)
                state.update(dict(fix))
            held, _, height, unknown = ctx.state_versions_info()
            assert (held, unknown) == mo.info(state) and height == 2 + b, b
            assert ctx.state_index_info()[0] == _public(state), b
            if b + S < n_blocks:
                make(b + S)
        assert decided[0] >= 3 and decided[11] >= 50, decided        # hot keys written ahead of their ranges: mostly conflicts
    finally:
        ctx.state_versions([], 0)


def test_growth_fold_bound_refusals_replace_and_removal(ctx, net):
    B = pkg().binding
    key = lambda s: (CC, "", s if isinstance(s, bytes) else s.encode())
    # refusals keep the table and the index
    ctx.state_versions_indexed([(key("s%05d" % i), (0, 1)) for i in range(100)] + [((CC, "c", b"p"), (0, 1))], 1)
    assert ctx.state_index_info()[:2] == (100, 100)
    with pytest.raises(B.FabGpuError, match="twice"):
        ctx.state_versions_update([(key("x"), (1, 1)), (key("x"), (2, 2))], 1)
    with pytest.raises(B.FabGpuError, match="below"):
        ctx.state_versions_update([(key("x"), (1, 1))], 0)
    assert ctx.state_index_info()[:2] == (100, 100)
    # growth of the delta past its first size, and a fold into the base: 12 blocks of 500 new keys
    for b in range(12):
        txs = [rangecases.w(*["n%02d_%03d_%d" % (b, t, j) for j in range(5)]) for t in range(100)]
        blk, _ = _block(net, txs, seed=900 + b)
        tv = ctx.validate_block(blk).tolist()
        assert tv == [0] * 100
        assert ctx.validate_mvcc(0, 1 + b, tv).tolist() == [0] * 100
    live, entries, nbytes = ctx.state_index_info()
    assert (live, entries) == (6100, 6100) and nbytes >= 6100 * 48
    # removed keys stay as dead entries and are skipped
    ctx.state_versions_update([(key("s%05d" % i), B.STATE_REMOVE) for i in range(50)], 13)
    assert ctx.state_index_info()[:2] == (6050, 6100)
    reads = [("n11_099_%d" % j, (12, 99)) for j in range(5)] + [("s%05d" % i, (0, 1)) for i in range(50, 100)]
    blk, _ = _block(net, [rangecases.q("n11_099", "", reads), rangecases.q("s00000", "s00051", [("s00050", (0, 1))])], seed=950)
    tv = ctx.validate_block(blk).tolist()
    assert ctx.validate_mvcc(0, 13, tv).tolist() == [0, 0]
    # a plain replace drops the index: ranges are 254 again
    ctx.state_versions([(key("a"), (1, 0))], 1)
    assert ctx.state_index_info() == (0, 0, 0)
    blk, _ = _block(net, [rangecases.q("a", "b", [("a", (1, 0))])], seed=951)
    tv = ctx.validate_block(blk).tolist()
    assert ctx.validate_mvcc(0, 1, tv).tolist() == [254]
    ctx.state_versions_indexed([(key("a"), (1, 0))], 1)
    ctx.validate_block(blk)
    assert ctx.validate_mvcc(0, 1, tv).tolist() == [0]
    # the byte bound: an index that would pass it breaks the table until a replace
    os.environ["FABGPU_STATE_MAX_BYTES"] = str(56 * 1024 + 48 * 1024)
    try:
        with pytest.raises(B.FabGpuError, match="FABGPU_STATE_MAX_BYTES"):
            ctx.state_versions_update([(key("y%04d" % i), (1, 1)) for i in range(300)], 2)
    finally:
        del os.environ["FABGPU_STATE_MAX_BYTES"]
    assert ctx.state_versions_info()[0] == 0 and ctx.state_index_info() == (0, 0, 0)
    with pytest.raises(B.FabGpuError, match="broken"):
        ctx.state_versions_update([], 2)
    ctx.validate_block(blk)
    assert ctx.validate_mvcc(0, 2, tv).tolist() == [254]
    ctx.state_versions_indexed([(key("a"), (1, 0))], 2)
    ctx.validate_block(blk)
    assert ctx.validate_mvcc(0, 2, tv).tolist() == [0]
    # removal
    ctx.state_versions([], 0)
    assert ctx.state_versions_info() == (0, 0, 0, 0) and ctx.state_index_info() == (0, 0, 0)
