"""GPU: the MVCC stage (fabgpu_validate_mvcc) over the world-state version table (fabgpu_state_versions / _update / _info) -- every case
through validate_block and validate_envelopes in both validator modes, a sequence of generated blocks over hot keys submitted three slots
deep (with the device's own flags and with the oracle's settled flags), and the refusals, growth and broken table through the library."""
import os

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from util import pkg
import mvcc_oracle as mo
import mvcccases
import mvccutil

pytestmark = pytest.mark.gpu

POLICIES = {mvcccases.CC: 0, mvcccases.OTHER: 0}
# faults that leave the read/write set reachable: the validator flags them (or leaves them at 254), the MVCC stage still enumerates them
SIG_FAULTS = ("bad_creator_sig", "bad_endorsement_sig", "dup_endorser", "unknown_endorser", "unknown_creator", "invalid_creator_cert",
              "high_s_endorsement", "two_bad_endorsements", "dup_txid", "bad_proposal_hash", "many_endorsements")


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
    c.namespace_versions({mvcccases.CC: "1.0"})
    c.channel_capability(cap)


def _block(net, txs, seed, faults=None):
    """a signed block whose transaction t carries txs[t]'s read/write set; None: a config-update transaction (no results reached)"""
    faults = dict(faults or {})
    faults.update({t: "config_update_type" for t, tx in enumerate(txs) if tx is None})
    hook = lambda t, part, b: mo.encode(txs[t]) if part == "TxReadWriteSet" and txs[t] is not None else b
    return blockgen.build_block(net, len(txs), 3, faults, seed=seed, mutate=hook)


def _entries(state):
    return [((k[0], k[1], k[2]), v) for k, v in mvccutil.state_entries(state)]


@pytest.mark.parametrize("entry", ["block", "envelopes"])
@pytest.mark.parametrize("mode", ["v20", "v13"])
def test_cases_on_the_device(ctx, net, entry, mode):
    """Every case: with the case's validator flags the device gives the codes written out; with the device's own flags it gives what the
    oracle gives for them; the table's counts follow the oracle's state."""
    B = pkg().binding
    _configure(ctx, net, B.CAP_V1_3 if mode == "v13" else B.CAP_V2_0)
    try:
        for name, state0, blocks in mvcccases.cases():
            for own in (False, True):
                state = dict(state0)
                ctx.state_versions(_entries(state), 1)
                for k, (txs, tv, codes) in enumerate(blocks):
                    blk, info = _block(net, txs, seed=31 + k)
                    dev_tv = ctx.validate_block(blk) if entry == "block" else ctx.validate_envelopes(info["env_blob"], info["env_off"])
                    use = dev_tv.tolist() if own else tv
                    got = ctx.validate_mvcc(0, 1 + k, use).tolist()
                    exp, state, is_open = mo.validate(state, 1 + k, txs, use)
                    assert got == exp, (name, own, k)
                    if not own:
                        assert got == codes, (name, k)
                    held, _, height, unknown = ctx.state_versions_info()
                    assert (held, unknown) == mo.info(state) and height == (1 + k if is_open else 2 + k), (name, own, k)
                    if is_open:
                        ctx.state_versions_update([], 2 + k)
                if name == "unknown_keys_cleared_by_update":
                    ctx.state_versions_update([((mvcccases.CC, "", b"u"), (2, 0))], 3)
                    assert ctx.state_versions_info()[3] == 0
                    blk, _ = _block(net, [mvcccases.r(("u", (2, 0)))], seed=77)
                    ctx.validate_block(blk)
                    assert ctx.validate_mvcc(0, 3, [0]).tolist() == [0]
    finally:
        _configure(ctx, net, B.CAP_V2_0)
        ctx.state_versions([], 0)


def _sequence(net, n_blocks, seed):
    rng = np.random.default_rng(seed)
    pool = ["hot%d" % i for i in range(10)]
    out = []
    for b in range(n_blocks):
        n = int(rng.integers(8, 24))
        txs = [mvccutil.random_tx(rng, pool, unreached=0.005) for _ in range(n)]
        faults = {t: SIG_FAULTS[int(rng.integers(len(SIG_FAULTS)))] for t in range(n) if txs[t] is not None and rng.random() < 0.1}
        blk, _ = _block(net, txs, seed=500 + b, faults=faults)
        out.append((txs, blk))
    return out


@pytest.mark.parametrize("settled", [False, True], ids=["device_flags", "settled_flags"])
def test_three_slots_deep_over_hot_keys(ctx, net, settled):
    """About 30 blocks submitted three slots deep; block k's MVCC stage runs after its wait while k+1 and k+2 are in flight.  Each block's
    flags equal the oracle's for the validator flags given (the device's own, or with the 254s settled by the validator oracle), and the
    table's counts follow the oracle's state; open blocks are closed, and unknown keys re-read every ten blocks, as a peer would."""
    seq = _sequence(net, 30, seed=11 if settled else 12)
    ids = _ids(net)
    pool_state = {(mvcccases.CC, "", ("hot%d" % i).encode()): (0, i % 3) for i in range(6)}
    state = dict(pool_state)
    ctx.state_versions(_entries(state), 1, capacity=64)
    S = pkg().binding.SLOTS
    try:
        for k in range(min(S, len(seq))):
            ctx.validate_block_async(k % S, seq[k][1])
        moved = 0
        for k, (txs, blk) in enumerate(seq):
            tv = ctx.validate_wait(k % S, len(txs) + 16)
            if settled:
                ref = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=[i[0] for i in ids])
                tv = np.where(tv == 254, ref, tv).astype(np.uint8)
            got = ctx.validate_mvcc(k % S, 1 + k, tv).tolist()
            exp, state, is_open = mo.validate(state, 1 + k, txs, tv.tolist())
            assert got == exp, k
            moved += sum(1 for x, y in zip(exp, tv.tolist()) if x != y)
            if is_open:
                ctx.state_versions_update([], 2 + k)
            if k % 10 == 9:
                fix = [(key, (1 + k, 0)) for key, v in state.items() if v == mo.UNKNOWN]
                ctx.state_versions_update(fix, 2 + k)
                state.update(dict(fix))
            held, _, height, unknown = ctx.state_versions_info()
            assert (held, unknown) == mo.info(state) and height == 2 + k, k
            if k + S < len(seq):
                ctx.validate_block_async(k % S, seq[k + S][1])
        assert moved >= 30
    finally:
        ctx.state_versions([], 0)


def test_refusals_growth_and_the_broken_table(ctx, net):
    B = pkg().binding
    blk, _ = _block(net, [mvcccases.r(("a", (1, 0))), mvcccases.w("a")], seed=3)
    tv = ctx.validate_block(blk).tolist()
    with pytest.raises(B.FabGpuError, match="no state version table"):
        ctx.validate_mvcc(0, 5, tv)
    key = (mvcccases.CC, "", b"a")
    ctx.state_versions([(key, (1, 0))], 5)
    _configure(ctx, net, B.CAP_V2_0)                                     # ledger state: msp_configure keeps the table
    assert ctx.state_versions_info() == (1, 1024, 5, 0)
    with pytest.raises(B.FabGpuError, match="height"):
        ctx.validate_mvcc(0, 4, tv)
    with pytest.raises(B.FabGpuError, match="transaction count"):
        ctx.validate_mvcc(0, 5, tv + [0])
    with pytest.raises(B.FabGpuError, match="no finished block"):
        ctx.validate_mvcc(2, 5, tv)
    with pytest.raises(B.FabGpuError, match="twice"):
        ctx.state_versions_update([(key, (1, 1)), (key, (2, 2))], 5)
    with pytest.raises(B.FabGpuError, match="below"):
        ctx.state_versions_update([], 4)
    assert ctx.state_versions_info() == (1, 1024, 5, 0)
    assert ctx.validate_mvcc(0, 5, tv).tolist() == [0, 0]
    with pytest.raises(B.FabGpuError, match="no finished block"):        # the slot's block was consumed
        ctx.validate_mvcc(0, 6, tv)
    assert ctx.state_versions_info() == (1, 1024, 6, 0)
    # an open block: refused until closed
    blk2, _ = _block(net, [None, mvcccases.r(("a", (5, 1)))], seed=4)
    tv2 = [0, 0]
    ctx.validate_block(blk2)
    assert ctx.validate_mvcc(0, 6, tv2).tolist() == [254, 254]
    ctx.validate_block(blk2)
    with pytest.raises(B.FabGpuError, match="open"):
        ctx.validate_mvcc(0, 6, tv2)
    ctx.state_versions_update([(key, B.STATE_REMOVE)], 7)
    assert ctx.state_versions_info() == (0, 1024, 7, 0)
    # growth past 1/2 load: 600 new keys of one block on a table of 1024 slots holding 0
    txs = [mvcccases.w(*["g%d_%d" % (t, j) for j in range(20)]) for t in range(30)]
    blk3, _ = _block(net, txs, seed=5)
    tv3 = ctx.validate_block(blk3).tolist()
    assert tv3 == [0] * 30
    assert ctx.validate_mvcc(0, 7, tv3).tolist() == [0] * 30
    assert ctx.state_versions_info() == (600, 2048, 8, 0)
    # the byte bound: a failed growth breaks the table until a replace
    os.environ["FABGPU_STATE_MAX_BYTES"] = str(56 * 2048)
    try:
        with pytest.raises(B.FabGpuError, match="FABGPU_STATE_MAX_BYTES"):
            ctx.state_versions_update([((mvcccases.CC, "", b"x%d" % i), (1, 1)) for i in range(600)], 8)
    finally:
        del os.environ["FABGPU_STATE_MAX_BYTES"]
    assert ctx.state_versions_info()[0] == 0
    with pytest.raises(B.FabGpuError, match="broken"):
        ctx.state_versions_update([], 8)
    blk4, _ = _block(net, [mvcccases.r(("q", None)), mvcccases.r(("q", None))], seed=6, faults={1: "bad_creator_sig"})
    tv4 = ctx.validate_block(blk4).tolist()
    assert tv4 == [0, 4]
    assert ctx.validate_mvcc(0, 8, tv4).tolist() == [254, 4]
    ctx.state_versions([], 8, capacity=10)
    ctx.validate_block(blk4)
    assert ctx.validate_mvcc(0, 8, tv4).tolist() == [0, 4]
    ctx.state_versions([], 0)
    assert ctx.state_versions_info() == (0, 0, 0, 0)
