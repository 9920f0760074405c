"""GPU: the committed tx-id set (fabgpu_committed_txids / _add / _info) in the device block validator -- the cases through every entry
point in both validator modes, with and without collection and key tables; three blocks in flight with each block's ids added right after
its submit, while the table grows; the broken state after a failed add; and removal."""
import os

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from util import pkg
import blockutil
import collcases
import klcases
import txid_oracle
import txidcases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    yield c
    c.close()


def _three_ways(ctx, blk, info):
    a = ctx.validate_block(blk).tolist()
    b = ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist()
    ctx.validate_block_async(1, blk)
    ctx.validate_envelopes_async(2, info["env_blob"], info["env_off"])
    c = ctx.validate_wait(1, len(a) + 16).tolist()
    d = ctx.validate_wait(2, len(a) + 16).tolist()
    assert a == b == c == d
    return a


@pytest.mark.parametrize("colls", [False, True], ids=["no_collections", "collections"])
@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
def test_txid_cases_on_the_device(ctx, use_bits, colls):
    """Every case: device == oracle == the codes written out, on every entry point."""
    B = pkg().binding
    names, bits = collcases.principals(use_bits)
    table_c = collcases.collection_table() if colls else None
    for case in txidcases.cases():
        net, blk, info, codes, calls, table = txidcases.materialize(case)
        ctx.msp_configure(net.identities(), collcases.forest()[0], names, net.channel, policies=txidcases.policies())
        if bits is not None:
            ctx.msp_principal_bits(bits)
        ctx.collection_policies(table_c)
        kt = klcases.key_table((case[0], False, {}, case[3])) if case[2] else None
        if kt:
            ctx.key_policies(*kt)
        ctx.namespace_versions(txidcases.versions())
        ctx.channel_capability(B.CAP_V1_3 if case[1] == txidcases.MODE_V13 else B.CAP_V2_0)
        for replace, ids, kinds in calls:
            (ctx.committed_txids if replace else ctx.committed_txids_add)(ids, kinds)
        exp = txidcases.oracle_flags(case, blk, net, names, bits, table, collections=table_c).tolist()
        assert exp == codes, case[0]
        assert _three_ways(ctx, blk, info) == codes, case[0]
        ctx.committed_txids([])
        base = txidcases.oracle_flags(case, blk, net, names, bits, None, collections=table_c).tolist()
        assert _three_ways(ctx, blk, info) == base, case[0]


def _blocks(n_blocks, n_tx):
    """n_blocks fault-free blocks of n_tx transactions (seeded), as (blob, env_off, ids)"""
    net = blockgen.Network()
    out = []
    for k in range(n_blocks):
        _, info = blockgen.build_block(net, n_tx, 3, None, seed=1000 + k, number=k + 1)
        n = info["env_off"].shape[0] - 1
        envs = [bytes(info["env_blob"][info["env_off"][t]:info["env_off"][t + 1]]) for t in range(n)]
        out.append(envs)
    return net, out


def _assemble(envs):
    off = np.zeros(len(envs) + 1, np.uint32)
    off[1:] = np.cumsum([len(e) for e in envs])
    return np.frombuffer(b"".join(envs), np.uint8).copy(), off


@pytest.mark.parametrize("growing", [False, True], ids=["presized", "growing"])
def test_pipeline_sees_exactly_the_ids_added_before_each_submit(ctx, growing):
    """Three 10 000-transaction blocks in flight on the three slots.  After each submit the block's ids are added; block k replays 500 of
    block k-1's envelopes and 500 of block k-3's.  Each block's own transactions stay VALID -- an add leaking into a block submitted before
    it would flag them 9 -- and the replays are 9.  'growing': the set starts at its smallest table and 20 000 filler ids per step force
    rehashes while blocks are in flight."""
    B = pkg().binding
    net, fresh = _blocks(7, 10000)
    ctx.msp_configure(blockutil.identities_of(net), net.policy_n_of(2), net.principals, net.channel)
    ctx.channel_capability(B.CAP_V2_0)
    ctx.committed_txids(["0" * 64], capacity=0 if growing else 400000)
    rng = np.random.default_rng(7)
    blocks, expect = [], []
    for k, envs in enumerate(fresh):
        rep = []
        if k >= 1:
            rep += [fresh[k - 1][i] for i in rng.choice(len(fresh[k - 1]), 500, replace=False)]
        if k >= 3:
            rep += [fresh[k - 3][i] for i in rng.choice(len(fresh[k - 3]), 500, replace=False)]
        blocks.append(_assemble(envs + rep))
        expect.append([ob.VALID] * len(envs) + [ob.DUPLICATE_TXID] * len(rep))
    sizes, got = [], [None] * len(blocks)
    for k, (blob, off) in enumerate(blocks):
        slot = k % B.SLOTS
        if k >= B.SLOTS:
            got[k - B.SLOTS] = ctx.validate_wait(slot, 20000).tolist()
        ctx.validate_envelopes_async(slot, blob, off)
        ids = [txid_oracle.txid_of(e) for e in fresh[k]]
        if growing:
            ids += [bytes(rng.integers(0, 256, 32, dtype=np.uint8)).hex() for _ in range(20000)]
        ctx.committed_txids_add(ids)
        sizes.append(ctx.committed_txids_info())
    for k in range(len(blocks) - B.SLOTS, len(blocks)):
        got[k] = ctx.validate_wait(k % B.SLOTS, 20000).tolist()
    for k in range(len(blocks)):
        assert got[k] == expect[k], k
    held = 1 + 7 * 10000 + (7 * 20000 if growing else 0)
    assert sizes[-1][0] == held
    if growing:
        assert len({s[1] for s in sizes}) >= 3 and sizes[-1][1] >= 2 * held
    else:
        assert len({s[1] for s in sizes}) == 1
    ctx.committed_txids([])


def test_broken_set_and_restore(ctx):
    """FABGPU_TXID_MAX_BYTES below what an add needs: the add fails, every transaction that reaches the ledger check is then 254 (earlier
    codes unchanged) and _add is refused, until a replacing call succeeds."""
    B = pkg().binding
    net = blockgen.Network()
    n = 3 * len(blockgen.FAULTS) + 4
    faults = blockutil.fault_map(n)
    blk, info = blockgen.build_block(net, n, 3, faults, seed=11, nthreads=2)
    ids = blockutil.identities_of(net)
    ctx.msp_configure(ids, net.policy_n_of(2), net.principals, net.channel)
    ctx.channel_capability(B.CAP_V2_0)
    ctx.committed_txids([])
    base = ctx.validate_block(blk).tolist()
    assert base == ob.validate_block(blk, ids, net.channel, net.policy_n_of(2), net.principals, known=[i[0] for i in ids]).tolist()
    saved = os.environ.get("FABGPU_TXID_MAX_BYTES")
    os.environ["FABGPU_TXID_MAX_BYTES"] = str(36 * 1024)
    try:
        ctx.committed_txids(["%064x" % k for k in range(300)])
        assert ctx.committed_txids_info() == (300, 1024)
        assert ctx.validate_block(blk).tolist() == base
        with pytest.raises(B.FabGpuError) as e:
            ctx.committed_txids_add(["%064x" % k for k in range(1000, 1400)])
        assert "FABGPU_TXID_MAX_BYTES" in str(e.value) and "broken" in str(e.value)
        broken = ctx.validate_block(blk).tolist()
        reaches = txid_oracle.committed(ob.validate_block, blk, ids, net.channel, net.policy_n_of(2), net.principals, known=[i[0] for i in ids],
                                        committed={txid_oracle.txid_of(bytes(info["env_blob"][info["env_off"][t]:info["env_off"][t + 1]])): 1
                                                   for t in range(n)})
        assert broken == reaches.tolist()
        assert sum(a != b for a, b in zip(broken, base)) >= n // 2
        with pytest.raises(B.FabGpuError, match="broken"):
            ctx.committed_txids_add(["%064x" % 1])
        ctx.committed_txids(["%064x" % k for k in range(10)])
    finally:
        if saved is None:
            os.environ.pop("FABGPU_TXID_MAX_BYTES", None)
        else:
            os.environ["FABGPU_TXID_MAX_BYTES"] = saved
    assert ctx.validate_block(blk).tolist() == base
    ctx.committed_txids([])


def test_removal_and_refusals(ctx):
    """n = 0 removes the set (flags of a context that never had one); refused calls keep the set; msp_configure keeps it."""
    B = pkg().binding
    net = blockgen.Network()
    blk, info = blockgen.build_block(net, 64, 3, blockutil.fault_map(64), seed=13, nthreads=2)
    ids = blockutil.identities_of(net)
    fresh = B.Context(max_batch=8192)
    try:
        for c in (ctx, fresh):
            c.msp_configure(ids, net.policy_n_of(2), net.principals, net.channel)
            c.channel_capability(B.CAP_V2_0)
        never = fresh.validate_block(blk).tolist()
        with pytest.raises(B.FabGpuError, match="no committed tx-id set"):
            fresh.committed_txids_add(["%064x" % 1])
    finally:
        fresh.close()
    tx_ids = [txid_oracle.txid_of(bytes(info["env_blob"][info["env_off"][t]:info["env_off"][t + 1]])) for t in range(64)]
    tx_ids = [i for i in tx_ids if i is not None]                    # an envelope whose header does not parse has no id
    ctx.committed_txids(tx_ids)
    with_set = ctx.validate_block(blk).tolist()
    assert with_set != never
    for bad in (lambda: ctx.committed_txids_add(tx_ids[:2], [0, 2]), lambda: ctx.committed_txids(tx_ids[:2], [3, 0])):
        with pytest.raises(B.FabGpuError, match="kind"):
            bad()
    assert ctx.validate_block(blk).tolist() == with_set
    ctx.msp_configure(ids, net.policy_n_of(2), net.principals, net.channel)
    assert ctx.validate_block(blk).tolist() == with_set
    ctx.committed_txids([])
    assert ctx.committed_txids_info() == (0, 0)
    assert ctx.validate_block(blk).tolist() == never
