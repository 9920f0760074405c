"""GPU: the block's private update batch (fabgpu_block_pvt_updates) -- every case through validate_block and validate_envelopes in both
validator modes and under LevelDB and CouchDB, with status and verdict equal to validate_pvtdata's with the stage's flags; seeded blocks
over hot private keys submitted three slots deep with the public, hashed and private batches applied after each; repeated calls, short
record buffers, and the refusals."""
import ctypes

import numpy as np
import pytest

from tools import blockgen
from util import pkg
import pvt_updates_oracle as puo
import pvtupdatecases as cases
import updates_oracle as uo

pytestmark = pytest.mark.gpu

POLICIES = {cases.CC: 0}


@pytest.fixture(scope="module")
def net():
    return blockgen.Network()


@pytest.fixture(scope="module")
def ctx(net):
    c = pkg().binding.Context(max_batch=8192)
    _configure(c, net, pkg().binding.CAP_V2_0)
    yield c
    c.close()


def _configure(c, net, cap):
    c.msp_configure([(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table], net.policy_n_of(3), net.principals, net.channel,
                    policies=POLICIES)
    c.namespace_versions({cases.CC: "1.0"})
    c.channel_capability(cap)


def _block(net, txs, seed):
    rws = cases.rwsets(txs)
    hook = lambda t, part, b: rws[t] if part == "TxReadWriteSet" else b
    return blockgen.build_block(net, len(txs), 3, {}, seed=seed, mutate=hook)


def _entries(versions):
    return sorted(versions.items())


@pytest.mark.parametrize("db", ["leveldb", "couchdb"])
@pytest.mark.parametrize("entry", ["block", "envelopes"])
@pytest.mark.parametrize("mode", ["v20", "v13"])
def test_cases_on_the_device(ctx, net, entry, mode, db):
    B = pkg().binding
    _configure(ctx, net, B.CAP_V1_3 if mode == "v13" else B.CAP_V2_0)
    ctx.state_database(B.STATEDB_COUCHDB if db == "couchdb" else B.STATEDB_LEVELDB)
    try:
        for k, (name, committed, tv, txs, want) in enumerate(cases.cases()):
            ctx.state_versions(_entries(committed[0]), 1, capacity=64)
            blk, info = _block(net, txs, seed=41 + k)
            ctx.validate_block(blk) if entry == "block" else ctx.validate_envelopes(info["env_blob"], info["env_off"])
            codes, hashed, verdict, status, recs = cases.run_oracle(committed, 1, txs, tv)
            assert recs == want, name
            assert ctx.validate_mvcc(0, 1, tv).tolist() == codes, name
            pvt = cases.pvt_of(txs)
            got = ctx.block_pvt_updates(0, 1, pvt)
            assert got == (verdict, status, want), name
            assert got[:2] == ctx.validate_pvtdata(0, codes, pvt), name
            assert ctx.block_pvt_updates(0, 1, pvt) == got, name            # rebuilt: the same records
            hw = ctx.block_updates(0, 1)                                      # the hashed batch is still there
            assert (hw is None) == (hashed is None), name
    finally:
        _configure(ctx, net, B.CAP_V2_0)
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions([], 0)


def _hashed_values(recs, values):
    """updates_oracle's committed values after the device's hashed batch (ns, coll decoded)"""
    conv = [(t, op, ns.decode(), coll.decode(), key, v, m) for t, op, ns, coll, key, v, m in recs]
    return uo.apply(values, conv), conv


def test_three_slots_deep_over_hot_private_keys(ctx, net):
    """Seeded blocks three slots deep: after each block's stage the private records equal the oracle's, and the private state the
    device's three batches leave (RENEW records resolved with the state before the block) equals the oracle's"""
    S = pkg().binding.SLOTS
    blocks = []
    for b in range(24):
        txs, tv = cases.seeded(3000 + b, 12 + b % 9)
        blocks.append((txs, tv, _block(net, txs, seed=800 + b)[0]))
    ctx.state_versions([], 1, capacity=1024)
    versions, values, pstate, dev_state = {}, {}, {}, {}
    counts = {"put": 0, "del": 0, "renew": 0, None: 0}
    try:
        for k in range(min(S, len(blocks))):
            ctx.validate_block_async(k % S, blocks[k][2])
        for k, (txs, tv, _) in enumerate(blocks):
            slot = k % S
            ctx.validate_wait(slot, len(txs) + 16)
            codes, versions2, _ = uo.flags(versions, 1 + k, [t["pub"] for t in txs], tv)
            assert ctx.validate_mvcc(slot, 1 + k, tv).tolist() == codes, k
            hashed = uo.batch(versions, values, 1 + k, [t["pub"] for t in txs], codes)
            verdict, status, want = puo.batch(1 + k, codes, cases.rwsets(txs), cases.pvt_of(txs), hashed)
            got = ctx.block_pvt_updates(slot, 1 + k, cases.pvt_of(txs))
            assert got == (verdict, status, want), k
            dev_h = ctx.block_updates(slot, 1 + k)
            if want is None:
                counts[None] += 1
                pstate, dev_state = {}, {}
            else:
                for r in want:
                    counts[r[1]] += 1
                pstate = puo.apply(pstate, 1 + k, want, hashed, values)
                dev_state = puo.apply(dev_state, 1 + k, got[2], [(t, op, ns, coll, key, v, m) for t, op, ns, coll, key, v, m in dev_h], values)
                assert dev_state == pstate, k
            values = uo.apply(values, hashed) if hashed is not None else {}
            versions = versions2
            if k + S < len(blocks):
                ctx.validate_block_async(slot, blocks[k + S][2])
        assert counts["put"] > 50 and counts["renew"] > 3, counts
    finally:
        ctx.state_versions([], 0)


def _raw(ctx, slot, block_num, pvt, rec_cap, status=True, n_pvt=None, off=None, seq=None):
    B = pkg().binding
    seqs = sorted(pvt)
    items = [pvt[s] for s in seqs]
    blob = np.frombuffer(b"".join(items) or b"\0", np.uint8).copy()
    off = np.array(off if off is not None else np.cumsum([0] + [len(x) for x in items]), np.uint32)
    sq = np.array(seq if seq is not None else (seqs or [0]), np.uint32)
    st = np.zeros(3 * max(len(seqs), 1) + 3, np.int32)
    out = np.zeros(4, np.int32)
    rec = np.full(B.PVT_UPDATE_WORDS * max(rec_cap, 1), 0xAAAAAAAA, np.uint32)
    n = ctypes.c_size_t(12345)
    complete = ctypes.c_int(-1)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = B.lib().fabgpu_block_pvt_updates(ctx._h, ctypes.c_int(slot), ctypes.c_uint64(block_num), p(blob), p(off), p(sq),
                                          ctypes.c_size_t(len(seqs) if n_pvt is None else n_pvt), p(st) if status else None, p(out), p(rec),
                                          ctypes.c_size_t(rec_cap), ctypes.byref(n), ctypes.byref(complete))
    return rc, rec, n.value, complete.value


def test_short_buffers_and_refusals(ctx, net):
    B = pkg().binding
    W = B.PVT_UPDATE_WORDS
    name, committed, tv, txs, want = cases.cases()[1]              # two records
    pvt = cases.pvt_of(txs)
    ctx.state_versions([], 1, capacity=64)
    try:
        blk, _ = _block(net, txs, seed=9)
        ctx.validate_block(blk)
        assert _raw(ctx, 0, 1, pvt, 4)[0] == B.E_ARG                 # before the stage ran
        assert ctx.validate_mvcc(0, 1, tv).tolist() == [0]
        rc, rec, n, complete = _raw(ctx, 0, 1, pvt, 1)
        assert rc == 0 and complete == 1 and n == 2 and (rec[W:] == 0xAAAAAAAA).all() and rec[1] == B.UPDATE_PUT
        rc, rec, n, complete = _raw(ctx, 0, 1, pvt, 0)
        assert rc == 0 and n == 2
        # refusals, each with nothing enqueued
        assert _raw(ctx, 1, 1, pvt, 4)[0] == B.E_ARG                 # another slot
        assert _raw(ctx, 0, 2, pvt, 4)[0] == B.E_ARG                 # another block
        assert _raw(ctx, 0, 1, {5: pvt[0]}, 4)[0] == B.E_ARG         # a seq past the block
        two = {0: pvt[0], 1: pvt[0]}
        assert _raw(ctx, 0, 1, two, 4, seq=[0, 0])[0] == B.E_ARG     # a seq given twice
        assert _raw(ctx, 0, 1, pvt, 4, off=[len(pvt[0]), 0])[0] == B.E_ARG   # offsets decrease
        assert _raw(ctx, 0, 1, pvt, 4, status=False)[0] == B.E_ARG   # NULL status with entries
        L = B.lib()
        assert L.fabgpu_block_pvt_updates(ctx._h, 0, ctypes.c_uint64(1), None, None, None, ctypes.c_size_t(0), None, None, None,
                                          ctypes.c_size_t(0), None, None) == B.E_ARG
        assert L.fabgpu_block_pvt_updates(ctx._h, 0, ctypes.c_uint64(1), None, None, None, ctypes.c_size_t(1), None,
                                          np.zeros(4, np.int32).ctypes.data_as(ctypes.c_void_p), None, ctypes.c_size_t(0),
                                          ctypes.byref(ctypes.c_size_t()), ctypes.byref(ctypes.c_int())) == B.E_ARG
        assert ctx.block_pvt_updates(0, 1, pvt)[2] == want            # still there
        assert ctx.block_pvt_updates(0, 1, {}) == ((0, -1, -1, -1), {}, [])
        ctx.validate_block_async(0, blk)                             # the slot's next submit
        assert _raw(ctx, 0, 1, pvt, 4)[0] == B.E_ARG
        ctx.validate_wait(0, 16)
        ctx.state_versions_update([], 2)
        ctx.validate_block(blk)
        assert ctx.validate_mvcc(0, 2, tv).tolist() == [0]
        ctx.state_versions_update([], 3)                             # a state call
        assert _raw(ctx, 0, 2, pvt, 4)[0] == B.E_ARG
    finally:
        ctx.state_versions([], 0)
