"""GPU: the block's update batch (fabgpu_block_updates) -- every case through validate_block and validate_envelopes in both validator
modes and under LevelDB and CouchDB, a sequence of seeded blocks over hot keys submitted three slots deep with the batch applied to a
state after each, repeated calls, short output buffers, and the refusals."""
import ctypes

import numpy as np
import pytest

from tools import blockgen
from util import pkg
import updatecases
import updates_oracle as uo
import updatesutil

pytestmark = pytest.mark.gpu

POLICIES = {updatecases.CC: 0}


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
    c.namespace_versions({updatecases.CC: "1.0"})
    c.channel_capability(cap)


def _block(net, txs, seed):
    faults = {t: "config_update_type" for t, tx in enumerate(txs) if tx is None}
    hook = lambda t, part, b: uo.encode(txs[t]) if part == "TxReadWriteSet" and txs[t] is not None else b
    return blockgen.build_block(net, len(txs), 3, faults, seed=seed, mutate=hook)


def _recs(got):
    return None if got is None else [(t, op, ns.decode(), coll.decode(), key, v, m) for t, op, ns, coll, key, v, m in got]


def _entries(versions):
    return sorted((k, v) for k, v in versions.items() if v != "unknown")


@pytest.mark.parametrize("db", ["leveldb", "couchdb"])
@pytest.mark.parametrize("entry", ["block", "envelopes"])
@pytest.mark.parametrize("mode", ["v20", "v13"])
def test_cases_on_the_device(ctx, net, entry, mode, db):
    B = pkg().binding
    couch = db == "couchdb"
    _configure(ctx, net, B.CAP_V1_3 if mode == "v13" else B.CAP_V2_0)
    ctx.state_database(B.STATEDB_COUCHDB if couch else B.STATEDB_LEVELDB)
    try:
        for name, state0, steps in updatecases.cases():
            versions, _ = updatecases.split(state0)
            ctx.state_versions(_entries(versions), 1)
            for k, step in enumerate(steps):
                txs, tv, want = step[:3]
                if couch and len(step) > 3:
                    want = step[3]
                blk, info = _block(net, txs, seed=41 + k)
                ctx.validate_block(blk) if entry == "block" else ctx.validate_envelopes(info["env_blob"], info["env_off"])
                codes, versions, is_open = uo.flags(versions, 1 + k, txs, tv, couch)
                assert ctx.validate_mvcc(0, 1 + k, tv).tolist() == codes, (name, k)
                got = ctx.block_updates(0, 1 + k)
                assert _recs(got) == want, (name, k)
                assert ctx.block_updates(0, 1 + k) == got, (name, k)
                if is_open:
                    ctx.state_versions_update([], 2 + k)
    finally:
        _configure(ctx, net, B.CAP_V2_0)
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions([], 0)


def _sequence(net, n_blocks, seed, versions):
    """seeded blocks over ten hot keys whose flags, all transactions VALID for the validator, hold no 254"""
    rng = np.random.default_rng(seed)
    pool = ["hot%d" % i for i in range(10)]
    out = []
    for b in range(n_blocks):
        for _ in range(50):
            n = int(rng.integers(8, 24))
            txs = [updatesutil.random_tx(rng, pool, t) for t in range(n)]
            codes, nv, _ = uo.flags(versions, 1 + b, txs, [0] * n)
            if 254 not in codes:
                break
        versions = nv
        out.append((txs, _block(net, txs, seed=700 + b)[0]))
    return out


def test_three_slots_deep_over_hot_keys(ctx, net):
    """About 30 blocks three slots deep: after each block's stage its batch equals the oracle's, and applied to a state (reading the
    committed sources from it) gives the oracle's state, value and metadata."""
    versions = {(updatecases.CC, "", ("hot%d" % i).encode()): (0, i % 3) for i in range(6)}
    values = {k: (b"c%d" % i, None) for i, k in enumerate(sorted(versions))}
    seq = _sequence(net, 30, 13, dict(versions))
    ctx.state_versions(_entries(versions), 1, capacity=64)
    S = pkg().binding.SLOTS
    state, oracle_state, records = dict(values), dict(values), 0
    try:
        for k in range(min(S, len(seq))):
            ctx.validate_block_async(k % S, seq[k][1])
        for k, (txs, blk) in enumerate(seq):
            tv = ctx.validate_wait(k % S, len(txs) + 16)
            assert tv.tolist() == [0] * len(txs)
            codes, versions2, _ = uo.flags(versions, 1 + k, txs, tv.tolist())
            assert ctx.validate_mvcc(k % S, 1 + k, tv).tolist() == codes, k
            want = uo.batch(versions, oracle_state, 1 + k, txs, codes)
            got = _recs(ctx.block_updates(k % S, 1 + k))
            assert got == want, k
            state = uo.apply(state, got)
            oracle_state = uo.apply(oracle_state, want)
            assert state == oracle_state, k
            versions = versions2
            records += len(got)
            if k + S < len(seq):
                ctx.validate_block_async(k % S, seq[k + S][1])
        assert records > 100
    finally:
        ctx.state_versions([], 0)


def _raw(ctx, slot, block_num, rec_cap, meta_cap):
    L = pkg().binding.lib()
    rec = np.full(pkg().binding.UPDATE_WORDS * max(rec_cap, 1), 0xAAAAAAAA, np.uint32)
    meta = np.full(max(meta_cap, 1), 0xAA, np.uint8)
    n = (ctypes.c_size_t * 2)()
    complete = ctypes.c_int(-1)
    rc = L.fabgpu_block_updates(ctx._h, ctypes.c_int(slot), ctypes.c_uint64(block_num), rec.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(rec_cap),
                                meta.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(meta_cap), n, ctypes.byref(complete))
    return rc, rec, meta, (int(n[0]), int(n[1])), complete.value


def test_short_buffers_and_refusals(ctx, net):
    B = pkg().binding
    W = B.UPDATE_WORDS
    versions, _ = updatecases.split(updatecases.ST)
    ctx.state_versions(_entries(versions), 1)
    try:
        txs = [updatecases.tx(writes=[("k%d" % t, b"v%d" % t)], md=[("k%d" % t, [("VALIDATION_PARAMETER", b"p%d" % t)])]) for t in range(6)]
        blk, _ = _block(net, txs, seed=9)
        tv = ctx.validate_block(blk)
        assert _raw(ctx, 0, 1, 4, 64)[0] == B.E_ARG                   # before the stage ran
        assert ctx.validate_mvcc(0, 1, tv).tolist() == [0] * 6
        full = ctx.block_updates(0, 1)
        per = len(uo.serialize([("VALIDATION_PARAMETER", b"p0")]))
        rc, rec, meta, n, complete = _raw(ctx, 0, 1, 2, 5)
        assert rc == 0 and complete == 1 and n == (6, 6 * per)
        assert (rec[2 * W:] == 0xAAAAAAAA).all() and (meta[5:] == 0xAA).all()
        assert rec[0] == 0 and bytes(meta[:5]) == full[0][6][:5]
        rc, rec, meta, n, complete = _raw(ctx, 0, 1, 0, 0)
        assert rc == 0 and n == (6, 6 * per)
        # refusals, each with nothing enqueued
        assert _raw(ctx, 1, 1, 4, 64)[0] == B.E_ARG                   # another slot
        assert _raw(ctx, 0, 2, 4, 64)[0] == B.E_ARG                   # another block
        L = B.lib()
        assert L.fabgpu_block_updates(ctx._h, 0, ctypes.c_uint64(1), None, ctypes.c_size_t(0), None, ctypes.c_size_t(0), None, None) == B.E_ARG
        assert L.fabgpu_block_updates(ctx._h, 0, ctypes.c_uint64(1), None, ctypes.c_size_t(4), None, ctypes.c_size_t(0), (ctypes.c_size_t * 2)(),
                                      ctypes.byref(ctypes.c_int())) == B.E_ARG
        assert ctx.block_updates(0, 1) == full                        # still there
        ctx.state_versions_update([], 2)                              # a state call
        assert _raw(ctx, 0, 1, 4, 64)[0] == B.E_ARG
        blk2, _ = _block(net, [updatecases.tx(writes=[("k0", b"w")])], seed=10)
        ctx.validate_block(blk2)
        assert ctx.validate_mvcc(0, 2, [0]).tolist() == [0]
        assert ctx.block_updates(0, 2) == [(0, "put", b"mycc", b"", b"k0", b"w", B.COMMITTED)]
        ctx.validate_block_async(1, blk2)                             # another slot's stage
        ctx.validate_wait(1, 16)
        assert ctx.validate_mvcc(1, 3, [0]).tolist() == [0]
        assert _raw(ctx, 0, 2, 4, 64)[0] == B.E_ARG
        assert ctx.block_updates(1, 3) is not None
        ctx.validate_block_async(1, blk2)                             # the slot's next submit
        assert _raw(ctx, 1, 3, 4, 64)[0] == B.E_ARG
        ctx.validate_wait(1, 16)
        # an empty envelope list: complete, no records
        ctx.validate_envelopes_async(2, np.zeros(1, np.uint8), np.zeros(1, np.uint32))
        ctx.validate_wait(2, 16)
        assert ctx.validate_mvcc(2, 4, []).tolist() == []
        assert ctx.block_updates(2, 4) == []
    finally:
        ctx.state_versions([], 0)
