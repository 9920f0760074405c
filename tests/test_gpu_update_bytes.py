"""GPU: the block's deterministic update bytes (fabgpu_block_update_bytes) -- every case through validate_block and validate_envelopes in
both validator modes and under LevelDB and CouchDB, a seeded sequence three slots deep whose commit hashes chained from the device's bytes
equal the oracle's chain, a block of over 100 000 records with a 1 MiB value, repeated calls, short output buffers, and the refusals."""
import ctypes
import hashlib

import numpy as np
import pytest

from tools import blockgen
from util import pkg
import update_bytes_oracle as bo
import updatebytescases as cases
import updates_oracle as uo

pytestmark = pytest.mark.gpu

POLICIES = {ns: 0 for ns in [cases.CC] + cases.NSS + ["ns%d" % i for i in range(4)]}


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
    c.namespace_versions({ns: "1.0" for ns in POLICIES})
    c.channel_capability(cap)


def _block(net, txs, seed):
    hook = lambda t, part, b: uo.encode(txs[t]) if part == "TxReadWriteSet" else b
    return blockgen.build_block(net, len(txs), 3, {}, seed=seed, mutate=hook)


def _entries(versions):
    return sorted((k, v) for k, v in versions.items() if v != "unknown")


def _committed(recs, values):
    """what the peer reads for the device's COMMITTED-value records, in record order"""
    B = pkg().binding
    return [values[(ns.decode(), coll.decode(), key)][0] for _t, _op, ns, coll, key, v, _m in recs or () if v == B.COMMITTED]


@pytest.mark.parametrize("db", ["leveldb", "couchdb"])
@pytest.mark.parametrize("entry", ["block", "envelopes"])
@pytest.mark.parametrize("mode", ["v20", "v13"])
def test_cases_on_the_device(ctx, net, entry, mode, db):
    B = pkg().binding
    couch = db == "couchdb"
    _configure(ctx, net, B.CAP_V1_3 if mode == "v13" else B.CAP_V2_0)
    ctx.state_database(B.STATEDB_COUCHDB if couch else B.STATEDB_LEVELDB)
    try:
        for case in cases.cases():
            name, block_num, state0, txs, tv, want = case[:6]
            if couch and len(case) > 6:
                want = case[6]
            versions, values = cases.split(state0)
            ctx.state_versions(_entries(versions), block_num, capacity=64)
            blk, info = _block(net, txs, seed=51)
            ctx.validate_block(blk) if entry == "block" else ctx.validate_envelopes(info["env_blob"], info["env_off"])
            codes, _, _ = uo.flags(versions, block_num, txs, tv, couch)
            assert ctx.validate_mvcc(0, block_num, tv).tolist() == codes, name
            recs = ctx.block_updates(0, block_num)
            got = ctx.block_update_bytes(0, block_num, _committed(recs, values))
            assert got == (None if want is None else bo.marshal(want)), name
            assert ctx.block_update_bytes(0, block_num, _committed(recs, values)) == got, name
    finally:
        _configure(ctx, net, B.CAP_V2_0)
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions([], 0)


def _sequence(net, n_blocks, seed, versions):
    """seeded blocks over hot keys in several namespaces and collections whose flags, all transactions VALID for the validator, hold no 254"""
    rng = np.random.default_rng(seed)
    pool = ["hot%d" % i for i in range(10)]
    out = []
    for b in range(n_blocks):
        for _ in range(50):
            n = int(rng.integers(8, 24))
            txs = [cases.random_tx(rng, pool, t) for t in range(n)]
            codes, nv, _ = uo.flags(versions, 1 + b, txs, [0] * n)
            if 254 not in codes:
                break
        versions = nv
        out.append((txs, _block(net, txs, seed=900 + b)[0]))
    return out


def test_commit_hash_chain_three_slots_deep(ctx, net):
    """About 30 blocks three slots deep: at every block the commit hash chained from block 1 with the device's bytes equals the one chained
    with the oracle's"""
    versions = {(ns, "", ("hot%d" % i).encode()): (0, i % 3) for ns in cases.NSS[:2] for i in range(6)}
    values = {k: (b"c%d" % i, None) for i, k in enumerate(sorted(versions))}
    seq = _sequence(net, 30, 23, dict(versions))
    ctx.state_versions(_entries(versions), 1, capacity=256)
    S = pkg().binding.SLOTS
    state, oracle_state = dict(values), dict(values)
    h_dev = h_oracle = b""
    total = 0
    try:
        for k in range(min(S, len(seq))):
            ctx.validate_block_async(k % S, seq[k][1])
        for k, (txs, blk) in enumerate(seq):
            tv = ctx.validate_wait(k % S, len(txs) + 16)
            assert len(tv) == len(txs)
            codes, versions2, _ = uo.flags(versions, 1 + k, txs, [0] * len(txs))
            flags = ctx.validate_mvcc(k % S, 1 + k, [0] * len(txs)).tolist()
            assert flags == codes, k
            recs = ctx.block_updates(k % S, 1 + k)
            dev = ctx.block_update_bytes(k % S, 1 + k, _committed(recs, state))
            want_recs = uo.batch(versions, oracle_state, 1 + k, txs, codes)
            want = bo.update_bytes(want_recs, 1 + k, bo.committed_values(want_recs, oracle_state))
            assert dev is not None and dev == want, k
            h_dev = bo.commit_hash(bytes(flags), dev, h_dev)
            h_oracle = bo.commit_hash(bytes(codes), want, h_oracle)
            assert h_dev == h_oracle, k
            state = uo.apply(state, [(t, op, ns.decode(), coll.decode(), key, v, m) for t, op, ns, coll, key, v, m in recs])
            oracle_state = uo.apply(oracle_state, want_recs)
            versions = versions2
            total += len(dev)
            if k + S < len(seq):
                ctx.validate_block_async(k % S, seq[k + S][1])
        assert total > 5000
    finally:
        ctx.state_versions([], 0)


def test_a_block_of_100000_records_with_a_1_mib_value(ctx, net):
    rng = np.random.default_rng(77)
    txs = []
    for t in range(10):
        writes = [(bytes(rng.integers(0, 256, int(rng.integers(1, 48)), dtype=np.uint8)) + b"%d.%d" % (t, j), b"v%d" % j) for j in range(9000)]
        if t == 3:
            writes.append((b"big", bytes(rng.integers(0, 256, 1 << 20, dtype=np.uint8))))
        colls = [("coll%d" % c, [], [(hashlib.sha256(b"%d.%d" % (t, q)).digest(), b"h%d" % q) for q in range(c * 400, c * 400 + 400)], [])
                 for c in range(3)]
        txs.append([cases.ns("ns%d" % (t % 4), writes=writes, colls=colls)])
    ctx.state_versions([], 1, capacity=1 << 18)
    try:
        blk, _ = _block(net, txs, seed=61)
        ctx.validate_block(blk)
        codes, _, _ = uo.flags({}, 1, txs, [0] * 10)
        assert ctx.validate_mvcc(0, 1, [0] * 10).tolist() == codes == [0] * 10
        recs = uo.batch({}, {}, 1, txs, codes)
        assert len(recs) >= 100_000
        want = bo.update_bytes(recs, 1)
        got = ctx.block_update_bytes(0, 1)
        assert got is not None and len(got) == len(want) and got == want
        assert ctx.block_update_bytes(0, 1) == got
    finally:
        ctx.state_versions([], 0)


def _raw(ctx, slot, block_num, vals, out_cap, n_val=None, off=None):
    B = pkg().binding
    blob = np.frombuffer(b"".join(vals) + b"\x00", np.uint8).copy()
    o = np.zeros(len(vals) + 1, np.uint32) if off is None else np.asarray(off, np.uint32)
    if off is None:
        o[1:] = np.cumsum([len(v) for v in vals])
    out = np.full(max(out_cap, 1), 0xAA, np.uint8)
    n = ctypes.c_size_t(12345)
    complete = ctypes.c_int(-1)
    rc = B.lib().fabgpu_block_update_bytes(ctx._h, ctypes.c_int(slot), ctypes.c_uint64(block_num), blob.ctypes.data_as(ctypes.c_void_p),
                                           o.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(vals) if n_val is None else n_val),
                                           out.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(out_cap), ctypes.byref(n), ctypes.byref(complete))
    return rc, out, n.value, complete.value


def test_short_buffers_and_refusals(ctx, net):
    B = pkg().binding
    L = B.lib()
    versions, values = cases.split(cases.ST)
    ctx.state_versions(_entries(versions), 1)
    try:
        txs = [cases.tx(cases.ns(cases.CC, md=[("a", cases.E1)], colls=[("c1", [], [], [(cases.hk(0x41), cases.E1)])])),
               cases.tx(cases.ns(cases.CC, writes=[("k%d" % t, b"v%d" % t) for t in range(6)]))]
        blk, _ = _block(net, txs, seed=9)
        tv = ctx.validate_block(blk)
        vals = [b"A0", b"HR0"]
        assert _raw(ctx, 0, 1, vals, 64)[0] == B.E_ARG                 # before the stage ran
        assert ctx.validate_mvcc(0, 1, [0, 0]).tolist() == [0, 0]
        full = ctx.block_update_bytes(0, 1, vals)
        recs = ctx.block_updates(0, 1)
        assert _committed(recs, values) == vals
        assert full == bo.update_bytes(uo.batch(versions, values, 1, txs, [0, 0]), 1, vals)
        rc, out, n, complete = _raw(ctx, 0, 1, vals, 5)
        assert rc == 0 and complete == 1 and n == len(full) and bytes(out[:5]) == full[:5] and (out[5:] == 0xAA).all()
        rc, out, n, complete = _raw(ctx, 0, 1, vals, 0)
        assert rc == 0 and complete == 1 and n == len(full)
        # refusals, each with nothing enqueued
        assert _raw(ctx, 0, 1, vals[:1], 64)[0] == B.E_ARG               # n_val below the COMMITTED records
        assert _raw(ctx, 0, 1, vals + [b"x"], 64)[0] == B.E_ARG          # above
        assert _raw(ctx, 0, 1, vals, 64, off=[0, 3, 2])[0] == B.E_ARG    # decreasing offsets
        assert _raw(ctx, 1, 1, vals, 64)[0] == B.E_ARG                   # another slot
        assert _raw(ctx, 0, 2, vals, 64)[0] == B.E_ARG                   # another block
        n, c = ctypes.c_size_t(0), ctypes.c_int(0)
        blob = (ctypes.c_uint8 * 8)()
        off = (ctypes.c_uint32 * 3)(0, 2, 5)
        u64 = ctypes.c_uint64(1)
        assert L.fabgpu_block_update_bytes(ctx._h, 0, u64, blob, off, ctypes.c_size_t(2), None, ctypes.c_size_t(0), None, ctypes.byref(c)) == B.E_ARG
        assert L.fabgpu_block_update_bytes(ctx._h, 0, u64, blob, off, ctypes.c_size_t(2), None, ctypes.c_size_t(0), ctypes.byref(n), None) == B.E_ARG
        assert L.fabgpu_block_update_bytes(ctx._h, 0, u64, blob, off, ctypes.c_size_t(2), None, ctypes.c_size_t(8), ctypes.byref(n),
                                           ctypes.byref(c)) == B.E_ARG         # NULL out with a capacity
        assert L.fabgpu_block_update_bytes(ctx._h, 0, u64, blob, None, ctypes.c_size_t(2), None, ctypes.c_size_t(0), ctypes.byref(n),
                                           ctypes.byref(c)) == B.E_ARG         # NULL offsets
        assert L.fabgpu_block_update_bytes(ctx._h, 0, u64, None, off, ctypes.c_size_t(2), None, ctypes.c_size_t(0), ctypes.byref(n),
                                           ctypes.byref(c)) == B.E_ARG         # NULL values
        assert ctx.block_update_bytes(0, 1, vals) == full                # still there
        # the slot's next submit
        blk2, _ = _block(net, [cases.tx(cases.ns(cases.CC, writes=[("k0", b"w")]))], seed=10)
        ctx.validate_block_async(0, blk2)
        assert _raw(ctx, 0, 1, vals, 64)[0] == B.E_ARG
        ctx.validate_wait(0, 16)
        assert ctx.validate_mvcc(0, 2, [0]).tolist() == [0]
        assert ctx.block_update_bytes(0, 2) == bo.marshal([bo.kvwrite(b"k0", b"w", version=bo.height(2, 0), namespace=cases.CC)])
        ctx.state_versions_update([], 3)                                 # a state call
        assert _raw(ctx, 0, 2, [], 64)[0] == B.E_ARG
        # an empty envelope list: complete, no bytes
        ctx.validate_envelopes_async(2, np.zeros(1, np.uint8), np.zeros(1, np.uint32))
        ctx.validate_wait(2, 16)
        assert ctx.validate_mvcc(2, 3, []).tolist() == []
        assert ctx.block_update_bytes(2, 3) == b""
    finally:
        ctx.state_versions([], 0)
