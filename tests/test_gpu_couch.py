"""GPU: the MVCC stage under CouchDB (fabgpu_state_database, couchval.cuh) -- every case through fabgpu_validate_mvcc in both modes, the
value check on the generated corpus and on long, deep and boundary-straddling values (fabgpu_test_couch_values), generated sequences
submitted three slots deep with the index installed and the mode switched between blocks, and the install refusals."""
import numpy as np
import pytest

from tools import blockgen
from util import pkg
import couch_oracle as co
import couchcases
import couchutil
import mvcc_oracle as mo

pytestmark = pytest.mark.gpu

CC = couchcases.CC
POLICIES = {CC: 0, "othercc": 0}


@pytest.fixture(scope="module")
def net():
    return blockgen.Network()


@pytest.fixture(scope="module")
def ctx(net):
    c = pkg().binding.Context(max_batch=8192)
    c.msp_configure([(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table], net.policy_n_of(3), net.principals, net.channel,
                    policies=POLICIES)
    c.namespace_versions({CC: "1.0"})
    c.channel_capability(pkg().binding.CAP_V2_0)
    yield c
    c.state_database(pkg().binding.STATEDB_LEVELDB)
    c.close()


def _block(net, txs, seed):
    hook = lambda t, part, b: co.encode(txs[t]) if part == "TxReadWriteSet" and txs[t] is not None else b
    return blockgen.build_block(net, len(txs), 3, {}, seed=seed, mutate=hook)


def _entries(state):
    return [(k, v) for k, v in sorted(state.items()) if v != mo.UNKNOWN]


@pytest.mark.parametrize("couch", [True, False], ids=["couchdb", "leveldb"])
def test_cases_on_the_device(ctx, net, couch):
    B = pkg().binding
    ctx.state_database(B.STATEDB_COUCHDB if couch else B.STATEDB_LEVELDB)
    try:
        for name, state0, steps in couchcases.cases():
            ctx.state_versions_indexed(_entries(state0), 1)
            state = dict(state0)
            for height, (txs, tv, codes) in enumerate(steps, 1):
                blk, _ = _block(net, txs, seed=60 + height)
                ctx.validate_block(blk)
                got = ctx.validate_mvcc(0, height, tv).tolist()
                exp, state, _ = co.validate(state, height, txs, tv, couch=couch)
                assert got == exp, (name, height)
                if couch:
                    assert got == codes, (name, height)
                held, _, _, unknown = ctx.state_versions_info()
                assert (held, unknown) == mo.info(state), (name, height)
    finally:
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions([], 0)


@pytest.mark.parametrize("path", [0, 1, 2], ids=["by_length", "one_thread", "cta"])
def test_generated_values_on_the_device(ctx, path):
    vals = couchutil.corpus(1, 100000)
    got = ctx.test_couch_values(vals, path).tolist()
    exp = [co.value_bits(v) for v in vals]
    bad = [(v, g, e) for v, g, e in zip(vals, got, exp) if g != e]
    assert not bad, bad[:5]


def test_long_deep_and_straddling_values_on_the_device(ctx):
    rng = np.random.default_rng(9)
    vals = []
    # escapes, backslash runs, strings, numbers and brackets straddling lane chunks, tiles and the length bound
    for L in (31, 32, 33, 63, 64, 65, 127, 128, 129, 4095, 4096, 4097, co.TILE_BYTES - 1, co.TILE_BYTES, co.TILE_BYTES + 1,
              co.SHORT_MAX + 1, 2 * co.TILE_BYTES + 3):
        for tail in (b'\\"', b"\\\\", b"\\u005f", b"\\\\\\"):
            pad = max(0, L - 14 - len(tail))
            vals.append(b'{"_id":1,"s":"' + b"x" * pad + tail + b'"}')
        vals.append(b'{"n":' + b"1" * max(1, L - 12) + b',"_a":1}')
        vals.append(b" " * (L - 2) + b"{}")
        vals.append(b'{"_b":' + b"[" * 30 + b" " * max(0, L - 36) + b"]" * 30 + b"}")
    deep = lambda d: b'{"k":' * d + b"1" + b"}" * d
    vals += [deep(co.DEPTH - 1), deep(co.DEPTH), deep(co.DEPTH + 1), b"[" * 1000 + b"]" * 1000]
    big = [couchutil.document(rng) for _ in range(60000)]
    vals.append(b'{"docs":[' + b",".join(big) + b'],"_id":1}')                                     # several MiB of documents
    vals.append(b'{"doc":"' + bytes(rng.integers(0x61, 0x7a, 8 << 20, dtype=np.uint8)) + b'","_id":1}')     # 8 MiB
    vals.append(b"[" + b"1," * (200 << 10) + b"1]")
    exp = [co.value_bits(v) for v in vals]
    assert ctx.test_couch_values(vals, 0).tolist() == exp
    assert ctx.test_couch_values(vals, 1).tolist() == exp
    assert ctx.test_couch_values(vals, 2).tolist() == exp


def test_unholdable_key_of_a_254_writer_is_settled_by_removal(ctx, net):
    B = pkg().binding
    ctx.state_database(B.STATEDB_COUCHDB)
    try:
        ctx.state_versions_indexed([((CC, "", b"b"), (0, 1))], 1)
        txs = [couchcases.wv("_a", b'{"v":1}'), couchcases.wv("b", b'{"v":2}')]
        blk, _ = _block(net, txs, seed=80)
        ctx.validate_block(blk)
        assert ctx.validate_mvcc(0, 1, [254, 0]).tolist() == [254, 0]
        assert ctx.state_versions_info()[3] == 1
        rng_tx = couchcases.rc.q("A", "z", [("b", (1, 1))])
        for h, want in ((2, 254), (3, 0)):
            if h == 3:
                with pytest.raises(B.FabGpuError, match="CouchDB"):
                    ctx.state_versions_update([((CC, "", b"_a"), (1, 0))], 3)
                ctx.state_versions_update([((CC, "", b"_a"), B.STATE_REMOVE), ((CC, "", b"b"), (1, 1))], 3)
                assert ctx.state_versions_info()[3] == 0
            blk, _ = _block(net, [rng_tx], seed=80 + h)
            ctx.validate_block(blk)
            assert ctx.validate_mvcc(0, h, [0]).tolist() == [want], h
    finally:
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions([], 0)


def _tx(rng, pool, vals):
    k = pool[int(rng.integers(0, len(pool)))]
    x = rng.random()
    if x < 0.3:
        return [dict(ns=CC, reads=[(k, (0, 1))])]
    writes = [(pool[int(rng.integers(0, len(pool)))], False, vals[int(rng.integers(0, len(vals)))]) for _ in range(int(rng.integers(1, 3)))]
    return [dict(ns=CC, reads=[(k, (0, 1))] if x < 0.6 else [], writes=writes)]


def test_three_slots_deep_with_the_mode_switched(ctx, net):
    """Generated blocks submitted three slots deep, the index installed; the mode is switched between blocks while other slots hold
    blocks in flight; each block's flags equal the oracle's for the mode set when its stage runs."""
    B = pkg().binding
    rng = np.random.default_rng(31)
    pool = ["k%d" % i for i in range(12)]
    vals = [b'{"a":1}', b'{"_id":1}', b'{"~version":2}', b"plain", b'["_id"]', b'{"_id":1,"n":1e10000}', b'{"b":{"_id":1}}']
    state = {(CC, "", k.encode()): (0, 1) for k in pool[:8]}
    ctx.state_versions_indexed(_entries(state), 1, capacity=64)
    S = pkg().binding.SLOTS
    n_blocks = 24
    seq = {}

    def make(b):
        txs = [_tx(rng, pool, vals) for _ in range(int(rng.integers(8, 20)))]
        blk, _ = _block(net, txs, seed=900 + b)
        seq[b] = txs
        ctx.validate_block_async(b % S, blk)
    try:
        for b in range(S):
            make(b)
        seen = {0: 0, 11: 0, 24: 0, 254: 0}
        for b in range(n_blocks):
            couch = (b // 3) % 2 == 0
            ctx.state_database(B.STATEDB_COUCHDB if couch else B.STATEDB_LEVELDB)
            txs = seq.pop(b)
            tv = ctx.validate_wait(b % S, len(txs) + 16)
            got = ctx.validate_mvcc(b % S, 1 + b, tv).tolist()
            exp, state, _ = co.validate(state, 1 + b, txs, tv.tolist(), couch=couch)
            assert got == exp, b
            for x in exp:
                seen[x] = seen.get(x, 0) + 1
            if b % 4 == 3:
                fix = [(key, (1 + b, 0)) for key, v in state.items() if v == mo.UNKNOWN]
                ctx.state_versions_update(fix, 2 + b)
                state.update(dict(fix))
            if b + S < n_blocks:
                make(b + S)
        assert seen[24] > 5 and seen[0] > 20, seen
    finally:
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions([], 0)


def test_install_refusals(ctx):
    B = pkg().binding
    key = lambda s: (CC, "", s)
    ctx.state_database(B.STATEDB_COUCHDB)
    try:
        for bad in (b"", b"_a", b"\xff", b"\xed\xa0\x80", b"\xc0\xaf"):
            with pytest.raises(B.FabGpuError, match="CouchDB"):
                ctx.state_versions([(key(bad), (1, 0))], 1)
        ctx.state_versions_indexed([(key(b"ok"), (1, 0)), ((CC, "coll", b"\xff" * 32), (1, 1))], 1)
        with pytest.raises(B.FabGpuError, match="CouchDB"):
            ctx.state_versions_update([(key(b"_x"), (1, 2))], 1)
        assert ctx.state_versions_info()[0] == 2 and ctx.state_index_info()[0] == 1
        with pytest.raises(B.FabGpuError):
            ctx.state_database(2)
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions_update([(key(b"_x"), (1, 2))], 1)
        assert ctx.state_versions_info()[0] == 3
    finally:
        ctx.state_database(B.STATEDB_LEVELDB)
        ctx.state_versions([], 0)
