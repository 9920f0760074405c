"""The update bytes (updatebytes.cuh) on the host build: the oracle against update_batch_bytes_test.go's three scenarios, the written-out
cases against the oracle and the host build, seeded blocks over a hot key pool with random namespaces, collections and key bytes, and
the same runs under AddressSanitizer / UndefinedBehaviorSanitizer."""
import ctypes
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from util import ROOT
from blockutil import _p
import mvcc_oracle as mo
import update_bytes_oracle as bo
import updatebytescases as cases
import updates_oracle as uo
import updatesutil
from update_bytes_oracle import kvwrite as K

SRC = os.path.join(ROOT, "tests", "host_sim", "update_bytes_host.cpp")
_LIB = None


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_ubytes_"), "libupdate_bytes_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, SRC])
        L = ctypes.CDLL(so)
        L.hs_new.restype = ctypes.c_void_p
        L.hs_new.argtypes = [ctypes.c_ulonglong]
        L.hs_free.argtypes = [ctypes.c_void_p]
        L.hs_apply.restype = ctypes.c_char_p
        L.hs_apply.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.c_size_t, ctypes.c_ulonglong, ctypes.c_size_t,
                                                                                           ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.hs_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.hs_update_bytes.restype = ctypes.c_char_p
        L.hs_update_bytes.argtypes = ([ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 2 + [ctypes.c_ulonglong]
                                      + [ctypes.c_void_p] * 2 + [ctypes.c_size_t] + [ctypes.c_void_p] * 2
                                      + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)])
        _LIB = L
    return _LIB


class HostBytes(updatesutil.HostUpdates):
    def __init__(self, seed=0x5EED):
        self.L = lib()
        self.h = ctypes.c_void_p(self.L.hs_new(seed))
        self.max_bytes = 0

    def update_bytes(self, block_num, txs, tv, committed, out_cap=1 << 22):
        """(flags, the bytes or None when incomplete, full length)"""
        blob, res, ht = updatesutil.block_of(txs)
        tv = np.ascontiguousarray(np.asarray(list(tv) or [0], np.uint8))
        flags = np.zeros(max(len(txs), 1), np.uint8)
        vals = [bytes(v) for v in committed]
        vb = np.frombuffer(b"".join(vals) + b"\x00", np.uint8).copy()
        vo = np.zeros(len(vals) + 1, np.uint32)
        vo[1:] = np.cumsum([len(v) for v in vals])
        out = np.zeros(max(out_cap, 1), np.uint8)
        n = ctypes.c_size_t(0)
        complete = ctypes.c_int(0)
        err = self.L.hs_update_bytes(self.h, _p(blob), blob.size, _p(res), _p(ht), block_num, _p(tv), _p(flags), len(txs), _p(vb), _p(vo), len(vals),
                                     _p(out), out_cap, ctypes.byref(n), ctypes.byref(complete))
        if err is not None:
            raise ValueError(err.decode())
        return flags[:len(txs)].tolist(), (out[:min(n.value, out_cap)].tobytes() if complete.value else None), n.value


# ---- the oracle against update_batch_bytes_test.go ---------------------------------------------------------------------------------
def _put(t, ns, key, value, coll=""):
    return (t, "put", ns, coll, key, value, None)


def _del(t, ns, key, coll=""):
    return (t, "del", ns, coll, key, None, None)


def test_oracle_only_public_writes():
    recs = [_put(1, "ns1", b"key1", b"value1"), _put(2, "ns1", b"key2", b"value2"), _put(3, "ns2", b"key3", b"value3"),
            _put(4, "ns3", b"key4", b"value4"), _put(5, "ns3", b"key5", b"value5"), _del(6, "ns3", b"key6")]
    want = [K(b"key1", b"value1", version=bo.height(1, 1), namespace="ns1"), K(b"key2", b"value2", version=bo.height(1, 2)),
            K(b"key3", b"value3", version=bo.height(1, 3), namespace="ns2"), K(b"key4", b"value4", version=bo.height(1, 4), namespace="ns3"),
            K(b"key5", b"value5", version=bo.height(1, 5)), K(b"key6", is_delete=True, version=bo.height(1, 6))]
    for order in (recs, recs[::-1]):
        assert bo.kvwrites(order, 1) == want
        assert bo.update_bytes(order, 1) == bo.marshal(want)
    # the first KVWrite by hand: 0a len (0a 03 "ns1" 1a 04 "key1" 2a 06 "value1" 32 04 01 01 01 01)
    body = b"\x0a\x03ns1\x1a\x04key1\x2a\x06value1\x32\x04\x01\x01\x01\x01"
    assert bo.update_bytes(recs, 1).startswith(b"\x0a" + bytes([len(body)]) + body)


def test_oracle_public_writes_and_collections():
    recs = [_put(1, "ns1", b"key1", b"value1"), _put(2, "ns1", b"key2", b"value2"), _put(3, "ns1", b"key3", b"value3", "coll1"),
            _put(4, "ns1", b"key4", b"value4", "coll1"), _put(5, "ns1", b"key5", b"value5", "coll2"), _del(6, "ns1", b"key6", "coll2"),
            _put(7, "ns2", b"key7", b"value7")]
    want = [K(b"key1", b"value1", version=bo.height(1, 1), namespace="ns1"), K(b"key2", b"value2", version=bo.height(1, 2)),
            K(b"key3", b"value3", version=bo.height(1, 3), collection="coll1"), K(b"key4", b"value4", version=bo.height(1, 4)),
            K(b"key5", b"value5", version=bo.height(1, 5), collection="coll2"), K(b"key6", is_delete=True, version=bo.height(1, 6)),
            K(b"key7", b"value7", version=bo.height(1, 7), namespace="ns2")]
    for order in (recs, recs[::-1]):
        assert bo.kvwrites(order, 1) == want
        assert bo.update_bytes(order, 1) == bo.marshal(want)


def test_oracle_only_channel_config():
    assert bo.update_bytes([_put(1, "", b"resourcesconfigtx.CHANNEL_CONFIG_KEY", b"value1")], 1) == b""
    assert bo.update_bytes([], 1) == b""


def test_oracle_height_and_commit_hash():
    assert bo.order_preserving(0) == b"\x00" and bo.order_preserving(256) == b"\x02\x01\x00" and bo.height(1, 300) == b"\x01\x01\x02\x01\x2c"
    import hashlib
    assert bo.commit_hash(b"\x00\x0b", b"xy", b"p") == hashlib.sha256(b"\x02\x00\x0bxyp").digest()


# ---- the host build ------------------------------------------------------------------------------------------------------------------
def _host(state0, height):
    versions, _ = cases.split(state0)
    s = HostBytes()
    s.replace([(k, v) for k, v in sorted(versions.items())], height, hint=64)
    return s


@pytest.mark.parametrize("couch", [False, True], ids=["leveldb", "couchdb"])
@pytest.mark.parametrize("case", cases.cases(), ids=lambda c: c[0])
def test_case_oracle_and_host_build(case, couch):
    name, block_num, state0, txs, tv, want = case[:6]
    if couch and len(case) > 6:
        want = case[6]
    versions, values = cases.split(state0)
    codes, _, _ = uo.flags(versions, block_num, txs, tv, couch)
    recs = uo.batch(versions, values, block_num, txs, codes)
    committed = bo.committed_values(recs, values)
    got = bo.update_bytes(recs, block_num, committed)
    if want is None:
        assert got is None, name
    else:
        assert bo.kvwrites(recs, block_num, committed) == want, name
        assert got == bo.marshal(want), name
    s = _host(state0, block_num)
    host_tv = uo.couch_flags(txs, tv) if couch else tv
    flags, dev, n = s.update_bytes(block_num, txs, host_tv, committed)
    assert flags == codes and dev == got, name
    if got is not None and len(got) > 10:                            # a short buffer: the full length, the first bytes
        s2 = _host(state0, block_num)
        _, part, n2 = s2.update_bytes(block_num, txs, host_tv, committed, out_cap=7)
        assert n2 == len(got) and part == got[:7]


def test_refusal_of_a_wrong_value_count():
    s = _host(cases.ST, 1)
    with pytest.raises(ValueError, match="n_val"):
        s.update_bytes(1, [cases.tx(cases.ns(cases.CC, md=[("a", cases.E1)]))], [0], [])


def _seeded(n_blocks, seed, versions, values, fix=True):
    """per block (block_num, txs, tv, flags, records, committed values, bytes, open, fixes), the oracle's state carried from block to
    block; fixes: the unknown keys a peer re-reads from its state database after the block (every 50th, with fix)"""
    rng = np.random.default_rng(seed)
    pool = ["k%d" % i for i in range(10)]
    for b in range(1, n_blocks + 1):
        n = int(rng.integers(1, 14))
        txs = [cases.random_tx(rng, pool, t) for t in range(n)]
        tv = [int(rng.choice([0, 0, 0, 0, 0, 10, 254] if b % 7 == 0 else [0, 0, 0, 0, 10])) for _ in range(n)]
        codes, versions2, is_open = uo.flags(versions, b, txs, tv)
        recs = uo.batch(versions, values, b, txs, codes)
        committed = bo.committed_values(recs, values)
        want = bo.update_bytes(recs, b, committed)
        if recs is not None:
            values = uo.apply(values, recs)
        versions = versions2
        fixes = [(k, (b, 0)) for k, v in versions.items() if v == mo.UNKNOWN] if fix and b % 50 == 0 else []
        versions.update(dict(fixes))
        values.update({k: (b"read%d" % b, None) for k, _ in fixes})    # what the peer reads with the version
        yield b, txs, tv, codes, recs, committed, want, is_open, fixes


def _state0():
    versions = {(ns, "", ("k%d" % i).encode()): (0, i % 3) for ns in cases.NSS[:2] for i in range(6)}
    return versions, {k: (b"c" + k[2], None) for k in versions}


def test_seeded_blocks_over_a_hot_key_pool():
    versions, values = _state0()
    s = HostBytes(seed=3)
    s.replace(sorted(versions.items()), 1)
    seen = {"complete": 0, "bytes": 0, "committed": 0, "multi_ns": 0, "colls": 0}
    for b, txs, tv, codes, recs, committed, want, is_open, fixes in _seeded(300, 5, versions, values):
        flags, got, _ = s.update_bytes(b, txs, tv, committed)
        assert flags == codes and got == want, b
        if want is not None:
            seen["complete"] += 1; seen["bytes"] += len(want); seen["committed"] += len(committed)
            seen["multi_ns"] += len({r[2] for r in recs}) > 1
            seen["colls"] += any(r[3] for r in recs)
        if is_open:
            s.update([], b + 1)
        if fixes:
            s.update(fixes, b + 1)
    assert seen["complete"] > 60 and seen["committed"] > 15 and seen["multi_ns"] > 15 and seen["colls"] > 10, seen


def _corpus_block(block_num, txs, tv, committed):
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    out = u32(block_num) + u32(block_num >> 32) + u32(len(txs))
    for t, tx in enumerate(txs):
        rw = uo.encode(tx)
        out += u32(3 | tv[t] << 8) + u32(len(rw)) + rw
    return out + u32(len(committed)) + b"".join(u32(len(v)) for v in committed) + b"".join(bytes(v) for v in committed)


def test_the_same_runs_under_sanitizers(tmp_path):
    """the cases that start from an empty state (LevelDB) and 300 seeded blocks from an empty table, in a program built with ASan and
    UBSan: the oracle's bytes"""
    exe = str(tmp_path / "update_bytes_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-DUPDATE_BYTES_MAIN", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-fno-omit-frame-pointer", "-o", exe, SRC])
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    runs = []
    for name, block_num, state0, txs, tv, _want in [c[:6] for c in cases.cases() if not c[2]]:
        codes, _, _ = uo.flags({}, block_num, txs, tv)
        recs = uo.batch({}, {}, block_num, txs, codes)
        runs.append((name, [(block_num, txs, tv, [], bo.update_bytes(recs, block_num, []))]))
    seq = [(b, txs, tv, committed, want) for b, txs, tv, _c, _r, committed, want, _o, _f in _seeded(300, 9, {}, {}, fix=False)]
    runs.append(("seeded", seq))
    complete = 0
    for name, blocks in runs:
        path = tmp_path / ("%s.bin" % name)
        path.write_bytes(struct.pack("<I", len(blocks)) + b"".join(_corpus_block(b, txs, tv, c) for b, txs, tv, c, _ in blocks))
        run = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env, timeout=900)
        assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
        lines = run.stdout.strip().split("\n")
        assert len(lines) == len(blocks), (name, run.stdout[-2000:])
        for i, (line, (b, _, _, _, want)) in enumerate(zip(lines, blocks)):
            f = line.split(" ")
            assert f[:4] in (["block", str(i), "complete", "1"], ["block", str(i), "complete", "0"]), line[:200]
            got = bytes.fromhex(f[4]) if f[3] == "1" else None
            assert got == want, (name, b)
            complete += want is not None
    assert complete > 20
