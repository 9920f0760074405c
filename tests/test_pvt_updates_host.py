"""The private update batch (pvtupdates.cuh) on the host build: the written-out cases against pvt_updates_oracle and the host build,
seeded blocks over a hot pool of private keys with the private state carried from block to block, and an AddressSanitizer /
UndefinedBehaviorSanitizer run over private data mutated at every private level."""
import ctypes
import os
import random
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from tools import fabricpb as pb
from util import ROOT
from blockutil import _blob, _p
import mvccutil
import pvt_updates_oracle as puo
import pvtupdatecases as cases
import pvtutil
import updates_oracle as uo
import updatesutil
import wiremut

WORDS = 11
_LIB = None
SRC = os.path.join(ROOT, "tests", "host_sim", "pvt_updates_host.cpp")


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_pu_"), "libpvt_updates_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, SRC])
        L, U = ctypes.CDLL(so), updatesutil.lib()
        for name in ("hs_new", "hs_free", "hs_apply", "hs_info", "hs_lookup"):
            f, g = getattr(L, name), getattr(U, name)
            f.restype, f.argtypes = g.restype, g.argtypes
        L.pu_host.restype = ctypes.c_char_p
        L.pu_host.argtypes = ([ctypes.c_void_p] * 4 + [ctypes.c_ulonglong] + [ctypes.c_void_p] * 2 + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                              ctypes.c_void_p] + [ctypes.c_void_p] * 3 + [ctypes.c_size_t] + [ctypes.c_void_p] * 3 + [ctypes.c_size_t] + [ctypes.c_void_p] * 2)
        _LIB = L
    return _LIB


def decode(words, blob):
    ops = {1: "put", 2: "del", 3: "renew"}
    src = bytes(blob)
    return [(w[0], ops[w[1]], src[w[2]:w[2] + w[3]], src[w[4]:w[4] + w[5]], src[w[6]:w[6] + w[7]], src[w[8]:w[8] + w[9]] if w[1] == 1 else None,
             w[10] if w[1] == 3 else None) for w in np.asarray(words, np.uint32).reshape(-1, WORDS).tolist()]


class HostPvt(mvccutil.HostState):
    def __init__(self, seed=0x5EED):
        self.L = lib()
        self.h = ctypes.c_void_p(self.L.hs_new(seed))
        self.max_bytes = 0

    def run(self, block_num, txs, tv, rec_cap=4096):
        """(flags, verdict, status, records or None, full record count)"""
        blob, res, ht = pvtutil.block_of(cases.rwsets(txs))
        pvt = cases.pvt_of(txs)
        seqs = sorted(pvt)
        pb_, off = _blob([pvt[s] for s in seqs])
        sq = np.array(seqs or [0], np.uint32)
        tv = np.ascontiguousarray(np.asarray(list(tv) or [0], np.uint8))
        flags = np.zeros(max(len(txs), 1), np.uint8)
        hrec = np.zeros(4096 * updatesutil.WORDS, np.uint32)
        st = np.zeros(3 * max(len(seqs), 1), np.int32)
        out = np.zeros(4, np.int32)
        rec = np.zeros(max(rec_cap, 1) * WORDS, np.uint32)
        n_h, n = ctypes.c_size_t(0), ctypes.c_size_t(0)
        complete = ctypes.c_int(0)
        err = self.L.pu_host(self.h, _p(blob), _p(res), _p(ht), block_num, _p(tv), _p(flags), len(txs), _p(hrec), 4096, ctypes.byref(n_h), _p(pb_),
                             _p(off), _p(sq), len(seqs), _p(st), _p(out), _p(rec), rec_cap, ctypes.byref(n), ctypes.byref(complete))
        if err is not None:
            raise mvccutil.StateError(err.decode(), False)
        status = {s: tuple(int(x) for x in st[3 * i:3 * i + 3]) for i, s in enumerate(seqs)}
        recs = decode(rec[:min(n.value, rec_cap) * WORDS], pb_) if complete.value else None
        return flags[:len(txs)].tolist(), tuple(int(x) for x in out), status, recs, n.value


def _host(versions):
    s = HostPvt()
    s.replace(sorted(versions.items()), 1, hint=64)
    return s


@pytest.mark.parametrize("case", cases.cases(), ids=lambda c: c[0])
def test_case_oracle_and_host_build(case):
    name, committed, tv, txs, want = case
    codes, hashed, verdict, status, recs = cases.run_oracle(committed, 1, txs, tv)
    assert recs == want, name
    flags, hv, hs, got, _ = _host(committed[0]).run(1, txs, tv)
    assert (flags, hv, hs, got) == (codes, verdict, status, want), name


def test_short_record_buffer_reports_the_full_count():
    name, committed, tv, txs, want = cases.cases()[1]
    _, _, _, got, n = _host(committed[0]).run(1, txs, tv, rec_cap=1)
    assert n == len(want) == 2 and got == want[:1]


def test_seeded_blocks_over_a_hot_key_pool():
    """300 seeded blocks: every block's records equal the oracle's, and the private state carried by applying them (renew records
    resolved as the peer would) stays the oracle's"""
    s = _host({})
    versions, values, pstate = {}, {}, {}
    seen = {"put": 0, "del": 0, "renew": 0, "incomplete": 0}
    for b in range(300):
        txs, tv = cases.seeded(1000 + b, 8 + b % 13)
        pubs = [t["pub"] for t in txs]
        codes, new_versions, is_open = uo.flags(versions, 1 + b, pubs, tv)
        hashed = uo.batch(versions, values, 1 + b, pubs, codes)
        verdict, status, want = puo.batch(1 + b, codes, cases.rwsets(txs), cases.pvt_of(txs), hashed)
        flags, hv, hs, got, _ = s.run(1 + b, txs, tv)
        assert (flags, hv, hs, got) == (codes, verdict, status, want), b
        assert not is_open
        if want is None:
            seen["incomplete"] += 1
            pstate = {}                            # the peer builds this block's batch itself
        else:
            for r in want:
                seen[r[1]] += 1
            pstate = puo.apply(pstate, 1 + b, want, hashed, values)
        values = uo.apply(values, hashed) if hashed is not None else {}
        versions = new_versions
    assert seen["put"] > 500 and seen["del"] > 100 and seen["renew"] > 20 and 0 < seen["incomplete"] < 150, seen
    assert pstate


# ---- sanitizers ------------------------------------------------------------------------------------------------------------------
LEVELS = ("TxPvtReadWriteSet", "NsPvtReadWriteSet", "CollectionPvtReadWriteSet", "KVRWSet", "KVWrite", "KVMetadataWrite", "KVMetadataEntry")


def _corpus(n_blocks=200, seed=9):
    r = random.Random(seed)
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    lb = lambda b: u32(len(b)) + bytes(b)
    out, mutated = u32(n_blocks), 0
    for b in range(n_blocks):
        n = r.randrange(1, 8)
        txs, tv = cases.seeded(5000 + b, n, pool=4)
        pvt = {}
        for t, x in enumerate(txs):
            target = r.choice(LEVELS)
            kind = r.choice([k for k in wiremut.KINDS if k != "chdr_int"])

            def mut(part, v):
                nonlocal mutated
                if part == target and r.random() < 0.6:
                    mutated += 1
                    return wiremut.mutate(r, kind, part, v)
                return v
            ws = [pb.f_bytes(3, mut("KVWrite", pb.f_bytes(1, b"k%d" % r.randrange(4)) + pb.f_uint(2, int(r.random() < 0.2)) +
                                    pb.f_bytes(3, b"v%d" % r.randrange(9)))) for _ in range(r.randrange(0, 3))]
            me = mut("KVMetadataEntry", pb.f_bytes(1, b"VALIDATION_PARAMETER") + pb.f_bytes(2, b"ep"))
            ms = [pb.f_bytes(4, mut("KVMetadataWrite", pb.f_bytes(1, b"k%d" % r.randrange(4)) + pb.f_bytes(2, me)))] if r.random() < 0.5 else []
            rw = mut("KVRWSet", b"".join(ws + ms))
            coll = pb.f_bytes(2, mut("CollectionPvtReadWriteSet", pb.f_bytes(1, b"c1") + pb.f_bytes(2, rw)))
            pvt[t] = mut("TxPvtReadWriteSet", pb.f_bytes(2, mut("NsPvtReadWriteSet", pb.f_bytes(1, cases.CC.encode()) + coll)))
            if r.random() < 0.5:                   # half: the public hash is that of the mutated rwset, so the write walk is reached
                x["hashes"] = {(cases.CC, "c1"): puo.sha(rw)}
        rws = cases.rwsets(txs)
        out += u32(n) + b"".join(u32(3 | tv[t] << 8) + lb(rw) for t, rw in enumerate(rws))
        out += u32(len(pvt)) + b"".join(u32(sq) + lb(e) for sq, e in sorted(pvt.items()))
    return out, mutated


def test_pvt_updates_under_sanitizers(tmp_path):
    exe = str(tmp_path / "pu_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-DPU_MAIN", "-o", exe, SRC])
    corpus, mutated = _corpus()
    assert mutated > 150
    path = tmp_path / "corpus.bin"
    path.write_bytes(corpus)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    res = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env)
    assert res.returncode == 0, res.stderr[-4000:]
    lines = res.stdout.splitlines()
    assert len(lines) == 200 and not any(x.startswith("refused") for x in lines)
    complete = [x for x in lines if " complete 1 " in x]
    assert len(complete) > 20 and any(not x.endswith(" 0") for x in complete), lines[:20]
