"""The private-data check's byte code under AddressSanitizer and UndefinedBehaviorSanitizer: tests/host_sim/pvt_host.cpp runs the scan,
the public-hash lookup and the decode over blocks whose private data carries wire-level mutations (tests/wiremut.py) at every private
level -- half of them with the public hash recomputed from the mutated bytes, so that the decoder is reached -- and its output equals
pvt_oracle's."""
import os
import random
import struct
import subprocess

from tools import fabricpb as pb
from util import ROOT
import pvt_oracle as po
import pvtcases
import wiremut

# the private levels, outermost first; the rwset levels are those of a KVRWSet with every nested message
LEVELS = ("TxPvtReadWriteSet", "NsPvtReadWriteSet", "CollectionPvtReadWriteSet", "KVRWSet", "KVRead", "Version", "RangeQueryInfo",
          "QueryReads", "QueryReadsMerkleSummary", "KVWrite", "KVMetadataWrite", "KVMetadataEntry")


def _rwset(r, mut):
    """a KVRWSet with every nested level, each passed through mut(level, bytes)"""
    ver = lambda: mut("Version", pb.f_uint(1, r.randrange(1, 9)) + pb.f_uint(2, r.randrange(9)))
    read = lambda k: mut("KVRead", pb.f_bytes(1, k) + pb.f_bytes(2, ver()))
    raw = mut("QueryReads", pb.f_bytes(1, read(b"q1")) + pb.f_bytes(1, read(b"q2")))
    mk = mut("QueryReadsMerkleSummary", pb.f_uint(1, 4) + pb.f_uint(2, 2) + pb.f_bytes(3, bytes(32)))
    rq = mut("RangeQueryInfo", pb.f_bytes(1, b"a") + pb.f_bytes(2, b"z") + pb.f_uint(3, 1) + pb.f_bytes(4 if r.random() < 0.5 else 5, raw if r.random() < 0.5 else mk))
    w = mut("KVWrite", pb.f_bytes(1, b"k%d" % r.randrange(99)) + pb.f_uint(2, 0) + pb.f_bytes(3, r.randbytes(r.randrange(40))))
    me = mut("KVMetadataEntry", pb.f_bytes(1, b"VALIDATION_PARAMETER") + pb.f_bytes(2, b"ep"))
    md = mut("KVMetadataWrite", pb.f_bytes(1, b"m") + pb.f_bytes(2, me))
    return mut("KVRWSet", pb.f_bytes(1, read(b"r")) + pb.f_bytes(2, rq) + pb.f_bytes(3, w) + pb.f_bytes(4, md))


def _corpus(n_blocks=250, seed=4):
    r = random.Random(seed)
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    lb = lambda b: u32(len(b)) + bytes(b)
    out, blocks, mutated = u32(n_blocks), [], 0
    for _ in range(n_blocks):
        n = r.randrange(1, 10)
        txs, flags, pvt = [], [], {}
        for t in range(n):
            target = r.choice(LEVELS)
            kind = r.choice([k for k in wiremut.KINDS if k != "chdr_int"])

            def mut(part, b):
                nonlocal mutated
                if part == target and r.random() < 0.5:
                    mutated += 1
                    return wiremut.mutate(r, kind, part, b)
                return b
            colls = [("c%d" % k, _rwset(r, mut)) for k in range(r.randrange(1, 3))]
            honest = [("c%d" % k, _rwset(random.Random(t * 10 + k), lambda p, b: b)) for k in range(len(colls))]
            # half: the public hashes are those of the mutated bytes (the decoder is reached); else of unmutated ones
            src = colls if r.random() < 0.5 else honest
            txs.append([(pvtcases.CC, [(c, pvtcases.sha(rw)) for c, rw in src])])
            flags.append(r.choice((0, 0, 254, 11)))
            coll_msgs = b"".join(pb.f_bytes(2, mut("CollectionPvtReadWriteSet", pb.f_bytes(1, c.encode()) + pb.f_bytes(2, rw))) for c, rw in colls)
            pvt[t] = mut("TxPvtReadWriteSet", pb.f_bytes(2, mut("NsPvtReadWriteSet", pb.f_bytes(1, pvtcases.CC.encode()) + coll_msgs)))
        rwsets = pvtcases.rwsets_of(txs)
        out += u32(n) + b"".join(u32(3 | flags[t] << 8) + lb(rw) for t, rw in enumerate(rwsets))
        out += u32(len(pvt)) + b"".join(u32(s) + lb(e) for s, e in sorted(pvt.items()))
        blocks.append(po.validate(rwsets, flags, pvt))
    return out, blocks, mutated


def test_pvt_stage_under_sanitizers(tmp_path):
    exe = str(tmp_path / "pvt_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-DPV_ASAN_MAIN", "-o", exe, os.path.join(ROOT, "tests", "host_sim", "pvt_host.cpp")])
    corpus, blocks, mutated = _corpus()
    assert mutated > 300
    path = tmp_path / "corpus.bin"
    path.write_bytes(corpus)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    res = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env)
    assert res.returncode == 0, res.stderr[-4000:]
    lines = res.stdout.splitlines()
    assert len(lines) == len(blocks)
    codes = []
    for line, (verdict, status) in zip(lines, blocks):
        exp = list(verdict) + [x for s in sorted(status) for x in status[s]]
        assert [int(x) for x in line.split()] == exp
        codes += [s[0] for s in status.values()]
    assert all(codes.count(c) > 20 for c in (po.OK, po.MISMATCH, po.UNDET)), [codes.count(c) for c in (0, 1, 254)]
