"""The MVCC stage's byte code under AddressSanitizer and UndefinedBehaviorSanitizer: tests/host_sim/mvcc_asan.cpp runs the scan, the key
table, the walk and the apply over random blocks whose read/write sets carry wire-level mutations (tests/wiremut.py) -- of the Version
messages above all, and of every other level of the set."""
import os
import random
import struct
import subprocess

import numpy as np

from util import ROOT
import mvcc_oracle as mo
import mvccutil
import wiremut

LEVELS = ("Version", "Version", "Version", "KVRead", "KVReadHash", "KVRWSet", "HashedRWSet", "NsReadWriteSet", "TxReadWriteSet")


def _corpus(n_blocks=300, seed=3):
    r = random.Random(seed)
    rng = np.random.default_rng(seed)
    pool = ["k%d" % i for i in range(10)]
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    u64 = lambda v: struct.pack("<Q", v)
    lb = lambda b: u32(len(b)) + bytes(b)
    keys = [("mycc", "", k.encode()) for k in pool[:6]] + [("mycc", "c", b"h" + k.encode()) for k in pool[:3]]
    out = u32(len(keys)) + b"".join(lb(a.encode()) + lb(c.encode()) + lb(k) + u64(0) + u64(i % 3) for i, (a, c, k) in enumerate(keys))
    out += u32(n_blocks)
    mutated = 0
    for _ in range(n_blocks):
        n = r.randrange(1, 12)
        out += u32(n)
        for _ in range(n):
            tx = mvccutil.random_tx(rng, pool, unreached=0.02)
            tv = r.choice((0, 0, 0, 254, 10))
            if tx is None:
                out += u32(1 | tv << 8) + lb(b"")
                continue
            target = r.choice(LEVELS) if r.random() < 0.6 else None
            kind = r.choice([k for k in wiremut.KINDS if k != "chdr_int"])

            def mut(part, b):
                nonlocal target, mutated
                if part == target and r.random() < 0.5:
                    mutated += 1
                    return wiremut.mutate(r, kind, part, b)
                return b
            out += u32(3 | tv << 8) + lb(mo.encode(tx, mut))
    return out, mutated


def test_mvcc_stage_under_sanitizers(tmp_path):
    exe = str(tmp_path / "mvcc_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-o", exe, os.path.join(ROOT, "tests", "host_sim", "mvcc_asan.cpp")])
    corpus, mutated = _corpus()
    assert mutated > 300
    path = tmp_path / "corpus.bin"
    path.write_bytes(corpus)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    run = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env, timeout=900)
    assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
    last = run.stdout.split("\n")[-2].split()
    assert last[:2] == ["blocks", "300"], last
    assert int(last[5]) > 100 and int(last[7]) > 20 and int(last[9]) > 50, last      # VALID, 11 and 254 all reached
