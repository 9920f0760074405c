"""The range stage's byte code under AddressSanitizer and UndefinedBehaviorSanitizer: tests/host_sim/range_asan.cpp runs the scan, the
range parser, the written-key sort, the range records, the walk, the apply and the index maintenance over random blocks whose range
queries carry wire-level mutations (tests/wiremut.py) of the RangeQueryInfo and of every other level of the read/write set."""
import os
import random
import struct
import subprocess

import numpy as np

from util import ROOT
import range_oracle as ro
import rangeutil
import wiremut


def _corpus(n_blocks=300, seed=4):
    r = random.Random(seed)
    rng = np.random.default_rng(seed)
    pool = ["k%d" % i for i in range(10)]
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    lb = lambda b: u32(len(b)) + bytes(b)
    keys = [("mycc", "", k.encode()) for k in pool[:6]] + [("mycc", "c", b"h" + k.encode()) for k in pool[:3]]
    state = {k: (0, i % 3) for i, k in enumerate(keys)}
    out = u32(len(keys)) + b"".join(lb(a.encode()) + lb(c.encode()) + lb(k) + u32(0) + u32(0) + u32(i % 3) + u32(0)
                                    for i, (a, c, k) in enumerate(keys))
    out += u32(n_blocks)
    mutated = 0
    kinds = [k for k in wiremut.KINDS if k != "chdr_int"]
    for _ in range(n_blocks):
        n = r.randrange(1, 12)
        out += u32(n)
        for _ in range(n):
            tx = rangeutil.random_range_tx(rng, pool, state)
            tv = r.choice((0, 0, 0, 254, 10))
            if tx is None:
                out += u32(1 | tv << 8) + lb(b"")
                continue
            rw = ro.encode(tx)
            if tx[0].get("ranges") and r.random() < 0.7:
                info = ro.range_info(*tx[0]["ranges"][0])
                tx[0]["ranges"] = [wiremut.mutate(r, r.choice(kinds), "RangeQueryInfo", info)]
                rw = ro.encode(tx)
                mutated += 1
            elif r.random() < 0.2:
                rw = wiremut.mutate(r, r.choice(kinds), "TxReadWriteSet", rw)
                mutated += 1
            out += u32(3 | tv << 8) + lb(rw)
    return out, mutated


def test_range_stage_under_sanitizers(tmp_path):
    exe = str(tmp_path / "range_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-o", exe, os.path.join(ROOT, "tests", "host_sim", "range_asan.cpp")])
    corpus, mutated = _corpus()
    assert mutated > 300
    path = tmp_path / "corpus.bin"
    path.write_bytes(corpus)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    run = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env, timeout=900)
    assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
    last = run.stdout.split("\n")[-3].split()
    assert last[:2] == ["blocks", "300"], last
    assert int(last[5]) > 100 and int(last[7]) > 5 and int(last[9]) > 50, last      # VALID, 11 and 254 all reached
