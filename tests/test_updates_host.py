"""The update batch (updates.cuh) on the host build: the written-out cases against updates_oracle and the host build, seeded blocks with
values and metadata over a hot key pool, and an AddressSanitizer / UndefinedBehaviorSanitizer run over mutated read/write sets."""
import os
import random
import struct
import subprocess

import numpy as np
import pytest

from util import ROOT
import mvcc_oracle as mo
import updatecases
import updates_oracle as uo
import updatesutil
import wiremut


def _host(state0):
    versions, _ = updatecases.split(state0)
    s = updatesutil.HostUpdates()
    s.replace([(k, v) for k, v in sorted(versions.items())], 1)
    return s


@pytest.mark.parametrize("couch", [False, True], ids=["leveldb", "couchdb"])
@pytest.mark.parametrize("case", updatecases.cases(), ids=lambda c: c[0])
def test_case_oracle_and_host_build(case, couch):
    name, state0, steps = case
    versions, values = updatecases.split(state0)
    s = _host(state0)
    for k, step in enumerate(steps):
        txs, tv, want = step[:3]
        if couch and len(step) > 3:
            want = step[3]
        codes, new_versions, is_open = uo.flags(versions, 1 + k, txs, tv, couch)
        got = uo.batch(versions, values, 1 + k, txs, codes)
        assert got == want, (name, k)
        host_tv = uo.couch_flags(txs, tv) if couch else tv
        flags, recs, _ = s.updates(1 + k, txs, host_tv)
        assert flags == codes and recs == want, (name, k)
        if got is not None:
            values = uo.apply(values, got)
        versions = new_versions
        if is_open:
            s.update([], 2 + k)


def test_seeded_blocks_over_a_hot_key_pool():
    rng = np.random.default_rng(5)
    pool = ["k%d" % i for i in range(10)]
    versions = {(updatecases.CC, "", k.encode()): (0, i % 3) for i, k in enumerate(pool[:6])}
    values = {k: (b"c" + k[2], None) for k in versions}
    s = updatesutil.HostUpdates(seed=3)
    s.replace(sorted(versions.items()), 1)
    seen = {"complete": 0, "records": 0, "committed": 0, "inherited_md": 0}
    for b in range(1, 300):
        n = int(rng.integers(1, 14))
        txs = [updatesutil.random_tx(rng, pool, t) for t in range(n)]
        tv = [int(rng.choice([0, 0, 0, 0, 0, 10, 254] if b % 7 == 0 else [0, 0, 0, 0, 10])) for _ in range(n)]
        codes, versions2, is_open = uo.flags(versions, b, txs, tv)
        want = uo.batch(versions, values, b, txs, codes)
        flags, recs, counts = s.updates(b, txs, tv)
        assert flags == codes and recs == want, b
        if want is not None:
            seen["complete"] += 1; seen["records"] += len(want)
            seen["committed"] += sum(r[5] == uo.COMMITTED for r in want)
            seen["inherited_md"] += sum(isinstance(r[6], bytes) and r[1] == "put" for r in want)
            values = uo.apply(values, want)
        versions = versions2
        if is_open:
            s.update([], b + 1)
        if b % 50 == 0:                                              # a peer re-reads the unknown keys from its state database
            fix = [(k, (b, 0)) for k, v in versions.items() if v == mo.UNKNOWN]
            s.update(fix, b + 1)
            versions.update(dict(fix))
    assert seen["complete"] > 60 and seen["records"] > 150 and seen["committed"] > 15 and seen["inherited_md"] > 25, seen


def test_caps_smaller_than_the_batch():
    s = _host(updatecases.ST)
    txs = [updatecases.tx(writes=[("k%d" % t, b"v%d" % t)], md=[("k%d" % t, [("VALIDATION_PARAMETER", b"p")])]) for t in range(6)]
    _, full, counts = s.updates(1, txs, [0] * 6)
    s2 = _host(updatecases.ST)
    _, part, counts2 = s2.updates(1, txs, [0] * 6, rec_cap=2, meta_cap=5)
    assert counts == counts2 == (6, 6 * len(uo.serialize([("VALIDATION_PARAMETER", b"p")])))
    assert part is not None and len(part) == 2 and [r[:5] for r in part] == [r[:5] for r in full[:2]]


def _corpus(n_blocks=300, seed=9):
    r = random.Random(seed)
    rng = np.random.default_rng(seed)
    pool = ["k%d" % i for i in range(8)]
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    out, mutated = u32(n_blocks), 0
    for _ in range(n_blocks):
        n = r.randrange(1, 12)
        out += u32(n)
        for t in range(n):
            rw = uo.encode(updatesutil.random_tx(rng, pool, t))
            if r.random() < 0.5:
                rw = wiremut.mutate(r, r.choice([k for k in wiremut.KINDS if k != "chdr_int"]), "TxReadWriteSet", rw)
                mutated += 1
            out += u32(3 | r.choice((0, 0, 0, 0, 10)) << 8) + u32(len(rw)) + rw
    return out, mutated


def test_update_batch_under_sanitizers(tmp_path):
    exe = str(tmp_path / "updates_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-DUPDATES_MAIN", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-fno-omit-frame-pointer", "-o", exe, os.path.join(ROOT, "tests", "host_sim", "updates_host.cpp")])
    corpus, mutated = _corpus()
    assert mutated > 300
    path = tmp_path / "corpus.bin"
    path.write_bytes(corpus)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    run = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env, timeout=900)
    assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
    last = run.stdout.strip().split("\n")[-1].split()
    assert last[:3] == ["done", "300", "blocks,"] and int(last[3]) > 10, last
