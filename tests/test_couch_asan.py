"""CouchDB's value and key checks (couchval.cuh) under AddressSanitizer and UndefinedBehaviorSanitizer: tests/host_sim/couch_asan.cpp
scans mutated documents, every truncation of a set of documents, nesting at and past the scan's bound, and escape, backslash, string,
number and bracket runs straddling every lane chunk and tile boundary of the CTA scan -- each value in a buffer of exactly its length,
through both scans -- and both verdicts equal couch_oracle's."""
import os
import struct
import subprocess

import numpy as np

from util import ROOT
import couch_oracle as co
import couchutil


def _values():
    rng = np.random.default_rng(12)
    vals = couchutil.corpus(6, 20000)
    for d in [couchutil.document(rng) for _ in range(40)] + [b'{"_id":"a\\"b","n":1.7976931348623157e308,"\\u005fx":[1,{"y":null}]}']:
        vals += [d[:i] for i in range(len(d) + 1)]
    deep = lambda d, o, c: o * d + b"1" + c * d
    for d in (co.DEPTH - 1, co.DEPTH, co.DEPTH + 1, 3 * co.DEPTH):
        vals += [deep(d, b'{"k":', b"}"), deep(d, b"[", b"]"), deep(d, b'{"k":', b"}")[:-1], b'{"_id":1,"d":' + deep(d, b"[", b"]") + b"}"]
    for L in list(range(1, 200)) + [co.SHORT_MAX - k for k in range(-3, 40)]:
        for run in (b"\\" * 1, b"\\" * 2, b"\\" * 3, b"\\u00", b"\\u005f", b'\\"'):
            pad = max(0, L - 10)
            vals.append(b'{"s":"' + b"a" * pad + run + b'"}')
            vals.append(b'{"' + b"_" * (pad % 7) + run + b'":1}')
        vals.append(b'{"n":' + b"9" * max(1, L - 6) + b"}")
    for edge in (co.LANE_BYTES, 2 * co.LANE_BYTES, co.TILE_BYTES, 2 * co.TILE_BYTES):
        for off in range(-7, 8):
            pad = edge + off
            for run in (b"\\", b"\\\\", b"\\\\\\", b"\\u005f", b'\\"', b"\\u00"):
                vals.append(b'{"s":"' + b"a" * max(0, pad - 6) + run + b'x","_id":1}')
            vals.append(b'{"_id":1,"n":' + b"7" * max(1, pad - 13) + b"}")
            vals.append(b" " * max(0, pad - 1) + b'{"_b":[' + b"[" * 20 + b"]" * 20 + b"]}")
            vals.append(b'{"a":"' + b"q" * max(0, pad - 6) + b'"}')
    vals.append(b"")
    return vals


def test_values_under_sanitizers(tmp_path):
    exe = str(tmp_path / "couch_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-o", exe, os.path.join(ROOT, "tests", "host_sim", "couch_asan.cpp")])
    vals = _values()
    path = tmp_path / "values.bin"
    path.write_bytes(struct.pack("<I", len(vals)) + b"".join(struct.pack("<I", len(v)) + v for v in vals))
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    run = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env, timeout=900)
    assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
    lines = run.stdout.split("\n")[:-1]
    assert len(lines) == len(vals)
    got = [tuple(int(x) for x in ln.split()) for ln in lines]
    exp = [(co.value_bits(v), co.value_bits(v), int(co.key_ok(v))) for v in vals]
    bad = [(v, g, e) for v, g, e in zip(vals, got, exp) if g != e]
    assert not bad, bad[:5]
