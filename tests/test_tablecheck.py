"""The table checker (tests/tablecheck.py) on host-built tables: it accepts what the table builders of ecdsa_verify.cuh make, and
it names exactly the entries of a corrupted copy -- what lets tests/test_gpu_table_contents.py vouch for the device-built tables."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import p256
from util import ROOT, hostsim
import tablecheck as tc

P = p256.P
G = (p256.GX, p256.GY)
W, WINDOWS = 8, 32                 # the host build's generator table (tests/util.py: FAB_WG=8, the same two-level builder)
WS, SWINDOWS = 8, 33               # small tables: signed 8-bit windows


def _gtable():
    p = ctypes.POINTER(ctypes.c_uint8)()
    n = hostsim().hostsim_gtable(ctypes.byref(p))
    return ctypes.string_at(p, n)


@pytest.fixture(scope="module")
def small_table(tmp_path_factory):
    """q -> the host build's small table of key q (tests/host_sim/smalltable_host.cpp, compiled outside the source tree)."""
    so = str(tmp_path_factory.mktemp("smalltable") / "libsmalltable_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host_sim", "smalltable_host.cpp")])
    lib = ctypes.CDLL(so)
    assert lib.host_small_window_bits() == WS

    def build(q):
        out = np.zeros(SWINDOWS * (1 << (WS - 1)) * 64, np.uint8)
        a = [np.frombuffer(int(v).to_bytes(32, "big"), np.uint8).copy() for v in q]
        lib.host_small_table(*[x.ctypes.data_as(ctypes.c_void_p) for x in a], out.ctypes.data_as(ctypes.c_void_p))
        return out.tobytes()
    return build


def _key_with_small_mont_x():
    """A curve point whose x, in Montgomery form, is below 2^256 - p: the only kind of entry that can be stored as x + p."""
    rinv = pow(1 << 256, -1, P)
    for s in range(1, 1000):
        x = s * rinv % P
        rhs = (x * x * x - 3 * x + p256.B) % P
        y = pow(rhs, (P + 1) // 4, P)
        if y * y % P == rhs:
            return x, y
    raise AssertionError("no such key")


def _coords(rows, i):
    o = 64 * i
    return int.from_bytes(rows[o:o + 32], "little"), int.from_bytes(rows[o + 32:o + 64], "little")


def _put(rows, i, X, Y):
    rows[64 * i:64 * i + 64] = X.to_bytes(32, "little") + Y.to_bytes(32, "little")


def _corrupt(rows, per, kind, j, d):
    """A copy of rows with entry (j, d) corrupted as `kind`; returns (copy, the entries that are now wrong)."""
    rows = bytearray(rows)
    i = j * per + d - 1
    X, Y = _coords(rows, i)
    if kind == "limb":
        rows[64 * i + 32 + 4 * 5] ^= 0x10
        return bytes(rows), [(j, d)]
    if kind == "neg_y":
        _put(rows, i, X, P - Y)
        return bytes(rows), [(j, d)]
    if kind == "unreduced":
        assert X + P < 1 << 256
        _put(rows, i, X + P, Y)
        return bytes(rows), [(j, d)]
    if kind == "swap":
        rows[64 * i:64 * i + 128] = rows[64 * i + 64:64 * i + 128] + rows[64 * i:64 * i + 64]
        return bytes(rows), [(j, d), (j, d + 1)]
    if kind == "segment":                                   # 32 entries normalised with the same wrong Z: (x, y) -> (x l^2, y l^3)
        lam = 0x1234567
        for k in range(32):
            Xk, Yk = _coords(rows, i + k)
            _put(rows, i + k, Xk * lam * lam % P, Yk * lam * lam * lam % P)
        return bytes(rows), [(j, d + k) for k in range(32)]
    raise ValueError(kind)


def test_checker_accepts_the_host_built_tables(small_table):
    assert tc.check_table(_gtable(), W, False, G, top=tc.top_digit(W, WINDOWS)) == []
    for q in (G, _key_with_small_mont_x(), p256.scalar_mult(p256.N - 1, G), p256.scalar_mult(1 << 200, G)):
        assert tc.check_table(small_table(q), WS, True, q) == []


# (kind, window, digit): a limb of the last entry, the doubling at d = 2, a pair across a chunk / low-high boundary of the two-level
# builder (d = 64, 65) and across a 32-entry segment of the small builder (d = 32, 33), a segment at the end of a window
GTABLE_CASES = [("limb", 5, 77), ("limb", 31, 255), ("neg_y", 0, 2), ("neg_y", 17, 1), ("swap", 3, 64), ("swap", 8, 15),
                ("segment", 9, 33), ("segment", 30, 224)]
SMALL_CASES = [("unreduced", 0, 1), ("limb", 32, 128), ("neg_y", 0, 2), ("neg_y", 4, 128), ("swap", 7, 32), ("segment", 20, 97),
               ("segment", 0, 1)]


@pytest.mark.parametrize("kind,j,d", GTABLE_CASES)
def test_checker_names_exactly_the_corrupted_generator_entries(kind, j, d):
    rows, want = _corrupt(_gtable(), (1 << W) - 1, kind, j, d)
    assert tc.check_table(rows, W, False, G, top=tc.top_digit(W, WINDOWS)) == want


@pytest.mark.parametrize("kind,j,d", SMALL_CASES)
def test_checker_names_exactly_the_corrupted_small_table_entries(small_table, kind, j, d):
    q = _key_with_small_mont_x()
    rows, want = _corrupt(small_table(q), 1 << (WS - 1), kind, j, d)
    assert tc.check_table(rows, WS, True, q) == want


def test_off_curve_key_is_exactly_the_zero_marker(small_table):
    bad = (G[0], G[1] ^ 1)
    rows = small_table(bad)
    assert rows[:64] == bytes(64)
    assert tc.check_table(rows, WS, True, bad) == []
    assert tc.check_table(small_table(G), WS, True, bad) == [(0, 1)]          # a table where the marker should be
    assert tc.check_table(rows, WS, True, G) != []                              # the marker where a table should be


def _seam_runs(rows, per, bases):
    runs = []
    for j in range(len(bases)):
        for a, b in tc.seam_spans(W, per, chunk=16):
            runs.append((j, a, rows[64 * (j * per + a - 1):64 * (j * per + b)], bases[j], False))
    return runs


def test_seam_pairs_name_the_corrupted_entry():
    """Pairs read at the seams only (the start of each pair unchecked, as for the device generator table): clean pairs pass, and a wrong
    entry in a pair is named alone once the pair's start has been computed."""
    per = (1 << W) - 1
    bases = tc.window_bases(G, W, WINDOWS)
    spans = tc.seam_spans(W, per, chunk=16)
    assert spans[:3] == [(1, 1), (14, 17), (30, 33)] and spans[-1] == (254, 255)
    assert tc.check_runs(_seam_runs(_gtable(), per, bases)) == []
    for kind, j, d in (("limb", 2, 16), ("neg_y", 6, 17), ("swap", 11, 32), ("limb", 31, 255), ("neg_y", 9, 1)):
        rows, want = _corrupt(_gtable(), per, kind, j, d)
        assert tc.check_runs(_seam_runs(rows, per, bases)) == want, (kind, j, d)
