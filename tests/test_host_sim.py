"""The verify algorithm the CUDA kernel runs (fabric-mod_b200/csrc/ecdsa_verify.cuh: fixed-base table, Booth
windows, complete Jacobian group law, inversion-free final check) compiled for the host and compared with the oracle.
Runs on the GPU-less build box; the PTX limb primitives themselves are covered by tests/test_gpu_*.py."""
import numpy as np
import pytest

from oracle import bccsp_sw as o
from oracle import fast
from tools import workload
from util import be32, from_be, hash_to_e32, hostsim_verify, pkg
import vectors

V_INVALID, V_VALID, V_OFFCURVE = 0, 1, 2
HOST_WIDTHS = (8, 8, 8)         # FAB_WG, FAB_WQ, FAB_WS of the host build (util.hostsim)
PRODUCT_WIDTHS = (22, 16, 8)    # the library's (binding.build_info, Context.small_table_info): the widths of the GPU tests' chain cases


@pytest.mark.parametrize("cached", [False, True, "ba", "small"])
def test_constructed_edge_cases(cached):
    b = pkg().binding
    for c in vectors.build():
        exp = vectors.expected_status(c)
        if c["expect"] is not None:
            assert exp == c["expect"], "oracle disagrees with the construction: " + c["name"]
        if len(c["sig"]) == 0:
            continue
        st, r, s = b.gate_signature(c["sig"])
        if st != o.VALID:
            assert st == exp, c["name"]
            continue
        out = hostsim_verify(be32(c["qx"] % (1 << 256)), be32(c["qy"] % (1 << 256)), hash_to_e32(c["digest"]),
                             np.frombuffer(r, np.uint8), np.frombuffer(s, np.uint8), cached=cached is True, ba=cached == "ba", small=cached == "small")[0]
        got = {V_VALID: o.VALID, V_INVALID: o.INVALID, V_OFFCURVE: o.ERR_OFF_CURVE}[int(out)]
        assert got == exp, c["name"]
    # the chain-collision cases of every order at the host build's widths, in one batch: this path's own order takes its doubling and
    # infinity branches at every reachable step, the other orders' cases are adversarial inputs all the same
    cases = vectors.chain_cases(*HOST_WIDTHS)
    exp = vectors.oracle_statuses(cases)
    out = hostsim_verify(*vectors.chain_soa(cases), cached=cached is True, ba=cached == "ba", small=cached == "small")
    bad = [c["name"] for c, e, g in zip(cases, exp, out) if g != (V_VALID if e == o.VALID else V_INVALID)]
    assert not bad, "%d of %d chain cases disagree with the oracle, e.g. %s" % (len(bad), len(cases), bad[:8])


_COVERAGE = [(HOST_WIDTHS, order) for order in vectors.CHAIN_ORDERS] + [(PRODUCT_WIDTHS, order) for order in vectors.CHAIN_ORDERS] + \
            [((8, 8, ws), "small") for ws in (5, 6, 7)]


def _chain_cases(widths):
    return vectors.chain_cases(*widths) if widths[2] == 8 else vectors.chain_cases(*widths, orders=("small",))


@pytest.mark.parametrize("widths,order", _COVERAGE, ids=["%d-%d-%d-%s" % (w + (order,)) for w, order in _COVERAGE])
def test_chain_cases_reach_every_exceptional_step(widths, order):
    """The chain-collision generator (vectors.chain_cases) against its scalar model (vectors.chain_events): every case takes exactly
    its intended branch under its own kernel's order, the cases reach every (step, kind) that order can reach at these widths, none
    collides inside the affine levels of the batch-affine kernels (where the per-signature fallback would run), and the oracle gives
    VALID for the doublings and mid-chain infinities, INVALID for the final infinities."""
    cases = [c for c in _chain_cases(widths) if c["order"] == order]
    for c in cases:
        assert vectors.chain_events(order, c["u1"], c["u2"], c["d"], widths) == [(c["step"], c["kind"])], c["name"]
        assert not [ev for ev in vectors.chain_events("ba", c["u1"], c["u2"], c["d"], widths) if ev[0][0] == "L"], c["name"]
    reached = {(c["step"], c["kind"]) for c in cases}
    assert len(reached) == len(cases) and reached == vectors.chain_steps(order, widths)
    assert {k for _, k in reached} == set(vectors.CHAIN_KINDS)
    st = vectors.oracle_statuses(cases)
    assert [int(s) for s in st] == [c["expect"] for c in cases]
    for kind in vectors.CHAIN_KINDS:                 # and the Python oracle agrees with its C restatement on these inputs
        c = next(c for c in cases if c["kind"] == kind)
        assert vectors.expected_status(c) == c["expect"], c["name"]


def test_chain_model_on_known_chains():
    """chain_events on chains worked out by hand at 8/8: u1 = 5, u2 = 1 meets the key's first window at the same point (dbl) in
    the key-table order and at the opposite point when the key is negated (final infinity); lanes and tail labels."""
    w = HOST_WIDTHS
    assert vectors.chain_events("jac", 5, 1, 5, w) == [("q0", "dbl")]
    assert vectors.chain_events("jac", 5, 1, N_ - 5, w) == [("q0", "final_inf")]
    assert vectors.chain_events("jac", 5, 1 + (1 << 8), N_ - 5, w) == [("q0", "opp")]       # window q1 follows: R = 256 Q
    assert vectors.chain_events("generic", 5, 1, 5, w) == [("g0", "dbl")]
    assert vectors.chain_events("small", 5, 1, 5, w) == [("q0", "dbl")]
    assert vectors.chain_events("small", 0x81, 0xFF, 0x81, w) == [("q0", "opp")]           # 0xFF recodes to -1 + 256
    # 8/8: windows 0..31 are G's, 32..63 the key's; lane 0 = g0 = 1, lane 1 = q1 (window 33) = 2^8 d = 1: the combine doubles
    assert vectors.chain_events("l2", 1, 1 << 8, pow(1 << 8, -1, N_), w) == [("c0.0", "dbl")]
    assert vectors.chain_events("ba", 3 << 24, 0, 1, w) == []                               # a G group never collides with its own windows
    assert vectors.chain_events("ba", 1, (N_ - 1), 1, w) == [("t0", "final_inf")]


N_ = vectors.N


def test_product_widths_are_the_librarys():
    b = pkg().binding
    assert b.build_info() + (b.Context.small_table_info()[0],) == PRODUCT_WIDTHS


def test_config1_1024_tuples():
    # BASELINE.json configs[0]: 1 024 synthetic tuples, K = 16 keys, all valid
    w = workload.Workload(1024, 16, seed=workload.DEFAULT_SEED, nthreads=4)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=4)
    assert (exp == o.VALID).all()
    out = hostsim_verify(w.qx(), w.qy(), w.digest, w.r, w.s)
    assert (out == V_VALID).all()


def test_tampered_matches_oracle_bit_for_bit():
    w = workload.Workload(768, 8, seed=7, nthreads=4)
    w.tamper_r(frac=0.25)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=4)
    out = hostsim_verify(w.qx(), w.qy(), w.digest, w.r, w.s)
    assert ((out == V_VALID) == (exp == o.VALID)).all()
    assert 100 < int((exp != o.VALID).sum()) < 300
    # the per-key-table path gives the same bits
    out_c = hostsim_verify(w.qx(), w.qy(), w.digest, w.r, w.s, cached=True)
    assert (out_c == out).all()
    # and so does the batch-affine accumulation with its shared inversions (groups of 64 with a ragged tail: 768 + 37)
    out_b = hostsim_verify(w.qx(), w.qy(), w.digest, w.r, w.s, ba=True)
    assert (out_b == out).all()
    # the small-table tier (signed windows, no doublings)
    out_s = hostsim_verify(w.qx(), w.qy(), w.digest, w.r, w.s, small=True)
    assert (out_s == out).all()
    k = 37
    out_b2 = hostsim_verify(w.qx()[:k], w.qy()[:k], w.digest[:k], w.r[:k], w.s[:k], ba=True)
    assert (out_b2 == out[:k]).all()


def test_field_inversion_by_division_steps():
    """fe_inv_safegcd (the shared inversion of the batch-affine levels) against the Fermat ladder and Python."""
    import ctypes
    from util import hostsim, from_be
    rng = np.random.default_rng(11)
    p = (1 << 256) - (1 << 224) + (1 << 192) + (1 << 96) - 1
    xs = [1, 2, p - 1, p - 2, (1 << 255), 3] + [int.from_bytes(rng.bytes(32), "big") % (p - 1) + 1 for _ in range(60)]
    a = np.concatenate([be32(x) for x in xs])
    outs = []
    for op in (4, 8):
        out = np.zeros_like(a)
        hostsim().hostsim_fieldop(ctypes.c_int(op), a.ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(len(xs)),
                                  out.ctypes.data_as(ctypes.c_void_p))
        outs.append(out.reshape(-1, 32))
    assert (outs[0] == outs[1]).all()
    R = 1 << 256
    for x, o_ in zip(xs, outs[1]):          # Montgomery in / out: x = a R  ->  a^-1 R = R^2 / x
        assert from_be(o_) == (R * R * pow(x, -1, p)) % p


def test_small_table_signed_recoding_on_crafted_scalars():
    """k * Q through the small table (signed FAB_WS-bit windows; the host build uses the product's width) for scalars that stress the recoding: runs of ones (carry through every
    window), digits exactly at the sign boundary (32 / 33), the largest values below 2^256 (the last window absorbs the carry)."""
    import ctypes
    import random
    from oracle import p256
    from util import hostsim
    hs = hostsim()
    Q = p256.scalar_mult(0x1234567, (p256.GX, p256.GY))
    rng = random.Random(99)
    ks = [1, 2, 31, 32, 33, 63, 64, 65, (1 << 256) - 1, (1 << 256) - 2, p256.N - 1, p256.N, p256.N + 1, (1 << 255), (1 << 255) - 1,
          int("100000" * 43, 2) & ((1 << 256) - 1), int("100001" * 43, 2) & ((1 << 256) - 1), int("011111" * 43, 2) & ((1 << 256) - 1),
          int("111111" * 42, 2), 0,
          int("10000000" * 32, 2), int("10000001" * 32, 2), int("01111111" * 32, 2), int("11111111" * 31 + "11111110", 2), int("10000000" * 31 + "01111111", 2)]
    ks += [rng.getrandbits(256) for _ in range(12)]
    for k in ks:
        ox = (ctypes.c_uint8 * 32)(); oy = (ctypes.c_uint8 * 32)()
        hs.hostsim_small_mul(k.to_bytes(32, "big"), Q[0].to_bytes(32, "big"), Q[1].to_bytes(32, "big"), ox, oy)
        exp = p256.scalar_mult(k % p256.N, Q)
        got = (int.from_bytes(bytes(ox), "big"), int.from_bytes(bytes(oy), "big"))
        assert got == ((0, 0) if exp is p256.INF else exp), hex(k)


@pytest.mark.parametrize("ws", [5, 6, 7])
def test_small_tables_at_other_window_widths(ws):
    """The small-table code is width-generic (FAB_WS; the product builds 8): the host build at 5, 6 and 7 bits multiplies crafted scalars
    correctly (signed recoding with the carry absorbed by the last window) and verifies a tampered batch like the generic path."""
    import ctypes
    import os
    import subprocess
    from oracle import p256
    from util import ROOT
    d = os.path.join(ROOT, "tests", "host_sim")
    so = os.path.join(d, "libhostsim_ws%d.so" % ws)
    src = os.path.join(d, "hostsim.cpp")
    hdr = os.path.join(ROOT, "fabric-mod_b200", "csrc", "ecdsa_verify.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-DFAB_WG=8", "-DFAB_WQ=8", "-DFAB_Q_TWO_LEVEL=1", "-DFAB_WS=%d" % ws, "-shared", "-fPIC", "-o", so, src])
    hs = ctypes.CDLL(so)
    Q = p256.scalar_mult(0x7654321, (p256.GX, p256.GY))
    half, full = 1 << (ws - 1), 1 << ws
    nw = (257 + ws - 1) // ws
    pat = lambda digit: sum(digit << (ws * j) for j in range(nw)) & ((1 << 256) - 1)      # the same digit in every window
    ks = [1, half, half + 1, full - 1, full, pat(half), pat(half + 1), pat(half - 1), pat(full - 1), (1 << 256) - 1, p256.N - 1, p256.N + 1, 1 << 255]
    for k in ks:
        ox = (ctypes.c_uint8 * 32)(); oy = (ctypes.c_uint8 * 32)()
        hs.hostsim_small_mul(k.to_bytes(32, "big"), Q[0].to_bytes(32, "big"), Q[1].to_bytes(32, "big"), ox, oy)
        exp = p256.scalar_mult(k % p256.N, Q)
        assert (int.from_bytes(bytes(ox), "big"), int.from_bytes(bytes(oy), "big")) == ((0, 0) if exp is p256.INF else exp), (ws, hex(k))
    w = workload.Workload(256, 4, seed=70 + ws, nthreads=2)
    w.tamper_r(frac=0.25)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=2)
    arrs = [np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32) for a in (w.qx(), w.qy(), w.digest, w.r, w.s)]
    out = np.zeros(w.n, np.uint8)
    hs.hostsim_verify_batch_small(*[a.ctypes.data_as(ctypes.c_void_p) for a in arrs], ctypes.c_int(w.n), out.ctypes.data_as(ctypes.c_void_p))
    assert ((out == V_VALID) == (exp == o.VALID)).all() and 30 < int((exp != o.VALID).sum()) < 100
    # the small-table order's chain-collision cases at this width: a doubling or an infinity at every signed window
    cases = vectors.chain_cases(8, 8, ws, orders=("small",))
    exp = vectors.oracle_statuses(cases)
    arrs = vectors.chain_soa(cases)
    out = np.zeros(len(cases), np.uint8)
    hs.hostsim_verify_batch_small(*[a.ctypes.data_as(ctypes.c_void_p) for a in arrs], ctypes.c_int(len(cases)), out.ctypes.data_as(ctypes.c_void_p))
    bad = [c["name"] for c, e, g in zip(cases, exp, out) if g != (V_VALID if e == o.VALID else V_INVALID)]
    assert not bad, (ws, bad[:8])


def test_field_ops_match_python_integers():
    """Every op of the shared test table (fieldops.cuh) in the host build, against Python integers: the same op codes and expectations
    as tests/test_gpu_field.py, so the host and device hooks agree op for op."""
    import ctypes
    import random
    from util import field_op_cases, hostsim
    hs = hostsim()
    for op, (a, b, exp) in field_op_cases(random.Random(5), 200).items():
        A = np.stack([be32(x) for x in a]); B = np.stack([be32(x) for x in b])
        out = np.zeros_like(A)
        assert hs.hostsim_fieldop(ctypes.c_int(op), A.ctypes.data_as(ctypes.c_void_p), B.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(len(a)),
                                  out.ctypes.data_as(ctypes.c_void_p)) == 0
        assert [from_be(row) for row in out] == exp, op
    z = np.zeros((1, 32), np.uint8)
    for op in (-1, 17):
        assert hs.hostsim_fieldop(ctypes.c_int(op), z.ctypes.data_as(ctypes.c_void_p), z.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(1),
                                  z.ctypes.data_as(ctypes.c_void_p)) == -1
