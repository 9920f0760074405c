"""Constructed edge-case inputs (SURVEY.md A.5 checklist) shared by the host-sim and GPU parity tests.

Each case is (name, qx, qy, digest: bytes, sig_der: bytes); the expected outcome is whatever the oracle says
(oracle.bccsp_sw.status) -- the cases are built so that the interesting branch is taken, and most also carry an
`expect` hint that the tests assert against the oracle itself (guards against a vacuous construction)."""
import functools
import hashlib
import random

from oracle import bccsp_sw as o
from oracle import goasn1, p256

G = (p256.GX, p256.GY)
N, P = p256.N, p256.P


def _inv(a):
    return pow(a, -1, N)


def _e_bytes(e):
    return (e % N).to_bytes(32, "big")


def build():
    cases = []

    def add(name, q, digest, r, s, expect=None, sig=None):
        cases.append(dict(name=name, qx=q[0], qy=q[1], digest=digest, sig=sig if sig is not None else goasn1.marshal_ecdsa_signature(r, s),
                          expect=expect))

    d = 0xC0FFEE1234567890ABCDEF
    Q = p256.scalar_mult(d, G)
    dg = hashlib.sha256(b"fabric").digest()
    r, s = p256.ecdsa_sign_lows(d, dg, 0x1111222233334444)
    add("plain_valid", Q, dg, r, s, o.VALID)
    add("wrong_digest", Q, hashlib.sha256(b"fabrik").digest(), r, s, o.INVALID)
    add("wrong_key", p256.scalar_mult(d + 1, G), dg, r, s, o.INVALID)
    add("high_s", Q, dg, r, N - s, o.ERR_HIGH_S)
    add("r_zero", Q, dg, 0, s, o.ERR_R_NOT_POSITIVE)
    add("s_zero", Q, dg, r, 0, o.ERR_S_NOT_POSITIVE)
    add("r_negative", Q, dg, -r, s, o.ERR_R_NOT_POSITIVE)
    add("r_eq_n", Q, dg, N, s, o.INVALID)
    add("r_eq_n_minus_1", Q, dg, N - 1, s, o.INVALID)
    add("r_plus_n", Q, dg, r + N, s, o.INVALID)            # > 2^256 or >= n: never valid
    add("r_huge", Q, dg, (1 << 300) + r, s, o.INVALID)
    add("s_eq_1", Q, dg, r, 1, o.INVALID)
    add("r_eq_1", Q, dg, 1, s, o.INVALID)

    # digest extremes: e = 0, e = 2^256-1 (>= n, not reduced before use), short digest, long digest
    for name, dgx in (("e_zero", b"\x00" * 32), ("e_all_ones", b"\xff" * 32), ("e_short", b"hello world"), ("e_long", b"\xa5" * 48)):
        rr, ss = p256.ecdsa_sign_lows(d, dgx, 0x5555AAAA5555)
        add(name, Q, dgx, rr, ss, o.VALID)
    # e == n exactly -> u1 = 0 -> result is u2*Q alone
    rr, ss = p256.ecdsa_sign_lows(d, N.to_bytes(32, "big"), 0x77778888)
    add("e_eq_n_u1_zero", Q, N.to_bytes(32, "big"), rr, ss, o.VALID)

    # s == floor(n/2) exactly (allowed) : choose k, r, then e = s*k - r*d
    k = 0xDEADBEEF0001
    rr = p256.scalar_mult(k, G)[0] % N
    ss = p256.HALF_N
    add("s_eq_half_n", Q, _e_bytes(ss * k - rr * d), rr, ss, o.VALID)
    add("s_eq_half_n_plus_1", Q, _e_bytes(ss * k - rr * d), rr, ss + 1, o.ERR_HIGH_S)

    # u1*G == u2*Q  (final addition is a doubling) with u1 = 5 (a single fixed-base window) and R = 10*G
    R10 = p256.scalar_mult(10, G)
    rr = R10[0] % N
    ss = 0x123456789ABCDEF
    u2 = rr * _inv(ss) % N
    dq = 5 * _inv(u2) % N
    Qd = p256.scalar_mult(dq, G)
    add("u1G_eq_u2Q_doubling", Qd, _e_bytes(5 * ss), rr, ss, o.VALID)
    # u1*G == -u2*Q -> infinity -> invalid
    add("u1G_eq_neg_u2Q_infinity", p256.point_neg(Qd), _e_bytes(5 * ss), rr, ss, o.INVALID)
    # same construction with a multi-window u1 (doubling met at the last window only if partial sums collide: generic path)
    u1 = 0x0102030405060708090A0B0C0D0E0F101112131415161718191A1B1C1D1E1F20 % N
    R2 = p256.scalar_mult(2 * u1 % N, G)
    rr2 = R2[0] % N
    u2b = rr2 * _inv(ss) % N
    Qe = p256.scalar_mult(u1 * _inv(u2b) % N, G)
    add("u1G_eq_u2Q_wide", Qe, _e_bytes(u1 * ss), rr2, ss, o.VALID)
    add("u1G_eq_neg_u2Q_wide", p256.point_neg(Qe), _e_bytes(u1 * ss), rr2, ss, o.INVALID)

    # x(R) >= n : the "r + n < p" second candidate (SURVEY A.5 item 8).  Find a curve point with x = n + t.
    t = 1
    while True:
        x = N + t
        y2 = (x * x * x - 3 * x + p256.B) % P
        y = pow(y2, (P + 1) // 4, P)
        if y * y % P == y2:
            break
        t += 1
    Rbig = (x, y)
    rr = t                                         # x mod n
    ss = 0x0BADC0DE0BADC0DE
    e_int = 0x1234567890ABCDEF1234567890ABCDEF
    u1 = e_int * _inv(ss) % N
    u2 = rr * _inv(ss) % N
    Qx = p256.scalar_mult(_inv(u2), p256.point_add(Rbig, p256.point_neg(p256.scalar_mult(u1, G))))
    add("x_ge_n_second_candidate", Qx, _e_bytes(e_int), rr, ss, o.VALID)
    add("x_ge_n_wrong_r", Qx, _e_bytes(e_int), rr + 1, ss, o.INVALID)
    # small r (< p - n) whose point's x is r itself, not r + n: first candidate must still win
    k = 3
    while p256.scalar_mult(k, G)[0] >= (P - N):
        k += 1
        if k > 50:
            break
    # (no small-x multiple of G exists in practice; keep a random small r as an INVALID probe instead)
    add("small_r_invalid", Q, dg, 0x1234, s, o.INVALID)

    # off-curve / out-of-range public keys (outside the reference's defined behaviour -> ERR_OFF_CURVE)
    add("q_off_curve", (Q[0], (Q[1] + 1) % P), dg, r, s, o.ERR_OFF_CURVE)
    add("q_zero_zero", (0, 0), dg, r, s, o.ERR_OFF_CURVE)
    # Q == G and Q == -G
    rr, ss = p256.ecdsa_sign_lows(1, dg, 0x4242424242)
    add("q_eq_G", G, dg, rr, ss, o.VALID)
    add("q_eq_negG", p256.point_neg(G), dg, rr, ss, o.INVALID)
    # u2*Q where the Booth recoding hits digit 16 / -16 and zero windows: scalars with long runs
    for name, kk in (("k_runs_ones", (1 << 255) - 1), ("k_pow2", 1 << 200), ("k_alt", int("10" * 128, 2))):
        kk %= N
        rr = p256.scalar_mult(kk, G)[0] % N
        ss = 0x7777
        add("sig_" + name, Q, _e_bytes(ss * kk - rr * d), rr, ss, o.VALID)

    # malformed DER (reference bccsp/sw/impl_test.go:931-959) and Go's leniency
    for i, v in enumerate((bytes([0x30, 0x07, 0x02, 0x01, 0x8F, 0x02, 0x02, 0xFF, 0xF1]),
                           bytes([0x30, 0x07, 0x02, 0x01, 0x8F, 0x02, 0x02, 0x00, 0x01]),
                           bytes([0x30, 0x07, 0x02, 0x01, 0x8F, 0x02, 0x81, 0x01, 0x01]),
                           bytes([0x30, 0x07, 0x02, 0x01, 0x8F, 0x02, 0x81, 0x01, 0x8F]),
                           bytes([0x30, 0x0A, 0x02, 0x01, 0x8F, 0x02, 0x05, 0x00, 0x00, 0x00, 0x00, 0x8F]))):
        add("der_malformed_%d" % i, Q, dg, 0, 0, o.ERR_UNMARSHAL, sig=v)
    good = goasn1.marshal_ecdsa_signature(r, s)
    add("der_trailing_garbage", Q, dg, 0, 0, o.VALID, sig=good + b"\x00\x01\x02")
    inner = good[2:] + b"\x02\x01\x09"
    add("der_extra_field_in_seq", Q, dg, 0, 0, o.VALID, sig=b"\x30" + bytes([len(inner)]) + inner)
    add("der_truncated", Q, dg, 0, 0, o.ERR_UNMARSHAL, sig=good[:-1])
    add("der_sig_dropped_first_byte", Q, dg, 0, 0, o.ERR_UNMARSHAL, sig=good[1:])   # msp/msp_test.go:532-535
    add("der_long_form_len", Q, dg, 0, 0, o.ERR_UNMARSHAL, sig=b"\x30\x81" + good[1:])
    add("der_wrong_outer_tag", Q, dg, 0, 0, o.ERR_UNMARSHAL, sig=b"\x31" + good[1:])
    add("der_empty", Q, dg, 0, 0, o.ERR_EMPTY_SIG, sig=b"")
    return cases


def expected_status(case):
    return o.status(o.P256PublicKey(case["qx"], case["qy"]), case["sig"], case["digest"])


def oracle_statuses(cases):
    """expected_status of many cases at once, through the oracle's C restatement (oracle/fast.py)."""
    import numpy as np
    from oracle import fast
    keys = np.stack([np.frombuffer((c["qx"] % (1 << 256)).to_bytes(32, "big") + (c["qy"] % (1 << 256)).to_bytes(32, "big"), np.uint8)
                     for c in cases])
    digs, sigs = [c["digest"] for c in cases], [c["sig"] for c in cases]
    doff = np.zeros(len(cases) + 1, np.uint32); doff[1:] = np.cumsum([len(x) for x in digs])
    soff = np.zeros(len(cases) + 1, np.uint32); soff[1:] = np.cumsum([len(x) for x in sigs])
    return fast.verify_batch(keys, np.arange(len(cases), dtype=np.int32), np.frombuffer(b"".join(digs), np.uint8), doff,
                             np.frombuffer(b"".join(sigs), np.uint8), soff, nthreads=4)


# ---- chain-collision signatures -----------------------------------------------------------------------------------------------
# Every verify kernel computes R = u1 G + u2 Q as a chain of point additions, in its own order.  An addition whose addend equals
# the running sum ("dbl") or its negative ("opp": the sum becomes infinity and the next addition starts from there; "final_inf"
# when nothing follows, so R is infinity and the signature is INVALID) takes the exceptional branch of the complete group law,
# which honest traffic never reaches.  The cases below put exactly one such event at a chosen step of a chosen kernel's chain.
#
# Method: Q = d G with d known, so every table entry is a known multiple of G and every partial sum is a known scalar.  Draw the
# digits, solve one linear equation mod n for the remaining free quantity (u1, u2 or d), then R = (u1 + u2 d) G, r = x(R) mod n,
# s = r / u2, e = u1 s; draw again while r = 0 or s > n/2.  A final_inf case has R = infinity, so its r is x(2 A) for the last
# addend A: the value a kernel would accept had it doubled instead of returning infinity.
#
# Orders (the step labels of chain_events):
#   generic  signed 5-bit Booth windows of u2 Q (doublings in between), then the G windows ascending      "g<j>"
#   jac      the G windows ascending, then the key's unsigned windows ascending                          "g<j>", "q<k>"
#   small    the G windows ascending, then the key's signed windows (carry into the next) ascending      "g<j>", "q<k>"
#   l2, l4   lane l adds windows l, l + L, ... of [G windows] ++ [key windows] ("w<j>"), then the lanes' sums are combined
#            pairwise with jac_add: level v adds lane l + 2^v into lane l ("c<v>.<l>")
#   ba       the leaves [G windows, padded to 4] ++ [key windows, padded to 4] summed pairwise in two affine levels
#            ("L1.<k>", "L2.<k>"), then the level-2 sums added k = last ... 0 into a Jacobian accumulator ("t<k>")
# A prefix of the windows of one reduced scalar never equals +- its next window (a P = +-b P with 0 < a + b < n, a != b cannot hold in
# a group of prime order n), so the G windows of jac / small, the Booth part of generic, the key groups of the ba tail and both ba
# levels never collide: chain_steps lists what is left.
CHAIN_ORDERS = ("generic", "jac", "small", "ba", "l2", "l4")
CHAIN_KINDS = ("dbl", "opp", "final_inf")
CHAIN_D = 0x5EC0DE5EC0DE0123456789ABCDEF0FEDCBA9876543210F00DF00D       # the key of every order that solves for u1 or u2


def _nwin(bits, w):
    return (bits + w - 1) // w


def _layout(widths):
    """(G windows, key windows, signed small-table windows) at widths = (wg, wq, ws)."""
    wg, wq, ws = widths
    return _nwin(256, wg), _nwin(256, wq), _nwin(257, ws)


def _unsigned_digits(k, w, count):
    return [(k >> (w * j)) & ((1 << w) - 1) for j in range(count)]


def _signed_digits(k, w, count):
    """The recoding of add_small_table: digits in (-2^(w-1), 2^(w-1)], a negative digit carries one into the next window."""
    out, carry = [], 0
    for j in range(count):
        v = ((k >> (w * j)) & ((1 << w) - 1)) + carry
        carry = 1 if v > (1 << (w - 1)) else 0
        out.append(v - (carry << w))
    return out


def _value(digits, w):
    return sum(dg << (w * j) for j, dg in enumerate(digits))


def _chain(s, addends, events):
    """Adds (label, scalar) addends one by one to the running sum s (a scalar of G; 0 = infinity); zero addends are skipped digits."""
    for label, v in addends:
        s = _pair(s, v, label, events)
    return s


def _pair(a, b, label, events):
    a, b = a % N, b % N
    if a and b:
        if a == b:
            events.append((label, "dbl"))
        elif (a + b) % N == 0:
            events.append((label, "opp"))
    return (a + b) % N


def chain_events(order, u1, u2, d, widths):
    """Scalar model of one kernel's addition chain for R = u1 G + u2 (d G): the (step, kind) of every addition whose operands are
    equal or opposite, in chain order.  When R is infinity the last "opp" is reported as "final_inf"."""
    wg, wq, ws = widths
    gw, qw, sw = _layout(widths)
    g = [("g%d" % j, dg << (wg * j)) for j, dg in enumerate(_unsigned_digits(u1, wg, gw))]
    q = [("q%d" % k, (dg << (wq * k)) * d) for k, dg in enumerate(_unsigned_digits(u2, wq, qw))]
    ev = []
    if order == "generic":
        total = _chain(u2 * d, g, ev)          # the Booth part is one scalar's prefix chain: it never collides
    elif order == "jac":
        total = _chain(0, g + q, ev)
    elif order == "small":
        total = _chain(0, g + [("q%d" % k, dg * (1 << (ws * k)) * d) for k, dg in enumerate(_signed_digits(u2, ws, sw))], ev)
    elif order in ("l2", "l4"):
        lanes = int(order[1])
        wins = [("w%d" % j, v) for j, (_, v) in enumerate(g + q)]
        acc = [_chain(0, wins[l::lanes], ev) for l in range(lanes)]
        level, dist = 0, 1
        while dist < lanes:
            for l in range(0, lanes, 2 * dist):
                acc[l] = _pair(acc[l], acc[l + dist], "c%d.%d" % (level, l), ev)
            level, dist = level + 1, 2 * dist
        total = acc[0]
    elif order == "ba":
        leaves = [v for _, v in g] + [0] * (-gw % 4) + [v for _, v in q] + [0] * (-qw % 4)
        l1 = [_pair(leaves[2 * k], leaves[2 * k + 1], "L1.%d" % k, ev) for k in range(len(leaves) // 2)]
        l2 = [_pair(l1[2 * k], l1[2 * k + 1], "L2.%d" % k, ev) for k in range(len(l1) // 2)]
        total = _chain(0, [("t%d" % k, l2[k]) for k in reversed(range(len(l2)))], ev)
    else:
        raise ValueError(order)
    if total == 0:
        last = max(i for i, (_, kind) in enumerate(ev) if kind == "opp")
        ev[last] = (ev[last][0], "final_inf")
    return ev


def chain_steps(order, widths):
    """Every (step, kind) the order's chain can reach with reduced scalars: dbl and final_inf at every step that can collide, opp
    wherever another addition follows it."""
    gw, qw, sw = _layout(widths)

    def seq(labels):
        return {(s, k) for i, s in enumerate(labels) for k in CHAIN_KINDS if k != "opp" or i + 1 < len(labels)}
    if order == "generic":
        return seq(["g%d" % j for j in range(gw)])
    if order == "jac":
        return seq(["q%d" % k for k in range(qw)])
    if order == "small":
        return seq(["q%d" % k for k in range(sw)])
    if order == "ba":
        return seq(["t%d" % k for k in reversed(range(_nwin(gw, 4)))])
    lanes = int(order[1])
    # inside a lane every key window can meet its lane's sum; opp also at a lane's last window (the other lanes keep R finite) and
    # final_inf when every other lane is zero
    out = {("w%d" % j, k) for j in range(gw, gw + qw) for k in CHAIN_KINDS}
    levels = lanes.bit_length() - 1
    for v in range(levels):
        for l in range(0, lanes, 2 << v):
            out |= {("c%d.%d" % (v, l), k) for k in (("dbl", "final_inf") if v + 1 == levels else ("dbl", "opp"))}
    return out


_G2 = None


def _mul_g(k):
    """k G (affine, None for infinity) in Jacobian coordinates over a table of 2^i G: the oracle's affine ladder is ~20x slower."""
    global _G2
    if _G2 is None:
        _G2 = [G]
        for _ in range(255):
            _G2.append(p256.point_add(_G2[-1], _G2[-1]))
    k %= N
    X, Y, Z = 1, 1, 0
    for i in range(256):
        if not (k >> i) & 1:
            continue
        x2, y2 = _G2[i]
        if Z == 0:
            X, Y, Z = x2, y2, 1
            continue
        z1z1 = Z * Z % P
        h = (x2 * z1z1 - X) % P
        rr = (y2 * Z * z1z1 - Y) % P
        if h == 0:                              # sum of distinct powers of two below n: never, but stay exact
            return p256.scalar_mult(k, G)
        hh = h * h % P
        hhh, v = h * hh % P, X * hh % P
        X3 = (rr * rr - hhh - 2 * v) % P
        Y, X, Z = (rr * (v - X3) - Y * hhh) % P, X3, Z * h % P
    if Z == 0:
        return p256.INF
    zi = pow(Z, -1, P)
    return (X * zi * zi % P, Y * zi * zi * zi % P)


def _draw_unsigned(rng, w, count, target, zero_above):
    top = 256 - w * (count - 1)
    ds = [rng.randrange(1 << (w if i + 1 < count else top)) for i in range(count)]
    if target is not None:
        while ds[target] == 0:
            ds[target] = rng.randrange(1 << (w if target + 1 < count else top))
        if zero_above:
            ds[target + 1:] = [0] * (count - target - 1)
    return ds


def _draw_signed(rng, w, count, target, zero_above):
    half = 1 << (w - 1)
    top = min(half, 1 << (256 - w * (count - 1)))          # the last window holds the carry of bit 255
    ds = [rng.randrange(-half + 1, half + 1) for _ in range(count - 1)] + [rng.randrange(top + 1)]
    hi = top if target + 1 == count else half
    while ds[target] == 0 or (zero_above and ds[target] < 0):
        ds[target] = rng.randrange(-half + 1, hi + 1)
    if zero_above:
        ds[target + 1:] = [0] * (count - target - 1)
    return ds


def _solve(order, step, kind, widths, rng):
    """One draw: (u1, u2, d, A) with the event at `step`, A the scalar of the addend there; None when the draw is unusable."""
    wg, wq, ws = widths
    gw, qw, sw = _layout(widths)
    fin = kind == "final_inf"
    sign = 1 if kind == "dbl" else -1                      # the running sum equals sign * addend
    d = CHAIN_D
    if order == "generic":                                 # before G window j the sum is u2 d + alpha: solve for u2
        j = int(step[1:])
        dg = _draw_unsigned(rng, wg, gw, j, fin)
        u1, alpha, gamma = _value(dg, wg), _value(dg[:j], wg), dg[j] << (wg * j)
        u2 = (sign * gamma - alpha) * pow(d, -1, N) % N
        return u1, u2, d, gamma
    if order in ("jac", "small"):                          # before key window k the sum is u1 + beta d: solve for u1
        k = int(step[1:])
        if order == "jac":
            dg = _draw_unsigned(rng, wq, qw, k, fin)
            u2, beta, gamma = _value(dg, wq), _value(dg[:k], wq), dg[k] << (wq * k)
        else:
            dg = _draw_signed(rng, ws, sw, k, fin)
            u2, beta, gamma = _value(dg, ws), _value(dg[:k], ws), dg[k] << (ws * k)
        u1 = (sign * gamma - beta) * d % N
        return u1, u2, d, gamma * d
    if order == "ba":                                      # before G group k the sum is u2 d + alpha: solve for d
        k = int(step[1:])
        dg = _draw_unsigned(rng, wg, gw, None, False)
        grp = range(4 * k, min(4 * k + 4, gw))
        while not any(dg[i] for i in grp):
            dg = _draw_unsigned(rng, wg, gw, None, False)
        if fin:
            dg[:4 * k] = [0] * (4 * k)
        u1 = _value(dg, wg)
        alpha = _value(dg, wg) - _value(dg[:4 * k + 4], wg)
        gamma = _value(dg[:4 * k + 4], wg) - _value(dg[:4 * k], wg)
        u2 = rng.randrange(1, N)
        return u1, u2, (sign * gamma - alpha) * pow(u2, -1, N) % N, gamma
    lanes = int(order[1])
    dg = _draw_unsigned(rng, wg, gw, None, False)
    dq = _draw_unsigned(rng, wq, qw, None, False)
    if step[0] == "w":                                     # inside lane l before window j: a + b d = sign * gamma d, solve for d
        j = int(step[1:])
        l, kq = j % lanes, j - gw
        while dq[kq] == 0:
            dq[kq] = rng.randrange(1, 1 << wq)
        if fin:                                            # every other lane empty, nothing after j in this one
            dg = [x if i % lanes == l else 0 for i, x in enumerate(dg)]
            dq = [x if (gw + i) % lanes == l and gw + i <= j else 0 for i, x in enumerate(dq)]
        a = sum(x << (wg * i) for i, x in enumerate(dg) if i % lanes == l)
        b = sum(x << (wq * i) for i, x in enumerate(dq) if (gw + i) % lanes == l and gw + i < j)
        gamma = dq[kq] << (wq * kq)
        den = (sign * gamma - b) % N
        if den == 0:
            return None
        d = a * pow(den, -1, N) % N
        return _value(dg, wg), _value(dq, wq), d, gamma * d
    v, l = (int(x) for x in step[1:].split("."))           # combine: lanes [l, l + 2^v) against [l + 2^v, l + 2^(v+1))

    def part(lo, hi):
        a = sum(x << (wg * i) for i, x in enumerate(dg) if lo <= i % lanes < hi)
        b = sum(x << (wq * i) for i, x in enumerate(dq) if lo <= (gw + i) % lanes < hi)
        return a, b
    aL, bL = part(l, l + (1 << v))
    aR, bR = part(l + (1 << v), l + (2 << v))
    den = (bL - bR) % N if sign > 0 else (bL + bR) % N
    if den == 0:
        return None
    d = ((aR - aL) if sign > 0 else -(aL + aR)) * pow(den, -1, N) % N
    return _value(dg, wg), _value(dq, wq), d, aR + bR * d


def _chain_case(order, step, kind, widths):
    rng = random.Random("chain/%s/%s/%s/%d/%d/%d" % ((order, step, kind) + tuple(widths)))
    for _ in range(1000):
        got = _solve(order, step, kind, widths, rng)
        if got is None:
            continue
        u1, u2, d, addend = got
        if not (0 < u1 < N and 0 < u2 < N and 0 < d < N) or chain_events(order, u1, u2, d, widths) != [(step, kind)]:
            continue
        if kind == "final_inf":
            assert (u1 + u2 * d) % N == 0
            r = _mul_g(2 * addend)[0] % N
        else:
            R = _mul_g(u1 + u2 * d)
            if R is p256.INF:
                continue
            r = R[0] % N
        if r == 0:
            continue
        s = r * pow(u2, -1, N) % N
        if s > p256.HALF_N:
            continue
        e = u1 * s % N
        Q = _mul_g(d)
        return dict(name="chain_%s_%s_%s" % (order, step, kind), qx=Q[0], qy=Q[1], digest=e.to_bytes(32, "big"),
                    sig=goasn1.marshal_ecdsa_signature(r, s), expect=o.INVALID if kind == "final_inf" else o.VALID,
                    order=order, step=step, kind=kind, u1=u1, u2=u2, d=d, r=r, s=s, e=e)
    raise AssertionError("no chain case for %s %s %s at %s" % (order, step, kind, widths))


@functools.lru_cache(maxsize=None)
def chain_cases(wg, wq, ws, orders=CHAIN_ORDERS):
    """One signature per reachable (order, step, kind) of chain_steps at window widths (wg, wq, ws), in the case format of build()
    plus order / step / kind and the scalars u1, u2, d, r, s, e.  `expect` is the construction's claim; the status is the oracle's."""
    widths = (wg, wq, ws)
    out = []
    for order in orders:
        for step, kind in sorted(chain_steps(order, widths)):
            out.append(_chain_case(order, step, kind, widths))
    return tuple(out)


def chain_soa(cases):
    """The pre-gated form of chain cases: (qx, qy, e, r, s), uint8[n, 32] big-endian each."""
    import numpy as np
    return tuple(np.stack([np.frombuffer(c[f].to_bytes(32, "big"), np.uint8) for c in cases]) for f in ("qx", "qy", "e", "r", "s"))


def mix_with_workload(cases, stride=29, first=11, keys=16, seed=0xC4A1):
    """A pre-gated batch of honest workload signatures (5 % tampered r) with the cases at rows first, first + stride, ...: at every
    lane position of a warp, a few per 256-signature CTA, and a batch size that is not a multiple of 32.  Returns a dict: soa = (qx, qy, e, r, s),
    keys_xy (the workload's keys, then each distinct key of the cases), kidx (row -> key), valid (the oracle's verdicts), pos."""
    import numpy as np
    from oracle import fast
    from tools import workload
    m = len(cases)
    n = stride * m + 5
    n += 1 if n % 32 == 0 else 0
    w = workload.Workload(n - m, keys, seed=seed)
    w.tamper_r(0.05)
    pos = np.arange(m) * stride + first
    honest = np.setdiff1d(np.arange(n), pos)
    soa = []
    for hon, crafted in zip((w.qx(), w.qy(), w.digest, w.r, w.s), chain_soa(cases)):
        a = np.zeros((n, 32), np.uint8)
        a[honest] = np.asarray(hon, np.uint8).reshape(-1, 32)
        a[pos] = crafted
        soa.append(a)
    ckeys = list(dict.fromkeys((c["qx"], c["qy"]) for c in cases))
    keys_xy = np.concatenate([w.keys_xy, np.stack([np.frombuffer(x.to_bytes(32, "big") + y.to_bytes(32, "big"), np.uint8) for x, y in ckeys])])
    kidx = np.zeros(n, np.int32)
    kidx[honest] = w.key_idx
    kidx[pos] = [keys + ckeys.index((c["qx"], c["qy"])) for c in cases]
    valid = np.zeros(n, bool)
    valid[honest] = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8) == o.VALID
    valid[pos] = oracle_statuses(cases) == o.VALID
    return dict(soa=tuple(soa), keys_xy=keys_xy, kidx=kidx, valid=valid, pos=pos)
