"""Independent CPU check of a device point table, entry by entry, with Python integers and oracle/p256 only.

A table holds, per window j, the multiples d * 2^(w j) * Q for d = 1 .. per (per = 2^w - 1 for an unsigned table, 2^(w-1) for a
signed one), stored affine in Montgomery form: 64 bytes per entry, x then y, each 8 little-endian 32-bit limbs.  An entry is right
when its coordinates are reduced (< p, as the kernels assume), the point is on the curve, and
- entry (j, 1) equals 2^(w j) * Q (the anchor, from the oracle);
- entry (j, d) equals entry (j, d-1) + entry (j, 1), checked without an inversion: with D = x1 - x_{d-1}, N = y1 - y_{d-1},
    x_d D^2 = N^2 - (x_{d-1} + x1) D^2   and   y_d D^3 = N (x_{d-1} - x_d) D^2 - y_{d-1} D^3.
The checks run on the stored Montgomery values (x R, y R): multiplied through by R^3 and R^4, the first equation gains a factor R on
N^2 and the second is unchanged; the curve equation becomes Y^2 R = X^3 - 3 X R^2 + b R^3.  Both addition equations pin x_d and y_d
down exactly, so a run of entries that starts at a known point is checked exactly.  After a wrong entry the walk goes on from the
true point (one affine addition), so each wrong entry is named once and its right neighbours are not.  A run that starts at an entry
no earlier run checked (a pair at a seam of the table) takes that entry as read; if anything in the run disagrees, the run's true
start is computed with a scalar multiplication and the run is walked again.

A small (signed) table of a key that is not a curve point is only the marker the builder writes: an all-zero first entry."""
from oracle import p256

P = p256.P
R = (1 << 256) % P
R2, R3 = R * R % P, R * R * R % P
RESOLVE_BUDGET = 64        # seam runs per call whose start is computed after a mismatch; past it, every entry of such a run is named


def entries_per_window(w, signed):
    return (1 << (w - 1)) if signed else (1 << w) - 1


def top_digit(w, windows):
    """The largest digit of a 256-bit scalar in the last of `windows` unsigned windows of w bits: the kernels read no entry past it."""
    return min((1 << w) - 1, (1 << (256 - w * (windows - 1))) - 1)


def window_bases(base, w, windows):
    """[2^(w j) * base for j in range(windows)], affine plain coordinates: the true entries (j, 1)."""
    out = [base]
    for _ in range(1, windows):
        out.append(p256.scalar_mult(1 << w, out[-1]))
    return out


def _mont(pt):
    return None if pt is None else (pt[0] * R % P, pt[1] * R % P)


def _plain(mpt):
    rinv = pow(R, -1, P)
    return None if mpt is None else (mpt[0] * rinv % P, mpt[1] * rinv % P)


def _stored(rows, i):
    """Entry i of rows as stored (Montgomery X, Y), or None when a coordinate is not reduced or the point is not on the curve."""
    o = 64 * i
    X, Y = int.from_bytes(rows[o:o + 32], "little"), int.from_bytes(rows[o + 32:o + 64], "little")
    if X >= P or Y >= P or (Y * Y * R - (X * X - 3 * R2) * X - p256.B * R3) % P:
        return None
    return X, Y


def _walk(j, d0, rows, p1, prev):
    """Entries d0, d0+1, ... of window j against `prev`, the true entry d0 - 1 (plain; None: infinity, for d0 == 1).  p1: the true
    entry (j, 1), plain.  Returns the wrong (j, d).  An entry that passes equals the true point, so it is on the curve: the curve
    equation is not evaluated again here."""
    X1, Y1 = _mont(p1)
    mprev = _mont(prev)
    bad = []
    for i in range(len(rows) // 64):
        o = 64 * i
        X, Y = int.from_bytes(rows[o:o + 32], "little"), int.from_bytes(rows[o + 32:o + 64], "little")
        if X >= P or Y >= P:
            ok = False
        elif mprev is None:
            ok = X == X1 and Y == Y1
        else:
            Xd, Yd = mprev
            dx = X1 - Xd
            if dx:                                             # the two equations of the module doc, the second divided by D^2
                n = Y1 - Yd
                ok = ((X + Xd + X1) * dx * dx - n * n * R) % P == 0 and ((Y + Yd) * dx - n * (Xd - X)) % P == 0
            else:                                              # prev == p1: the doubling of d = 2
                ok = (X, Y) == _mont(p256.point_add(_plain(mprev), p1))
        if ok:
            mprev = X, Y
        else:
            bad.append((j, d0 + i))
            mprev = _mont(p256.point_add(_plain(mprev), p1))
    return bad


def check_runs(runs):
    """runs: iterable of (j, d0, rows, p1, known): rows = the raw entries d0, d0+1, ... of window j, p1 = the true entry (j, 1).
    known: walk from the true entry d0 - 1 (one scalar multiplication); else the run's first entry is taken as read (see the module
    doc).  A run from d0 = 1 always starts at a known point, infinity.  Returns the wrong (window, digit), sorted."""
    bad, budget = [], RESOLVE_BUDGET
    for j, d0, rows, p1, known in runs:
        if not known and d0 > 1:
            first = _stored(rows, 0)
            if first is not None and not _walk(j, d0 + 1, rows[64:], p1, _plain(first)):
                continue
            if not budget:
                bad += [(j, d0 + i) for i in range(len(rows) // 64)]
                continue
            budget -= 1
        bad += _walk(j, d0, rows, p1, p256.scalar_mult(d0 - 1, p1) if d0 > 1 else None)
    return sorted(set(bad))


def table_runs(rows, w, signed, bases, top=None, run=1 << 14):
    """Runs (for check_runs) over a whole table read into `rows` (windows x entries_per_window rows), digits past `top` of the last
    window excepted, each run at most `run` entries and starting at a known point.  bases: window_bases of the table's point."""
    per = entries_per_window(w, signed)
    windows = len(rows) // (64 * per)
    assert len(rows) == 64 * per * windows and windows == len(bases)
    out = []
    for j in range(windows):
        n = per if top is None or j < windows - 1 else top
        out += [(j, 1 + k, rows[64 * (per * j + k):64 * (per * j + min(n, k + run))], bases[j], True) for k in range(0, n, run)]
    return out


def seam_spans(w, last, chunk=64):
    """Digit spans [a, b] that cover every pair (d - 1, d), d <= last, with d at a seam of the two-level builder: a chunk boundary
    (d = 0, 1, -1 mod chunk, one thread's chunk ending at 0 mod chunk) or a boundary between its low and high tables (d = 0, 1, -1
    mod 2^(w/2)); for d = 1, the span [1, 1] (the anchor).  Overlapping pairs are merged into one span."""
    half = 1 << (w // 2)
    ds = sorted({m + k for step in (chunk, half) for m in range(0, last + 2, step) for k in (-1, 0, 1) if 1 <= m + k <= last})
    spans = []
    for d in ds:
        if spans and d - 1 <= spans[-1][1]:
            spans[-1][1] = d
        else:
            spans.append([max(d - 1, 1), d])
    return [tuple(s) for s in spans]


def check_table(rows, w, signed, base, top=None):
    """The wrong (window, digit) of a whole table (see table_runs).  base: the key (x, y) as plain integers.  A signed table whose key is
    not a curve point must be exactly the zero marker in its first entry (nothing else of it is read by the kernels)."""
    rows = bytes(rows)
    if not p256.is_on_curve(*base):
        assert signed, "only the small tables mark a key that is not a curve point"
        return [] if rows[:64] == bytes(64) else [(0, 1)]
    per = entries_per_window(w, signed)
    return check_runs(table_runs(rows, w, signed, window_bases(base, w, len(rows) // (64 * per)), top))


def tasks_of(runs, entries=1 << 14):
    """runs grouped into lists of about `entries` entries: one check_runs call each, for a process pool."""
    tasks, cur, n = [], [], 0
    for r in runs:
        cur.append(r)
        n += len(r[2]) // 64
        if n >= entries:
            tasks.append(cur)
            cur, n = [], 0
    return tasks + ([cur] if cur else [])
