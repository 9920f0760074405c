"""GPU: the point tables the device builds, read back entry by entry (fabgpu_test_table_entries) and checked against the group law on
the CPU (tests/tablecheck.py, itself checked against host-built tables by tests/test_tablecheck.py).  Every verification reads its
points from these tables, and a signature touches a few dozen entries out of millions, so one wrong entry would only show as a valid
signature rejected now and then.  Read whole: every small table (including recycled slots), whole per-key window tables, and
generator windows 0, 6 and the useful part of the top one; read as pairs: every seam of the two-level builder in every window of the
other per-key tables and of the generator table.  Each test prints how many entries it checked."""
import collections
import multiprocessing
import os
import time

import numpy as np
import pytest

from oracle import p256
from tools import workload
from util import from_be, pkg
import tablecheck as tc
import vectors

pytestmark = pytest.mark.gpu

G = (p256.GX, p256.GY)
PIECE = 1 << 20                     # entries per read: the readback never holds more than 64 MiB
RUN = 1 << 14                       # entries per run of a whole window (each starts with one scalar multiplication)


@pytest.fixture(scope="module")
def pool():
    with multiprocessing.get_context("spawn").Pool(os.cpu_count()) as p:
        yield p


def _context(**env):
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return pkg().binding.Context(max_batch=4096)
    finally:
        for k in env:
            del os.environ[k]


def _xy(q):
    return np.frombuffer(q[0].to_bytes(32, "big") + q[1].to_bytes(32, "big"), np.uint8)


def _read(ctx, key_slot, window, digit):
    """Raw bytes of entries (window[i], digit[i]), 64 per entry."""
    window, digit = np.asarray(window, np.uint32), np.asarray(digit, np.uint32)
    assert window.shape[0] <= PIECE
    return ctx.test_table_entries(key_slot, window, digit).tobytes()


class _Checks:
    """Runs handed to the pool as they are read; at most three reads' worth waits in the pool at a time."""

    def __init__(self, pool):
        self.pool, self.pending, self.bad, self.entries = pool, collections.deque(), [], collections.Counter()

    def submit(self, kind, runs):
        self.entries[kind] += sum(len(r[2]) // 64 for r in runs)
        self.pending.append(self.pool.map_async(tc.check_runs, tc.tasks_of(runs)))
        while len(self.pending) > 3:
            self._collect()

    def _collect(self):
        self.bad += [b for part in self.pending.popleft().get() for b in part]

    def wrong(self):
        while self.pending:
            self._collect()
        return list(dict.fromkeys(self.bad))           # an entry both in a whole window and at a seam is named once

    def whole(self, kind, ctx, key_slot, per, bases, windows, top):
        """Windows `windows` of a table, every entry (digits past `top` of the last window excepted), in reads of at most PIECE."""
        for j in windows:
            n = top if j == len(bases) - 1 else per
            for d0 in range(1, n + 1, PIECE):
                cnt = min(PIECE, n - d0 + 1)
                rows = _read(ctx, key_slot, np.full(cnt, j), np.arange(d0, d0 + cnt))
                self.submit(kind, [(j, d0 + k, rows[64 * k:64 * min(cnt, k + RUN)], bases[j], True) for k in range(0, cnt, RUN)])

    def seams(self, kind, ctx, key_slot, w, bases, last):
        """Every seam pair (tablecheck.seam_spans) of every window, digits up to last[j]."""
        for j in range(len(bases)):
            spans = tc.seam_spans(w, last[j])
            while spans:
                k, n = 0, 0
                while k < len(spans) and n + spans[k][1] - spans[k][0] + 1 <= PIECE:
                    n += spans[k][1] - spans[k][0] + 1
                    k += 1
                part, spans = spans[:k], spans[k:]
                digits = np.concatenate([np.arange(a, b + 1) for a, b in part])
                rows = _read(ctx, key_slot, np.full(len(digits), j), digits)
                runs, o = [], 0
                for a, b in part:
                    runs.append((j, a, rows[64 * o:64 * (o + b - a + 1)], bases[j], False))
                    o += b - a + 1
                self.submit(kind, runs)


def _small_keys():
    n = p256.N
    structured = [G, p256.point_neg(G), p256.scalar_mult(2, G), p256.scalar_mult(n - 1, G), p256.scalar_mult(3, G)]
    structured += [p256.scalar_mult(1 << k, G) for k in (7, 8, 9, 31, 32, 64, 128, 200, 248, 255)]
    widths = pkg().binding.build_info() + (pkg().binding.Context.small_table_info()[0],)
    chain = [(c["qx"], c["qy"]) for c in vectors.chain_cases(*widths, orders=("small",))]
    w = workload.Workload(128, 96, seed=0x7AB1)
    rnd = [(from_be(k[:32]), from_be(k[32:])) for k in w.keys_xy]
    keys = list(dict.fromkeys(structured + chain + rnd))
    assert all(p256.is_on_curve(*q) for q in keys)
    return keys + [(G[0], G[1] ^ 1)]                                  # last: not a curve point


def _check_small(ck, ctx, handles, keys):
    ws, windows, _ = pkg().binding.Context.small_table_info()
    per = 1 << (ws - 1)
    window, digit = np.repeat(np.arange(windows), per), np.tile(np.arange(1, per + 1), windows)
    for h, q in zip(handles, keys):
        rows = _read(ctx, int(h), window, digit)
        if not p256.is_on_curve(*q):
            ck.entries["small"] += 1
            if tc.check_table(rows, ws, True, q):
                ck.bad.append(("off-curve key", int(h)))
            continue
        ck.submit("small", tc.table_runs(rows, ws, True, tc.window_bases(q, ws, windows)))


def test_small_tables_every_entry(pool):
    t0 = time.time()
    keys = _small_keys()
    assert len(keys) >= 97
    ctx = _context(FABGPU_SMALL_SLOTS=256, FABGPU_KEY_SLOTS=1)
    try:
        handles = ctx.keys_register_small(np.stack([_xy(q) for q in keys]))
        assert (handles <= -2).all()
        n0 = ctx.launch_count()
        ck = _Checks(pool)
        _check_small(ck, ctx, handles, keys)                       # read at once: the hook waits for the builds it reads
        assert ctx.launch_count() == n0 + len(keys)
        for j, d in ((33, 1), (0, 0), (0, 129)):                   # outside the small table's shape
            with pytest.raises(pkg().binding.FabGpuError):
                ctx.test_table_entries(int(handles[0]), [j], [d])
        bad = ck.wrong()
    finally:
        ctx.close()
    assert not bad, bad[:20]
    print("small tables: %d keys, %d entries checked in %.1f s" % (len(keys), ck.entries["small"], time.time() - t0))


def test_small_table_recycling(pool):
    """A pool of 16 small tables: a second registration recycles 8 slots.  The new tables belong wholly to their new keys (one of them
    not a curve point: the marker lands in a recycled slot), the survivors are intact, and the evicted keys' handles are refused."""
    t0 = time.time()
    keys = _small_keys()
    first, second = keys[:16], keys[16:23] + keys[-1:]
    ctx = _context(FABGPU_SMALL_SLOTS=16, FABGPU_KEY_SLOTS=1)
    try:
        h1 = ctx.keys_register_small(np.stack([_xy(q) for q in first]))
        h2 = ctx.keys_register_small(np.stack([_xy(q) for q in second]))
        assert (h1 <= -2).all() and (h2 <= -2).all() and ctx.key_table_stats()["small_recycled"] == 8
        live, evicted = [], []
        for h, q in zip(h1, first):
            try:
                ctx.test_table_entries(int(h), [0], [1])
                live.append((h, q))
            except pkg().binding.FabGpuError:
                evicted.append(h)
        slot = lambda h: (-2 - int(h)) & 0xFFFFF
        assert len(evicted) == 8 and sorted(map(slot, evicted)) == sorted(map(slot, h2))
        ck = _Checks(pool)
        _check_small(ck, ctx, h2, second)
        _check_small(ck, ctx, [h for h, _ in live], [q for _, q in live])
        bad = ck.wrong()
    finally:
        ctx.close()
    assert not bad, bad[:20]
    print("recycled small tables: %d entries checked in %.1f s" % (ck.entries["small"], time.time() - t0))


def _key_bases(q):
    wq = pkg().binding.build_info()[1]
    return tc.window_bases(q, wq, (256 + wq - 1) // wq)


def test_key_tables_whole_and_at_every_seam(pool):
    """Two per-key tables read whole, two more at every seam of every window."""
    t0 = time.time()
    wq = pkg().binding.build_info()[1]
    per = (1 << wq) - 1
    w = workload.Workload(8, 2, seed=0x7AB2)
    keys = [(from_be(k[:32]), from_be(k[32:])) for k in w.keys_xy] + [G, p256.scalar_mult(p256.N - 1, G)]
    ctx = _context(FABGPU_KEY_SLOTS=4, FABGPU_SMALL_SLOTS=0)
    try:
        slots = ctx.keys_register(np.stack([_xy(q) for q in keys])) & 0xFFF
        ck = _Checks(pool)
        for k in (0, 2):
            bases = _key_bases(keys[k])
            ck.whole("key, whole", ctx, int(slots[k]), per, bases, range(len(bases)), top=tc.top_digit(wq, len(bases)))
        for k in (1, 3):
            bases = _key_bases(keys[k])
            ck.seams("key, seams", ctx, int(slots[k]), wq, bases, [per] * (len(bases) - 1) + [tc.top_digit(wq, len(bases))])
        bad = ck.wrong()
    finally:
        ctx.close()
    assert not bad, bad[:20]
    print("key tables: %s checked in %.1f s" % (dict(ck.entries), time.time() - t0))


def test_key_table_recycling(pool):
    """FABGPU_KEY_SLOTS=4: keys 4 and 5 take the slots of keys 0 and 1 (as in test_key_table_eviction_and_off_curve_keys); windows 0,
    7 and 15 of both recycled slots hold the new keys' points, every entry."""
    t0 = time.time()
    wq = pkg().binding.build_info()[1]
    per = (1 << wq) - 1
    w = workload.Workload(12, 6, seed=47)
    keys = [(from_be(k[:32]), from_be(k[32:])) for k in w.keys_xy]
    ctx = _context(FABGPU_KEY_SLOTS=4, FABGPU_SMALL_SLOTS=0)
    try:
        s1 = ctx.keys_register(w.keys_xy[:4])
        s2 = ctx.keys_register(w.keys_xy[2:6])
        assert sorted((s2[2:] & 0xFFF).tolist()) == sorted(s1[:2].tolist())
        ck = _Checks(pool)
        for k, h in ((4, s2[2]), (5, s2[3])):
            bases = _key_bases(keys[k])
            ck.whole("key, recycled", ctx, int(h) & 0xFFF, per, bases, [0, 7, len(bases) - 1], top=tc.top_digit(wq, len(bases)))
        bad = ck.wrong()
    finally:
        ctx.close()
    assert not bad, bad[:20]
    print("recycled key tables: %s checked in %.1f s" % (dict(ck.entries), time.time() - t0))


def test_generator_table_windows_and_seams(pool):
    """Windows 0 and 6 whole, the top window's useful digits whole, and every seam pair of all windows."""
    t0 = time.time()
    wg = pkg().binding.build_info()[0]
    per, windows = (1 << wg) - 1, (256 + wg - 1) // wg
    top = tc.top_digit(wg, windows)
    bases = tc.window_bases(G, wg, windows)
    ctx = _context(FABGPU_KEY_SLOTS=1, FABGPU_SMALL_SLOTS=0)
    try:
        ck = _Checks(pool)
        ck.whole("generator, whole windows", ctx, -1, per, bases, [0, 6, windows - 1], top=top)
        ck.seams("generator, seams", ctx, -1, wg, bases, [per] * (windows - 1) + [top])
        bad = ck.wrong()
    finally:
        ctx.close()
    assert not bad, bad[:20]
    print("generator table: %s checked in %.1f s" % (dict(ck.entries), time.time() - t0))
