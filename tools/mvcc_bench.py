"""Cost of the MVCC stage (fabgpu_validate_mvcc) over the world-state version table (development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction by the peers of 4 orgs, NOutOf(3) chaincode
policy -- with two reads and two writes per transaction over a pool of installed keys (every read carries the installed version), and the
hot-key block, where every transaction reads and writes one key.  Legs alternated `--rounds` times in one process:
  (a) mvcc_1e6 / mvcc_1e7: the stage on the random block with 10^6 / 10^7 keys installed -- ms per call (it returns with the block
      applied), the install time and the table's bytes;
  (b) hot_key: the stage on the hot-key block;
  (c) loop_plain / loop_mvcc: ms per block of the three-in-flight loop (submit k+3 after waiting k) without and with validate_mvcc + apply
      between the wait and the next submit.
Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402
import mvcc_oracle as mo  # noqa: E402

NS = "mycc"


def key(i):
    return b"k%08d" % i


def install(ctx, n, capacity):
    """n keys k00000000.. of NS with version (0, i % 1000), built as arrays: seconds for the call"""
    L = pkg.binding.lib()
    nb = np.frombuffer(NS.encode() * n, np.uint8)
    no = (np.arange(n + 1, dtype=np.uint64) * len(NS)).astype(np.uint32)
    cb = np.zeros(1, np.uint8)
    co = np.zeros(n + 1, np.uint32)
    idx = np.arange(n, dtype=np.int64)
    kb = np.empty((n, 9), np.uint8)
    kb[:, 0] = ord("k")
    for p in range(8):
        kb[:, 8 - p] = ord("0") + (idx // 10 ** p) % 10
    kb = np.ascontiguousarray(kb.reshape(-1))
    ko = (np.arange(n + 1, dtype=np.uint64) * 9).astype(np.uint32)
    ver = np.zeros((n, 2), np.uint64)
    ver[:, 1] = idx % 1000
    ver = np.ascontiguousarray(ver.reshape(-1))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    t0 = time.perf_counter()
    ctx._ck(L.fabgpu_state_versions(ctx._h, p(nb), p(no), p(cb), p(co), p(kb), p(ko), p(ver), ctypes.c_size_t(n), ctypes.c_uint64(1),
                                    ctypes.c_size_t(capacity)))
    return time.perf_counter() - t0


def random_block(net, n_tx, pool, rng):
    txs = []
    for _ in range(n_tx):
        r = rng.integers(0, pool, 2)
        w = rng.integers(0, pool, 2)
        txs.append([dict(ns=NS, reads=[(key(int(i)), (0, int(i) % 1000)) for i in r], writes=[(key(int(i)), False) for i in w])])
    return txs


def build(net, txs, seed):
    hook = lambda t, part, b: mo.encode(txs[t]) if part == "TxReadWriteSet" else b
    _, info = blockgen.build_block(net, len(txs), 3, {}, seed=seed, mutate=hook)
    return info


def stage_ms(ctx, info, reps):
    """ms per validate_mvcc call on the block (validated on slot 0 first, outside the timing); the flags of the first call"""
    out, first = [], None
    for _ in range(reps):
        tv = ctx.validate_envelopes(info["env_blob"], info["env_off"])
        h = ctx.state_versions_info()[2]
        t0 = time.perf_counter()
        f = ctx.validate_mvcc(0, h, tv)
        out.append((time.perf_counter() - t0) * 1e3)
        first = f if first is None else first
    return out, first


def loop_ms(ctx, pinned, eoff, n_tx, slots, blocks, mvcc):
    t0 = time.perf_counter()
    for k in range(slots):
        ctx.validate_envelopes_async(k, pinned[k], eoff)
    for k in range(blocks):
        tv = ctx.validate_wait(k % slots, n_tx)
        if mvcc:
            ctx.validate_mvcc(k % slots, ctx.state_versions_info()[2], tv)
        if k + slots < blocks:
            ctx.validate_envelopes_async(k % slots, pinned[k % slots], eoff)
    return (time.perf_counter() - t0) / blocks * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--big", type=int, default=10_000_000, help="keys of the large table")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    rng = np.random.default_rng(5)
    net = blockgen.Network()
    rand = build(net, random_block(net, args.txs, 1_000_000, rng), 17)
    hot = build(net, [[dict(ns=NS, reads=[(key(0), (0, 0))], writes=[(key(0), False)])] for _ in range(args.txs)], 18)
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    n = rand["env_off"].shape[0] - 1
    pinned = []
    for k in range(slots):
        b = ctx.block_buffer(len(rand["env_blob"]), slot=k)
        b[:] = np.frombuffer(rand["env_blob"], np.uint8)
        pinned.append(b)
    runs = {"mvcc_1e6": [], "mvcc_1e7": [], "hot_key": [], "loop_plain": [], "loop_mvcc": []}
    for _ in range(args.rounds):
        for name, keys in (("mvcc_1e6", 1_000_000), ("mvcc_1e7", args.big)):
            r = {"install_s": install(ctx, keys, keys + 200_000)}
            ms, f = stage_ms(ctx, rand, 10)
            held, slots_n, _, _ = ctx.state_versions_info()
            r.update(ms_median=float(np.median(ms)), ms_min=float(np.min(ms)), ms_max=float(np.max(ms)), keys_held=held,
                     table_bytes=slots_n * 56, first_flags={str(c): int((f == c).sum()) for c in np.unique(f)})
            runs[name].append(r)
        install(ctx, 1_000_000, 0)
        ms, f = stage_ms(ctx, hot, 10)
        runs["hot_key"].append(dict(ms_median=float(np.median(ms)), ms_min=float(np.min(ms)), ms_max=float(np.max(ms)),
                                    first_flags={str(c): int((f == c).sum()) for c in np.unique(f)}))
        loop_ms(ctx, pinned, rand["env_off"], n, slots, 6, False)       # warm-up
        for leg in ("loop_plain", "loop_mvcc"):
            runs[leg].append(loop_ms(ctx, pinned, rand["env_off"], n, slots, 30, leg == "loop_mvcc"))
    ctx.state_versions([], 0)
    ctx.close()
    res = {"tool": "mvcc_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures, 2 reads + 2 writes per transaction over 10^6 keys; hot-key block; "
           "%d blocks in flight" % (args.txs, slots), "runs": runs}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
