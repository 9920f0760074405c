"""Cost of the deterministic update bytes (fabgpu_block_update_bytes) after the MVCC stage and the batch export (development tool).

updates_bench.py's 10k-transaction block, spread over 8 namespaces and 4 collections: each transaction reads two installed keys of the
first namespace, writes one key there and one in another namespace, and a third of them write a hashed key in a collection of a
namespace; 1 % put a metadata write on their own key and 1 % a blind metadata write alone on an installed key, which makes its value COMMITTED (the
caller passes 64 bytes for each).  Legs alternated `--rounds` times in one process:
  (a) bytes_first / bytes_again: ms of the first fabgpu_block_update_bytes call after fabgpu_block_updates (it also sorts the batch)
      and of a repeated call, each a host clock around the C call (into a preallocated buffer), which returns synchronised;
  (b) loop_plain / loop_bytes: ms per block of the three-in-flight loop with validate_mvcc and the fabgpu_block_updates export between
      the wait and the next submit, without and with the bytes call after them.
--profile: one separate run under torch.profiler, the ub_* kernels' device times summed per name.
Prints one JSON line, with the card's name and power limit read in the same run.  The Go committer's own cost of
deterministicBytesForPubAndHashUpdates is not measured here: there is no Go toolchain."""
import argparse
import ctypes
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.mvcc_bench import NS, install, key  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402
from tools.updates_bench import META, build, export_c, _REC  # noqa: E402
from tools import blockgen  # noqa: E402

NSS = [NS] + ["ns%d" % i for i in range(1, 8)]
COLLS = ["coll%d" % i for i in range(4)]


def spread_block(n_tx, pool, rng):
    txs = []
    for t in range(n_tx):
        r, w = rng.integers(0, pool, 2), rng.integers(0, pool, 2)
        home = dict(ns=NS, reads=[(key(int(i)), (0, int(i) % 1000)) for i in r], writes=[(key(int(w[0])), b"value-%d-0" % t)])
        if t % 100 == 0:
            home["md"] = [(key(int(w[0])), META)]
        elif t % 100 == 50:
            home["md"] = [(key(int(rng.integers(0, pool))), META)]
        other = dict(ns=NSS[1 + t % 7], writes=[(key(int(w[1])), b"value-%d-1" % t)])
        if t % 3 == 0:
            other["colls"] = [(COLLS[t % 4], [], [(hashlib.sha256(b"pk%d" % t).digest(), hashlib.sha256(b"pv%d" % t).digest())], [])]
        txs.append([home, other])
    return txs


_OUT = np.zeros(1 << 24, np.uint8)
_VALS = np.frombuffer(b"\x5a" * (64 * 40_000), np.uint8).copy()
_VOFF = (np.arange(40_001, dtype=np.uint32) * 64)


def committed_count(n_rec):
    return int(np.count_nonzero(_REC[: n_rec * pkg.binding.UPDATE_WORDS].reshape(-1, pkg.binding.UPDATE_WORDS)[:, 2] == pkg.binding.SRC_COMMITTED))


def bytes_c(ctx, slot, h, n_val):
    """fabgpu_block_update_bytes into a preallocated buffer, 64 bytes per committed value: (length, complete)"""
    n = ctypes.c_size_t(0)
    complete = ctypes.c_int(0)
    ctx._ck(pkg.binding.lib().fabgpu_block_update_bytes(ctx._h, ctypes.c_int(slot), ctypes.c_uint64(h), _VALS.ctypes.data_as(ctypes.c_void_p),
                                                        _VOFF.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(n_val),
                                                        _OUT.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(_OUT.size), ctypes.byref(n),
                                                        ctypes.byref(complete)))
    return int(n.value), complete.value


def bytes_ms(ctx, info, reps):
    first, again, n = [], [], None
    for _ in range(reps):
        tv = ctx.validate_envelopes(info["env_blob"], info["env_off"])
        h = ctx.state_versions_info()[2]
        ctx.validate_mvcc(0, h, tv)
        n_rec = export_c(ctx, 0, h)[0]
        nv = committed_count(n_rec)
        t0 = time.perf_counter()
        n = bytes_c(ctx, 0, h, nv)
        t1 = time.perf_counter()
        bytes_c(ctx, 0, h, nv)
        t2 = time.perf_counter()
        first.append((t1 - t0) * 1e3); again.append((t2 - t1) * 1e3)
        n = (n_rec, nv) + n
    return dict(first_ms_median=float(np.median(first)), first_ms_min=float(np.min(first)), first_ms_max=float(np.max(first)),
                again_ms_median=float(np.median(again)), records_committed_bytes_complete=n)


def loop_ms(ctx, pinned, eoff, n_tx, slots, blocks, with_bytes):
    t0 = time.perf_counter()
    for k in range(slots):
        ctx.validate_envelopes_async(k, pinned[k], eoff)
    for k in range(blocks):
        tv = ctx.validate_wait(k % slots, n_tx)
        h = ctx.state_versions_info()[2]
        ctx.validate_mvcc(k % slots, h, tv)
        n_rec = export_c(ctx, k % slots, h)[0]
        if with_bytes:
            bytes_c(ctx, k % slots, h, committed_count(n_rec))
        if k + slots < blocks:
            ctx.validate_envelopes_async(k % slots, pinned[k % slots], eoff)
    return (time.perf_counter() - t0) / blocks * 1e3


def profile(ctx, info, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    bytes_ms(ctx, info, 2)                                             # warm
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        bytes_ms(ctx, info, 3)
        torch.cuda.synchronize()
    k = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "ub_" in e.name:
            short = e.name.split("(")[0].split("::")[-1]
            k.setdefault(short, []).append(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "update_bytes_trace.json"))
    return {n: dict(calls=len(v), us_mean=float(np.mean(v)), us_total_per_rep=float(np.sum(v)) / 3) for n, v in sorted(k.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="the torch.profiler run instead of the timed legs")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file (the trace beside it)")
    args = ap.parse_args()
    rng = np.random.default_rng(5)
    net = blockgen.Network()
    info = build(net, spread_block(args.txs, 1_000_000, rng), 17)
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel, policies={n: 0 for n in NSS})
    install(ctx, 1_000_000, 1_400_000)
    res = {"tool": "update_bytes_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures over %d namespaces and %d collections, 2 reads + 2 writes per "
           "transaction over 10^6 keys, a hashed write in a third, 1 %% with a metadata write and 1 %% with a COMMITTED value; %d blocks "
           "in flight" % (args.txs, len(NSS), len(COLLS), slots)}
    if args.profile:
        res["kernels"] = profile(ctx, info, os.path.dirname(args.out) if args.out else None)
    else:
        n = info["env_off"].shape[0] - 1
        pinned = []
        for k in range(slots):
            b = ctx.block_buffer(len(info["env_blob"]), slot=k)
            b[:] = np.frombuffer(info["env_blob"], np.uint8)
            pinned.append(b)
        runs = {"bytes": [], "loop_plain": [], "loop_bytes": []}
        for _ in range(args.rounds):
            runs["bytes"].append(bytes_ms(ctx, info, 10))
            loop_ms(ctx, pinned, info["env_off"], n, slots, 6, False)   # warm-up
            for leg in ("loop_plain", "loop_bytes"):
                runs[leg].append(loop_ms(ctx, pinned, info["env_off"], n, slots, 30, leg == "loop_bytes"))
        res["runs"] = runs
    ctx.state_versions([], 0)
    ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
