"""Cost of the update-batch export (fabgpu_block_updates) after the MVCC stage (development tool).

mvcc_bench.py's shape: a 10k-transaction block, 3 endorsements per transaction, two reads and two writes per transaction over 10^6
installed keys, with a metadata write (a VALIDATION_PARAMETER entry) on one of its keys in 1 % of the transactions; and the hot-key
block, where every transaction writes one key blind (a metadata write in 1 % of them).  Legs alternated `--rounds` times in one process:
  (a) export_rand / export_hot: ms of the first fabgpu_block_updates call after the stage (it builds the batch) and of a repeated call
      (copies only), each a host clock around the C call (into preallocated buffers), which returns synchronised; the record and
      metadata counts; and, apart, ms of the binding's block_updates, which also reads every record's bytes back into Python objects;
  (b) loop_plain / loop_export: ms per block of the three-in-flight loop with validate_mvcc between the wait and the next submit, without
      and with the C call after it.
--profile: one separate run of each export under torch.profiler, the ud_* kernels' device times summed per name.
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
from tools.mvcc_bench import NS, install, key  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402
import updates_oracle as uo  # noqa: E402

META = [("VALIDATION_PARAMETER", b"\x12\x04policy")]


def random_block(n_tx, pool, rng):
    txs = []
    for t in range(n_tx):
        r, w = rng.integers(0, pool, 2), rng.integers(0, pool, 2)
        ns = dict(ns=NS, reads=[(key(int(i)), (0, int(i) % 1000)) for i in r], writes=[(key(int(i)), b"value-%d-%d" % (t, j)) for j, i in enumerate(w)])
        if t % 100 == 0:
            ns["md"] = [(key(int(w[0])), META)]
        txs.append([ns])
    return txs


def hot_block(n_tx):
    return [[dict(ns=NS, writes=[(key(0), b"hot-%d" % t)], md=[(key(0), META)] if t % 100 == 0 else [])] for t in range(n_tx)]


def build(net, txs, seed):
    hook = lambda t, part, b: uo.encode(txs[t]) if part == "TxReadWriteSet" else b
    _, info = blockgen.build_block(net, len(txs), 3, {}, seed=seed, mutate=hook)
    return info


_REC = np.zeros(pkg.binding.UPDATE_WORDS * 40_000, np.uint32)
_META = np.zeros(1 << 22, np.uint8)


def export_c(ctx, slot, h):
    """fabgpu_block_updates into preallocated buffers (as a peer's caller would): (records, metadata bytes, complete)"""
    n = (ctypes.c_size_t * 2)()
    complete = ctypes.c_int(0)
    ctx._ck(pkg.binding.lib().fabgpu_block_updates(ctx._h, ctypes.c_int(slot), ctypes.c_uint64(h), _REC.ctypes.data_as(ctypes.c_void_p),
                                                   ctypes.c_size_t(_REC.size // pkg.binding.UPDATE_WORDS), _META.ctypes.data_as(ctypes.c_void_p),
                                                   ctypes.c_size_t(_META.size), n, ctypes.byref(complete)))
    return int(n[0]), int(n[1]), complete.value


def export_ms(ctx, info, reps):
    """per rep: the block validated and staged on slot 0 (untimed), then the first and a repeated C call (timed), then the binding's"""
    first, again, py, n = [], [], [], None
    for _ in range(reps):
        tv = ctx.validate_envelopes(info["env_blob"], info["env_off"])
        h = ctx.state_versions_info()[2]
        ctx.validate_mvcc(0, h, tv)
        t0 = time.perf_counter()
        n = export_c(ctx, 0, h)
        t1 = time.perf_counter()
        export_c(ctx, 0, h)
        t2 = time.perf_counter()
        ctx.block_updates(0, h)
        t3 = time.perf_counter()
        first.append((t1 - t0) * 1e3); again.append((t2 - t1) * 1e3); py.append((t3 - t2) * 1e3)
    return dict(first_ms_median=float(np.median(first)), first_ms_min=float(np.min(first)), first_ms_max=float(np.max(first)),
                again_ms_median=float(np.median(again)), binding_ms_median=float(np.median(py)), records_meta_bytes_complete=n)


def loop_ms(ctx, pinned, eoff, n_tx, slots, blocks, export):
    t0 = time.perf_counter()
    for k in range(slots):
        ctx.validate_envelopes_async(k, pinned[k], eoff)
    for k in range(blocks):
        tv = ctx.validate_wait(k % slots, n_tx)
        h = ctx.state_versions_info()[2]
        ctx.validate_mvcc(k % slots, h, tv)
        if export:
            export_c(ctx, k % slots, h)
        if k + slots < blocks:
            ctx.validate_envelopes_async(k % slots, pinned[k % slots], eoff)
    return (time.perf_counter() - t0) / blocks * 1e3


def profile(ctx, infos, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    res = {}
    for name, info in infos.items():
        export_ms(ctx, info, 2)                                        # warm
        with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            export_ms(ctx, info, 3)
            torch.cuda.synchronize()
        k = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "ud_" in e.name:
                short = e.name.split("(")[0].split("::")[-1]
                k.setdefault(short, []).append(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
        res[name] = {n: dict(calls=len(v), us_mean=float(np.mean(v))) for n, v in sorted(k.items())}
        if out_dir:
            prof.export_chrome_trace(os.path.join(out_dir, "updates_%s_trace.json" % name))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="the torch.profiler run instead of the timed legs")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file (traces beside it)")
    args = ap.parse_args()
    rng = np.random.default_rng(5)
    net = blockgen.Network()
    infos = {"rand": build(net, random_block(args.txs, 1_000_000, rng), 17), "hot": build(net, hot_block(args.txs), 18)}
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    install(ctx, 1_000_000, 1_400_000)
    res = {"tool": "updates_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures, 2 reads + 2 writes per transaction over 10^6 keys, 1 %% with a "
           "metadata write; hot-key block (every transaction writes one key); %d blocks in flight" % (args.txs, slots)}
    if args.profile:
        res["kernels"] = profile(ctx, infos, os.path.dirname(args.out) if args.out else None)
    else:
        rand = infos["rand"]
        n = rand["env_off"].shape[0] - 1
        pinned = []
        for k in range(slots):
            b = ctx.block_buffer(len(rand["env_blob"]), slot=k)
            b[:] = np.frombuffer(rand["env_blob"], np.uint8)
            pinned.append(b)
        runs = {"export_rand": [], "export_hot": [], "loop_plain": [], "loop_export": []}
        for _ in range(args.rounds):
            runs["export_rand"].append(export_ms(ctx, rand, 10))
            runs["export_hot"].append(export_ms(ctx, infos["hot"], 10))
            loop_ms(ctx, pinned, rand["env_off"], n, slots, 6, False)   # warm-up
            for leg in ("loop_plain", "loop_export"):
                runs[leg].append(loop_ms(ctx, pinned, rand["env_off"], n, slots, 30, leg == "loop_export"))
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
