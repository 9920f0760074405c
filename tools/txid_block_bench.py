"""The per-block step of the committed tx-id set: host _add against add_block (development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction, NOutOf(3) chaincode policy -- with a set of 10^6
random ids installed.  Two legs alternated `--rounds` times in one process, each the loop a peer runs with every slot in flight (submit
block k, add its ids, submit block k+1):
  (a) add:        fabgpu_committed_txids_add with 10^4 fresh random ids staged before the loop (tools/txid_bench.py's loop: the
                  peer's own parse of the block for its ids is not counted);
  (b) add_block:  fabgpu_committed_txids_add_block(slot).
Each submitted block carries the same envelopes, so from the second block on every transaction of leg (b) is DUPLICATE_TXID.  Reports
ms per block, the host time per call, and the device time of the two add_block kernels from torch.profiler.  Prints one JSON line, with
the card's name and power limit read in the same run."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402
from tools.txid_bench import install, random_ids  # noqa: E402


def loop(ctx, pinned, eoff, n_tx, slots, blocks, per_block):
    """blocks submitted round-robin, per_block(slot) right after each submit: ms per block and each call's ms"""
    t_call = []
    t0 = time.perf_counter()
    for k in range(blocks):
        if k >= slots:
            ctx.validate_wait(k % slots, n_tx)
        ctx.validate_envelopes_async(k % slots, pinned[k % slots], eoff)
        ta = time.perf_counter()
        per_block(k % slots)
        t_call.append((time.perf_counter() - ta) * 1e3)
    for k in range(max(0, blocks - slots), blocks):
        ctx.validate_wait(k % slots, n_tx)
    return (time.perf_counter() - t0) / blocks * 1e3, t_call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=30)
    ap.add_argument("--installed", type=int, default=1_000_000)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    _, info = blockgen.build_block(net, args.txs, 3, {}, seed=17)
    n = info["env_off"].shape[0] - 1
    eoff = info["env_off"]
    env_blob = bytes(info["env_blob"])
    L = pkg.binding.lib()

    def host_add(ctx, rng):
        adds = [random_ids(rng, n) for _ in range(args.blocks)]
        seq = iter(adds)

        def call(slot):
            b, o = next(seq)
            ctx._ck(L.fabgpu_committed_txids_add(ctx._h, b.ctypes.data_as(ctypes.c_void_p), o.ctypes.data_as(ctypes.c_void_p), None,
                                                 ctypes.c_size_t(n)))
        return call

    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    ctx.msp_configure([(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table], net.policy_n_of(3), net.principals, net.channel)
    pinned = []
    for k in range(slots):
        b = ctx.block_buffer(len(env_blob), slot=k)
        b[:] = np.frombuffer(env_blob, np.uint8)
        pinned.append(b)
    rng = np.random.default_rng(23)
    blob, off = random_ids(rng, args.installed)
    runs = {"add": [], "add_block": []}
    for _ in range(args.rounds):
        for name in runs:
            r = {"install_s": install(ctx, blob, off, args.installed + (args.blocks + 1) * args.txs)}
            call = host_add(ctx, rng) if name == "add" else ctx.committed_txids_add_block
            r["ms_per_block"], calls = loop(ctx, pinned, eoff, n, slots, args.blocks, call)
            r["call_ms_median"], r["call_ms_max"] = float(np.median(calls)), float(np.max(calls))
            r["ids_held"] = ctx.committed_txids_info()[0]
            runs[name].append(r)
    kernels = {}
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        install(ctx, blob, off, args.installed + (args.blocks + 1) * args.txs)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            loop(ctx, pinned, eoff, n, slots, 10, ctx.committed_txids_add_block)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if "txid_block" in ev.key:
                kernels[ev.key.split("(")[0]] = {"calls": ev.count, "us_avg": ev.device_time_total / max(ev.count, 1)}
    except Exception as e:                               # the profile is an extra: the legs above stand without it
        kernels = {"error": str(e)}
    ctx.committed_txids([])
    ctx.close()
    res = {"tool": "txid_block_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures, %d blocks in flight, %d blocks per leg; %d random ids installed"
           % (args.txs, slots, args.blocks, args.installed), "runs": runs, "kernels": kernels}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
