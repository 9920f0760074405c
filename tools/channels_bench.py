"""Channel contexts of one table group (fabgpu_init_shared) against separate contexts (development tool).

Reports, in one process:
  (1) the device memory an extra context takes: a second fabgpu_init beside the first, and a fabgpu_init_shared context;
  (2) the time to create each;
  (3) bench.py's block_replay block -- 10k transactions, 3 endorsements each, NOutOf(3) policy -- validated on ONE context with every
      slot in flight, as ms per block;
  (4) the same on THREE channel contexts of one group, each driven by its own host thread with every slot in flight.  Channels x and y
      have the same endorsers (one network seed, two channel names); channel z has others.  Reported as the aggregate ms per block and
      blocks per second of the three, and per channel;
  (5) the window tables built for each case.
Legs (3) and (4) alternate `--rounds` times; the first context of the group is the one context of leg (3).  Prints one JSON line, with
the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402

MAX_BATCH = 8192


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def channel(ctx, net, txs, seed):
    """configures the context for the network's channel and stages its block in the slots' pinned buffers: (pinned, eoff, n)"""
    _, info = blockgen.build_block(net, txs, 3, {}, seed=seed)
    ctx.msp_configure([(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table], net.policy_n_of(3), net.principals, net.channel)
    blob = bytes(info["env_blob"])
    pinned = []
    for k in range(pkg.binding.SLOTS):
        b = ctx.block_buffer(len(blob), slot=k)
        b[:] = np.frombuffer(blob, np.uint8)
        pinned.append(b)
    return pinned, info["env_off"], info["env_off"].shape[0] - 1


def loop(ctx, ch, blocks):
    """blocks submitted round-robin over the slots, every slot in flight; every flag must be VALID.  Seconds."""
    pinned, eoff, n = ch
    S = pkg.binding.SLOTS
    bad = 0
    t0 = time.perf_counter()
    for k in range(blocks):
        if k >= S:
            bad += int(ctx.validate_wait(k % S, n).any())
        ctx.validate_envelopes_async(k % S, pinned[k % S], eoff)
    for k in range(max(0, blocks - S), blocks):
        bad += int(ctx.validate_wait(k % S, n).any())
    dt = time.perf_counter() - t0
    if bad:
        raise RuntimeError("a block of valid transactions came back with invalid flags")
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=30, help="blocks per channel per leg")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    torch.cuda.init()
    Context = pkg.binding.Context
    res = {"tool": "channels_bench", "card": card()}

    free0 = free_bytes()
    t = time.perf_counter()
    parent = Context(max_batch=MAX_BATCH)
    t_parent = time.perf_counter() - t
    free1 = free_bytes()
    t = time.perf_counter()
    extra = Context(max_batch=MAX_BATCH)
    t_full = time.perf_counter() - t
    free2 = free_bytes()
    extra.close()
    free3 = free_bytes()
    t = time.perf_counter()
    extra = Context(max_batch=MAX_BATCH, share_tables_with=parent)
    t_shared = time.perf_counter() - t
    free4 = free_bytes()
    extra.close()
    mib = 1 << 20
    res["memory_mib"] = {"first_context": (free0 - free1) / mib, "extra_fabgpu_init": (free1 - free2) / mib,
                         "extra_fabgpu_init_shared": (free3 - free4) / mib,
                         "note": "an extra fabgpu_init caps its pools by the memory the first context left (half of it for window tables, "
                                 "an eighth for small tables)"}
    res["create_s"] = {"first_context": t_parent, "extra_fabgpu_init": t_full, "extra_fabgpu_init_shared": t_shared}

    nets = {"x": blockgen.Network(channel="channel-x"), "y": blockgen.Network(channel="channel-y"),
            "z": blockgen.Network(seed=0xC0FFEE, channel="channel-z")}
    ctxs = {"x": parent, "y": Context(max_batch=MAX_BATCH, share_tables_with=parent), "z": Context(max_batch=MAX_BATCH, share_tables_with=parent)}
    chans, built = {}, {}
    for name, seed in (("x", 17), ("y", 18), ("z", 19)):
        before = parent.key_table_stats()["big"]
        chans[name] = channel(ctxs[name], nets[name], args.txs, seed)
        built[name] = parent.key_table_stats()["big"] - before
    res["window_tables_built"] = {"one_context": built["x"], "three_channels_one_group": sum(built.values()),
                                  "per_channel": built, "three_separate_contexts_would_build": 3 * built["x"]}
    for name in chans:                                     # warm-up: every slot of every channel once
        loop(ctxs[name], chans[name], pkg.binding.SLOTS)

    runs = {"one_context": [], "three_channels": []}
    for _ in range(args.rounds):
        dt = loop(parent, chans["x"], args.blocks)
        runs["one_context"].append({"ms_per_block": dt / args.blocks * 1e3, "blocks_per_s": args.blocks / dt})
        per, errors = {}, []

        def drive(name):
            try:
                per[name] = loop(ctxs[name], chans[name], args.blocks)
            except Exception as e:                      # reported on the main thread
                errors.append(e)
        th = [threading.Thread(target=drive, args=(name,)) for name in chans]
        t0 = time.perf_counter()
        for x in th:
            x.start()
        for x in th:
            x.join()
        wall = time.perf_counter() - t0
        if errors:
            raise errors[0]
        total = args.blocks * len(chans)
        runs["three_channels"].append({"aggregate_ms_per_block": wall / total * 1e3, "aggregate_blocks_per_s": total / wall,
                                       "per_channel_ms_per_block": {k: v / args.blocks * 1e3 for k, v in per.items()}})
    res["runs"] = runs
    one = float(np.median([r["blocks_per_s"] for r in runs["one_context"]]))
    three = float(np.median([r["aggregate_blocks_per_s"] for r in runs["three_channels"]]))
    res["summary"] = {"one_context_blocks_per_s_median": one, "three_channels_aggregate_blocks_per_s_median": three, "ratio": three / one}
    res["workload"] = ("%d txs x (1 creator + 3 endorsement) signatures per block, NOutOf(3) policy, %d blocks in flight per context, "
                       "%d blocks per channel per leg, %d rounds" % (args.txs, pkg.binding.SLOTS, args.blocks, args.rounds))
    res["key_table_stats"] = parent.key_table_stats()
    for name in ("z", "y", "x"):
        ctxs[name].close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
