"""The block's private update batch, fabgpu_block_pvt_updates, against the private-data check alone (development tool).

A 10k-transaction block (3 endorsements per transaction, NOutOf(3) chaincode policy) whose transactions each carry one collection of
about 1 KiB of private data holding two private writes, with their hashed writes and pvt_rwset_hash in the public read/write set, in two
shapes:
  random  fresh keys, and 1 % of the transactions write metadata on a committed private key instead (RENEW records);
  hot     the writes overwrite a pool of 64 keys, and 1 % of the transactions write metadata only, on a key written earlier in the block
          (renewals the device decides).
Per shape, alternated over `--rounds` rounds in one process:
  - a host clock around validate_pvtdata and around block_pvt_updates on the same block after its MVCC stage (both return synchronised);
  - ms per block of a loop with three blocks in flight (submit, wait, validate_mvcc, block_updates), with and without block_pvt_updates.
Kernel times come from a separate torch.profiler run.  Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402
import pvtupdatecases as cases  # noqa: E402

ENT = [("VALIDATION_PARAMETER", b"p")]


def shape(n_tx, hot):
    """(transactions in pvtupdatecases' form, committed hashed versions)"""
    r = random.Random(11)
    txs, committed = [], {}
    for t in range(n_tx):
        if r.random() < 0.01:
            if hot and t > 0:
                k = "h%d" % r.randrange(64)
            else:
                k = "c%d" % t
                committed[cases.hkey(k)] = (0, t)
            txs.append(cases.tx(cases.one(md=[(k, ENT)])))
            continue
        keys = ["h%d" % r.randrange(64) for _ in range(2)] if hot else ["k%d.%d" % (t, i) for i in range(2)]
        txs.append(cases.tx(cases.one([(k, r.randbytes(480)) for k in keys])))
    return txs, committed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=12)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    B = pkg.binding
    ctx = B.Context(max_batch=8192)
    ctx.msp_configure([(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table], net.policy_n_of(3), net.principals, net.channel,
                      policies={cases.CC: 0})
    S = B.SLOTS
    out = {}
    for name in ("random", "hot"):
        txs, committed = shape(args.txs, name == "hot")
        rws = cases.rwsets(txs)
        pvt = cases.pvt_of(txs)
        hook = lambda t, part, b: rws[t] if part == "TxReadWriteSet" else b
        blk, info = blockgen.build_block(net, args.txs, 3, {}, seed=17, mutate=hook)
        entries = sorted(committed.items())
        height = [1]

        def fresh():
            ctx.state_versions(entries, 1, capacity=1 << 16)
            height[0] = 1

        fresh()
        flags = ctx.validate_envelopes(info["env_blob"], info["env_off"])
        codes = ctx.validate_mvcc(0, 1, flags).tolist()
        verdict, status, recs = ctx.block_pvt_updates(0, 1, pvt)
        assert verdict == (0, -1, -1, -1) and recs is not None, verdict
        kinds = {k: sum(1 for r in recs if r[1] == k) for k in ("put", "del", "renew")}
        check_ms, upd_ms, loop = [], [], {"with": [], "without": []}
        for _ in range(args.rounds):
            for leg in ("check", "updates"):
                for _ in range(args.calls):
                    t0 = time.perf_counter()
                    if leg == "check":
                        ctx.validate_pvtdata(0, codes, pvt)
                    else:
                        ctx.block_pvt_updates(0, height[0], pvt)
                    (check_ms if leg == "check" else upd_ms).append((time.perf_counter() - t0) * 1e3)
            for leg in ("without", "with"):
                fresh()
                t0 = time.perf_counter()
                for k in range(S):
                    ctx.validate_envelopes_async(k, info["env_blob"], info["env_off"])
                for k in range(args.blocks):
                    slot = k % S
                    tv = ctx.validate_wait(slot, args.txs + 16)
                    ctx.validate_mvcc(slot, height[0], tv)
                    ctx.block_updates(slot, height[0])
                    if leg == "with":
                        ctx.block_pvt_updates(slot, height[0], pvt)
                    height[0] += 1
                    if k + S < args.blocks:
                        ctx.validate_envelopes_async(slot, info["env_blob"], info["env_off"])
                loop[leg].append((time.perf_counter() - t0) * 1e3 / args.blocks)
            # leave slot 0 in the call window of a finished block for the next round's single calls
            fresh()
            ctx.validate_envelopes(info["env_blob"], info["env_off"])
            ctx.validate_mvcc(0, 1, flags)
        kernels = {}
        try:
            import torch
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    ctx.block_pvt_updates(0, 1, pvt)
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                if "pu_" in ev.key or "pv_" in ev.key or "sha256" in ev.key:
                    kernels[ev.key.split("(")[0]] = {"calls": ev.count, "us_avg": ev.device_time_total / max(ev.count, 1)}
        except Exception as e:                           # the profile is an extra: the timings above stand without it
            kernels = {"error": str(e)}
        q = lambda xs: {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}
        out[name] = {"records": kinds, "entries": len(pvt), "valid": codes.count(0),
                     "validate_pvtdata_ms": q(check_ms), "block_pvt_updates_ms": q(upd_ms),
                     "loop_ms_per_block_without": q(loop["without"]), "loop_ms_per_block_with": q(loop["with"]), "kernels": kernels}
    ctx.close()
    res = {"tool": "pvt_updates_bench", "card": card(), "workload": "%d txs, 3 endorsements, %d rounds" % (args.txs, args.rounds), "shapes": out}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
