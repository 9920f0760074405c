"""The private-data check of a block, fabgpu_validate_pvtdata (development tool).

A 10k-transaction block (3 endorsements per transaction, NOutOf(3) chaincode policy) whose public read/write sets carry the
pvt_rwset_hash of each transaction's private data, in three shapes:
  (a) one collection of about 1 KiB of private data per transaction;
  (b) two collections of about 4 KiB each per transaction;
  (c) (a) with one transaction's rwset replaced by one of about 1 MiB -- one thread hashes it, the known cost of the stage.
Per shape: the median and spread of ms per call over `--calls` calls (host clock around the call, which returns with the stream
synchronised), the device time per kernel from torch.profiler, and, as a CPU reference point (not the Go peer, which is not measured),
the host time of hashing the same rwset bytes with hashlib on one thread.  Prints one JSON line, with the card's name and power limit
read in the same run."""
import argparse
import hashlib
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
import pvtcases  # noqa: E402


def shape(n_tx, sizes, big_at=None):
    """(public TxReadWriteSet bytes per transaction, {seq: TxPvtReadWriteSet}, every rwset)"""
    r = random.Random(5)
    rwsets, pvt, all_rw = [], {}, []
    for t in range(n_tx):
        colls = []
        for k, size in enumerate(sizes):
            n_w = 1 if t != big_at else 16
            sz = size if t != big_at else 1 << 16
            colls.append(("c%d" % k, pvtcases.kvrwset(r.randrange(1 << 30), n_writes=n_w, size=sz)))
        nss = [(pvtcases.CC, colls)]
        pvt[t] = pvtcases.entry(nss)
        rwsets.append(pvtcases.public([(pvtcases.CC, [(c, pvtcases.sha(rw)) for c, rw in colls])], dict(((pvtcases.CC, c), rw) for c, rw in colls)))
        all_rw += [rw for _, rw in colls]
    return rwsets, pvt, all_rw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    ctx = pkg.binding.Context(max_batch=8192)
    ctx.msp_configure([(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table], net.policy_n_of(3), net.principals, net.channel,
                      policies={pvtcases.CC: 0})
    shapes = {"one_1KiB_collection": ([1000], None), "two_4KiB_collections": ([4000, 4000], None), "one_1MiB_rwset_among_1KiB": ([1000], 1234)}
    out = {}
    for name, (sizes, big) in shapes.items():
        rwsets, pvt, all_rw = shape(args.txs, sizes, big)
        hook = lambda t, part, b: rwsets[t] if part == "TxReadWriteSet" else b
        _, info = blockgen.build_block(net, args.txs, 3, {}, seed=17, mutate=hook)
        flags = ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist()
        zeros = [0] * len(flags)
        verdict, status = ctx.validate_pvtdata(0, zeros, pvt)
        assert verdict == (0, -1, -1, -1) and all(s[0] == 0 for s in status.values()), (verdict, [s for s in status.values() if s[0]][:3])
        ms = []
        for _ in range(args.calls):
            t0 = time.perf_counter()
            ctx.validate_pvtdata(0, zeros, pvt)
            ms.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        for rw in all_rw:
            hashlib.sha256(rw).digest()
        cpu_ms = (time.perf_counter() - t0) * 1e3
        kernels = {}
        try:
            import torch
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    ctx.validate_pvtdata(0, zeros, pvt)
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                if "pv_" in ev.key or "sha256" in ev.key:
                    kernels[ev.key.split("(")[0]] = {"calls": ev.count, "us_avg": ev.device_time_total / max(ev.count, 1)}
        except Exception as e:                           # the profile is an extra: the timings above stand without it
            kernels = {"error": str(e)}
        out[name] = {"ms_per_call_median": float(np.median(ms)), "ms_per_call_min": float(np.min(ms)), "ms_per_call_max": float(np.max(ms)),
                     "private_bytes": int(sum(len(e) for e in pvt.values())), "rwsets": len(all_rw),
                     "device_flags_valid": int(sum(1 for f in flags if f == 0)), "kernels": kernels,
                     "cpu_reference_hashlib_one_thread_ms": cpu_ms}
    ctx.close()
    res = {"tool": "pvt_bench", "card": card(), "workload": "%d txs, 3 endorsements each, %d calls per shape" % (args.txs, args.calls), "shapes": out}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
