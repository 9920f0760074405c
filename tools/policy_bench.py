"""Decide-stage cost of role principals and ImplicitMeta policies (development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction by the peers of 4 orgs, created by a client --
validated under two configurations, alternated `--rounds` times in one process:
  (a) member: today's MSP-id principals, NOutOf(3) over SignedBy of every org, no principal bits;
  (b) stock:  ImplicitMeta MAJORITY over each org's OR('OrgN.peer'), with principal bits (fabgpu_msp_principal_bits).
Every flag must be VALID under both.  For each leg: ms per block with every slot in flight, one blocking call, and the
block_decide_kernel stage (fabgpu_block_timing out[9], FABGPU_BLOCK_EVENTS=1).  Prints one JSON line, with the card's name and
power limit read in the same run."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("fabric-mod_b200")
from tools import blockgen  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, limit = [x.strip() for x in out.splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as ex:                       # the numbers stay meaningful only with the card named: say why it is missing
        return {"error": repr(ex)}


def configs(net):
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    n = net.n_orgs
    # ImplicitMeta(n // 2 + 1) over n NOutOf(1) nodes, each over SignedBy(org o's peer principal)
    stock = np.array([(2, n // 2 + 1, 1, n)] + [(0, 1, 1 + n + o, 1) for o in range(n)] + [(1, o, 0, 0) for o in range(n)], np.int32)
    peer_of = {i.serialized: i.mspid for i in net.peers + net.peers_alt}
    bits = np.array([[peer_of.get(i.serialized) == net.principals[o] and i.valid for o in range(n)] for i in net.msp_table], bool)
    return {"member": (ids, net.policy_n_of(3), net.principals, None),
            "stock": (ids, stock, ["%s.peer" % p for p in net.principals], bits)}


def leg(ctx, cfg, net, pinned, eoff, n_tx, slots, reps_single, reps_flight):
    ids, nodes, principals, bits = cfg
    ctx.msp_configure(ids, nodes, principals, net.channel)
    if bits is not None:
        ctx.msp_principal_bits(bits)
    return timed(ctx, pinned, eoff, n_tx, slots, reps_single, reps_flight)


def timed(ctx, pinned, eoff, n_tx, slots, reps_single, reps_flight):
    """The configuration ctx holds, on the block in `pinned` (one copy per slot): every flag must be VALID."""
    os.environ["FABGPU_BLOCK_EVENTS"] = "1"
    decide = []
    for _ in range(3):
        assert not ctx.validate_envelopes(pinned[0], eoff).any()
    for _ in range(reps_single):
        ctx.validate_envelopes(pinned[0], eoff)
        decide.append(ctx.block_timing()[9])
    os.environ["FABGPU_BLOCK_EVENTS"] = "0"
    t0 = time.perf_counter()
    for _ in range(reps_single):
        fl = ctx.validate_envelopes(pinned[0], eoff)
    single = (time.perf_counter() - t0) / reps_single * 1e3
    assert not fl.any()
    for k in range(slots):
        ctx.validate_envelopes_async(k, pinned[k], eoff)
        assert not ctx.validate_wait(k, n_tx).any()
    t0 = time.perf_counter()
    for k in range(reps_flight):
        if k >= slots:
            assert not ctx.validate_wait(k % slots, n_tx).any()
        ctx.validate_envelopes_async(k % slots, pinned[k % slots], eoff)
    for k in range(max(0, reps_flight - slots), reps_flight):
        assert not ctx.validate_wait(k % slots, n_tx).any()
    flight = (time.perf_counter() - t0) / reps_flight * 1e3
    return {"ms_per_block_in_flight": flight, "single_call_ms": single, "block_decide_kernel_us_median": float(np.median(decide)),
            "block_decide_kernel_us_min": float(np.min(decide))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    _, info = blockgen.build_block(net, args.txs, 3, {}, seed=17)
    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    eblob, eoff = info["env_blob"], info["env_off"]
    pinned = []
    for k in range(slots):
        b = ctx.block_buffer(len(eblob), slot=k)
        b[:] = np.frombuffer(eblob, np.uint8)
        pinned.append(b)
    cfgs = configs(net)
    runs = {"member": [], "stock": []}
    for _ in range(args.rounds):
        for name in ("member", "stock"):
            runs[name].append(leg(ctx, cfgs[name], net, pinned, eoff, args.txs, slots, 10, 30))
    ctx.close()
    res = {"tool": "policy_bench", "card": card(), "workload": "%d txs x (1 creator + 3 endorsement) signatures, 4 orgs + 1 client, %d blocks in flight"
           % (args.txs, slots), "legs": {"member": "NOutOf(3) over MSP-id principals, no bits", "stock": "ImplicitMeta MAJORITY of OR('OrgN.peer'), bits"},
           "runs": runs}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
