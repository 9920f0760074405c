"""Block cost of the v1.3 mode (fabgpu_channel_capability(FABGPU_CAP_V1_3); development tool).

bench.py's block_replay block -- 10k transactions, 3 endorsements each by the peers of 4 orgs, created by a client, NOutOf(3) chaincode
policy -- validated in v2.0 mode and in v1.3 mode with the chaincode's lscc version installed, the two legs alternated `--rounds` times
in one process.  For each leg: ms per block with every slot in flight, one blocking call, and the device stages (fabgpu_block_timing
out[5..9], FABGPU_BLOCK_EVENTS=1; out[9] is block_decide_kernel).  Prints one JSON line, with the card's name and power limit read in
the same run, and each leg's spread (min, max) over the rounds."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import blockgen  # noqa: E402
from tools.keylevel_bench import timed  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    _, info = blockgen.build_block(net, args.txs, 3, {}, seed=11)
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    B = pkg.binding
    ctx = B.Context(max_batch=8192)
    slots = B.SLOTS
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel, policies={blockgen.CHAINCODE: 0})
    ctx.namespace_versions({blockgen.CHAINCODE: "1.0"})
    pinned = []
    for k in range(slots):
        b = ctx.block_buffer(len(info["env_blob"]), slot=k)
        b[:] = np.frombuffer(info["env_blob"], np.uint8)
        pinned.append(b)
    runs = {"v20": [], "v13": []}
    for _ in range(args.rounds):
        for name, cap in (("v20", B.CAP_V2_0), ("v13", B.CAP_V1_3)):
            ctx.channel_capability(cap)
            runs[name].append(timed(ctx, pinned, info["env_off"], args.txs, slots, 10, 30))
    ctx.close()
    assert runs["v20"][0]["flags"] == runs["v13"][0]["flags"], "the two validators disagree on the block_replay block"
    spread = {name: {k: [min(r[k] for r in rs), max(r[k] for r in rs)] for k in ("ms_per_block_in_flight", "single_call_ms")} |
              {"decide_us": [min(r["stage_us_median"]["decide_resolve"] for r in rs), max(r["stage_us_median"]["decide_resolve"] for r in rs)]}
              for name, rs in runs.items()}
    res = {"tool": "legacy_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures, %d blocks in flight" % (args.txs, slots), "spread": spread, "runs": runs}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
