"""Block cost of a private-data collection policy table (fabgpu_collection_policies; development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction by the peers of 4 orgs, created by a client --
except that every transaction writes one public key and one key of collection _implicit_org_<MSPID> of an org that endorses it.  The
chaincode policy is NOutOf(3) over the orgs; each implicit collection maps to its org's OR('OrgN.peer').  Two legs alternated
`--rounds` times in one process:
  (a) no_table: the chaincode policy alone (the collection write falls under it, as without fabgpu_collection_policies);
  (b) table:    the collection table installed: 4 implicit collections of the chaincode plus those of 20 more chaincodes x 10 orgs
                (204 entries), so every transaction satisfies its chaincode policy and one collection policy.
Every flag must be VALID under both.  For each leg: ms per block with every slot in flight, one blocking call, and the
block_decide_kernel stage (fabgpu_block_timing out[9], FABGPU_BLOCK_EVENTS=1).  Prints one JSON line, with the card's name and
power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg, timed  # noqa: E402


def configuration(net):
    """(identities, nodes, {(namespace, collection): root}): root 0 = NOutOf(3) over SignedBy of every org, root 5 + 2o = OR(org o)"""
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    n = net.n_orgs
    nodes = np.concatenate([net.policy_n_of(3), np.array([r for o in range(n) for r in ((0, 1, n + 2 + 2 * o, 1), (1, o, 0, 0))], np.int32)])
    org_root = lambda o: n + 1 + 2 * o
    table = {(blockgen.CHAINCODE, "_implicit_org_%s" % net.principals[o]): org_root(o) for o in range(n)}
    for k in range(20):
        for o in range(10):
            table[("cc%02d" % k, "_implicit_org_Org%dMSP" % (o + 1))] = org_root(o % n)
    return ids, nodes, table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    # build_block's endorsers of transaction t are the peers of orgs t, t + 1, t + 2 (mod 4): org t % 4 always endorses
    coll = lambda t: [(blockgen.CHAINCODE, 1, 1, [("_implicit_org_%s" % net.principals[t % net.n_orgs], 1, 0, 0)])]
    _, info = blockgen.build_block(net, args.txs, 3, {}, seed=17, namespaces=coll)
    ids, nodes, table = configuration(net)
    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    eblob, eoff = info["env_blob"], info["env_off"]
    pinned = []
    for k in range(slots):
        b = ctx.block_buffer(len(eblob), slot=k)
        b[:] = np.frombuffer(eblob, np.uint8)
        pinned.append(b)
    ctx.msp_configure(ids, nodes, net.principals, net.channel)
    runs = {"no_table": [], "table": []}
    for _ in range(args.rounds):
        for name in ("no_table", "table"):
            ctx.collection_policies(table if name == "table" else None)
            runs[name].append(timed(ctx, pinned, eoff, args.txs, slots, 10, 30))
    ctx.close()
    res = {"tool": "collection_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures, 4 orgs + 1 client, 1 public + 1 collection write each, %d blocks in flight"
           % (args.txs, slots), "table_entries": len(table),
           "legs": {"no_table": "NOutOf(3) chaincode policy only", "table": "chaincode policy + the written implicit collection's OR('OrgN.peer')"},
           "runs": runs}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
