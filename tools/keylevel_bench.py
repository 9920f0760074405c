"""Block cost of a key policy table (fabgpu_key_policies; development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction by the peers of 4 orgs, created by a client,
NOutOf(3) chaincode policy -- except that every transaction writes two public keys drawn from a pool of 2 000.  Three legs alternated
`--rounds` times in one process:
  (a) no_table: no key policy table (every flag as without fabgpu_key_policies);
  (b) table:    a 10^5-entry table in which half of the pool carries a validation parameter every endorsement set satisfies;
  (c) deps:     (b), plus 1 % of the transactions metadata-writing a key that later transactions write (in-block dependencies);
  (d) hot:      (b), every transaction also writing and metadata-writing one hot key (asset-transfer with per-asset owners on one
                asset): every transaction depends on every earlier one, the resolve stage's worst case.
For each leg: ms per block with every slot in flight, one blocking call, and the device stages (fabgpu_block_timing out[5..9],
FABGPU_BLOCK_EVENTS=1; out[9] includes the resolve kernel).  Also the cost of a 10^3-entry update into a 10^6-entry table.  Prints one
JSON line, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402


def timed(ctx, pinned, eoff, n_tx, slots, reps_single, reps_flight):
    os.environ["FABGPU_BLOCK_EVENTS"] = "1"
    ref = ctx.validate_envelopes(pinned[0], eoff).copy()
    stages = []
    for _ in range(reps_single):
        assert (ctx.validate_envelopes(pinned[0], eoff) == ref).all()
        stages.append(list(ctx.block_timing()[5:10]))
    os.environ["FABGPU_BLOCK_EVENTS"] = "0"
    t0 = time.perf_counter()
    for _ in range(reps_single):
        fl = ctx.validate_envelopes(pinned[0], eoff)
    single = (time.perf_counter() - t0) / reps_single * 1e3
    assert (fl == ref).all()
    for k in range(slots):
        ctx.validate_envelopes_async(k, pinned[k], eoff)
        ctx.validate_wait(k, n_tx)
    t0 = time.perf_counter()
    for k in range(reps_flight):
        if k >= slots:
            assert (ctx.validate_wait(k % slots, n_tx) == ref).all()
        ctx.validate_envelopes_async(k % slots, pinned[k % slots], eoff)
    for k in range(max(0, reps_flight - slots), reps_flight):
        assert (ctx.validate_wait(k % slots, n_tx) == ref).all()
    flight = (time.perf_counter() - t0) / reps_flight * 1e3
    med = np.median(np.array(stages), axis=0).tolist()
    return {"ms_per_block_in_flight": flight, "single_call_ms": single, "stage_us_median": dict(zip(["walk", "creator", "endorsement", "verify", "decide_resolve"], med)),
            "flags": {int(c): int((ref == c).sum()) for c in np.unique(ref)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    rng = np.random.default_rng(5)
    pool = ["key%d" % i for i in range(2000)]
    keys = [list(rng.choice(pool, 2, replace=False)) for _ in range(args.txs)]
    md = {t: [keys[t + 1 + int(rng.integers(0, 50)) if t + 51 < args.txs else t][0]] for t in range(args.txs) if rng.random() < 0.01}
    blocks = {}
    hot = {t: ["hotkey"] for t in range(args.txs)}
    for name, mdw in (("plain", {}), ("deps", md), ("hot", hot)):
        extra = ["hotkey"] if name == "hot" else []
        _, info = blockgen.build_block(net, args.txs, 3, {}, seed=17,
                                       namespaces=lambda t: [(blockgen.CHAINCODE, 1, keys[t] + extra, [], mdw.get(t, []))])
        blocks[name] = info
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    n = net.n_orgs
    # validation parameters: NOutOf(1) over every org (satisfied by any endorsement set), appended after the chaincode policy
    vp_nodes = np.array([(0, 1, 1, n)] + [(1, o, 0, 0) for o in range(n)], np.int32)
    table = {("cc%02d" % (k % 20), "", b"asset%d" % k): 0 for k in range(100000 - 1000)}
    table.update({(blockgen.CHAINCODE, "", k.encode()): 0 for k in pool[:1000]})
    table[(blockgen.CHAINCODE, "", b"hotkey")] = 0
    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)

    def stage(blk):                                    # the block in every slot's pinned buffer
        out = []
        for k in range(slots):
            b = ctx.block_buffer(len(blocks[blk]["env_blob"]), slot=k)
            b[:] = np.frombuffer(blocks[blk]["env_blob"], np.uint8)
            out.append(b)
        return out
    runs = {"no_table": [], "table": [], "deps": [], "hot": []}
    for _ in range(args.rounds):
        for name in ("no_table", "table", "deps", "hot"):
            ctx.key_policies(vp_nodes, table) if name != "no_table" else ctx.key_policies([], {})
            blk = name if name in ("deps", "hot") else "plain"
            runs[name].append(timed(ctx, stage(blk), blocks[blk]["env_off"], args.txs, slots, 10, 30))
    # update cost: 10^3 entries into a 10^6-entry table
    big = {("cc%02d" % (k % 20), "", b"asset%d" % k): 0 for k in range(1000000)}
    t0 = time.perf_counter(); ctx.key_policies(vp_nodes, big); install = time.perf_counter() - t0
    upd = []
    for r in range(5):
        chg = {("cc%02d" % (k % 20), "", b"asset%d" % k): (0 if r % 2 else -1) for k in range(r * 1000, r * 1000 + 1000)}
        chg.update({("new", "", b"n%d-%d" % (r, k)): 0 for k in range(500)})
        t0 = time.perf_counter(); ctx.key_policies_update(vp_nodes, chg); upd.append((time.perf_counter() - t0) * 1e3)
    ctx.close()
    res = {"tool": "keylevel_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures, 2 public writes each from a pool of 2000 keys, %d blocks in flight"
           % (args.txs, slots), "table_entries": len(table), "deps_metadata_writers": len(md),
           "runs": runs, "install_1e6_s": install, "update_1e3_into_1e6_ms": upd}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
