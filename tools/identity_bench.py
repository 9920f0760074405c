"""Identity admission against reconfiguration (development tool): what a channel that gains client certificates costs per block.

Workload: blocks of `--txs` transactions (default 10 000), 3 endorsements each under NOutOf(3); an MSP of 4 endorsing peers and 2 000
clients, with principal bits and de-duplication groups installed; each block has `--new` transactions (default 100) created by
clients the table does not hold yet, one each, and one transaction by each client that was new in an earlier block (the clients keep
transacting), the rest by the 2 000.  Three legs, alternated in one process over `--rounds` rounds,
each starting from the 2 000-client table:
  (a) no admission: three blocks in flight; every block keeps its new clients' transactions at 254;
  (b) list + add: three blocks in flight; after each wait, fabgpu_block_unknown_identities and fabgpu_msp_identities_add of what it
      listed (bits and groups included) -- a block submitted after the add decides those clients;
  (c) reconfigure per block: fabgpu_msp_configure with the new clients (its groups and namespace policies) + principal bits, then the
      block, which drains the slots.
Per leg: ms per block (host clock around the whole run of blocks, which ends synchronised), and the 254s over all blocks; for (b)
the host time per list and per add call.  --profile instead runs leg (b) once under torch.profiler and reports device time per
kernel.  Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import copy
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402

N_BASE = 2000


def ids_of(idents):
    return [(i.serialized, i.mspid, i.xy, i.valid) for i in idents]


def bits_of(net, idents):
    """principal bits of MSP-id member matching (what SatisfiesPrincipal answers for these identities)"""
    return np.array([[i.mspid == p and i.valid for p in net.principals] for i in idents], bool).reshape(len(idents), len(net.principals))


def build(net, n_blocks, n_tx, n_new):
    rng = np.random.default_rng(7)
    blocks = []
    for b in range(n_blocks):
        creators = [net.clients[int(c)] for c in rng.integers(0, N_BASE, n_tx)]
        fresh = net.clients[N_BASE + n_new * b:N_BASE + n_new * (b + 1)]
        earlier = net.clients[N_BASE:N_BASE + n_new * b]
        for t, c in zip(rng.choice(n_tx, len(fresh) + len(earlier), replace=False), fresh + earlier):
            creators[int(t)] = c
        n2 = copy.copy(net)
        n2.clients = creators
        blk, info = blockgen.build_block(n2, n_tx, 3, {}, seed=50 + b)
        blocks.append((info, fresh))
    return blocks


class Leg:
    def __init__(self, P, net):
        self.P, self.net = P, net
        self.base = net.peers + net.clients[:N_BASE]
        self.ctx = P.Context(max_batch=65536)
        self.nodes = net.policy_n_of(3)
        self.pol = {blockgen.CHAINCODE: 0}

    def configure(self, idents):
        self.ctx.msp_configure(ids_of(idents), self.nodes, self.net.principals, self.net.channel, policies=self.pol)
        self.ctx.msp_principal_bits(bits_of(self.net, idents))

    def pipelined(self, blocks, admit):
        """three blocks in flight; admit: list and add after each wait.  Returns (ms per block, 254s over all blocks, list ms, add ms)"""
        self.configure(self.base)
        by_ser = {i.serialized: i for i in self.net.clients}
        # every certificate is its own: a new client's group is any id no other identity has
        group_of = {i.serialized: len(self.base) + k for k, i in enumerate(self.net.clients[N_BASE:])}
        t_list, t_add, admitted = [], [], set()
        n, n254 = len(blocks), 0
        t0 = time.perf_counter()
        for j in range(min(2, n)):
            self.ctx.validate_envelopes_async(j % 3, blocks[j][0]["env_blob"], blocks[j][0]["env_off"])
        for k in range(n):
            if k + 2 < n:
                self.ctx.validate_envelopes_async((k + 2) % 3, blocks[k + 2][0]["env_blob"], blocks[k + 2][0]["env_off"])
            n254 += int((self.ctx.validate_wait(k % 3, len(blocks[k][0]["env_off"])) == 254).sum())
            if admit:
                a = time.perf_counter()
                listed = self.ctx.block_unknown_identities(k % 3)
                t_list.append((time.perf_counter() - a) * 1e3)
                # a block submitted before an earlier add lists what that add admitted: those are in the table already
                new = [by_ser[s] for s, _ in listed if s in by_ser and s not in admitted]
                admitted.update(i.serialized for i in new)
                if new:
                    groups = [group_of[i.serialized] for i in new]
                    bits = bits_of(self.net, new)
                    a = time.perf_counter()
                    self.ctx.msp_identities_add(ids_of(new), groups=groups, bits=bits)
                    t_add.append((time.perf_counter() - a) * 1e3)
        ms = (time.perf_counter() - t0) * 1e3 / n
        return ms, n254, t_list, t_add

    def reconfigure(self, blocks):
        table = list(self.base)
        t0 = time.perf_counter()
        n254 = 0
        for info, fresh in blocks:
            table += fresh
            self.configure(table)
            n254 += int((self.ctx.validate_envelopes(info["env_blob"], info["env_off"]) == 254).sum())
        return (time.perf_counter() - t0) * 1e3 / len(blocks), n254


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))} if xs else None


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--new", type=int, default=100, help="transactions per block created by clients the table does not hold")
    ap.add_argument("--blocks", type=int, default=6, help="blocks per leg")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="run leg (b) once under torch.profiler instead")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    P = pkg.binding
    net = blockgen.Network(n_orgs=4, n_clients=N_BASE + args.new * args.blocks, seed=0x1DE7)
    blocks = build(net, args.blocks, args.txs, args.new)
    leg = Leg(P, net)
    leg.pipelined(blocks[:3], True)                                  # warm-up: tables, buffers, module loads
    res = {"tool": "identity_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsements), NOutOf(3), MSP of 4 peers + %d clients with principal bits and groups, %d new "
                       "clients per block, %d blocks per leg" % (args.txs, N_BASE, args.new, args.blocks)}
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            leg.pipelined(blocks, True)
            torch.cuda.synchronize()
        res["kernels_us_per_call"] = {ev.key.split("(")[0]: {"calls": ev.count, "us_avg": ev.device_time_total / max(ev.count, 1)}
                                      for ev in prof.key_averages() if ev.device_time_total > 0}
    else:
        rounds = []
        for r in range(args.rounds):
            a_ms, a_254, _, _ = leg.pipelined(blocks, False)
            b_ms, b_254, t_list, t_add = leg.pipelined(blocks, True)
            c_ms, c_254 = leg.reconfigure(blocks)
            rounds.append({"a_no_admission": {"ms_per_block": a_ms, "total_254": a_254},
                           "b_list_add": {"ms_per_block": b_ms, "total_254": b_254, "list_ms": stats(t_list), "add_ms": stats(t_add)},
                           "c_reconfigure": {"ms_per_block": c_ms, "total_254": c_254}})
        res["rounds"] = rounds
    leg.ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
