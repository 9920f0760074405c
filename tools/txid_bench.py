"""Block cost of the committed tx-id set (fabgpu_committed_txids; development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction by the peers of 4 orgs, created by a client,
NOutOf(3) chaincode policy.  Three legs alternated `--rounds` times in one process:
  (a) no_set:  no set installed (every flag as without fabgpu_committed_txids);
  (b) set_1e6: 10^6 random ids, none of the block's;
  (c) set_1e7: 10^7 random ids plus 1 % of the block's ids (those transactions are DUPLICATE_TXID).
For each leg: ms per block with every slot in flight and with one blocking call, the device stages (fabgpu_block_timing out[5..9],
FABGPU_BLOCK_EVENTS=1; out[9] is block_decide_kernel), and for (b) / (c) the pipelined loop a peer runs -- submit block k, add 10^4 ids,
submit block k+1 -- with the time of each add call, the install time of the set and the table's bytes.  Prints one JSON line, with the
card's name and power limit read in the same run."""
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
from tools.keylevel_bench import timed  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402

_HEX = np.frombuffer(b"0123456789abcdef", np.uint8)


def random_ids(rng, n):
    """n random canonical ids as (blob, offsets): 64 lowercase hex characters each"""
    raw = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    hexa = np.empty((n, 64), np.uint8)
    hexa[:, 0::2] = _HEX[raw >> 4]
    hexa[:, 1::2] = _HEX[raw & 15]
    return np.ascontiguousarray(hexa.reshape(-1)), (np.arange(n + 1, dtype=np.uint64) * 64).astype(np.uint32)


def with_ids(blob, off, extra):
    """(blob, off) followed by the id strings `extra`"""
    b = np.concatenate([blob, np.frombuffer(b"".join(x.encode() for x in extra), np.uint8)]) if extra else blob
    o = np.concatenate([off, off[-1] + 64 * np.arange(1, len(extra) + 1, dtype=np.uint32)]) if extra else off
    return np.ascontiguousarray(b), np.ascontiguousarray(o.astype(np.uint32))


def install(ctx, blob, off, capacity):
    L = pkg.binding.lib()
    t0 = time.perf_counter()
    ctx._ck(L.fabgpu_committed_txids(ctx._h, blob.ctypes.data_as(ctypes.c_void_p), off.ctypes.data_as(ctypes.c_void_p), None,
                                     ctypes.c_size_t(off.shape[0] - 1), ctypes.c_size_t(capacity)))
    ctx.committed_txids_info()                        # waits for the insert to finish
    return time.perf_counter() - t0


def pipelined_adds(ctx, pinned, eoff, n_tx, slots, blocks, rng):
    """blocks submitted round-robin, 10^4 fresh ids added after each submit: ms per block and each add's ms"""
    L = pkg.binding.lib()
    adds = [random_ids(rng, 10000) for _ in range(blocks)]
    t_add = []
    t0 = time.perf_counter()
    for k in range(blocks):
        if k >= slots:
            ctx.validate_wait(k % slots, n_tx)
        ctx.validate_envelopes_async(k % slots, pinned[k % slots], eoff)
        b, o = adds[k]
        ta = time.perf_counter()
        ctx._ck(L.fabgpu_committed_txids_add(ctx._h, b.ctypes.data_as(ctypes.c_void_p), o.ctypes.data_as(ctypes.c_void_p), None, ctypes.c_size_t(10000)))
        t_add.append((time.perf_counter() - ta) * 1e3)
    for k in range(max(0, blocks - slots), blocks):
        ctx.validate_wait(k % slots, n_tx)
    return (time.perf_counter() - t0) / blocks * 1e3, t_add


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--big", type=int, default=10_000_000, help="ids of leg (c)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    net = blockgen.Network()
    _, info = blockgen.build_block(net, args.txs, 3, {}, seed=17)
    n = info["env_off"].shape[0] - 1
    from oracle import blockval as ob
    from tools import fabricpb as pb

    def txid_of(env):
        hdr = pb.parse(pb.parse(pb.parse(env, ob.S_ENVELOPE)["payload"], ob.S_PAYLOAD)["header"], ob.S_HEADER)
        return pb.parse(hdr["channel_header"], ob.S_CHDR)["tx_id"].decode()
    block_ids = [txid_of(bytes(info["env_blob"][info["env_off"][t]:info["env_off"][t + 1]])) for t in range(n)]
    matching = block_ids[:: 100]                      # 1 % of the block's transactions
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    ctx = pkg.binding.Context(max_batch=8192)
    slots = pkg.binding.SLOTS
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    pinned = []
    for k in range(slots):
        b = ctx.block_buffer(len(info["env_blob"]), slot=k)
        b[:] = np.frombuffer(info["env_blob"], np.uint8)
        pinned.append(b)
    rng = np.random.default_rng(23)
    small = random_ids(rng, 1_000_000)
    big = with_ids(*random_ids(rng, args.big), matching)
    runs = {"no_set": [], "set_1e6": [], "set_1e7": []}
    for _ in range(args.rounds):
        for name in runs:
            r = {}
            if name == "no_set":
                ctx.committed_txids([])
            else:
                blob, off = small if name == "set_1e6" else big
                r["install_s"] = install(ctx, blob, off, off.shape[0] - 1 + 1_000_000)
            r.update(timed(ctx, pinned, info["env_off"], n, slots, 10, 30))
            if name != "no_set":
                r["pipelined_ms_per_block"], adds = pipelined_adds(ctx, pinned, info["env_off"], n, slots, 30, rng)
                r["add_1e4_ms_median"] = float(np.median(adds))
                r["add_1e4_ms_max"] = float(np.max(adds))
                held, slots_n = ctx.committed_txids_info()
                r["ids_held"], r["table_bytes"] = held, slots_n * 36
            runs[name].append(r)
    ctx.committed_txids([])
    ctx.close()
    res = {"tool": "txid_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures, %d blocks in flight; sets of 1e6 random ids and %d random ids + 1 %% "
           "of the block's" % (args.txs, slots, args.big), "runs": runs}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
