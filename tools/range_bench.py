"""Cost of range queries in the MVCC stage (fabgpu_validate_mvcc) over the ordered key index (development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction by the peers of 4 orgs, NOutOf(3) chaincode
policy -- over installed keys k00000000.. of one namespace.  Legs, alternated `--rounds` times in one process, each with 10^6 and with
`--big` keys installed:
  composite: half the transactions run a prefix range of 10 results (start k<7 digits>, end the prefix + U+10FFFF, as
      GetStateByPartialCompositeKey records one) with raw reads; the other half read and write one key;
  merkle:    half the transactions run a 200-result range recorded as a Merkle summary of max_degree 50;
  contended: transaction 2j writes a new key inside the range of transaction 2j + 1;
  each leg with the index installed (ms per call, install seconds, index bytes) and without one (`*_noindex`: the range transactions
  come back 254 -- the stage's own baseline; the CPU time those 254s then cost the committer is not measured here).
  maintain: 100 blocks of 1000 transactions that each write 10 new keys (10^4 new keys per block), over 10^6 installed keys: ms per
      call with and without the index.
Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import blockgen  # noqa: E402
from tools.policy_bench import card, pkg  # noqa: E402
import range_oracle as ro  # noqa: E402

NS = "mycc"
TOP = "\U0010ffff".encode()


def key(i):
    return b"k%08d" % i


def ver(i):
    return (0, i % 1000)


def install(ctx, n, indexed):
    """n keys of NS with version (0, i % 1000), built as arrays: seconds for the call"""
    L = pkg.binding.lib()
    nb = np.frombuffer(NS.encode() * n, np.uint8)
    no = (np.arange(n + 1, dtype=np.uint64) * len(NS)).astype(np.uint32)
    cb = np.zeros(1, np.uint8)
    co = np.zeros(n + 1, np.uint32)
    idx = np.arange(n, dtype=np.int64)
    kb = np.empty((n, 9), np.uint8)
    kb[:, 0] = ord("k")
    for p in range(8):
        kb[:, 8 - p] = ord("0") + (idx // 10 ** p) % 10
    kb = np.ascontiguousarray(kb.reshape(-1))
    ko = (np.arange(n + 1, dtype=np.uint64) * 9).astype(np.uint32)
    v = np.zeros((n, 2), np.uint64)
    v[:, 1] = idx % 1000
    v = np.ascontiguousarray(v.reshape(-1))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    fn = L.fabgpu_state_versions_indexed if indexed else L.fabgpu_state_versions
    t0 = time.perf_counter()
    ctx._ck(fn(ctx._h, p(nb), p(no), p(cb), p(co), p(kb), p(ko), p(v), ctypes.c_size_t(n), ctypes.c_uint64(1), ctypes.c_size_t(n + 2_000_000)))
    return time.perf_counter() - t0


def composite_block(n_tx, pool, rng):
    txs = []
    for t in range(n_tx):
        if t % 2:
            base = int(rng.integers(0, pool // 10)) * 10
            pre = b"k%07d" % (base // 10)
            txs.append([dict(ns=NS, ranges=[(pre, pre + TOP, True, [(key(i), ver(i)) for i in range(base, base + 10)])])])
        else:
            i = int(rng.integers(0, pool))
            txs.append([dict(ns=NS, reads=[(key(i), ver(i))], writes=[(key(i), False)])])
    return txs


def merkle_block(n_tx, pool, rng):
    txs, cache = [], {}
    for t in range(n_tx):
        if t % 2:
            base = int(rng.integers(0, pool // 200)) * 200
            if base not in cache:
                cache[base] = ro.summary_of([(key(i), ver(i)) for i in range(base, base + 200)], 50)
            txs.append([dict(ns=NS, ranges=[(key(base), key(base + 200), True, cache[base])])])
        else:
            i = int(rng.integers(0, pool))
            txs.append([dict(ns=NS, reads=[(key(i), ver(i))], writes=[(key(i), False)])])
    return txs


def contended_block(n_tx, pool, rng):
    txs = []
    for t in range(0, n_tx, 2):
        base = int(rng.integers(0, pool // 10)) * 10
        pre = b"k%07d" % (base // 10)
        txs.append([dict(ns=NS, writes=[(pre + b"5x%d" % t, False)])])
        txs.append([dict(ns=NS, ranges=[(pre, pre + TOP, True, [(key(i), ver(i)) for i in range(base, base + 10)])])])
    return txs


def insert_block(n_tx, b):
    return [[dict(ns=NS, writes=[(b"n%03d_%05d_%d" % (b, t, j), False) for j in range(10)])] for t in range(n_tx)]


def build(net, txs, seed):
    hook = lambda t, part, b: ro.encode(txs[t]) if part == "TxReadWriteSet" else b
    _, info = blockgen.build_block(net, len(txs), 3, {}, seed=seed, mutate=hook)
    return info


def stage_ms(ctx, info, reps):
    """ms per validate_mvcc call on the block (validated first, outside the timing); the flags of the first call"""
    out, first = [], None
    for _ in range(reps):
        tv = ctx.validate_envelopes(info["env_blob"], info["env_off"])
        h = ctx.state_versions_info()[2]
        t0 = time.perf_counter()
        f = ctx.validate_mvcc(0, h, tv)
        out.append((time.perf_counter() - t0) * 1e3)
        first = f if first is None else first
    return out, first


def summary(ms, f=None):
    r = dict(ms_median=float(np.median(ms)), ms_min=float(np.min(ms)), ms_max=float(np.max(ms)))
    if f is not None:
        r["first_flags"] = {str(c): int((f == c).sum()) for c in np.unique(f)}
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--big", type=int, default=10_000_000, help="keys of the large install")
    ap.add_argument("--maintain", type=int, default=100, help="blocks of the maintenance sequence")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    rng = np.random.default_rng(5)
    net = blockgen.Network()
    pool = 1_000_000
    blocks = {"composite": build(net, composite_block(args.txs, pool, rng), 17), "merkle": build(net, merkle_block(args.txs, pool, rng), 18),
              "contended": build(net, contended_block(args.txs, pool, rng), 19)}
    ins = [build(net, insert_block(1000, b), 100 + b) for b in range(args.maintain)]
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    ctx = pkg.binding.Context(max_batch=8192)
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    runs = {}
    for _ in range(args.rounds):
        for keys in (1_000_000, args.big):
            tag = "1e6" if keys == 1_000_000 else "big"
            for indexed in (True, False):
                inst = install(ctx, keys, indexed)
                info = ctx.state_index_info()
                runs.setdefault("install_%s%s" % (tag, "" if indexed else "_noindex"), []).append(
                    dict(install_s=inst, index_bytes=info[2], index_entries=info[1]))
                for leg, blk in blocks.items():
                    if leg != "composite":
                        install(ctx, keys, indexed)
                    ms, f = stage_ms(ctx, blk, 5)
                    runs.setdefault("%s_%s%s" % (leg, tag, "" if indexed else "_noindex"), []).append(summary(ms, f))
        for indexed in (True, False):
            install(ctx, 1_000_000, indexed)
            ms = []
            for info in ins:
                m, _ = stage_ms(ctx, info, 1)
                ms += m
            r = summary(ms)
            r["index_entries_after"] = ctx.state_index_info()[1]
            runs.setdefault("maintain_1e6%s" % ("" if indexed else "_noindex"), []).append(r)
    ctx.state_versions([], 0)
    ctx.close()
    res = {"tool": "range_bench", "card": card(),
           "workload": "%d txs x (1 creator + 3 endorsement) signatures; half of them a 10-result prefix range (composite), a 200-result "
           "Merkle range of max_degree 50 (merkle), or a range after an in-range write (contended); %d insert blocks of 10^4 new keys" % (args.txs, args.maintain),
           "runs": runs}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
