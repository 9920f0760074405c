"""Cost of CouchDB's key and value checks in the MVCC stage (fabgpu_state_database, development tool).

bench.py's block_replay shape -- a 10k-transaction block, 3 endorsements per transaction by the peers of 4 orgs, NOutOf(3) chaincode
policy -- over 10^6 installed keys of one namespace.  Every transaction reads one key and writes two seeded JSON documents of about
1 KiB.  Legs, each alternating LevelDB and CouchDB mode `--rounds` times in one process (ms per fabgpu_validate_mvcc call, and for
CouchDB the GB/s of JSON values over the whole call):
  docs:     the documents carry no reserved name;
  reserved: 5 % of the transactions carry an "_id" field (INVALID_WRITESET under CouchDB);
  big:      as docs, with one transaction writing an 8 MiB document, which takes the CTA scan (the others take the one-thread scan).
The GB/s counts the value bytes the scans read: every value here is scanned to its end.
  paths:    the crossover of the two scans: about 20 MB of flat documents of one size, through fabgpu_test_couch_values with each scan
            forced (ms per call, median of `--rounds`, the same host-to-device copy in both), per size.
Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
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
from tools.range_bench import NS, install, key, ver  # noqa: E402
import couch_oracle as co  # noqa: E402


def document(rng, size, reserved=False):
    """a flat JSON object of about `size` bytes with string and number members"""
    parts = ['"_id":"doc%d"' % int(rng.integers(1 << 30))] if reserved else []
    n = 0
    while n < size:
        f = "f%d" % len(parts)
        v = '"%s"' % ("x" * int(rng.integers(8, 48))) if rng.random() < 0.6 else "%d.%d" % (int(rng.integers(1 << 30)), int(rng.integers(1000)))
        parts.append('"%s":%s' % (f, v))
        n += len(parts[-1]) + 1
    return ("{" + ",".join(parts) + "}").encode()


def block(n_tx, pool, rng, p_reserved=0.0, big=0):
    txs, nbytes = [], 0
    for t in range(n_tx):
        i, j = (int(x) for x in rng.integers(0, pool, 2))
        docs = [document(rng, 1024, rng.random() < p_reserved), document(rng, 1024)]
        if big and t == n_tx // 2:
            docs[0] = document(rng, big)
        nbytes += sum(len(d) for d in docs)
        txs.append([dict(ns=NS, reads=[(key(i), ver(i))], writes=[(key(i), False, docs[0]), (key(j) + b"w", False, docs[1])])])
    return txs, nbytes


def build(net, txs, seed):
    hook = lambda t, part, b: co.encode(txs[t]) if part == "TxReadWriteSet" else b
    _, info = blockgen.build_block(net, len(txs), 3, {}, seed=seed, mutate=hook)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--txs", type=int, default=10000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    rng = np.random.default_rng(7)
    net = blockgen.Network()
    pool = 1_000_000
    legs = {"docs": block(args.txs, pool, rng), "reserved": block(args.txs, pool, rng, p_reserved=0.05), "big": block(args.txs, pool, rng, big=8 << 20)}
    infos = {name: build(net, txs, 30 + k) for k, (name, (txs, _)) in enumerate(legs.items())}
    ids = [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]
    ctx = pkg.binding.Context(max_batch=8192)
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    B = pkg.binding
    out = dict(card=card(), txs=args.txs, keys=pool)
    for name, info in infos.items():
        ms = {"leveldb": [], "couchdb": []}
        flags = {}
        for r in range(args.rounds + 1):                       # round 0 warms up
            for mode in ("leveldb", "couchdb"):
                install(ctx, pool, False)
                ctx.state_database(B.STATEDB_COUCHDB if mode == "couchdb" else B.STATEDB_LEVELDB)
                tv = ctx.validate_envelopes(info["env_blob"], info["env_off"])
                t0 = time.perf_counter()
                f = ctx.validate_mvcc(0, 1, tv)
                dt = (time.perf_counter() - t0) * 1e3
                if r:
                    ms[mode].append(dt)
                flags[mode] = {str(c): int((f == c).sum()) for c in np.unique(f)}
        nbytes = legs[name][1]
        out[name] = {mode: dict(ms_median=float(np.median(v)), ms_min=float(np.min(v)), ms_max=float(np.max(v)), flags=flags[mode])
                     for mode, v in ms.items()}
        out[name]["json_bytes"] = nbytes
        out[name]["couchdb"]["json_gb_per_s"] = nbytes / (out[name]["couchdb"]["ms_median"] * 1e-3) / 1e9
    out["paths"] = {}
    for size in (512, 2048, 8192, 16384, 32768, 131072):
        vals = [document(rng, size) for _ in range(max(64, (20 << 20) // size))]
        row = {}
        for path, name in ((1, "one_thread_ms"), (2, "cta_ms")):
            ctx.test_couch_values(vals, path)
            t = []
            for _ in range(args.rounds):
                t0 = time.perf_counter()
                ctx.test_couch_values(vals, path)
                t.append((time.perf_counter() - t0) * 1e3)
            row[name] = float(np.median(t))
        out["paths"][str(size)] = row
    ctx.state_database(B.STATEDB_LEVELDB)
    ctx.state_versions([], 0)
    ctx.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
