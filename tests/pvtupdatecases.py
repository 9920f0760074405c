"""The private update batch's cases with their expected records written out, and the builders of their blocks.

A transaction is made by `tx(spec)` from a private entry spec [(ns, [(coll, writes, md)])] (pvt_updates_oracle's form): its public
read/write set carries, per collection, the hashed writes and hashed metadata writes of the private ones (key_hash = SHA-256 of the key,
value_hash = SHA-256 of the value -- of b"" when the value field is absent) and the rwset's pvt_rwset_hash; `hw` / `hm` replace the
hashed side, `hash_ok=False` leaves the pvt_rwset_hash out (containsPvtWrites is false), `entry=False` gives no private entry.

A case is (name, committed, tv, txs, want): committed = (versions, values, private state) -- updates_oracle's {(ns, coll, key): version}
and {(ns, coll, key): (value, metadata)} with the key hash for hashed keys, and {(ns, coll, key): (value, version)}; tv the validator's
flags; want the records (pvt_updates_oracle's form) at block 1, or None."""
import random

import pvt_updates_oracle as puo
import updates_oracle as uo

CC = "mycc"
DEL = uo.DEL
sha = puo.sha
B = lambda s: s.encode()


def tx(spec, hw=None, hm=None, hash_ok=True, entry=True, flip=False):
    """{"pub": updates_oracle transaction, "hashes": {(ns, coll): pvt_rwset_hash}, "entry": entry bytes or None}"""
    pub = []
    hashes = puo.hashes_of(spec) if hash_ok else {}
    for ns, colls in spec:
        cs = []
        for c, writes, md in colls:
            w = hw.get((ns, c)) if hw and (ns, c) in hw else [(sha(B(k)), v if v is DEL else sha(v or b"")) for k, v in writes]
            m = hm.get((ns, c)) if hm and (ns, c) in hm else [(sha(B(k)), e) for k, e in md]
            cs.append((c, [], w, m))
        pub.append(dict(ns=ns, colls=cs))
    e = puo.entry(spec) if entry else None
    if flip and e:
        e = e[:-1] + bytes([e[-1] ^ 1])
    return dict(pub=pub, hashes=hashes, entry=e)


def rwsets(txs):
    return [puo.encode(t["pub"], t["hashes"]) for t in txs]


def pvt_of(txs):
    return {i: t["entry"] for i, t in enumerate(txs) if t["entry"] is not None}


def hkey(k):
    return (CC, "c1", sha(B(k)))


def one(writes=(), md=(), coll="c1"):
    return [(CC, [(coll, list(writes), list(md))])]


EMPTY = ({}, {}, {})
ENT = [("VALIDATION_PARAMETER", b"p")]


def cases():
    out = []
    k1, k2, k4, k9 = b"k1", b"k2", b"k4", b"k9"
    r = lambda t, op, key, value=None, h=None: (t, op, B(CC), b"c1", key, value, h)
    out.append(("last_writer_across_transactions", EMPTY, [0, 0], [tx(one([("k1", b"a")])), tx(one([("k1", b"b")]))],
                [r(1, "put", k1, b"b")]))
    out.append(("last_writer_within_one_kvrwset", EMPTY, [0], [tx(one([("k1", b"a"), ("k2", b"x"), ("k1", b"b")]))],
                [r(0, "put", k1, b"b"), r(0, "put", k2, b"x")]))
    twice = [(CC, [("c1", [("k2", b"x"), ("k1", b"a")], [])]), (CC, [("c1", [("k2", b"x"), ("k1", b"a")], [])])]
    out.append(("repeated_namespace_entry", EMPTY, [0], [tx(twice)], [r(0, "put", k2, b"x"), r(0, "put", k1, b"a")]))
    committed1 = ({hkey("k1"): (0, 0)}, {hkey("k1"): (sha(b"old"), None)}, {(B(CC), b"c1", k1): (b"old", (0, 0))})
    out.append(("delete", committed1, [0], [tx(one([("k1", DEL)]))], [r(0, "del", k1)]))
    out.append(("present_empty_value", EMPTY, [0], [tx(one([("k1", b"")]))], [r(0, "put", k1, b"")]))
    out.append(("absent_value_incomplete", EMPTY, [0], [tx(one([("k1", None)]))], None))
    out.append(("not_valid_skipped_and_missing_entries", EMPTY, [11, 0, 0, 0],
                [tx(one([("k1", b"a")])), tx(one([("k2", b"b")]), hash_ok=False), tx(one([("k9", b"c")]), entry=False), tx(one([("k4", b"d")]))],
                [r(3, "put", k4, b"d")]))
    committed2 = ({hkey("k1"): (0, 0), hkey("k2"): (0, 1)}, {hkey("k1"): (sha(b"old"), None), hkey("k2"): (sha(b"w0"), None)},
                  {(B(CC), b"c1", k1): (b"old", (0, 0)), (B(CC), b"c1", k2): (b"w0", (0, 1))})
    # k1: a hashed metadata-only write, the value hash the committed one; k2: the hashed side puts SHA-256(w0) from the block
    out.append(("renew_committed_keys", committed2, [0, 0],
                [tx(one(md=[("k1", ENT)])), tx(one(md=[("k2", ENT)]), hw={(CC, "c1"): [(sha(k2), sha(b"w0"))]})],
                [r(0, "renew", k1, None, 0), r(1, "renew", k2, None, 1)]))
    out.append(("in_block_renewal_matching_hash", EMPTY, [0, 0], [tx(one([("k1", b"a")])), tx(one(md=[("k1", ENT)]))],
                [r(1, "put", k1, b"a")]))
    out.append(("in_block_renewal_mismatched_hash", EMPTY, [0, 0],
                [tx(one([("k1", b"a")]), hw={(CC, "c1"): [(sha(k1), sha(b"other"))]}), tx(one(md=[("k1", ENT)]))],
                [r(0, "put", k1, b"a")]))
    out.append(("metadata_write_then_hashed_delete", committed1, [0, 0], [tx(one(md=[("k1", ENT)])), tx(one([("k1", DEL)]))],
                [r(1, "del", k1)]))
    out.append(("metadata_write_dropped_in_hashed_space", EMPTY, [0], [tx(one(md=[("k9", ENT)]))], []))
    out.append(("metadata_delete_without_entries", committed1, [0], [tx(one(md=[("k1", None)]))], [r(0, "renew", k1, None, 0)]))
    # the latest private value is a Delete, the hashed PUT's value hash is SHA-256 of nothing: Put(nil) panics in the reference
    out.append(("delete_versus_empty_value_hash", committed1, [0, 0],
                [tx(one([("k1", DEL)]), hw={(CC, "c1"): [(sha(k1), sha(b""))]}), tx(one(md=[("k1", ENT)]))], None))
    out.append(("mismatch_verdict", EMPTY, [0, 0], [tx(one([("k1", b"a")])), tx(one([("k2", b"b")]), flip=True)], None))
    garbage = dict(tx(one([("k2", b"b")])))
    g = puo.pb.f_bytes(2, puo.pb.f_bytes(1, B(CC)) + puo.pb.f_bytes(2, puo.pb.f_bytes(1, b"c1") + puo.pb.f_bytes(2, b"\x0a\xff\x01ab")))
    garbage.update(entry=g, hashes={(CC, "c1"): sha(b"\x0a\xff\x01ab")})
    out.append(("undetermined_verdict", EMPTY, [0, 0], [tx(one([("k1", b"a")])), garbage], None))
    out.append(("incomplete_public_batch", EMPTY, [0, 254], [tx(one([("k1", b"a")])), tx(one([("k2", b"b")]))], None))
    return out


def run_oracle(committed, block_num, txs, tv):
    """(flags, hashed records, verdict, status, records) of one block"""
    versions, values, _ = committed
    codes, _, _ = uo.flags(versions, block_num, [t["pub"] for t in txs], tv)
    hashed = uo.batch(versions, values, block_num, [t["pub"] for t in txs], codes)
    verdict, status, recs = puo.batch(block_num, codes, rwsets(txs), pvt_of(txs), hashed)
    return codes, hashed, verdict, status, recs


def seeded(seed, n, pool=12):
    """a seeded block over a hot pool of private keys: puts, deletes, empty values, metadata writes (some on keys written earlier in the
    block), now and then a mismatched hashed value, a transaction without an entry or with a flag other than VALID"""
    rg = random.Random(seed)
    txs, tv = [], []
    for t in range(n):
        writes, md = [], []
        for _ in range(rg.randrange(0, 3)):
            k = "k%d" % rg.randrange(pool)
            x = rg.random()
            writes.append((k, DEL if x < 0.2 else b"" if x < 0.25 else b"v%d.%d.%d" % (seed, t, len(writes))))
        if rg.random() < 0.3:
            md.append(("k%d" % rg.randrange(pool), None if rg.random() < 0.2 else [("VALIDATION_PARAMETER", b"s%d" % t)]))
        if not writes and not md:
            md.append(("k%d" % rg.randrange(pool), ENT))
        hw = None
        if writes and rg.random() < 0.1:
            hw = {(CC, "c1"): [(sha(B(k)), v if v is DEL else sha(b"x" + (v or b""))) for k, v in writes]}
        txs.append(tx(one(writes, md), hw=hw, entry=rg.random() > 0.05))
        tv.append(rg.choice((0, 0, 0, 0, 0, 0, 11)))
    return txs, tv
