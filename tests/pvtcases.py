"""The private-data check's cases with their expected per-entry and block codes written out, and the builders of the public read/write
sets (pvt_rwset_hash included) and the private data they check.

A transaction is [(namespace, [(collection, hash)])] with hash None (absent), b"" (present, empty) or the 32 bytes to carry, or None for
a non-endorser transaction.  Each collection also carries the HashedRWSet of its private writes, key_hash and value_hash derived as
rwset_builder.go derives them (SHA-256 of the key, SHA-256 of the value).  A case is (name, txs, flags, pvt, status, verdict): pvt maps
SeqInBlock to a marshalled TxPvtReadWriteSet, status to (code, ns, coll) per entry, verdict is (code, seq, ns, coll)."""
import hashlib
import random

from tools import fabricpb as pb
import pvt_oracle

CC, OTHER = "mycc", "othercc"
OK, MISMATCH, SKIP, UNDET = 0, 1, 2, 254
NONE = (OK, -1, -1, -1)
sha = lambda b: hashlib.sha256(b).digest()


def kvrwset(seed, n_writes=2, size=24, reads=1, key_prefix=b"pk"):
    """a private KVRWSet{reads = 1, writes = 3}: KVRead{key = 1, version = 2}, KVWrite{key = 1, value = 3}, values from the seed"""
    r = random.Random(seed)
    out = b""
    for i in range(reads):
        out += pb.f_bytes(1, pb.f_bytes(1, key_prefix + b"-r%d" % i) + pb.f_bytes(2, pb.f_uint(1, r.randrange(1, 9)) + pb.f_uint(2, r.randrange(9))))
    for i in range(n_writes):
        out += pb.f_bytes(3, pb.f_bytes(1, key_prefix + b"-w%d-%d" % (seed, i)) + pb.f_bytes(3, r.randbytes(size)))
    return out


def _hashed(rw):
    """the HashedRWSet{hashed_writes = 2} of a private KVRWSet: KVWriteHash{key_hash = 1, value_hash = 3} per write that decodes"""
    out = b""
    try:
        for f, wt, v in pb.fields(rw):
            if f == 3 and wt == 2:
                w = pb.parse(bytes(v), {1: ("k", "bytes"), 3: ("v", "bytes")})
                out += pb.f_bytes(2, pb.f_bytes(1, sha(w["k"] or b"")) + pb.f_bytes(3, sha(w["v"] or b"")))
    except pb.PbError:
        pass
    return out


def public(tx, rws=None):
    """TxReadWriteSet bytes of a transaction; rws: {(ns, coll): private rwset} whose hashed writes the collection carries"""
    if tx is None:
        return None
    rws = rws or {}
    out = b""
    for ns, colls in tx:
        body = pb.f_bytes(1, ns.encode()) + pb.f_bytes(2, pb.f_bytes(1, pb.f_bytes(1, b"pub-" + ns.encode())))
        for cname, h in colls:
            c = pb.f_bytes(1, cname.encode()) + pb.f_bytes(2, _hashed(rws.get((ns, cname), b"")))
            if h is not None:
                c += pb.f_bytes(3, h)
            body += pb.f_bytes(3, c)
        out += pb.f_bytes(2, body)
    return out


def entry(nss):
    """TxPvtReadWriteSet bytes: [(namespace, [(collection, rwset)])]"""
    return b"".join(pb.f_bytes(2, pb.f_bytes(1, ns.encode()) + b"".join(pb.f_bytes(2, pb.f_bytes(1, c.encode()) + pb.f_bytes(2, rw)) for c, rw in colls))
                    for ns, colls in nss)


def flip(rw, at=-1):
    b = bytearray(rw)
    b[at] ^= 1
    return bytes(b)


def _tx_for(nss, hashes=None):
    """a transaction whose public hashes are those of the rwsets of nss (an entry's layout), unless `hashes` overrides one"""
    hashes = hashes or {}
    return [(ns, [(c, hashes.get((ns, c), sha(rw))) for c, rw in colls]) for ns, colls in nss]


def cases():
    out = []
    a, b, c = kvrwset(1), kvrwset(2), kvrwset(3)
    one = [(CC, [("c1", a)])]
    out.append(("match", [_tx_for(one)], [0], {0: entry(one)}, {0: (OK, -1, -1)}, NONE))
    bad = [(CC, [("c1", flip(a))])]
    out.append(("flipped_byte", [_tx_for(one)], [0], {0: entry(bad)}, {0: (MISMATCH, 0, 0)}, (MISMATCH, 0, 0, 0)))
    extra = [(CC, [("c1", a), ("c2", b)])]
    out.append(("collection_not_in_public_set", [_tx_for(one)], [0], {0: entry(extra)}, {0: (MISMATCH, 0, 1)}, (MISMATCH, 0, 0, 1)))
    absent = [(CC, [("c1", None)])]
    out.append(("hashes_absent_skip", [absent], [0], {0: entry(bad)}, {0: (SKIP, -1, -1)}, NONE))
    empty = [(CC, [("c1", b""), ("c2", None)])]
    out.append(("empty_hashes_with_collections", [empty], [0], {0: entry(one)}, {0: (UNDET, -1, -1)}, (UNDET, 0, -1, -1)))
    out.append(("empty_hashes_without_collections", [empty, empty], [0, 0], {0: b"", 1: entry([(CC, [])])},
                {0: (OK, -1, -1), 1: (OK, -1, -1)}, NONE))
    out.append(("flag_not_valid_ignored", [_tx_for(one), _tx_for(one)], [11, 10], {0: entry(bad), 1: entry(bad)},
                {0: (MISMATCH, 0, 0), 1: (MISMATCH, 0, 0)}, NONE))
    out.append(("undetermined_before_valid_mismatch", [_tx_for(one), _tx_for(one)], [254, 0], {0: entry(bad), 1: entry(bad)},
                {0: (MISMATCH, 0, 0), 1: (MISMATCH, 0, 0)}, (UNDET, 0, -1, -1)))
    out.append(("undetermined_after_valid_mismatch", [_tx_for(one), _tx_for(one), _tx_for(one)], [0, 0, 254],
                {0: entry(one), 1: entry(bad), 2: entry(bad)}, {0: (OK, -1, -1), 1: (MISMATCH, 0, 0), 2: (MISMATCH, 0, 0)}, (MISMATCH, 1, 0, 0)))
    # two namespaces with one collection name: retrieveHash takes the collection of the entry's namespace
    two = [(CC, [("c1", a)]), (OTHER, [("c1", b)])]
    swapped = [(OTHER, [("c1", a)])]
    out.append(("two_namespaces_same_collection", [_tx_for(two), _tx_for(two)], [0, 0], {0: entry(list(reversed(two))), 1: entry(swapped)},
                {0: (OK, -1, -1), 1: (MISMATCH, 0, 0)}, (MISMATCH, 1, 0, 0)))
    # several namespaces and collections: the first failure in entry order is the one reported
    many = [(CC, [("c1", a), ("c2", b)]), (OTHER, [("c3", c)])]
    many_bad = [(CC, [("c1", a), ("c2", flip(b, 5))]), (OTHER, [("c3", flip(c))])]
    late_bad = [(CC, [("c1", a), ("c2", b)]), (OTHER, [("c3", flip(c))])]
    out.append(("order_decides_the_reported_failure", [_tx_for(many), _tx_for(many), _tx_for(many)], [11, 0, 0],
                {0: entry(many_bad), 1: entry(late_bad), 2: entry(many_bad)},
                {0: (MISMATCH, 0, 1), 1: (MISMATCH, 1, 0), 2: (MISMATCH, 0, 1)}, (MISMATCH, 1, 1, 0)))
    # an undecodable rwset whose hash matches, before a mismatching collection of the same entry: the mismatch wins
    garbage = b"\x0a\xff\x01ab"
    gm = [(CC, [("c1", garbage), ("c2", flip(b))])]
    g_only = [(CC, [("c1", garbage)])]
    gtx = _tx_for([(CC, [("c1", garbage), ("c2", b)])])
    out.append(("undecodable_before_mismatch", [gtx, gtx], [0, 0], {0: entry(gm), 1: entry(g_only)},
                {0: (MISMATCH, 0, 1), 1: (UNDET, 0, 0)}, (MISMATCH, 0, 0, 1)))
    out.append(("undecodable_alone", [gtx], [0], {0: entry(g_only)}, {0: (UNDET, 0, 0)}, (UNDET, 0, -1, -1)))
    bad_key = pb.f_bytes(3, pb.f_bytes(1, b"k\xff\xfe") + pb.f_bytes(3, b"v"))
    bk = [(CC, [("c1", a), ("c2", bad_key)])]
    out.append(("invalid_utf8_private_key", [_tx_for(bk)], [0], {0: entry(bk)}, {0: (UNDET, 0, 1)}, (UNDET, 0, -1, -1)))
    out.append(("empty_entry", [_tx_for(one)], [0], {0: b""}, {0: (OK, -1, -1)}, NONE))
    out.append(("non_endorser_transaction", [None, _tx_for(one)], [0, 0], {0: entry(one), 1: entry(one)},
                {0: (UNDET, -1, -1), 1: (OK, -1, -1)}, (UNDET, 0, -1, -1)))
    big = kvrwset(9, n_writes=16, size=1 << 16)
    assert len(big) > 1 << 20
    bigs = [(CC, [("c1", big)])]
    out.append(("one_mib_rwset", [_tx_for(bigs), _tx_for(bigs), _tx_for(one)], [0, 0, 0],
                {0: entry(bigs), 1: entry([(CC, [("c1", flip(big, len(big) // 2))])]), 2: entry(one)},
                {0: (OK, -1, -1), 1: (MISMATCH, 0, 0), 2: (OK, -1, -1)}, (MISMATCH, 1, 0, 0)))
    return out


def rwsets_of(txs, pvt=None):
    """the public TxReadWriteSet bytes of each transaction, hashed writes from the private rwsets the entries hold"""
    out = []
    for t, tx in enumerate(txs):
        rws = {}
        if pvt and t in pvt:
            try:
                rws = {(ns.decode(), c.decode()): rw for _, _, ns, c, rw in pvt_oracle.entry_colls(pvt[t])}
            except (pb.PbError, UnicodeDecodeError):
                rws = {}
        out.append(public(tx, rws))
    return out


def seeded(seed, n, p_pvt=0.7):
    """a seeded block's transactions, flags and private data: one to three collections over up to two namespaces per transaction, some
    hashes absent or empty, some private data flipped, undecodable or with an extra collection, some flags other than VALID"""
    r = random.Random(seed)
    txs, flags, pvt = [], [], {}
    for t in range(n):
        if r.random() < 0.03:
            txs.append(None); flags.append(r.choice((0, 254))); pvt[t] = entry([(CC, [("c1", kvrwset(t))])])
            continue
        nss = []
        for ns in ([CC] if r.random() < 0.7 else [CC, OTHER]):
            nss.append((ns, [("c%d" % k, kvrwset(seed * 7919 + t * 31 + k, r.randrange(0, 4), r.randrange(1, 200))) for k in range(r.randrange(1, 3))]))
        hashes = {}
        x = r.random()
        if x < 0.05:
            hashes = {(ns, c): None for ns, cs in nss for c, _ in cs}
        elif x < 0.08:
            hashes = {(ns, c): b"" for ns, cs in nss for c, _ in cs}
        txs.append(_tx_for(nss, hashes))
        flags.append(r.choice((0, 0, 0, 0, 254, 11, 10)))
        if r.random() > p_pvt:
            continue
        y = r.random()
        if y < 0.08:
            ns, cs = nss[-1]
            nss[-1] = (ns, cs[:-1] + [(cs[-1][0], flip(cs[-1][1] or b"\x00"))])
        elif y < 0.11:
            nss[0] = (nss[0][0], nss[0][1] + [("extra", kvrwset(t + 1))])
        elif y < 0.13:
            nss = [(nss[0][0], [(nss[0][1][0][0], b"\x1a\x05ab")])]
            txs[-1] = _tx_for(nss)
        elif y < 0.15:
            nss = []
        pvt[t] = entry(nss)
    return txs, flags, pvt
