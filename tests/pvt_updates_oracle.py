"""The block's private update batch, restated: validateAndPreparePvtBatch's batch half (core/ledger/kvledger/txmgmt/validation/
batch_preparer.go:119-160, 341-410) -- addPvtRWSetToPvtUpdateBatch, addEntriesToMetadataUpdates and incrementPvtdataVersionIfNeeded --
over the flags mvcc_oracle leaves, the hashed records updates_oracle.batch gives and the check pvt_oracle.validate makes, as
fabgpu_block_pvt_updates reports it.

Public transactions are in updates_oracle's form; their collections carry a pvt_rwset_hash when `hashes` names them (encode).  A private
entry is [(ns, [(coll, writes, md)])] with writes [(key, value)] (value bytes, None for no value field, DEL) and md [(key, entries)], as
updates_oracle writes a KVRWSet.  The committed private state is {(ns, coll, key): (value, (block, tx))}.  A record is
(tx, op, ns, coll, key, value, hashed_index): op "put" / "del" / "renew"; value a put's bytes, else None; hashed_index a renew's index in
the hashed records, else None."""
import hashlib

from tools import fabricpb as pb
import pvt_oracle as po
import updates_oracle as uo

DEL = uo.DEL
sha = lambda b: hashlib.sha256(b).digest()


# ---- wire form -------------------------------------------------------------------------------------------------------------------
def kvrwset(writes=(), md=()):
    """a private KVRWSet{writes = 3, metadata_writes = 4}"""
    return (b"".join(pb.f_bytes(3, uo._write(uo._b(k), v)) for k, v in writes) +
            b"".join(pb.f_bytes(4, uo._md(uo._b(k), e)) for k, e in md))


def entry(spec):
    """TxPvtReadWriteSet bytes of [(ns, [(coll, writes, md)])]"""
    return b"".join(pb.f_bytes(2, pb.f_bytes(1, ns.encode()) + b"".join(
        pb.f_bytes(2, pb.f_bytes(1, c.encode()) + pb.f_bytes(2, kvrwset(w, m))) for c, w, m in colls)) for ns, colls in spec)


def hashes_of(spec):
    """{(ns, coll): SHA-256 of the collection's rwset} of an entry spec: the pvt_rwset_hash a matching public set carries"""
    return {(ns, c): sha(kvrwset(w, m)) for ns, colls in spec for c, w, m in colls}


def encode(tx, hashes=None):
    """updates_oracle.encode, with CollectionHashedReadWriteSet.pvt_rwset_hash = hashes[(ns, coll)] where given"""
    if tx is None:
        return None
    hashes = hashes or {}
    out = b""
    for ns in tx:
        one = uo.encode([dict(ns, colls=[])])
        body = pb.parse(one, {2: ("ns", "rep_bytes")})["ns"][0]
        for name, hr, hw, hm in ns.get("colls", ()):
            h = b"".join(pb.f_bytes(1, pb.f_bytes(1, uo._b(k)) + uo.mo._version(v, uo.mo._same_part)) for k, v in hr)
            h += b"".join(pb.f_bytes(2, uo._write(uo._b(k), v)) for k, v in hw)
            h += b"".join(pb.f_bytes(3, uo._md(uo._b(k), e)) for k, e in hm)
            c = pb.f_bytes(1, name.encode()) + pb.f_bytes(2, h)
            if (ns["ns"], name) in hashes:
                c += pb.f_bytes(3, hashes[(ns["ns"], name)])
            body += pb.f_bytes(3, c)
        out += pb.f_bytes(2, body)
    return out


# ---- the batch -------------------------------------------------------------------------------------------------------------------
def _walk(e):
    """(writes, metadata-written keys) of an entry that decodes, in wire order: [(ns, coll, key, is_delete, value or None)]"""
    writes, md = [], []
    for _, _, ns, coll, rw in po.entry_colls(e):
        d = pb.parse(rw, {3: ("w", "rep_bytes"), 4: ("md", "rep_bytes")})
        for w in d["w"]:
            x = pb.parse(w, {1: ("k", "bytes"), 2: ("d", "uint"), 3: ("v", "bytes")})
            writes.append((ns, coll, x["k"] or b"", bool(x["d"]), x["v"]))
        for m in d["md"]:
            md.append((ns, coll, pb.parse(m, {1: ("k", "bytes")})["k"] or b""))
    return writes, md


def batch(block_num, codes, rwsets, pvt, hashed):
    """(verdict, status, records or None): codes the stage's final flags, hashed updates_oracle.batch's records (None: incomplete)"""
    verdict, status = po.validate(rwsets, codes, pvt)
    if hashed is None or verdict[0] != po.OK:
        return verdict, status, None
    upd, order, metas = {}, {}, {}                    # key -> [tx, op, value]; key -> (tx, first position in tx); key -> first seen
    for t in sorted(pvt):
        if codes[t] != uo.VALID or status[t][0] != po.OK:
            continue
        writes, md = _walk(pvt[t])
        first = {}
        for pos, (ns, coll, key, is_del, value) in enumerate(writes):
            k = (ns, coll, key)
            if not is_del and value is None:
                return verdict, status, None              # PutValAndMetadata(nil) panics
            upd[k] = [t, "del" if is_del else "put", None if is_del else value]
            first.setdefault(k, pos)
            order[k] = (t, first[k])
        for k in md:
            metas.setdefault(k, len(metas))
    hrec = {(r[2].encode() if isinstance(r[2], str) else r[2], r[3].encode() if isinstance(r[3], str) else r[3], r[4]): (i, r)
            for i, r in enumerate(hashed)}
    renews = []
    for k in metas:                                       # incrementPvtdataVersionIfNeeded, each key on its own
        ns, coll, key = k
        h = hrec.get((ns, coll, sha(key)))
        if h is None or h[1][1] != "put":
            continue                                      # no hashed record, or a DELETE (bytes.Equal(hash, nil) is false)
        i, r = h
        if k not in upd:
            renews.append((r[0], "renew", ns, coll, key, None, i))
            continue
        e = upd[k]
        if e[0] == r[0]:
            continue                                      # the same version
        if r[5] == uo.COMMITTED:
            return verdict, status, None                  # the hashed value hash is the committed one
        if sha(e[2] or b"") == r[5]:
            if e[1] == "del":
                return verdict, status, None              # Put of a nil value: the reference panics
            e[0] = r[0]
    recs = sorted(((e[0], e[1], k[0], k[1], k[2], e[2], None) for k, e in upd.items()), key=lambda x: order[(x[2], x[3], x[4])])
    return verdict, status, recs + sorted(renews, key=lambda x: x[6])


def apply(state, block_num, records, hashed, hashed_values):
    """the committed private state after the batch; renew records resolved as the peer would: GetPrivateData, its version, and
    SHA-256 of the value against the hashed record's value hash (COMMITTED: from hashed_values, updates_oracle's committed values)"""
    new = dict(state)
    for tx, op, ns, coll, key, value, hi in records:
        k = (ns, coll, key)
        if op == "put":
            new[k] = (value, (block_num, tx))
        elif op == "del":
            new.pop(k, None)
        else:
            latest = state.get(k)
            r = hashed[hi]
            vh = hashed_values.get((ns.decode(), coll.decode(), sha(key)), (None,))[0] if r[5] == uo.COMMITTED else r[5]
            if latest is not None and latest[1] != (block_num, tx) and sha(latest[0]) == vh:
                new[k] = (latest[0], (block_num, tx))
    return new
