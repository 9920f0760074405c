"""Reference restatement of the ledger's private-data check, validateAndPreparePvtBatch's check path
(core/ledger/kvledger/txmgmt/validation/batch_preparer.go:119-188), over a block's public read/write sets and the private data a caller
holds: one marshalled rwset.TxPvtReadWriteSet per SeqInBlock.

Each entry gets its outcome as if its transaction were VALID:
  SKIP      containsPvtWrites (types.go:49-58) is false: no CollectionHashedReadWriteSet carries a pvt_rwset_hash (:136-138).  A present
            but empty hash is non-nil under golang/protobuf v1.3.3 (recalled, unverified): a transaction whose only hashes are such is
            UNDET when the entry holds a collection, OK when it holds none.
  MISMATCH  validatePvtdata (:166-181): the first collection, through the namespaces and their collections in order, whose
            SHA-256(rwset) differs from retrieveHash(ns, coll) (types.go:62-78).  All hashes before any decode (:146-156).
  UNDET     TxPvtRwSetFromProtoMsg (rwset_proto_util.go:266-303) decoding an rwset as a KVRWSet fails (wire rules of tools/fabricpb.py,
            strings must be valid UTF-8); the entry's outer levels do not parse; the transaction's read/write set is not reached (None).
The block's verdict: the entry with the smallest seq whose outcome is MISMATCH or UNDET and whose flag is VALID or 254 (:133-135 skips
every other flag) decides -- MISMATCH at (seq, ns, coll) when its flag is VALID, else UNDET at seq."""
import hashlib

from tools import fabricpb as pb

OK, MISMATCH, SKIP, UNDET = 0, 1, 2, 254
VALID, NOT_VALIDATED = 0, 254


def _utf8(b):
    try:
        bytes(b).decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def _strs(*items):
    if not all(_utf8(x) for x in items):
        raise pb.PbError("invalid UTF-8")


def public_colls(rwset):
    """TxReadWriteSet{ns_rwset = 2}: [(namespace, [(collection_name, has_hash, hash)])]; NsReadWriteSet{namespace = 1,
    collection_hashed_rwset = 3}, CollectionHashedReadWriteSet{collection_name = 1, pvt_rwset_hash = 3}, the last occurrence winning"""
    out = []
    for nsb in pb.parse(rwset, {1: ("dm", "uint"), 2: ("ns", "rep_bytes")})["ns"]:
        ns = pb.parse(nsb, {1: ("name", "bytes"), 2: ("kv", "bytes"), 3: ("colls", "rep_bytes")})
        colls = []
        for cb in ns["colls"]:
            c = pb.parse(cb, {1: ("name", "bytes"), 2: ("h", "bytes"), 3: ("hash", "bytes")})
            colls.append((c["name"] or b"", c["hash"] is not None, c["hash"]))
        out.append((ns["name"] or b"", colls))
    return out


def contains_pvt_writes(pub):
    """types.go:49-58 -> OK (a non-empty hash), 'empty' (present hashes, all empty) or SKIP"""
    hashes = [h for _, colls in pub for _, has, h in colls if has]
    return OK if any(hashes) else "empty" if hashes else SKIP


def retrieve_hash(pub, ns, coll):
    """types.go:62-78"""
    for name, colls in pub:
        if name != ns:
            continue
        for cname, has, h in colls:
            if cname == coll:
                return h if has else None
    return None


def entry_colls(entry):
    """TxPvtReadWriteSet{data_model = 1, ns_pvt_rwset = 2}, NsPvtReadWriteSet{namespace = 1, collection_pvt_rwset = 2},
    CollectionPvtReadWriteSet{collection_name = 1, rwset = 2}: [(ns_i, coll_i, ns, coll, rwset)]; PbError when a level does not parse"""
    out = []
    for i, nsb in enumerate(pb.parse(entry, {1: ("dm", "uint"), 2: ("ns", "rep_bytes")})["ns"]):
        ns = pb.parse(nsb, {1: ("name", "rep_bytes"), 2: ("colls", "rep_bytes")})
        _strs(*ns["name"])
        name = ns["name"][-1] if ns["name"] else b""
        for j, cb in enumerate(ns["colls"]):
            c = pb.parse(cb, {1: ("name", "rep_bytes"), 2: ("rw", "bytes")})
            _strs(*c["name"])
            out.append((i, j, name, c["name"][-1] if c["name"] else b"", c["rw"] or b""))
    return out


def _read(b):
    r = pb.parse(b, {1: ("key", "rep_bytes"), 2: ("ver", "rep_bytes")})
    _strs(*r["key"])
    for v in r["ver"]:
        pb.parse(v, {1: ("blk", "uint"), 2: ("tx", "uint")})


def decodes(rw):
    """proto.Unmarshal of a KVRWSet with every nested level (DESIGN section 2's field numbers), strings valid UTF-8"""
    try:
        d = pb.parse(rw, {1: ("reads", "rep_bytes"), 2: ("rq", "rep_bytes"), 3: ("w", "rep_bytes"), 4: ("md", "rep_bytes")})
        for r in d["reads"]:
            _read(r)
        for q in d["rq"]:
            x = pb.parse(q, {1: ("s", "rep_bytes"), 2: ("e", "rep_bytes"), 3: ("x", "uint"), 4: ("raw", "rep_bytes"), 5: ("mk", "rep_bytes")})
            _strs(*x["s"], *x["e"])
            for raw in x["raw"]:
                for kv in pb.parse(raw, {1: ("kv", "rep_bytes")})["kv"]:
                    _read(kv)
            for mk in x["mk"]:
                pb.parse(mk, {1: ("d", "uint"), 2: ("l", "uint"), 3: ("h", "rep_bytes")})
        for w in d["w"]:
            x = pb.parse(w, {1: ("k", "rep_bytes"), 2: ("d", "uint"), 3: ("v", "bytes")})
            _strs(*x["k"])
        for m in d["md"]:
            x = pb.parse(m, {1: ("k", "rep_bytes"), 2: ("e", "rep_bytes")})
            _strs(*x["k"])
            for e in x["e"]:
                _strs(*pb.parse(e, {1: ("n", "rep_bytes"), 2: ("v", "bytes")})["n"])
        return True
    except pb.PbError:
        return False


def entry_outcome(rwset, entry):
    """(code, ns_i, coll_i) of one entry; rwset: the transaction's public TxReadWriteSet bytes, None when the walk never reaches it"""
    if rwset is None:
        return (UNDET, -1, -1)
    try:
        pub = public_colls(rwset)
        colls = entry_colls(entry)
    except pb.PbError:
        return (UNDET, -1, -1)
    has = contains_pvt_writes(pub)
    if has == SKIP:
        return (SKIP, -1, -1)
    if has == "empty" and colls:
        return (UNDET, -1, -1)
    for i, j, ns, coll, rw in colls:                                       # validatePvtdata: every hash first
        if hashlib.sha256(rw).digest() != retrieve_hash(pub, ns, coll):
            return (MISMATCH, i, j)
    for i, j, ns, coll, rw in colls:                                       # then TxPvtRwSetFromProtoMsg
        if not decodes(rw):
            return (UNDET, i, j)
    return (OK, -1, -1)


def validate(rwsets, flags, pvt):
    """rwsets[t]: public TxReadWriteSet bytes or None; flags: final flags; pvt: {seq: entry bytes} ->
    ((code, seq, ns, coll), {seq: (code, ns, coll)})"""
    status = {s: entry_outcome(rwsets[s], e) for s, e in pvt.items()}
    for s in sorted(status):
        code, i, j = status[s]
        if code in (MISMATCH, UNDET) and flags[s] in (VALID, NOT_VALIDATED):
            if code == MISMATCH and flags[s] == VALID:
                return (MISMATCH, s, i, j), status
            return (UNDET, s, -1, -1), status
    return (OK, -1, -1, -1), status
