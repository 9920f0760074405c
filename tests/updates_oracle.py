"""The block's public and hashed update batch, restated: prepareTxOps and applyWriteSet (core/ledger/kvledger/txmgmt/validation/tx_ops.go:18-232,
types.go:81-111) over the transactions mvcc_oracle.validate leaves VALID, as fabgpu_block_updates reports it.

A transaction is a list of namespaces, each a dict with optional entries
  reads  [(key, version)]                  as mvcc_oracle
  writes [(key, value)]                    value: bytes (an upsert, b"" present but empty), None (an upsert without a value), DEL
  md     [(key, entries)]                  entries: None or [] (no entry: metadataDelete), else a list of (name, value) -- marshalled as
                                           KVMetadataEntry{name = 1, value = 2}, empty fields left out -- or raw entry bytes
  colls  [(name, hreads, hwrites, hmd)]    with key hashes in place of keys, value hashes in place of values
None instead of the list: a transaction whose write set cannot be enumerated.

The committed state is (versions, values): mvcc_oracle's {(ns, coll, key): version or UNKNOWN} and {(ns, coll, key): (value, metadata)}.
A record is (tx, op, ns, coll, key, value, metadata): op "put" / "del"; value bytes, COMMITTED or None (a delete); metadata bytes (the
Serialize form), None (nil) or COMMITTED."""
from tools import fabricpb as pb
import couch_oracle as co
import mvcc_oracle as mo

DEL = "del"
COMMITTED = "committed"
VALID, NOT_VALIDATED = mo.VALID, mo.NOT_VALIDATED
_UNDET = "undet"          # a value, metadata or whole entry that depends on a key the table marks unknown
_NONCANON = "noncanon"    # metadata whose entries golang/protobuf would not re-marshal unchanged


# ---- wire form -------------------------------------------------------------------------------------------------------------------
def _b(k):
    return k.encode() if isinstance(k, str) else bytes(k)


def entry_bytes(e):
    if isinstance(e, (bytes, bytearray)):
        return bytes(e)
    name, value = _b(e[0]), _b(e[1])
    return (pb.f_bytes(1, name) if name else b"") + (pb.f_bytes(2, value) if value else b"")


def canonical(e):
    """name = 1 then value = 2, each at most once and non-empty, minimal lengths, nothing else: what golang/protobuf v1.3.3 re-marshals
    unchanged (recalled, not verified)"""
    b, p = entry_bytes(e), 0
    for tag in (0x0A, 0x12):
        if p < len(b) and b[p] == tag:
            n, q = pb.read_varint(b, p + 1)
            if n == 0 or q + n > len(b) or pb.varint(n) != b[p + 1:q]:
                return False
            p = q + n
    return p == len(b)


def serialize(entries):
    """statemetadata.Serialize (metadata.go:15-18): proto.Marshal(KVMetadataWrite{Entries}) -- field 2 per entry"""
    return b"".join(pb.f_bytes(2, entry_bytes(e)) for e in entries)


def _write(key, value):
    if value is DEL:
        return pb.f_bytes(1, key) + pb.f_uint(2, 1)
    return pb.f_bytes(1, key) + (pb.f_bytes(3, value) if value is not None else b"")


def _md(key, entries):
    return pb.f_bytes(1, key) + b"".join(pb.f_bytes(2, entry_bytes(e)) for e in entries or ())


def encode(tx) -> bytes:
    """rwset.TxReadWriteSet{ns_rwset = 2}, laid out as mvcc_oracle.encode lays it out"""
    out = b""
    for ns in tx:
        kv = b"".join(pb.f_bytes(1, pb.f_bytes(1, _b(k)) + mo._version(v, mo._same_part)) for k, v in ns.get("reads", ()))
        if ns.get("range"):
            kv += pb.f_bytes(2, pb.f_bytes(1, b"a") + pb.f_bytes(2, b"z") + pb.f_uint(3, 1))
        kv += b"".join(pb.f_bytes(3, _write(_b(k), v)) for k, v in ns.get("writes", ()))
        kv += b"".join(pb.f_bytes(4, _md(_b(k), e)) for k, e in ns.get("md", ()))
        body = pb.f_bytes(1, ns["ns"].encode()) + pb.f_bytes(2, kv)
        for name, hr, hw, hm in ns.get("colls", ()):
            h = b"".join(pb.f_bytes(1, pb.f_bytes(1, _b(k)) + mo._version(v, mo._same_part)) for k, v in hr)
            h += b"".join(pb.f_bytes(2, _write(_b(k), v)) for k, v in hw)
            h += b"".join(pb.f_bytes(3, _md(_b(k), e)) for k, e in hm)
            body += pb.f_bytes(3, pb.f_bytes(1, name.encode()) + pb.f_bytes(2, h))
        out += pb.f_bytes(2, body)
    return out


def as_mvcc_tx(tx):
    """the transaction in mvcc_oracle's form (only whether a write has a value, a metadata write entries)"""
    if tx is None:
        return None
    out = []
    for ns in tx:
        n = dict(ns=ns["ns"], reads=list(ns.get("reads", ())), range=ns.get("range", False))
        n["writes"] = [(k, v is DEL, v is not None) for k, v in ns.get("writes", ())]
        n["md"] = [(k, bool(e)) for k, e in ns.get("md", ())]
        n["colls"] = [(c, hr, [(k, v is DEL, v is not None) for k, v in hw], [(k, bool(e)) for k, e in hm]) for c, hr, hw, hm in ns.get("colls", ())]
        out.append(n)
    return out


def couch_flags(txs, tv):
    """CouchDB's pre-pass (couch_oracle.tx_code) over the validator's flags: INVALID_WRITESET or 254 for a VALID transaction"""
    out = list(tv)
    for t, tx in enumerate(txs):
        if out[t] == VALID and tx is not None:
            c = co.tx_code([dict(ns=ns["ns"], reads=ns.get("reads", ()),
                                 writes=[(k, v is DEL, None if v is DEL else v) for k, v in ns.get("writes", ())]) for ns in tx])
            if c is not None:
                out[t] = c
    return out


def flags(versions, block_num, txs, tv, couch=False):
    """mvcc_oracle.validate, after CouchDB's pre-pass when couch: (flags, new versions, open)"""
    if couch:
        tv = couch_flags(txs, tv)
    return mo.validate(versions, block_num, [as_mvcc_tx(tx) for tx in txs], tv)


# ---- the batch -------------------------------------------------------------------------------------------------------------------
def _ops(tx):
    """applyTxRwset (tx_ops.go:59-120): per (ns, coll, key) the flag sum (a uint8: :185-205), the last upsert's value, the last
    metadataUpdate's Serialize bytes, and the wire position of the first write"""
    ops, pos = {}, 0

    def get(k):
        nonlocal pos
        if k not in ops:
            ops[k] = [0, None, None, pos]
        pos += 1
        return ops[k]
    for ns in tx:
        n = ns["ns"]
        groups = [("", ns.get("writes", ()), ns.get("md", ()))] + [(c, hw, hm) for c, _, hw, hm in ns.get("colls", ())]
        for coll, writes, mds in groups:
            for k, v in writes:
                o = get((n, coll, _b(k)))
                if v is DEL:
                    o[0] = (o[0] + mo.KEY_DELETE) & 0xFF
                else:
                    o[0] = (o[0] + mo.UPSERT_VAL) & 0xFF
                    o[1] = v
            for k, e in mds:
                o = get((n, coll, _b(k)))
                if e:
                    o[0] = (o[0] + mo.METADATA_UPDATE) & 0xFF
                    o[2] = serialize(e) if all(canonical(x) for x in e) else _NONCANON
                else:
                    o[0] = (o[0] + mo.METADATA_DELETE) & 0xFF
    return ops


def batch(versions, values, block_num, txs, codes):
    """applyWriteSet (types.go:81-111) of every VALID transaction in order, over the final flags `codes`: the records in fabgpu_block_updates'
    order, or None when the device leaves the batch to the peer (a 254, a non-canonical deciding metadata write, a record that depends on
    a key the table marks unknown).  A 254 also stands for an open block (the unenumerable transaction is 254)."""
    if NOT_VALIDATED in codes:
        return None
    updates = {}                                   # key -> [tx, op, value, metadata, first position], or _UNDET (exists or dropped)

    def latest(k):
        """retrieveLatestState (tx_ops.go:127-144): the entry of updates, else the committed value; None absent"""
        if k in updates:
            return updates[k]
        v = versions.get(k)
        return None if v is None else _UNDET if v == mo.UNKNOWN else [None, "put", COMMITTED, COMMITTED, None]
    for t, tx in enumerate(txs):
        if codes[t] != VALID:
            continue
        for k, (f, value, meta, pos) in _ops(tx).items():
            if f & mo.KEY_DELETE:                                            # isDelete
                updates[k] = [t, "del", None, None, pos]
            elif f & mo.UPSERT_VAL and f & (mo.METADATA_UPDATE | mo.METADATA_DELETE):   # isUpsertAndMetadataUpdate
                updates[k] = [t, "put", value if value is not None else _UNDET, meta, pos]
            elif f | mo.UPSERT_VAL == mo.UPSERT_VAL:                       # isOnlyUpsert: retrieveLatestMetadata (:146-160)
                e = updates.get(k)
                md = COMMITTED if e is None else _UNDET if e is _UNDET else e[3]
                updates[k] = [t, "put", value if value is not None else _UNDET, md, pos]
            else:                                                          # the metadata path (:41-51)
                e = latest(k)
                if e is None:
                    continue                                               # absent: dropped
                if e is _UNDET:
                    updates[k] = _UNDET
                    continue
                assert e[2] is not None, "a deleted value: PutValAndMetadata panics, the stage gives 254"
                updates[k] = [t, "put", e[2], meta, pos]
    out = []
    for k, e in updates.items():
        if e is _UNDET or _UNDET in (e[2], e[3]) or e[3] is _NONCANON:
            return None
        out.append((e[0], e[1], k[0], k[1], k[2], e[2], e[3]))
    order = {k: (e[0], e[4]) for k, e in updates.items()}
    return sorted(out, key=lambda r: order[(r[2], r[3], r[4])])


def apply(values, records):
    """the committed values after the batch: COMMITTED sources read from `values` (GetState / GetStateMetadata)"""
    new = dict(values)
    for tx, op, ns, coll, key, value, meta in records:
        k = (ns, coll, key)
        if op == "del":
            new.pop(k, None)
            continue
        old = values.get(k, (None, None))
        new[k] = (old[0] if value == COMMITTED else value, old[1] if meta == COMMITTED else meta)
    return new
