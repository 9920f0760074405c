"""The ledger's MVCC check and write-set application, restated over a dict state (Fabric 2.2.1, LevelDB state database).

A transaction is a list of namespaces, each a dict with optional entries
  reads  [(key, version)]           KVRead{key = 1, version = 2}
  range  bool                       one RangeQueryInfo in KVRWSet.range_queries_info = 2
  writes [(key, is_delete[, has_value])]   KVWrite{key = 1, is_delete = 2, value = 3}; has_value False: no value field (a nil value)
  md     [key or (key, has_entries)]      KVMetadataWrite{key = 1, entries = 2}; has_entries False: no entry (Entries == nil)
  colls  [(name, hreads, hwrites, hmd)] with key hashes in place of keys
version None = no Version message (nil), () = an empty Version (block 0, tx 0, not nil), (b, t).  None instead of the list: a transaction
whose write set cannot be enumerated (no ChaincodeAction.results, a non-endorser transaction).

State: {(ns, coll, key): (block, tx) or UNKNOWN}; coll "" for public keys."""
from tools import fabricpb as pb

VALID, MVCC_READ_CONFLICT, NOT_VALIDATED = 0, 11, 254
UNKNOWN = "unknown"
REMOVE = (2 ** 64 - 1, 2 ** 64 - 1)


# ---- wire form -------------------------------------------------------------------------------------------------------------------
def _version(v, mut):
    if v is None:
        return b""
    b, t = (0, 0) if v == () else v
    return pb.f_bytes(2, mut("Version", (pb.f_uint(1, b) if b else b"") + (pb.f_uint(2, t) if t else b"")))


def _same_part(part, b):
    return b


def _write(key, delete, has_value=True):
    return pb.f_bytes(1, key) + (pb.f_uint(2, 1) if delete else b"") + (pb.f_bytes(3, b"value") if has_value and not delete else b"")


def _w(x):
    """(key, is_delete, has_value) of a writes entry"""
    return (x[0], x[1], x[2] if len(x) > 2 else True)


def _m(x):
    """(key, has_entries) of an md entry"""
    return (x, True) if isinstance(x, (str, bytes)) else tuple(x)


def _md(key, has_entries):
    return pb.f_bytes(1, key) + (_MD if has_entries else b"")


_MD = pb.f_bytes(2, pb.f_bytes(1, b"VALIDATION_PARAMETER") + pb.f_bytes(2, b"ep"))


def encode(tx, mut=_same_part) -> bytes:
    """rwset.TxReadWriteSet{data_model = 1, ns_rwset = 2} of a transaction; mut(part, bytes) may rewrite each "Version", "KVRead",
    "KVReadHash", "KVRWSet", "HashedRWSet", "NsReadWriteSet" and the "TxReadWriteSet" as it is assembled"""
    out = b""
    for ns in tx:
        kv = b"".join(pb.f_bytes(1, mut("KVRead", pb.f_bytes(1, _b(k)) + _version(v, mut))) for k, v in ns.get("reads", ()))
        if ns.get("range"):
            kv += pb.f_bytes(2, pb.f_bytes(1, b"a") + pb.f_bytes(2, b"z") + pb.f_uint(3, 1))
        kv += b"".join(pb.f_bytes(3, _write(_b(k), d, v)) for k, d, v in map(_w, ns.get("writes", ())))
        kv += b"".join(pb.f_bytes(4, _md(_b(k), e)) for k, e in map(_m, ns.get("md", ())))
        body = pb.f_bytes(1, ns["ns"].encode()) + pb.f_bytes(2, mut("KVRWSet", kv))
        for name, hr, hw, hm in ns.get("colls", ()):
            h = b"".join(pb.f_bytes(1, mut("KVReadHash", pb.f_bytes(1, _b(k)) + _version(v, mut))) for k, v in hr)
            h += b"".join(pb.f_bytes(2, _write(_b(k), d, v)) for k, d, v in map(_w, hw))
            h += b"".join(pb.f_bytes(3, _md(_b(k), e)) for k, e in map(_m, hm))
            body += pb.f_bytes(3, pb.f_bytes(1, name.encode()) + pb.f_bytes(2, mut("HashedRWSet", h)))
        out += pb.f_bytes(2, mut("NsReadWriteSet", body))
    return mut("TxReadWriteSet", out)


def _b(k):
    return k.encode() if isinstance(k, str) else bytes(k)


# ---- the check -------------------------------------------------------------------------------------------------------------------
# keyOpsFlag (tx_ops.go:162-169)
UPSERT_VAL, METADATA_UPDATE, METADATA_DELETE, KEY_DELETE = 1, 2, 4, 8


def _ops(tx):
    """prepareTxOps' key operations of one transaction: {key: (flag, value is nil)}.  applyTxRwset visits, per namespace, its writes, its
    metadata writes, then per collection its hashed writes and hashed metadata writes (tx_ops.go:59-98).  applyKVWrite deletes or upserts
    (:100-107); applyMetadata updates, or deletes when Entries is nil (:109-120).  Each ADDS its flag to the key's uint8 (:185-205), so
    a kind given twice carries: two upserts make 2, two deletes 16.  upsert keeps the last value (:185-189)."""
    ops = {}

    def add(key, flag, nil=None):
        f, was_nil = ops.get(key, (0, False))
        ops[key] = ((f + flag) & 0xff, was_nil if nil is None else nil)
    for ns in tx:
        n = ns["ns"]
        for k, d, v in map(_w, ns.get("writes", ())):
            add((n, "", _b(k)), KEY_DELETE) if d else add((n, "", _b(k)), UPSERT_VAL, not v)
        for k, e in map(_m, ns.get("md", ())):
            add((n, "", _b(k)), METADATA_UPDATE if e else METADATA_DELETE)
        for name, _, hw, hm in ns.get("colls", ()):
            for k, d, v in map(_w, hw):
                add((n, name, _b(k)), KEY_DELETE) if d else add((n, name, _b(k)), UPSERT_VAL, not v)
            for k, e in map(_m, hm):
                add((n, name, _b(k)), METADATA_UPDATE if e else METADATA_DELETE)
    return ops


def _class(flag):
    """'del' for isDelete (tx_ops.go:218-220); 'put' for isUpsertAndMetadataUpdate (:222-228) and isOnlyUpsert (:230-232), which keep
    the transaction's own value; 'md' for every other flag, whose value prepareTxOps takes from the latest state (:35-51)"""
    if flag & KEY_DELETE == KEY_DELETE:
        return "del"
    if (flag & UPSERT_VAL and flag & (METADATA_UPDATE | METADATA_DELETE)) or flag | UPSERT_VAL == UPSERT_VAL:
        return "put"
    return "md"


def _reads(tx):
    """(key, version) in validateTx's order (validator.go:121-147): per namespace its public reads, then each collection's hashed reads"""
    for ns in tx:
        for k, v in ns.get("reads", ()):
            yield (ns["ns"], "", _b(k)), v
        for name, hr, _, _ in ns.get("colls", ()):
            for k, v in hr:
                yield (ns["ns"], name, _b(k)), v


def _same(committed, v):
    """version.AreSame over rwsetutil.NewVersion (validator.go:186): nil equals only nil"""
    if committed is None or v is None:
        return committed is None and v is None
    return committed == ((0, 0) if v == () else tuple(v))


def validate(state, block_num, txs, tv):
    """validateAndPrepareBatch (validator.go:82-110) over the validator's flags tv: returns (flags, new state, open).  Only VALID
    transactions are checked (batch_preparer.go:192-284); every other flag is copied.  Handed back as 254: a range query (phantom reads are
    not restated), a read of a key an undetermined transaction wrote or the table marks unknown, a VALID transaction after one whose write
    set cannot be enumerated, and a metadata-only write of a key an earlier transaction of the block deleted (retrieveLatestState returns
    the deletion, and PutValAndMetadata panics on its nil value: statedb.go:202-205).  The writes of a 254 transaction leave their keys
    unknown; a transaction whose writes cannot be enumerated leaves the block open."""
    updates = {}                     # validator.go:176-193 updates.Exists: key -> 'put' / 'del' / 'undet'
    final = {}
    flags = []
    open_at = None
    for t, (tx, f) in enumerate(zip(txs, tv)):
        if f not in (VALID, NOT_VALIDATED):
            flags.append(f)
            continue
        if tx is None:
            open_at = t if open_at is None else open_at
            flags.append(NOT_VALIDATED)
            continue
        code = f
        ops = _ops(tx)
        if f == VALID:
            undet = fail = nil_put = False
            for key, v in _reads(tx):
                if key in updates:
                    undet |= updates[key] == "undet"
                    fail |= updates[key] != "undet"
                else:
                    c = state.get(key)
                    undet |= c == UNKNOWN
                    fail |= c != UNKNOWN and not _same(c, v)
            # PutValAndMetadata panics on a nil value (statedb.go:202-205): an upsert whose last write had no value, or the latest value
            # of a key an earlier transaction deleted (retrieveLatestState returns the deletion) -- or may have deleted
            nil_put = any((_class(f) == "put" and nil) or (_class(f) == "md" and updates.get(k) in ("del", "undet")) for k, (f, nil) in ops.items())
            has_range = any(ns.get("range") for ns in tx)
            after_open = open_at is not None and t > open_at
            code = NOT_VALIDATED if has_range or after_open or undet else MVCC_READ_CONFLICT if fail else NOT_VALIDATED if nil_put else VALID
        flags.append(code)
        if code == VALID:                                              # applyWriteSet (types.go:81-111) at height (block_num, t)
            for k, (f, _) in ops.items():
                op = _class(f)
                if op == "del":
                    updates[k] = "del"; final[k] = None
                elif op == "put":
                    updates[k] = "put"; final[k] = (block_num, t)
                elif updates.get(k) == "put":
                    final[k] = (block_num, t)
                elif state.get(k) == UNKNOWN:
                    updates[k] = "undet"; final[k] = UNKNOWN
                elif state.get(k) is not None:
                    updates[k] = "put"; final[k] = (block_num, t)
                # absent: the metadata-only operation is dropped (tx_ops.go:41-51)
        elif code == NOT_VALIDATED:
            for k in ops:
                updates[k] = "undet"; final[k] = UNKNOWN
    new = dict(state)
    for k, v in final.items():
        if v is None:
            new.pop(k, None)
        else:
            new[k] = v
    return flags, new, open_at is not None


def info(state):
    """(keys held, keys unknown) of a state"""
    return len(state), sum(1 for v in state.values() if v == UNKNOWN)
