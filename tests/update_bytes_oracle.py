"""The block's deterministic update bytes, restated: deterministicBytesForPubAndHashUpdates (core/ledger/kvledger/txmgmt/txmgr/
update_batch_bytes.go:29-105) over updates_oracle.batch's records, as fabgpu_block_update_bytes returns them, and the commit hash of
kvLedger.addBlockCommitHash (kv_ledger.go:621-632).

The encoder is google.protobuf's, over message classes built at run time from txmgr/updates.proto's field numbers: independent of the
device's hand encoder.  A KVWrite here is a dict with namespace, collection (str, "" when left out), key, value (bytes, b"" when left
out), is_delete (bool) and version (Height.ToBytes())."""
import hashlib

from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

import updates_oracle as uo

_UPDATES = None


def _updates_class():
    """txmgr.Updates{repeated KVWrite kvwrites = 1}, KVWrite{namespace = 1 string, collection = 2 string, key = 3 bytes, isDelete = 4
    bool, value = 5 bytes, version_bytes = 6 bytes}, proto3"""
    global _UPDATES
    if _UPDATES is None:
        F = descriptor_pb2.FieldDescriptorProto
        fd = descriptor_pb2.FileDescriptorProto(name="fabgpu_test_txmgr_updates.proto", package="fabgpu_test_txmgr", syntax="proto3")
        kv = fd.message_type.add(name="KVWrite")
        for name, number, kind in (("namespace", 1, F.TYPE_STRING), ("collection", 2, F.TYPE_STRING), ("key", 3, F.TYPE_BYTES),
                                   ("isDelete", 4, F.TYPE_BOOL), ("value", 5, F.TYPE_BYTES), ("version_bytes", 6, F.TYPE_BYTES)):
            kv.field.add(name=name, number=number, type=kind, label=F.LABEL_OPTIONAL)
        up = fd.message_type.add(name="Updates")
        up.field.add(name="kvwrites", number=1, type=F.TYPE_MESSAGE, label=F.LABEL_REPEATED, type_name=".fabgpu_test_txmgr.KVWrite")
        pool = descriptor_pool.DescriptorPool()
        pool.Add(fd)
        _UPDATES = message_factory.GetMessageClass(pool.FindMessageTypeByName("fabgpu_test_txmgr.Updates"))
    return _UPDATES


def order_preserving(n):
    """EncodeOrderPreservingVarUint64 (common/ledger/util/util.go:32-52): a length byte, then the big-endian bytes without leading zeros"""
    b = n.to_bytes(8, "big").lstrip(b"\x00")
    return bytes([len(b)]) + b


def height(block_num, tx):
    """Height{block_num, tx}.ToBytes() (core/ledger/internal/version/version.go:50-54)"""
    return order_preserving(block_num) + order_preserving(tx)


def _b(s):
    """a name's wire bytes: sort.Strings compares those"""
    return s.encode() if isinstance(s, str) else bytes(s)


def kvwrite(key, value=b"", is_delete=False, version=b"", namespace="", collection=""):
    return dict(namespace=namespace, collection=collection, key=bytes(key), is_delete=is_delete, value=bytes(value), version=version)


def kvwrites(records, block_num, committed=()):
    """The KVWrite list of the batch `records` (updates_oracle's form; a record with collection "" is public), COMMITTED values taken
    from `committed` in record order"""
    values = iter(committed)
    pub, hashed = {}, {}
    for tx, op, ns, coll, key, value, _meta in records:
        if value == uo.COMMITTED:
            value = bytes(next(values))
        v = None if op == "del" else value
        target = pub.setdefault(ns, {}) if coll == "" else hashed.setdefault(ns, {}).setdefault(coll, {})
        target[bytes(key)] = (v, height(block_num, tx))

    def gen(updates):                                                 # genKVs (:80-96): keys sorted
        return [kvwrite(k, updates[k][0] or b"", updates[k][0] is None, updates[k][1]) for k in sorted(updates)]
    out = []
    for ns in sorted(set(pub) | set(hashed), key=_b):                 # dedupAndSort (:98-107)
        if ns == "":
            continue                                                  # the channel config (:39-44)
        kvs = gen(pub.get(ns, {}))
        for coll in sorted(hashed.get(ns, {}), key=_b):              # genKVsFromCollsUpdates (:66-78)
            c = gen(hashed[ns][coll])
            c[0]["collection"] = coll
            kvs += c
        kvs[0]["namespace"] = ns
        out += kvs
    return out


def _utf8(s):
    try:
        _b(s).decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def marshal(kvs):
    """proto.Marshal(&Updates{Kvwrites: kvs}) with google.protobuf; None when a name is not valid UTF-8 (golang/protobuf v1.3.3 fails
    Marshal on a proto3 string that is not: recalled, not verified)"""
    if not all(_utf8(w["namespace"]) and _utf8(w["collection"]) for w in kvs):
        return None
    u = _updates_class()()
    for w in kvs:
        m = u.kvwrites.add()
        if w["namespace"]:
            m.namespace = _b(w["namespace"]).decode()
        if w["collection"]:
            m.collection = _b(w["collection"]).decode()
        m.key = w["key"]
        m.isDelete = w["is_delete"]
        m.value = w["value"]
        m.version_bytes = w["version"]
    return u.SerializeToString(deterministic=True)


def update_bytes(records, block_num, committed=()):
    """fabgpu_block_update_bytes' answer: the bytes, or None when the batch is incomplete (records None) or a name is not UTF-8"""
    return None if records is None else marshal(kvwrites(records, block_num, committed))


def committed_values(records, values):
    """the values of the COMMITTED-value records in record order, read from the state `values` ({(ns, coll, key): (value, metadata)}):
    GetState / GetValueHash"""
    return [values[(ns, coll, bytes(key))][0] for _tx, _op, ns, coll, key, value, _m in records or () if value == uo.COMMITTED]


def varint(n):
    out = b""
    while n >= 0x80:
        out += bytes([n & 0x7F | 0x80])
        n >>= 7
    return out + bytes([n])


def commit_hash(flags, update_bytes_, prev):
    """addBlockCommitHash: SHA-256(varint(len(flags)) || flags || update bytes || previous commit hash)"""
    flags = bytes(flags)
    return hashlib.sha256(varint(len(flags)) + flags + bytes(update_bytes_) + bytes(prev or b"")).digest()
