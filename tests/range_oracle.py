"""Range queries (phantom reads) in the ledger's MVCC check, restated over mvcc_oracle's dict state (Fabric 2.2, LevelDB state database):
validateRangeQuery (validator.go:216-237), the combined iterator (combined_iterator.go), rangeQueryResultsValidator and
rangeQueryHashValidator (rangequery_validator.go), and RangeQueryResultsHelper with its merkleTree (rwsetutil/query_results_helper.go).

mvcc_oracle's transaction form, each namespace with an optional
  ranges [(start, end, exhausted, reads)]   one RangeQueryInfo each, in KVRWSet.range_queries_info = 2
where reads is None (neither oneof field: no reads), a list [(key, version)] (raw_reads; version None / () / (b, t) as for reads) or
Merkle(max_degree, max_level, [hash bytes]) (reads_merkle_hashes); a range given as bytes is a RangeQueryInfo's wire form as it stands,
one this check does not decode (254).  Keys are str or bytes."""
import hashlib
from collections import namedtuple

from tools import fabricpb as pb
import mvcc_oracle as mo

VALID, MVCC_READ_CONFLICT, NOT_VALIDATED = mo.VALID, mo.MVCC_READ_CONFLICT, mo.NOT_VALIDATED
UNKNOWN = mo.UNKNOWN
Merkle = namedtuple("Merkle", "max_degree max_level hashes")


# ---- wire form -------------------------------------------------------------------------------------------------------------------
def _b(k):
    return k.encode() if isinstance(k, str) else bytes(k)


def kv_read(key, version):
    """KVRead{key = 1, version = 2} as proto.Marshal writes it: an empty key is omitted, a Version is present even when empty"""
    return (pb.f_bytes(1, key) if key else b"") + (b"" if version is None else pb.f_bytes(2, _ver(version)))


def _ver(v):
    b, t = (0, 0) if v == () else v
    return (pb.f_uint(1, b) if b else b"") + (pb.f_uint(2, t) if t else b"")


def range_info(start, end, exhausted, reads):
    """RangeQueryInfo{start_key = 1, end_key = 2, itr_exhausted = 3, oneof {raw_reads = 4, reads_merkle_hashes = 5}}"""
    out = (pb.f_bytes(1, _b(start)) if start else b"") + (pb.f_bytes(2, _b(end)) if end else b"") + (pb.f_uint(3, 1) if exhausted else b"")
    if isinstance(reads, Merkle):
        body = (pb.f_uint(1, reads.max_degree) if reads.max_degree else b"") + (pb.f_uint(2, reads.max_level) if reads.max_level else b"")
        out += pb.f_bytes(5, body + b"".join(pb.f_bytes(3, h) for h in reads.hashes))
    elif reads is not None:
        out += pb.f_bytes(4, b"".join(pb.f_bytes(1, kv_read(_b(k), v)) for k, v in reads))
    return out


def encode(tx) -> bytes:
    """TxReadWriteSet of a transaction, as mvcc_oracle.encode with each namespace's ranges after its reads (KVRWSet field order)"""
    out = b""
    for ns in tx:
        kv = b"".join(pb.f_bytes(1, pb.f_bytes(1, _b(k)) + mo._version(v, mo._same_part)) for k, v in ns.get("reads", ()))
        for r in ns.get("ranges", ()):
            kv += pb.f_bytes(2, r if isinstance(r, bytes) else range_info(*r))
        kv += b"".join(pb.f_bytes(3, mo._write(_b(k), d, v)) for k, d, v in map(mo._w, ns.get("writes", ())))
        kv += b"".join(pb.f_bytes(4, mo._md(_b(k), e)) for k, e in map(mo._m, ns.get("md", ())))
        body = pb.f_bytes(1, ns["ns"].encode()) + pb.f_bytes(2, kv)
        for name, hr, hw, hm in ns.get("colls", ()):
            h = b"".join(pb.f_bytes(1, pb.f_bytes(1, _b(k)) + mo._version(v, mo._same_part)) for k, v in hr)
            h += b"".join(pb.f_bytes(2, mo._write(_b(k), d, v)) for k, d, v in map(mo._w, hw))
            h += b"".join(pb.f_bytes(3, mo._md(_b(k), e)) for k, e in map(mo._m, hm))
            body += pb.f_bytes(3, pb.f_bytes(1, name.encode()) + pb.f_bytes(2, h))
        out += pb.f_bytes(2, body)
    return out


# ---- RangeQueryResultsHelper (hashing enabled) -----------------------------------------------------------------------------------
def _sha(b):
    return hashlib.sha256(b).digest()


class ResultsHelper:
    """NewRangeQueryResultsHelper(true, max_degree, sha256): AddResult, GetMerkleSummary and Done as the reference writes them"""

    def __init__(self, max_degree):
        if max_degree < 2:
            raise ValueError("maxDegree [%d] should not be less than 2 in the merkle tree" % max_degree)
        self.d, self.pending, self.tree, self.max_level = max_degree, [], {}, 1

    def add(self, key, version):
        self.pending.append((key, version))
        if len(self.pending) > self.d:
            self._process()

    def _process(self):
        b = b"".join(pb.f_bytes(1, kv_read(k, v)) for k, v in self.pending)       # proto.Marshal(QueryReads{kv_reads})
        self.pending = []
        self._update(_sha(b))

    def _update(self, h):
        self.tree.setdefault(1, []).append(h)
        level = 1
        while len(self.tree.get(level, [])) > self.d:
            nxt = _sha(b"".join(self.tree.pop(level)))
            self.tree.setdefault(level + 1, []).append(nxt)
            self.max_level = max(self.max_level, level + 1)
            level += 1

    def summary(self):
        return Merkle(self.d, self.max_level, list(self.tree.get(self.max_level, [])))

    def done(self):
        """the summary, or None when the tree is empty (max_degree or fewer results)"""
        if self.max_level == 1 and not self.tree.get(1):
            return None
        if self.pending:
            self._process()
        level = 1
        while level < self.max_level:
            hs = self.tree.get(level, [])
            if not hs:
                level += 1
                continue
            h = hs[0] if len(hs) == 1 else _sha(b"".join(hs))
            del self.tree[level]
            level += 1
            self.tree.setdefault(level, []).append(h)
        final = self.tree.get(self.max_level, [])
        if len(final) > self.d:
            del self.tree[self.max_level]
            self.max_level += 1
            self.tree[self.max_level] = [_sha(b"".join(final))]
        return self.summary()


def summary_of(results, max_degree):
    """Done()'s summary over (key, version) results"""
    h = ResultsHelper(max_degree)
    for k, v in results:
        h.add(k, v)
    return h.done()


class Panic(Exception):
    """where the reference panics, failing the commit"""


def hash_validate_reference(results, rec):
    """rangeQueryHashValidator.validate with its early exits (rangequery_validator.go:110-141), drawing results from an iterable.
    Raises Panic where it indexes MaxLevelHashes[lastMatchedIndex] out of range: after lastMatchedIndex passed 0, the max level rises
    and the new level holds a single hash."""
    h = ResultsHelper(rec.max_degree)
    last = -1
    for k, v in results:
        h.add(k, v)
        m = h.summary()
        if m.max_level < rec.max_level:
            continue
        if last == len(m.hashes) - 1:
            continue
        if len(m.hashes) > len(rec.hashes):
            return False
        last += 1
        if last >= len(m.hashes):
            raise Panic("index out of range [%d] with length %d" % (last, len(m.hashes)))
        if m.hashes[last] != rec.hashes[last]:
            return False
    return h.done() == rec


# ---- the combined iterator and the check -----------------------------------------------------------------------------------------
class Undetermined(Exception):
    """a result candidate whose state is unknown"""


def results(state, upd, block_num, ns, start, end, exhausted):
    """combinedIterator over the committed state and upd {key: ("put", (b, t)) | ("del",) | ("undet",)} of [start, end) in ns (an
    empty end: the rest of the namespace); then the end key once, when exhausted is False.  Yields (key, version); raises Undetermined
    when it reaches a candidate of unknown state."""
    start, end = _b(start), _b(end)
    inr = lambda k: k >= start and (end == b"" or k < end)
    keys = sorted({k for (n, c, k) in state if n == ns and c == "" and inr(k)} | {k for (n, c, k) in upd if n == ns and c == "" and inr(k)})

    def one(k):
        key = (ns, "", k)
        if key in upd:
            u = upd[key]
            if u[0] == "undet":
                raise Undetermined(k)
            return (k, u[1]) if u[0] == "put" else None
        v = state.get(key)
        if v == UNKNOWN:
            raise Undetermined(k)
        return None if v is None else (k, tuple(v))
    for k in keys:
        r = one(k)
        if r is not None:
            yield r
    if not exhausted:
        r = one(end)
        if r is not None:
            yield r


def _as_ver(v):
    return (0, 0) if v == () else tuple(v)


def check_range(state, upd, block_num, ns, rng):
    """'ok', 'fail' or 'undet' for one RangeQueryInfo of a VALID transaction"""
    if isinstance(rng, bytes):
        return "undet"
    start, end, exhausted, reads = rng
    it = results(state, upd, block_num, ns, start, end, exhausted)
    try:
        if isinstance(reads, Merkle):
            if reads.max_degree < 2:
                return "undet"
            return "ok" if hash_validate_reference(it, reads) else "fail"
        r = next(it, None)
        for k, v in reads or ():
            if r is None or r[0] != _b(k):
                return "fail"
            if v is None:                       # convertToVersionHeight dereferences the nil Version (rangequery_validator.go:165-166)
                return "undet"
            if r[1] != _as_ver(v):
                return "fail"
            r = next(it, None)
        return "ok" if r is None else "fail"
    except (Undetermined, Panic):
        return "undet"


def validate(state, block_num, txs, tv):
    """mvcc_oracle.validate with range queries decided (an index installed): (flags, new state, open)"""
    upd = {}
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
        ops = mo._ops(tx)
        if f == VALID:
            undet = fail = False
            for key, v in mo._reads(tx):
                if key in upd:
                    undet |= upd[key][0] == "undet"
                    fail |= upd[key][0] != "undet"
                else:
                    c = state.get(key)
                    undet |= c == UNKNOWN
                    fail |= c != UNKNOWN and not mo._same(c, v)
            for ns in tx:
                for rng in ns.get("ranges", ()):
                    c = check_range(state, upd, block_num, ns["ns"], rng)
                    undet |= c == "undet"
                    fail |= c == "fail"
            nil_put = any((mo._class(fl) == "put" and nil) or (mo._class(fl) == "md" and upd.get(k, ("",))[0] in ("del", "undet"))
                          for k, (fl, nil) in ops.items())
            after_open = open_at is not None and t > open_at
            code = NOT_VALIDATED if after_open or undet else MVCC_READ_CONFLICT if fail else NOT_VALIDATED if nil_put else VALID
        flags.append(code)
        if code == VALID:
            for k, (fl, _) in ops.items():
                op = mo._class(fl)
                if op == "del":
                    upd[k] = ("del",); final[k] = None
                elif op == "put":
                    upd[k] = ("put", (block_num, t)); final[k] = (block_num, t)
                elif upd.get(k, ("",))[0] == "put":
                    upd[k] = ("put", (block_num, t)); final[k] = (block_num, t)
                elif state.get(k) == UNKNOWN:
                    upd[k] = ("undet",); final[k] = UNKNOWN
                elif state.get(k) is not None:
                    upd[k] = ("put", (block_num, t)); final[k] = (block_num, t)
        elif code == NOT_VALIDATED:
            for k in ops:
                upd[k] = ("undet",); final[k] = UNKNOWN
    new = dict(state)
    for k, v in final.items():
        if v is None:
            new.pop(k, None)
        else:
            new[k] = v
    return flags, new, open_at is not None

