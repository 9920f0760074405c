"""CouchDB's key and value checks in the ledger's commit path, restated (Fabric 2.2, Go 1.14.4): validateWriteset
(validation/batch_preparer.go:317-330) over the CouchDB state database's ValidateKeyValue (statecouchdb.go:427, couchdoc_conv.go:37-57,
278-297), and the MVCC stage's flags with them (range_oracle.validate after the INVALID_WRITESET pre-pass).

A key is invalid when it is not valid UTF-8, starts with "_", or is empty.  Python's strict UTF-8 decoder rejects exactly what Go's
utf8.ValidString rejects: overlong forms, surrogates (ED A0..BF xx), code points above U+10FFFF and truncated sequences.

A value is invalid when json.Unmarshal(b, &map[string]interface{}{}) succeeds and a top-level member name is "~version" or starts with
"_".  It succeeds when the bytes pass encoding/json's checkValid scanner (restated by Scanner below), the top-level value is an object
or null, and no number anywhere fails strconv.ParseFloat(s, 64).  Rules the device answers with 254 (UNDET):
  - a number with an exponent of 10000 or more (readFloat stops accumulating the exponent there, as recalled);
  - a number whose 40 leading significant digits equal those of the overflow bound 2^1024 - 2^970, with decimal exponent 309;
  - a value nested deeper than DEPTH containers (a container opening past DEPTH before any syntax error) whose top-level value is an
    object.
Values of at most SHORT_MAX bytes take the device's one-thread scan, longer ones its CTA scan; both give value_bits.

The transaction form is range_oracle's, with a write's third element the value: bytes (the value field as given, also on a delete),
True (b"value", as mvcc_oracle writes it) or False / None / b"" (no value field: proto.Marshal omits an empty one)."""
import re

from tools import fabricpb as pb
import mvcc_oracle as mo
import range_oracle as ro

VALID, NOT_VALIDATED, INVALID_WRITESET = 0, 254, 24
OK, INVALID, UNDET = 0, 1, 2
SHORT_MAX = 16384
LANE_BYTES, TILE_BYTES = 64, 64 * 256       # the CTA scan's chunk per thread and tile
DEPTH = 128
# verdict bits, as fabgpu_test_couch_values reports them
SYNTAX_OK, TOP_OBJECT, NUM_ERR, NUM_UNDET, RESERVED, CUT = 1, 2, 4, 8, 16, 32
H = (2 ** 54 - 1) * 2 ** 970            # the least value ParseFloat(s, 64) rounds to +Inf
H_DIGITS = str(H)[:40]


def utf8_valid(b: bytes) -> bool:
    try:
        bytes(b).decode("utf-8", "strict")
        return True
    except UnicodeDecodeError:
        return False


def key_ok(k) -> bool:
    k = ro._b(k)
    return len(k) > 0 and k[:1] != b"_" and utf8_valid(k)


# ---- numbers ---------------------------------------------------------------------------------------------------------------------
def _decimal(tok: bytes):
    """(significant digits, x) with the token's magnitude = 0.digits x 10^x; digits "" for zero"""
    mant, _, exp = tok.decode().lower().partition("e")
    ip, _, fp = mant.lstrip("-").partition(".")
    digits = (ip + fp).lstrip("0")
    x = (len(ip.lstrip("0")) if ip.lstrip("0") else -(len(fp) - len(fp.lstrip("0")))) + (int(exp) if exp else 0)
    return digits, x


def number_verdict(tok: bytes):
    """0 (ParseFloat succeeds), NUM_ERR (it overflows) or NUM_UNDET for a number token of the grammar"""
    digits, x = _decimal(tok)
    if not digits:
        return 0
    if abs(int(tok.decode().lower().partition("e")[2] or "0")) >= 10000:
        return NUM_UNDET
    if x == 309 and len(digits) >= 40 and digits[:40] == H_DIGITS:
        return NUM_UNDET
    return NUM_ERR if overflows(tok) else 0


def overflows(tok: bytes) -> bool:
    """exact: the number's magnitude is at least H (compared digit by digit: H has 309 integer digits)"""
    digits, x = _decimal(tok)
    if not digits or x != 309:
        return bool(digits) and x > 309
    h = str(H)
    n = max(len(digits), len(h))
    return digits.ljust(n, "0") >= h.ljust(n, "0")


# ---- the scanner and the decode rules --------------------------------------------------------------------------------------------
_PLAIN = re.compile(rb'[^"\\\x00-\x1f]*')


class _Stop(Exception):
    pass


class Scanner:
    """encoding/json's grammar, left to right: whitespace is space, tab, CR and LF; strings take any byte >= 0x20 (no UTF-8 check) and the
    escapes \\" \\\\ \\/ \\b \\f \\n \\r \\t \\uXXXX; numbers -?(0|[1-9][0-9]*)(.[0-9]+)?([eE][+-]?[0-9]+)?; literals true, false, null.
    Collects the verdict bits: NUM_ERR / NUM_UNDET over every number, RESERVED over the top object's member names (unescaped, an
    invalid byte standing for U+FFFD), CUT when a container opens past DEPTH."""

    def __init__(self, b: bytes, depth_bound=DEPTH):
        self.b, self.i, self.bits, self.depth, self.bound = bytes(b), 0, 0, 0, depth_bound

    def peek(self):
        return self.b[self.i] if self.i < len(self.b) else None

    def ws(self):
        while self.peek() in (0x20, 0x09, 0x0D, 0x0A):
            self.i += 1

    def fail(self):
        raise _Stop("syntax")

    def value(self):
        self.ws()
        c = self.peek()
        if c is None:
            self.fail()
        if c in (0x7B, 0x5B):
            if self.depth == 0 and c == 0x7B:
                self.bits |= TOP_OBJECT
            if self.depth == self.bound:
                raise _Stop("cut")
            self.depth += 1
            self.i += 1
            self.obj() if c == 0x7B else self.arr()
            self.depth -= 1
        elif c == 0x22:
            self.string()
        elif c == 0x2D or 0x30 <= c <= 0x39:
            self.number()
        else:
            for lit in (b"true", b"false", b"null"):
                if c == lit[0]:
                    for k in lit:
                        if self.peek() != k:
                            self.fail()
                        self.i += 1
                    return
            self.fail()

    def obj(self):
        top = self.depth == 1
        self.ws()
        if self.peek() == 0x7D:
            self.i += 1
            return
        while True:
            self.ws()
            if self.peek() != 0x22:
                self.fail()
            name = self.string()
            if top and (name == "~version" or name.startswith("_")):
                self.bits |= RESERVED
            self.ws()
            if self.peek() != 0x3A:
                self.fail()
            self.i += 1
            self.value()
            self.ws()
            c = self.peek()
            self.i += 1
            if c == 0x7D:
                return
            if c != 0x2C:
                self.fail()

    def arr(self):
        self.ws()
        if self.peek() == 0x5D:
            self.i += 1
            return
        while True:
            self.value()
            self.ws()
            c = self.peek()
            self.i += 1
            if c == 0x5D:
                return
            if c != 0x2C:
                self.fail()

    def string(self):
        """the unescaped string (an invalid or non-ASCII byte as U+FFFD, a \\u escape as its code unit)"""
        self.i += 1
        out = []
        while True:
            c = self.peek()
            if c is None or c < 0x20:
                self.fail()
            self.i += 1
            if c == 0x22:
                return "".join(out)
            if c != 0x5C:
                out.append(chr(c) if c < 0x80 else "�")
                m = _PLAIN.match(self.b, self.i)             # a run of plain bytes at once
                if m.end() > self.i:
                    out.append("".join(chr(x) if x < 0x80 else "�" for x in m.group()[:10]))   # names: the first chars decide
                    self.i = m.end()
                continue
            e = self.peek()
            self.i += 1
            simple = {0x22: '"', 0x5C: "\\", 0x2F: "/", 0x62: "\b", 0x66: "\f", 0x6E: "\n", 0x72: "\r", 0x74: "\t"}
            if e in simple:
                out.append(simple[e])
            elif e == 0x75:
                h = self.b[self.i:self.i + 4]
                if len(h) < 4 or any(x not in b"0123456789abcdefABCDEF" for x in h):
                    self.fail()
                self.i += 4
                out.append(chr(int(h, 16)))
            else:
                self.fail()

    def number(self):
        s = self.i
        if self.peek() == 0x2D:
            self.i += 1
        dig = lambda: self.peek() is not None and 0x30 <= self.peek() <= 0x39
        if self.peek() == 0x30:
            self.i += 1
        elif dig():
            while dig():
                self.i += 1
        else:
            self.fail()
        if self.peek() == 0x2E:
            self.i += 1
            if not dig():
                self.fail()
            while dig():
                self.i += 1
        if self.peek() in (0x65, 0x45):
            self.i += 1
            if self.peek() in (0x2B, 0x2D):
                self.i += 1
            if not dig():
                self.fail()
            while dig():
                self.i += 1
        self.bits |= number_verdict(self.b[s:self.i])

    def run(self):
        """the verdict bits of the whole input"""
        try:
            self.value()
            self.ws()
            if self.i != len(self.b):
                self.fail()
            return self.bits | SYNTAX_OK
        except _Stop as e:
            return (self.bits & TOP_OBJECT) | CUT if str(e) == "cut" else 0


def scan_ok(b: bytes) -> bool:
    """checkValid (no depth bound)"""
    return bool(Scanner(b, depth_bound=10 ** 9).run() & SYNTAX_OK)


def value_bits(b: bytes) -> int:
    """the device's verdict bits (fabgpu_test_couch_values), on either path"""
    return Scanner(bytes(b)).run()


def code_of_bits(v: int) -> int:
    if v & CUT:
        return UNDET if v & TOP_OBJECT else OK
    if not v & SYNTAX_OK or not v & TOP_OBJECT or v & NUM_ERR or not v & RESERVED:
        return OK
    return UNDET if v & NUM_UNDET else INVALID


def value_code(b: bytes) -> int:
    """OK, INVALID (validateValue fails) or UNDET"""
    return code_of_bits(value_bits(b))


# ---- the stage ---------------------------------------------------------------------------------------------------------------------
def _wv(x):
    """(key, is_delete, value bytes or None) of a writes entry"""
    v = x[2] if len(x) > 2 else True
    v = b"value" if v is True else (None if v is False or v is None or v == b"" else bytes(v))
    return x[0], x[1], v


def _write(key, delete, value):
    return pb.f_bytes(1, key) + (pb.f_uint(2, 1) if delete else b"") + (pb.f_bytes(3, value) if value is not None else b"")


def encode(tx) -> bytes:
    """range_oracle.encode with each write's value as given (a delete's too)"""
    out = b""
    for ns in tx:
        kv = b"".join(pb.f_bytes(1, pb.f_bytes(1, ro._b(k)) + mo._version(v, mo._same_part)) for k, v in ns.get("reads", ()))
        for r in ns.get("ranges", ()):
            kv += pb.f_bytes(2, r if isinstance(r, bytes) else ro.range_info(*r))
        kv += b"".join(pb.f_bytes(3, _write(ro._b(k), d, v)) for k, d, v in map(_wv, ns.get("writes", ())))
        kv += b"".join(pb.f_bytes(4, mo._md(ro._b(k), e)) for k, e in map(mo._m, ns.get("md", ())))
        body = pb.f_bytes(1, ns["ns"].encode()) + pb.f_bytes(2, kv)
        for name, hr, hw, hm in ns.get("colls", ()):
            h = b"".join(pb.f_bytes(1, pb.f_bytes(1, ro._b(k)) + mo._version(v, mo._same_part)) for k, v in hr)
            h += b"".join(pb.f_bytes(2, mo._write(ro._b(k), d, v)) for k, d, v in map(mo._w, hw))
            h += b"".join(pb.f_bytes(3, mo._md(ro._b(k), e)) for k, e in map(mo._m, hm))
            body += pb.f_bytes(3, pb.f_bytes(1, name.encode()) + pb.f_bytes(2, h))
        out += pb.f_bytes(2, body)
    return out


def _as_range_tx(tx):
    """the transaction as range_oracle reads it: a write's value is only whether it has one"""
    if tx is None:
        return None
    out = []
    for ns in tx:
        n = dict(ns)
        if "writes" in ns:
            n["writes"] = [(k, d, v is not None) for k, d, v in map(_wv, ns["writes"])]
        out.append(n)
    return out


def tx_code(tx):
    """INVALID_WRITESET, NOT_VALIDATED or None (unchanged) for a VALID transaction under CouchDB"""
    inv = undet = False
    for ns in tx:
        for k, _, v in map(_wv, ns.get("writes", ())):
            if not key_ok(k):
                inv = True
            elif v:
                c = value_code(v)
                inv |= c == INVALID
                undet |= c == UNDET
        for k, _ in ns.get("reads", ()):
            undet |= not key_ok(k)
        for r in ns.get("ranges", ()):
            if isinstance(r, bytes):
                continue                            # a form the stage does not decode: 254 there
            start, end, exhausted, _ = r
            undet |= not utf8_valid(ro._b(start)) or not utf8_valid(ro._b(end)) or (not exhausted and not key_ok(end))
    return INVALID_WRITESET if inv else NOT_VALIDATED if undet else None


def validate(state, block_num, txs, tv, couch=True):
    """range_oracle.validate (an index installed), after CouchDB's pre-pass when couch: (flags, new state, open)"""
    tv = list(tv)
    if couch:
        for t, tx in enumerate(txs):
            if tv[t] == VALID and tx is not None:
                c = tx_code(tx)
                if c is not None:
                    tv[t] = c
    return ro.validate(state, block_num, [_as_range_tx(tx) for tx in txs], tv)
