"""Protobuf wire-level mutations of one serialized message, and a seeded corpus of mutated transactions built with them.

Each mutation takes a well-formed message (what tools/blockgen.py assembles at one level) and returns other bytes for it.  The
mutated bytes go back into build_block through its `mutate` hook, so every enclosing length prefix, the tx id, the proposal hash
and the signatures are computed from them: a mutation inside a signed message reaches the check it is aimed at instead of
stopping at the creator signature.

Kinds (KINDS; "chdr_int" applies to ChannelHeader only):
  tags       alias (field number + k * 2^32), big_field (2^29 - 1, 2^29, 2^32 - 1, 2^32, 2^61 - 1, 2^61), field_zero,
             padded_tag (non-minimal tag varints, up to the 11 bytes that overflow)
  varints    padded_varint (non-minimal lengths and values), varint10_high (10 bytes: the last one 0 or 1, valid, or with higher
             bits set, an overflow), varint11,
             chdr_int (ChannelHeader.type = 3 + 2^32, 3 + 2^63, -1 as 10 bytes, ...; epoch = 2^64 - 1, ...)
  wire types wire_type (a known field under each wire type 0-7), unknown_field (an unknown field of wire type 0-7, groups
             included, before, between or after the known ones)
  structure  repeat (a singular field twice, the changed copy first or last), empty_or_absent, len_off (+-1), truncate,
             huge_len (length varints >= 2^32)
  bytes      flip (seeded flips, inserts and deletes)
"""
import functools
import random

import numpy as np

from oracle import blockval as ob
from tools import blockgen
from tools import fabricpb as pb
import blockutil

KINDS = ("alias", "big_field", "field_zero", "padded_tag", "padded_varint", "varint10_high", "varint11", "chdr_int", "wire_type",
         "unknown_field", "repeat", "empty_or_absent", "len_off", "truncate", "huge_len", "flip")
TX_PARTS = tuple(p for p in blockgen.PARTS if p != "Block")


def uvarint(v: int, width: int = 0) -> bytes:
    """Base-128 varint of v (any size), padded with continuation bytes to `width` bytes when that is longer."""
    out = bytearray()
    while True:
        b, v = v & 0x7F, v >> 7
        if v or len(out) + 1 < width:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def varint10_high(v: int, high: int) -> bytes:
    """v's low 64 bits as a 10-byte varint whose last byte also carries `high`.  With high = 0 the last byte is 0 or 1 (bit 63)
    and the varint is valid; any other last byte overflows 64 bits, which golang/protobuf's decodeVarint rejects."""
    v &= (1 << 64) - 1
    return bytes(((v >> (7 * i)) & 0x7F) | 0x80 for i in range(9)) + bytes([(v >> 63) | (high & 0x7E)])


def split(msg: bytes):
    """[(field, wire_type, value)]: value is an int (varint), raw bytes (fixed64 / fixed32) or the payload (length-delimited)."""
    out = []
    for f, wt, v in pb.fields(msg):
        if wt in (1, 5):
            v = int(v).to_bytes(8 if wt == 1 else 4, "little")
        out.append((f, wt, bytes(v) if wt == 2 else v))
    return out


def body(wt: int, v, ln: bytes = None) -> bytes:
    if wt == 0:
        return uvarint(v if isinstance(v, int) else len(v))
    if wt == 1:
        return (v if isinstance(v, bytes) else int(v).to_bytes(8, "little"))[:8].ljust(8, b"\0")
    if wt == 5:
        return (v if isinstance(v, bytes) else int(v).to_bytes(8, "little"))[:4].ljust(4, b"\0")
    if wt == 2:
        v = v if isinstance(v, bytes) else uvarint(v)
        return (ln if ln is not None else uvarint(len(v))) + v
    return b""                                                     # 3 / 4: group start / end; 6 / 7: no such wire type


def enc(f: int, wt: int, v, tag: bytes = None, ln: bytes = None) -> bytes:
    return (tag if tag is not None else uvarint((f << 3) | wt)) + body(wt, v, ln)


def _other(r, v):
    """A value of the same kind as v but different from it."""
    if isinstance(v, int):
        return v + 1 + r.randrange(5)
    return bytes(r.getrandbits(8) for _ in range(max(1, min(len(v), 40)))) if r.random() < 0.5 else v[::-1] + b"x"


def _unknown(r, f=None, wt=None):
    f = f if f is not None else r.choice((9, 15, 16, 127, 128, 2047, 1 << 20))
    wt = wt if wt is not None else r.randrange(8)
    if wt == 3:                                                    # a group: start, one field, end (or no end)
        inner = enc(1, 0, r.randrange(300)) if r.random() < 0.5 else b""
        return enc(f, 3, None) + inner + (enc(f, 4, None) if r.random() < 0.7 else b"")
    return enc(f, wt, r.choice((0, 1, 300, b"", b"xyz", bytes(9))) if wt in (0, 2) else bytes(8))


def mutate(r: random.Random, kind: str, part: str, msg: bytes) -> bytes:
    """One mutation of `kind` applied to the well-formed message `msg` of level `part`."""
    fs = split(msg)
    ch = [enc(*x) for x in fs]
    pos = lambda: r.randrange(len(ch) + 1)
    if not fs or kind == "unknown_field":                          # before, between or after the known fields
        ch.insert(r.choice((0, len(ch), pos())), _unknown(r))
        return b"".join(ch)
    i = r.randrange(len(fs))
    f, wt, v = fs[i]
    if kind == "alias":
        k = r.choice((1, 2, 7, r.randrange(1, 1 << 28)))
        mode = r.randrange(3)
        if mode == 0:                                              # the known field becomes field f + k * 2^32
            ch[i] = enc(f + (k << 32), wt, v)
        elif mode == 1:                                            # an extra field f + k * 2^32 with other contents
            ch.insert(pos(), enc(f + (k << 32), wt, _other(r, v)))
        else:                                                      # field f garbled, its true value under f + k * 2^32
            ch[i] = enc(f, wt, _other(r, v))
            ch.insert(pos(), enc(f + (k << 32), wt, v))
    elif kind == "big_field":
        F = r.choice(((1 << 29) - 1, 1 << 29, (1 << 32) - 1, 1 << 32, (1 << 61) - 1, 1 << 61))
        w = r.choice((0, 1, 2, 5))
        ch.insert(pos(), enc(F, w, r.choice((1, b"xyz")) if w in (0, 2) else bytes(8)))
    elif kind == "field_zero":
        ch.insert(pos(), enc(0, r.choice((0, 2)), r.choice((0, b"zero"))))
    elif kind == "padded_tag":
        key = (f << 3) | wt
        ch[i] = enc(f, wt, v, tag=uvarint(key, r.randint(len(uvarint(key)) + 1, 11)))
    elif kind == "padded_varint":
        n = v if wt == 0 else len(v) if wt == 2 else None
        if n is None:
            ch[i] = enc(f, wt, v, tag=uvarint((f << 3) | wt, r.randint(2, 11)))
        elif wt == 0:
            ch[i] = uvarint((f << 3) | wt) + uvarint(n, r.randint(len(uvarint(n)) + 1, 11))
        else:
            ch[i] = enc(f, wt, v, ln=uvarint(n, r.randint(len(uvarint(n)) + 1, 11)))
    elif kind == "varint10_high":                                  # a valid 10-byte varint (last byte 0 / 1) or an overflowing one
        high = r.choice((0, 0, 0x02, 0x40, 0x7E))
        b63 = (1 << 63) if r.random() < 0.3 else 0
        if r.randrange(2) == 0 or wt not in (0, 2):               # the tag (bit 63: a field number >= 2^60)
            ch[i] = enc(f, wt, v, tag=varint10_high(((f << 3) | wt) | b63, high))
        elif wt == 0:
            ch[i] = uvarint((f << 3) | wt) + varint10_high(v | b63, high)
        else:
            ch[i] = enc(f, wt, v, ln=varint10_high(len(v) | b63, high))
    elif kind == "varint11":                                       # one byte past what a 64-bit varint may take
        if r.random() < 0.5 or wt not in (0, 2):
            ch[i] = uvarint((f << 3) | wt, 11) + body(wt, v)
        else:
            ch[i] = uvarint((f << 3) | wt) + (uvarint(v, 11) if wt == 0 else uvarint(len(v), 11) + v)
    elif kind == "chdr_int":
        if part != "ChannelHeader":
            raise ValueError("chdr_int applies to ChannelHeader")
        ch = [c for c, x in zip(ch, fs) if x[0] not in (1, 6)] if r.random() < 0.5 else ch
        if r.random() < 0.7:                                       # int32 type: Go keeps the low 32 bits
            t = r.choice((3 + (1 << 32), 3 + (1 << 63), (1 << 64) - 1, 1 + (1 << 32), 2 + (1 << 32), 3 + (1 << 31), (1 << 32) - 3, 4 + (1 << 32)))
            ch.insert(pos() if ch else 0, enc(1, 0, t))
        else:                                                      # uint64 epoch
            ch.insert(pos() if ch else 0, enc(6, 0, r.choice(((1 << 64) - 1, 1 << 32, 1 << 63, 0))))
    elif kind == "wire_type":
        w = r.randrange(8)
        ch[i] = enc(f, w, v if w in (0, 2) or not isinstance(v, int) else v.to_bytes(8, "little"))
    elif kind == "repeat":
        dup = enc(f, wt, _other(r, v))
        ch.insert(i + 1 if r.random() < 0.5 else i, dup)           # the changed copy last (it wins) or first (the original wins)
    elif kind == "empty_or_absent":
        j = r.choice([k for k, x in enumerate(fs) if x[1] == 2] or [i])
        ch[j] = enc(fs[j][0], 2, b"") if r.random() < 0.5 else b""
    elif kind == "len_off":
        j = r.choice([k for k, x in enumerate(fs) if x[1] == 2] or [i])
        g, _, w = fs[j]
        if fs[j][1] == 2:
            ch[j] = enc(g, 2, w, ln=uvarint(max(0, len(w) + r.choice((-1, 1)))))
    elif kind == "truncate":
        m = b"".join(ch)
        return m[: r.randrange(len(m))]
    elif kind == "huge_len":
        j = r.choice([k for k, x in enumerate(fs) if x[1] == 2] or [i])
        if fs[j][1] == 2:
            g, _, w = fs[j]
            # len + 2^32 reads as the true length once cut to 32 bits
            ch[j] = enc(g, 2, w, ln=uvarint(r.choice((len(w) + (1 << 32), len(w) + (1 << 33), (1 << 32) - 1, 1 << 63))))
    elif kind == "flip":
        m = bytearray(b"".join(ch))
        for _ in range(r.choice((1, 1, 2, 4))):
            op = r.random()
            if op < 0.6 and m:
                m[r.randrange(len(m))] ^= 1 << r.randrange(8)
            elif op < 0.8 and m:
                del m[r.randrange(len(m))]
            else:
                m.insert(r.randrange(len(m) + 1), r.getrandbits(8))
        return bytes(m)
    else:
        raise ValueError(kind)
    return b"".join(ch)


def plan(n_tx: int, seed: int, start: int = 0):
    """[(part, kind) or None] for n_tx transactions: every (level, kind) pair in turn, one transaction in eight left alone."""
    combos = [(p, k) for p in TX_PARTS for k in KINDS if k != "chdr_int" or p == "ChannelHeader"]
    random.Random(seed).shuffle(combos)
    out = []
    for t in range(n_tx):
        g = start + t
        out.append(None if g % 8 == 7 else combos[(g - g // 8) % len(combos)])
    return out


# fields leading from a level down to its ChannelHeader (Envelope.payload, Payload.header, Header.channel_header)
_CHDR_PATH = {"ChannelHeader": (), "Header": (1,), "Payload": (1, 1), "Envelope": (1, 1, 1)}


def _makes_config(part, data):
    """True when `data` of level `part` holds a ChannelHeader that decodes as a CONFIG transaction (type 1): config transactions
    are outside the oracle's restated scope."""
    if part not in _CHDR_PATH:
        return False
    try:
        for f in _CHDR_PATH[part]:
            data = pb.parse(data, {f: ("x", "bytes")})["x"] or b""
        return ob.int32_field(pb.parse(data, {1: ("type", "uint")})["type"] or 0) == 1
    except pb.PbError:
        return False


class Mutator:
    """build_block's `mutate` hook for one block: transaction t gets labels[t] = (part, kind), applied to the first occurrence of
    that level, with a random stream of its own (seed, t).  A mutation that would make a config transaction is drawn again."""

    def __init__(self, labels, seed):
        self.labels, self.seed, self.done = labels, seed, set()

    def __call__(self, t, part, data):
        lab = self.labels[t] if t is not None else None
        if lab is None or lab[0] != part or t in self.done:
            return data
        self.done.add(t)
        r = random.Random(self.seed * 1000003 + t)
        while True:
            out = mutate(r, lab[1], part, data)
            if not _makes_config(part, out):
                return out


def shape_namespaces(t):
    """Every corpus transaction has a private-data collection, so that the hashed read/write-set levels exist."""
    return [(blockgen.CHAINCODE, 2, 2, 1)]


def corpus_block(net, n_tx, seed, start=0, nthreads=2):
    """(block, info, labels): n_tx transactions, each mutated at one level (or left alone), each with a chaincode event and a
    private-data collection so that every level of blockgen.PARTS but Block occurs."""
    labels = plan(n_tx, seed, start)
    m = Mutator(labels, seed)
    blk, info = blockgen.build_block(net, n_tx, 3, {}, seed=seed, nthreads=nthreads, mutate=m, namespaces=shape_namespaces, events=lambda t: True)
    assert m.done == {t for t, lab in enumerate(labels) if lab is not None}, "a label names a level the transaction does not have"
    return blk, info, labels


CORPUS_BLOCKS, CORPUS_TX = 8, 440      # 3 520 transactions, 3 080 of them mutated


@functools.lru_cache(maxsize=None)
def corpus():
    """CORPUS_BLOCKS blocks of CORPUS_TX transactions, each mutated at one level (one in eight left alone), with the oracle's flags."""
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    nodes, pol = net.policies_for(2)
    out = []
    for b in range(CORPUS_BLOCKS):
        blk, info, labels = corpus_block(net, CORPUS_TX, seed=101 + b, start=b * CORPUS_TX)
        exp = ob.validate_block(blk, ids, net.channel, nodes, net.principals, policies=pol, known=[i[0] for i in ids])
        out.append((blk, info, labels, exp))
    return net, ids, nodes, pol, out


def block_mutants(n_per_kind=60):
    """[(kind, Block bytes)]: a 3-transaction block mutated n_per_kind times per kind, at the Block level and at the BlockData level."""
    net = blockgen.Network()
    blk, _ = blockgen.build_block(net, 3, 3, {}, seed=5, nthreads=2)
    blk_fields = split(blk)
    data = [v for f, wt, v in blk_fields if f == 2][0]
    out = []
    for kind in KINDS:
        if kind == "chdr_int":
            continue
        for s in range(n_per_kind):
            r = random.Random(s * 7919 + len(kind))
            if s % 2 == 0:
                out.append((kind, mutate(r, kind, "Block", blk)))
            else:
                d = mutate(r, kind, "BlockData", data)
                out.append((kind, b"".join(enc(f, wt, d if f == 2 else v) for f, wt, v in blk_fields)))
    return out


def ten_byte_varint(v, last):
    """v's low 63 bits in 10 bytes, the 10th byte being `last`."""
    return bytes(((v >> (7 * i)) & 0x7F) | 0x80 for i in range(9)) + bytes([last])


# (ChannelHeader field, value's low 63 bits, 10th byte, expected flag): the 10th byte may only be 0 or 1 (bit 63)
TEN_BYTE_CASES = [(1, 3, 0, ob.VALID), (1, 3, 1, ob.VALID), (1, 3, 2, ob.BAD_COMMON_HEADER), (1, 3, 0x7E, ob.BAD_COMMON_HEADER),
                  (6, 0, 0, ob.VALID), (6, 0, 1, ob.BAD_COMMON_HEADER), (6, 0, 2, ob.BAD_COMMON_HEADER), (6, 0, 0x40, ob.BAD_COMMON_HEADER)]


def ten_byte_block(net, field, v, last):
    """A 2-transaction block whose ChannelHeaders carry `field` (type = 1, epoch = 6) as a 10-byte varint ending in `last`."""
    def mut(t, part, b):
        if part != "ChannelHeader":
            return b
        return b"".join(enc(*f) for f in split(b) if f[0] != field) + uvarint(field << 3) + ten_byte_varint(v, last)
    return blockgen.build_block(net, 2, 3, {}, seed=5, nthreads=2, mutate=mut)
