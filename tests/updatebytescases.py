"""Update-bytes cases with their KVWrite lists written out: (name, block_num, state before, transactions, validator flags, KVWrites[,
CouchDB KVWrites]).  The state is {(ns, coll, key): (version, value, metadata)} and the table's height is block_num; transactions are in
updates_oracle's form; KVWrites is update_bytes_oracle's list, or None where the bytes are left to the peer.  The CouchDB list, when
given, is the one under CouchDB's pre-pass."""
import numpy as np

import updates_oracle as uo
import updatesutil
from update_bytes_oracle import height, kvwrite as K

V, N = 0, 254
CC = "mycc"
DEL = uo.DEL


class RawName(str):
    """a name whose wire bytes are `raw` (not UTF-8): updates_oracle.encode writes name.encode()"""
    def __new__(cls, raw):
        o = str.__new__(cls, raw.decode("latin-1"))
        o.raw = raw
        return o

    def encode(self, *args, **kwargs):
        return self.raw

    def __hash__(self):
        return str.__hash__(self)

    def __eq__(self, other):
        return str.__eq__(self, other)


def ns(name, writes=(), md=(), reads=(), colls=()):
    return dict(ns=name, reads=list(reads), writes=list(writes), md=list(md), colls=list(colls))


def tx(*namespaces):
    return list(namespaces)


def hk(first, last=0):
    """a 32-byte key hash: `first`, 30 zero bytes, `last`"""
    return bytes([first]) + bytes(30) + bytes([last])


B1 = 1
ST = {(CC, "", b"a"): ((0, 1), b"A0", None), (CC, "", b"gone"): ((0, 2), b"G0", None),
      (CC, "c1", hk(0x40)): ((0, 3), b"HQ0", None), (CC, "c1", hk(0x41)): ((0, 4), b"HR0", None)}
E1 = [("VALIDATION_PARAMETER", b"ep1")]


def H(tx_, block_num=B1):
    return height(block_num, tx_)


def cases():
    long_key = lambda c: b"p" * 35 + bytes([c]) + b"qqqq"
    return [
        ("namespaces_out_of_order", B1, ST,
         [tx(ns("zz", writes=[("k1", b"v1")]), ns("aa", writes=[("k2", b"v2")])),
          tx(ns("mm", writes=[("k3", b"v3")]), ns("aa", writes=[("k1", b"v4")]))], [V, V],
         [K(b"k1", b"v4", version=H(1), namespace="aa"), K(b"k2", b"v2", version=H(0)), K(b"k3", b"v3", version=H(1), namespace="mm"),
          K(b"k1", b"v1", version=H(0), namespace="zz")]),
        ("namespace_with_collection_writes_only", B1, ST,
         [tx(ns("beta", colls=[("c1", [], [(hk(0x20), b"hv1")], [])]), ns("alpha", writes=[("a", b"v1")]))], [V],
         [K(b"a", b"v1", version=H(0), namespace="alpha"), K(hk(0x20), b"hv1", version=H(0), namespace="beta", collection="c1")]),
        ("several_collections", B1, ST,
         [tx(ns(CC, writes=[("b", b"vb")], colls=[("c2", [], [(hk(0x10), b"x")], [])])),
          tx(ns(CC, writes=[("a", b"va")], colls=[("c1", [], [(hk(0x90), b"y"), (hk(0x05), b"z")], []), ("c10", [], [(hk(0x01), b"w")], [])]))],
         [V, V],
         [K(b"a", b"va", version=H(1), namespace=CC), K(b"b", b"vb", version=H(0)),
          K(hk(0x05), b"z", version=H(1), collection="c1"), K(hk(0x90), b"y", version=H(1)),
          K(hk(0x01), b"w", version=H(1), collection="c10"), K(hk(0x10), b"x", version=H(0), collection="c2")]),
        ("prefix_keys", B1, ST, [tx(ns(CC, writes=[("ab", b"1"), ("a\x00", b"2"), ("a", b"3")]))], [V],
         [K(b"a", b"3", version=H(0), namespace=CC), K(b"a\x00", b"2", version=H(0)), K(b"ab", b"1", version=H(0))]),
        ("high_bytes", B1, ST,
         [tx(ns("écc", writes=[(b"\xff", b"1")]), ns(CC, writes=[(b"\x80", b"2"), (b"\x7f", b"3"), (b"\xff\x00", b"4"), (b"\x01", b"5")],
                                                             colls=[("c1", [], [(hk(0xf0), b"h1"), (hk(0x70), b"h2")], [])]))], [V],
         [K(b"\x01", b"5", version=H(0), namespace=CC), K(b"\x7f", b"3", version=H(0)), K(b"\x80", b"2", version=H(0)), K(b"\xff\x00", b"4", version=H(0)),
          K(hk(0x70), b"h2", version=H(0), collection="c1"), K(hk(0xf0), b"h1", version=H(0)),
          K(b"\xff", b"1", version=H(0), namespace="écc")], []),
        ("keys_differing_after_32_bytes", B1, ST,
         [tx(ns(CC, writes=[(long_key(0x62), b"1"), (long_key(0x61), b"2")], colls=[("c1", [], [(hk(7, 0xff), b"h1"), (hk(7, 0x01), b"h2")], [])]))],
         [V],
         [K(long_key(0x61), b"2", version=H(0), namespace=CC), K(long_key(0x62), b"1", version=H(0)),
          K(hk(7, 0x01), b"h2", version=H(0), collection="c1"), K(hk(7, 0xff), b"h1", version=H(0))]),
        ("deletes_public_and_hashed", B1, ST,
         [tx(ns(CC, writes=[("gone", DEL)], colls=[("c1", [], [(hk(0x40), DEL)], [])]))], [V],
         [K(b"gone", is_delete=True, version=H(0), namespace=CC), K(hk(0x40), is_delete=True, version=H(0), collection="c1")]),
        ("put_with_an_empty_value", B1, ST, [tx(ns(CC, writes=[("a", b"")]))], [V],
         [K(b"a", version=H(0), namespace=CC)]),
        ("committed_values_public_and_hashed", B1, ST,
         [tx(ns(CC, md=[("a", E1)], colls=[("c1", [], [], [(hk(0x41), E1)])])), tx(ns(CC, writes=[("new", b"n1")]))], [V, V],
         [K(b"a", b"A0", version=H(0), namespace=CC), K(b"new", b"n1", version=H(1)), K(hk(0x41), b"HR0", version=H(0), collection="c1")]),
        ("block_0", 0, {}, [tx(ns(CC, writes=[("a", b"v")]))], [V], [K(b"a", b"v", version=b"\x00\x00", namespace=CC)]),
        ("block_255", 255, {}, [tx(ns(CC, writes=[("a", b"v")]))], [V], [K(b"a", b"v", version=b"\x01\xff\x00", namespace=CC)]),
        ("block_256", 256, {}, [tx(ns(CC, writes=[("a", b"v")])), tx(ns(CC, writes=[("b", b"w")]))], [V, V],
         [K(b"a", b"v", version=b"\x02\x01\x00\x00", namespace=CC), K(b"b", b"w", version=b"\x02\x01\x00\x01\x01")]),
        ("block_2_32", 1 << 32, {}, [tx(ns(CC, writes=[("a", b"v")]))], [V],
         [K(b"a", b"v", version=b"\x05\x01\x00\x00\x00\x00\x00", namespace=CC)]),
        ("block_2_56", 1 << 56, {}, [tx(ns(CC, writes=[("a", b"v")]))], [V],
         [K(b"a", b"v", version=b"\x08\x01\x00\x00\x00\x00\x00\x00\x00\x00", namespace=CC)]),
        ("lengths_around_varint_steps", B1, ST,
         [tx(ns(CC, writes=[(b"k" * 127, b"v" * 127), (b"l" * 128, b"w" * 128), (b"m", b"x" * 16383), (b"n", b"y" * 16384),
                            (b"o" * 16383, b"1"), (b"p" * 16384, b"2"), (b"q", b"z" * 40000)]))], [V],
         [K(b"k" * 127, b"v" * 127, version=H(0), namespace=CC), K(b"l" * 128, b"w" * 128, version=H(0)), K(b"m", b"x" * 16383, version=H(0)),
          K(b"n", b"y" * 16384, version=H(0)), K(b"o" * 16383, b"1", version=H(0)), K(b"p" * 16384, b"2", version=H(0)),
          K(b"q", b"z" * 40000, version=H(0))]),
        ("empty_batch", B1, ST, [tx(ns(CC, reads=[("a", (0, 1))]))], [V], []),
        ("empty_namespace_skipped", B1, ST, [tx(ns("", writes=[("cfg", b"c")]), ns(CC, writes=[("a", b"v")]))], [V],
         [K(b"a", b"v", version=H(0), namespace=CC)]),
        ("only_the_empty_namespace", B1, ST, [tx(ns("", writes=[("cfg", b"c")]))], [V], []),
        ("incomplete_batch", B1, ST, [tx(ns(CC, writes=[("a", b"v1")])), tx(ns(CC, writes=[("b", b"v2")]))], [V, N], None),
        ("collection_name_not_utf8", B1, ST, [tx(ns(CC, writes=[("a", b"v")], colls=[(RawName(b"c\xff"), [], [(hk(1), b"h")], [])]))], [V],
         None),
    ]


NSS = ["mycc", "cc2", "a", "zzé"]
COLLS = ["c1", "c2", "coll10"]


def random_tx(rng, pool, t):
    """updatesutil.random_tx's shape over several namespaces and collections, with random key bytes now and then"""
    out = []
    for name in rng.choice(NSS, size=int(rng.integers(1, 3)), replace=False):
        n = updatesutil.random_tx(rng, pool, t)[0]
        n["ns"] = str(name)
        if rng.random() < 0.3:
            n["writes"].append((bytes(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8)), b"r%d" % t))
        n["colls"] = [(str(rng.choice(COLLS)), hr, hw, hm) for _, hr, hw, hm in n["colls"]]
        out.append(n)
    return out


def split(state):
    """(versions, values) of a case state"""
    return {k: v[0] for k, v in state.items()}, {k: (v[1], v[2]) for k, v in state.items()}
