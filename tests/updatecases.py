"""Update-batch cases with their batches written out: (name, state before, [(transactions, validator flags, batch[, CouchDB batch])]).
The state is {(ns, coll, key): (version, value, metadata)}; transactions are in updates_oracle's form; a batch is updates_oracle's record
list, or None where the peer builds the batch itself.  The blocks run in order from height 1; the CouchDB batch, when given, is the one
under CouchDB's pre-pass."""
import hashlib

import updates_oracle as uo

V, C, N = 0, 11, 254
CC = "mycc"
DEL, COM = uo.DEL, uo.COMMITTED


def h(k):
    return hashlib.sha256(k.encode()).digest()


def tx(writes=(), md=(), reads=(), colls=(), ns=CC):
    return [dict(ns=ns, reads=list(reads), writes=list(writes), md=list(md), colls=list(colls))]


def put(t, key, value, meta, coll=""):
    return (t, "put", CC, coll, key if isinstance(key, bytes) else key.encode(), value, meta)


def dele(t, key, coll=""):
    return (t, "del", CC, coll, key if isinstance(key, bytes) else key.encode(), None, None)


E0 = [("VALIDATION_PARAMETER", b"ep0")]
E1 = [("VALIDATION_PARAMETER", b"ep1")]
E2 = [("n2", b"v2"), ("n3", b"")]                 # an entry with an empty value: only its name is marshalled
M0, M1, M2 = uo.serialize(E0), uo.serialize(E1), uo.serialize(E2)
ST = {(CC, "", b"a"): ((1, 0), b"A0", M0), (CC, "", b"b"): ((0, 3), b"B0", None), (CC, "c1", h("q")): ((1, 1), b"HQ0", None)}


def cases():
    hot = [tx(writes=[("hot", b"h%d" % t)], md=[("hot", [("VALIDATION_PARAMETER", b"p%d" % t)])] if t % 5 == 0 else []) for t in range(40)]
    return [
        ("put_put", ST, [([tx(writes=[("a", b"v1"), ("a", b"v2"), ("x", b"v3"), ("x", b"v4")])], [V], [put(0, "a", COM, None)])]),
        ("del_del", ST, [([tx(writes=[("a", DEL), ("a", DEL)])], [V], [put(0, "a", COM, None)])]),
        ("put_mdel", ST, [([tx(writes=[("a", b"v1")], md=[("a", None)])], [V], [put(0, "a", b"v1", None)])]),
        ("meta_then_mdel", ST, [([tx(md=[("a", E1), ("a", None)])], [V], [put(0, "a", COM, M1)])]),
        ("put_meta_mdel", ST, [([tx(writes=[("a", b"v1")], md=[("a", E1), ("a", None)])], [V], [put(0, "a", b"v1", M1)])]),
        ("put_only_inherits_metadata", ST, [([tx(md=[("a", E1)]), tx(writes=[("a", b"v1")]), tx(writes=[("b", b"v2")])], [V] * 3,
                                             [put(1, "a", b"v1", M1), put(2, "b", b"v2", COM)])]),
        ("meta_only_committed_absent_after_put", ST, [([tx(md=[("a", E1), ("x", E2)]), tx(writes=[("y", b"v1")]), tx(md=[("y", E2)])], [V] * 3,
                                                       [put(0, "a", COM, M1), put(2, "y", b"v1", M2)])]),
        ("delete_then_put", ST, [([tx(writes=[("a", DEL)]), tx(writes=[("a", b"v1")]), tx(writes=[("b", DEL)])], [V] * 3,
                                  [put(1, "a", b"v1", None), dele(2, "b")])]),
        ("hashed_writes_and_metadata", ST, [([tx(colls=[("c1", [], [(h("p"), b"hv1")], [(h("p"), E1)])]),
                                              tx(colls=[("c1", [], [], [(h("q"), E2)])]), tx(colls=[("c2", [], [(h("p"), DEL)], [])])], [V] * 3,
                                             [put(0, h("p"), b"hv1", M1, "c1"), put(1, h("q"), COM, M2, "c1"), dele(2, h("p"), "c2")])]),
        ("empty_value_and_empty_entry", ST, [([tx(writes=[("a", b"")], md=[("b", [b""])])], [V], [put(0, "a", b"", COM), put(0, "b", COM, b"\x12\x00")])]),
        ("non_canonical_entry", ST, [([tx(md=[("a", [b"\x12\x00"])])], [V], None),
                                     ([tx(md=[("a", [b"\x12\x01v\x0a\x01n"])])], [V], None),
                                     ([tx(md=[("a", [b"\x0a\x81\x00n"])]), tx(writes=[("a", b"v1")], md=[("a", None)])], [V, V],
                                      [put(1, "a", b"v1", None)])]),
        ("written_by_an_11", ST, [([tx(reads=[("a", (9, 9))], writes=[("a", b"v1"), ("y", b"v2")]), tx(writes=[("a", b"v3")])], [V, V],
                                   [put(1, "a", b"v3", COM)])]),
        ("couch_24_writer", ST, [([tx(writes=[("a", b'{"_id":1}')]), tx(md=[("a", E1)])], [V, V],
                                  [put(1, "a", b'{"_id":1}', M1)], [put(1, "a", COM, M1)])]),
        ("hot_key", ST, [(hot, [V] * 40, [put(39, "hot", b"h39", uo.serialize([("VALIDATION_PARAMETER", b"p35")]))])]),
        ("no_writes", ST, [([tx(reads=[("a", (1, 0))])], [V], [])]),
        ("a_254_and_an_open_block", ST, [([tx(writes=[("a", b"v1")]), tx(writes=[("b", b"v2")])], [V, N], None),
                                         ([None, tx(writes=[("b", b"v3")])], [V, V], None)]),
    ]


def split(state):
    """(versions, values) of a case state"""
    return {k: v[0] for k, v in state.items()}, {k: (v[1], v[2]) for k, v in state.items()}
