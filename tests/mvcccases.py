"""MVCC cases with their codes written out.  A case is (name, state before, [(transactions, validator flags, expected flags)]): the blocks
run in order from height 1 on, each one's flags through the MVCC check (mvcc_oracle's transaction form).  ns "mycc" is the chaincode
every generated transaction invokes; "othercc" is only read."""
import hashlib

V, C, N = 0, 11, 254          # VALID, MVCC_READ_CONFLICT, NOT_VALIDATED
CC, OTHER = "mycc", "othercc"


def h(k):
    return hashlib.sha256(k.encode()).digest()


def r(*reads, **kw):
    return [dict(ns=kw.get("ns", CC), reads=list(reads), writes=kw.get("writes", []), md=kw.get("md", []), range=kw.get("range", False),
                 colls=kw.get("colls", []))]


def w(*keys, **kw):
    return r(writes=[(k, False) for k in keys], **kw)


def d(*keys):
    return r(writes=[(k, True) for k in keys])


def md(*keys):
    return r(md=list(keys))


S0 = {(CC, "", b"a"): (1, 0), (CC, "", b"b"): (0, 3), (CC, "coll", h("p")): (1, 1)}


def cases():
    return [
        ("absent_nil_read", S0, [([r(("x", None))], [V], [V])]),
        ("absent_versioned_read", S0, [([r(("x", (1, 0)))], [V], [C])]),
        ("version_equal", S0, [([r(("a", (1, 0)), ("b", (0, 3)))], [V], [V])]),
        ("version_unequal", S0, [([r(("a", (1, 1)))], [V], [C])]),
        ("empty_version_vs_absent", {(CC, "", b"z"): (0, 0)}, [([r(("z", ())), r(("z", None)), r(("q", ()))], [V, V, V], [V, C, C])]),
        ("read_after_valid_put", S0, [([w("a"), r(("a", (1, 0)))], [V, V], [V, C])]),
        ("read_after_valid_delete", S0, [([d("a"), r(("a", (1, 0)))], [V, V], [V, C])]),
        ("read_after_validator_invalid_write", S0, [([w("a"), r(("a", (1, 0)))], [10, V], [10, V])]),
        ("read_after_mvcc_failed_write", S0, [([r(("a", (9, 9)), writes=[("a", False)]), r(("a", (1, 0)))], [V, V], [C, V])]),
        ("three_deep_chain", S0, [([r(("a", (1, 0)), writes=[("b", False)]), r(("b", (0, 3)), writes=[("c", False)]),
                                    r(("c", None), writes=[("a", False)]), r(("a", (1, 0)))], [V, V, V, V], [V, C, V, C])]),
        ("metadata_write_absent_then_read", S0, [([md("x"), r(("x", None))], [V, V], [V, V])]),
        ("metadata_write_present_then_read", S0, [([md("a"), r(("a", (1, 0)))], [V, V], [V, C])]),
        ("metadata_write_after_delete", S0, [([d("a"), md("a"), r(("a", None))], [V, V, V], [V, N, N])]),
        ("other_namespace_or_collection", S0, [([w("a"), r(("a", None), ns=OTHER),
                                                 r(colls=[("coll", [(h("a"), None)], [], [])]), r(colls=[("other", [(h("p"), None)], [], [])])],
                                                [V, V, V, V], [V, V, V, V])]),
        ("hashed_reads", S0, [([r(colls=[("coll", [(h("p"), (1, 1))], [], [])]), r(colls=[("coll", [(h("p"), (1, 2))], [], [])]),
                                r(colls=[("coll", [], [(h("p"), False)], [])]), r(colls=[("coll", [(h("p"), (1, 1))], [], [])])],
                               [V, V, V, V], [V, C, V, C])]),
        ("range_query", S0, [([r(("a", (1, 0)), range=True, writes=[("k", False)]), r(("k", None)), r(("a", (1, 0)))], [V, V, V], [N, N, V])]),
        ("unknown_keys_cleared_by_update", S0, [([w("u")], [N], [N]), ([r(("u", None)), r(("a", (1, 0)))], [V, V], [N, V])]),
        ("hot_key", S0, [([r(("a", (1, 0)), writes=[("a", False)]) for _ in range(5)], [V] * 5, [V, C, C, C, C])]),
        # one key written more than once by one transaction: the reference adds the operations' flags (tx_ops.go:185-205), so two
        # writes (2) and two writes + metadata (4) take the metadata path -- the key is dropped when absent, re-put with its latest value
        # when present -- and two deletes (16) do not delete
        ("duplicate_write_absent", S0, [([r(writes=[("x", False), ("x", False)]), r(("x", None))], [V, V], [V, V])]),
        ("duplicate_write_present", S0, [([r(writes=[("a", False), ("a", False)]), r(("a", (1, 0)))], [V, V], [V, C])]),
        ("duplicate_delete", S0, [([d("b", "b"), r(("b", (0, 3))), r(("q", None))], [V, V, V], [V, C, V]),
                                  ([r(("b", (1, 0)))], [V], [V])]),
        ("duplicate_write_and_metadata", S0, [([r(writes=[("x", False), ("x", False)], md=["x"]), r(("x", None))], [V, V], [V, V])]),
        ("write_and_metadata", S0, [([r(writes=[("x", False)], md=["x"]), r(("x", None))], [V, V], [V, C])]),
        # a write without a value is a nil value, on which PutValAndMetadata panics (statedb.go:202-205)
        ("write_without_value", S0, [([r(writes=[("x", False, False)]), r(("x", None)), r(writes=[("y", True, False)])], [V, V, V], [N, N, V])]),
        ("metadata_delete_absent_and_present", S0, [([md(("x", False)), md(("a", False)), r(("x", None)), r(("a", (1, 0)))],
                                                     [V, V, V, V], [V, V, V, C])]),
        ("metadata_after_undetermined_writer", S0, [([w("a"), md("a"), md("x")], [N, V, V], [N, N, V])]),
        ("open_block", S0, [([w("a"), None, r(("b", (0, 3)))], [V, V, V], [V, N, N])]),
    ]
