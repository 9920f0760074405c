"""Range-query cases with their codes written out, for the MVCC stage with an ordered key index.  A case is (name, state before, steps): a
step is a block (transactions, validator flags, expected flags) in range_oracle's transaction form, or ("update", entries) -- a
fabgpu_state_versions_update at the current height.  Blocks run from height 1 on; the state is installed with its index."""
from tools import fabricpb as pb
import range_oracle as ro

V, C, N = 0, 11, 254
CC = "mycc"
M = ro.Merkle


def k(s):
    return s.encode("utf-8") if isinstance(s, str) else s


def tx(ranges=(), reads=(), writes=(), md=(), ns=CC):
    return [dict(ns=ns, reads=list(reads), writes=list(writes), md=list(md), ranges=list(ranges))]


def q(start, end, reads, exhausted=True):
    """one range query; reads: [(key, version)], None or a Merkle"""
    return tx(ranges=[(start, end, exhausted, reads)])


def w(*keys):
    return tx(writes=[(x, False) for x in keys])


def dl(*keys):
    return tx(writes=[(x, True) for x in keys])


def state(**kv):
    return {(CC, "", k(x)): v for x, v in kv.items()}


S = state(a=(1, 0), b=(1, 1), c=(2, 0), d=(0, 5))
A, B, Cv, D = ("a", (1, 0)), ("b", (1, 1)), ("c", (2, 0)), ("d", (0, 5))
# composite keys: "\x00owner\x00alice\x00" ... "\x00owner\x00alice\x00" + U+10FFFF, as GetStateByPartialCompositeKey records them
OWN = "\x00owner\x00alice\x00"
SC = {**S, (CC, "", k(OWN + "a1")): (1, 2), (CC, "", k(OWN + "a2")): (1, 3), (CC, "", k("\x00owner\x00bob\x00b1")): (1, 4)}
# keys that are prefixes of one another, and bytes >= 0x80
SP = {(CC, "", x): (0, i) for i, x in enumerate([b"p", b"pa", b"pab", b"p\x80", b"p\xff", b"q"])}
# many keys, for Merkle trees
MANY = {(CC, "", b"m%02d" % i): (3, i) for i in range(20)}
MK = [(b"m%02d" % i, (3, i)) for i in range(20)]
# the key "" (an empty end key served when itr_exhausted is false)
SE = {**S, (CC, "", b""): (3, 3)}


def merkle(results, d):
    return ro.summary_of([(k(x), v) for x, v in results], d)


def _bad(*parts):
    return [dict(ns=CC, ranges=[b"".join(parts)])]


BOTH = pb.f_bytes(1, b"a") + pb.f_bytes(2, b"z") + pb.f_uint(3, 1) + pb.f_bytes(4, b"") + pb.f_bytes(5, pb.f_uint(1, 2))
TWICE = pb.f_bytes(1, b"a") + pb.f_bytes(4, b"") + pb.f_bytes(4, b"")
TRUNC = pb.f_bytes(1, b"a") + b"\x12\x05zz"


def cases():
    m3 = merkle(MK[:3], 2)
    m7 = merkle(MK[:7], 2)
    m20 = merkle(MK, 2)
    m20_3 = merkle(MK, 3)
    return [
        # ---- range shape
        ("empty_range", S, [([q("x", "y", []), q("x", "y", [A]), q("x", "y", None)], [V, V, V], [V, C, V])]),
        ("exhausted", S, [([q("a", "d", [A, B, Cv]), q("", "", [A, B, Cv, D]), q("b", "", [B, Cv, D])], [V, V, V], [V, V, V])]),
        ("not_exhausted_end_present", S, [([q("a", "c", [A, B, Cv], False), q("a", "c", [A, B], False), q("a", "c", [A, B])],
                                           [V, V, V], [V, C, V])]),
        ("not_exhausted_end_absent", S, [([q("a", "x", [A, B, Cv, D], False), q("a", "x", [A, B, Cv, D, ("x", (0, 0))], False)],
                                          [V, V], [V, C])]),
        ("not_exhausted_end_deleted_in_block", S, [([dl("c"), q("a", "c", [A, B], False), q("a", "c", [A, B, Cv], False)],
                                                    [V, V, V], [V, V, C])]),
        ("not_exhausted_end_put_in_block", S, [([w("x"), q("a", "x", [A, B, Cv, D, ("x", (1, 0))], False), q("a", "x", [A, B, Cv, D], False)],
                                                [V, V, V], [V, V, C])]),
        ("start_after_end", S, [([q("d", "b", [B], False), q("d", "b", [], False), q("d", "b", []), q("d", "b", [D])],
                                 [V, V, V, V], [V, C, V, C])]),
        ("empty_end_not_exhausted", SE, [([q("", "", [("", (3, 3)), A, B, Cv, D, ("", (3, 3))], False), q("", "", [("", (3, 3)), A, B, Cv, D], False),
                                           q("c", "", [Cv, D, ("", (3, 3))], False)], [V, V, V], [V, C, V])]),
        ("composite_key_bounds", SC, [([q(OWN, OWN + "\U0010ffff", [(OWN + "a1", (1, 2)), (OWN + "a2", (1, 3))]),
                                        q(OWN, OWN + "\U0010ffff", [(OWN + "a1", (1, 2))]),
                                        q("\x00owner\x00", "\x00owner\x00\U0010ffff", [(OWN + "a1", (1, 2)), (OWN + "a2", (1, 3)), ("\x00owner\x00bob\x00b1", (1, 4))])],
                                       [V, V, V], [V, C, V])]),
        ("prefix_keys_and_high_bytes", SP, [([q(b"p", b"q", [(b"p", (0, 0)), (b"pa", (0, 1)), (b"pab", (0, 2)), (b"p\x80", (0, 3)), (b"p\xff", (0, 4))]),
                                              q(b"p", b"q", [(b"p", (0, 0)), (b"p\x80", (0, 3)), (b"pa", (0, 1)), (b"pab", (0, 2)), (b"p\xff", (0, 4))]),
                                              q(b"pa", b"p\x80", [(b"pa", (0, 1)), (b"pab", (0, 2))]),
                                              q(b"p\x80", b"", [(b"p\x80", (0, 3)), (b"p\xff", (0, 4)), (b"q", (0, 5))])],
                                             [V, V, V, V], [V, C, V, V])]),
        # ---- result mismatches
        ("version_mismatch", S, [([q("a", "d", [A, ("b", (1, 2)), Cv]), q("a", "d", [A, ("b", ()), Cv])], [V, V], [C, C])]),
        # a raw read without a Version: the reference dereferences it once it is reached with a result of its key (254); a mismatching
        # key, or no result, returns false first
        ("raw_read_without_version", {**S, (CC, "", b"z"): (0, 0)},
         [([q("a", "d", [A, ("b", None), Cv]), q("z", "", [("z", None)]), q("a", "d", [A, ("bb", None), Cv]), q("x", "y", [("x", None)]),
            q("a", "d", [("b", None)])], [V, V, V, V, V], [N, N, C, C, C])]),
        ("missing_result", S, [([q("a", "d", [A, Cv])], [V], [C])]),
        ("extra_result", S, [([q("a", "d", [A, B, Cv, D]), q("a", "d", [A, B, ("bb", (1, 1)), Cv])], [V, V], [C, C])]),
        # ---- earlier writers in the block
        ("put_in_range", S, [([w("bb"), q("a", "d", [A, B, Cv])], [V, V], [V, C])]),
        ("delete_in_range", S, [([dl("b"), q("a", "d", [A, B, Cv]), q("a", "d", [A, Cv])], [V, V, V], [V, C, V])]),
        ("metadata_write_in_range", S, [([tx(md=["b"]), q("a", "d", [A, B, Cv]), q("a", "d", [A, ("b", (1, 0)), Cv])], [V, V, V], [V, C, V])]),
        ("metadata_write_on_absent_key_in_range", S, [([tx(md=["bb"]), q("a", "d", [A, B, Cv])], [V, V], [V, V])]),
        ("writer_flagged_invalid", S, [([w("bb"), dl("b"), q("a", "d", [A, B, Cv])], [10, 4, V], [10, 4, V])]),
        ("writer_undetermined", S, [([w("bb"), q("a", "d", [A, B, Cv]), q("x", "y", [])], [N, V, V], [N, N, V])]),
        ("writer_mvcc_conflict", S, [([tx(reads=[("a", (9, 9))], writes=[("bb", False)]), q("a", "d", [A, B, Cv])], [V, V], [C, V])]),
        ("crafted_read_of_in_block_version", S, [([w("bb"), q("a", "d", [A, B, ("bb", (1, 0)), Cv]), w("b"),
                                                   q("a", "d", [A, ("b", (1, 2)), ("bb", (1, 0)), Cv])], [V, V, V, V], [V, V, V, V])]),
        ("writer_after_the_range", S, [([q("a", "d", [A, B, Cv]), w("bb")], [V, V], [V, V])]),
        ("chain_of_ranges", S, [([q("a", "c", [A, B], False), w("bb"), q("a", "c", [A, B, ("bb", (1, 1))]), dl("a"),
                                  q("a", "c", [B, ("bb", (1, 1)), Cv], False)], [V, V, V, V, V], [C, V, V, V, V])]),
        # ---- Merkle summaries
        ("merkle_max_degree_results", MANY, [([q("m00", "m02", merkle(MK[:3], 2)), q("m00", "m03", m3), q("m00", "m02", M(2, 1, []))],
                                              [V, V, V], [C, V, C])]),
        ("merkle_deeper_trees", MANY, [([q("m00", "m07", m7), q("m00", "", m20), q("m00", "", m20_3), q("m00", "m19", m20)],
                                        [V, V, V, V], [V, V, V, C])]),
        ("merkle_wrong_shape", MANY, [([q("m00", "", M(2, m20.max_level + 1, m20.hashes)), q("m00", "", M(2, m20.max_level, m20.hashes + [m20.hashes[0]])),
                                        q("m00", "", M(2, m20.max_level, m20.hashes[:-1] or [b"x" * 32])),
                                        q("m00", "", M(2, m20.max_level, [h[:31] + b"\x00" for h in m20.hashes]))],
                                       [V, V, V, V], [C, C, C, C])]),
        # the reference's early-exit loop indexes past the top level when it rises after lastMatchedIndex passed 0 (a panic: 254);
        # max_degree 2: the summary of 6 results, then 9 results with the same first 6 -- or 7, where the loop returns false first
        ("merkle_early_exit_out_of_range", MANY, [([q("m00", "m09", merkle(MK[:6], 2)), q("m00", "m07", merkle(MK[:6], 2)),
                                                    q("m00", "m06", merkle(MK[:6], 2)), q("m00", "m12", merkle(MK[:9], 2))],
                                                   [V, V, V, V], [N, C, V, C])]),
        ("merkle_small_degree", MANY, [([q("m00", "m05", M(0, 1, [])), q("m00", "m05", M(1, 1, [])), q("x", "y", M(1, 1, []))],
                                        [V, V, V], [N, N, N])]),
        ("merkle_with_block_writes", MANY, [([w("m03x"), q("m00", "m07", m7), q("m00", "m07", merkle(MK[:4] + [("m03x", (1, 0))] + MK[4:7], 2))],
                                             [V, V, V], [V, C, V])]),
        # ---- wire forms not decoded, unknown keys
        ("both_oneof_fields", S, [([_bad(BOTH)], [V], [N])]),
        ("oneof_field_twice", S, [([_bad(TWICE)], [V], [N])]),
        ("unparsable_range_info", S, [([_bad(TRUNC)], [V], [N])]),
        ("unknown_key_in_range", S, [([w("bq")], [N], [N]),
                                     ([q("a", "d", [A, B, Cv]), q("c", "e", [Cv, D]), q("a", "b", [A, B], False), q("a", "bq", [A, B], False)],
                                      [V, V, V, V], [N, V, V, N]),
                                     ("update", [((CC, "", b"bq"), (2, 7))]),
                                     ([q("a", "d", [A, B, ("bq", (2, 7)), Cv])], [V], [V])]),
        # ---- index maintenance
        ("dead_entries_skipped", S, [("update", [((CC, "", b"b"), ro.mo.REMOVE)]), ([q("a", "d", [A, Cv]), q("a", "d", [A, B, Cv])], [V, V], [V, C])]),
        ("block_keys_seen_next_block", S, [([w("bz"), dl("c")], [V, V], [V, V]),
                                           ([q("a", "d", [A, B, ("bz", (1, 0))]), q("a", "d", [A, B])], [V, V], [V, C])]),
        ("update_keys_seen", S, [("update", [((CC, "", b"by"), (5, 5)), ((CC, "", b"bx"), ro.mo.REMOVE), ((CC, "coll", b"bw"), (5, 6))]),
                                 ([q("a", "d", [A, B, ("by", (5, 5)), Cv]), q("a", "d", [A, B, Cv])], [V, V], [V, C])]),
        ("other_namespace_untouched", S, [([w("bb"), tx(writes=[("bb", False)], ns="othercc"), q("a", "d", [A, B, Cv, D], False)],
                                           [10, V, V], [10, V, V])]),
    ]
