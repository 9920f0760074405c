"""Test infrastructure (not product code): the v1.3-mode cases (fabgpu_channel_capability(FABGPU_CAP_V1_3): the v1.4 validator with the
builtin v13 VSCC) that the oracle, the host build and the device are all held to, with every expected code written out.

The channel, node array and principals are collcases'.  The namespace table holds signature policies only (lscc chaincode definitions):
mycc wants 2 of 4 orgs, othercc 1 of 4, strictcc 3 of 4, qscc and cscc 1 of 4 (SignedByAnyMember), novercc 1 of 4 without an lscc
version; ghostcc has no entry.  Each endorsing org signs with its first peer.
"""
from oracle import blockval as ob
from tools import blockgen
import collcases
import klcases
import v13_oracle

V, F, NV, BAD = ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.NOT_VALIDATED, ob.ILLEGAL_WRITESET
EXP, OTHERR = v13_oracle.EXPIRED_CHAINCODE, ob.INVALID_OTHER_REASON
CC, OTHER, STRICT, NOVER, GHOST = collcases.CC, collcases.OTHER, "strictcc", "novercc", "ghostcc"
kh = blockgen.key_hash


def policies():
    _, r = collcases.forest()
    return {CC: r["cc"], OTHER: r["loose"], STRICT: r["strict"], NOVER: r["loose"], "qscc": r["loose"], "cscc": r["loose"], "lscc": r["loose"]}


def versions():
    return {CC: "1.0", OTHER: "2.0", STRICT: "1.0", "qscc": "1.0", "cscc": "1.0", "lscc": "1.0"}


def tx(orgs, namespaces, code, cc=(CC, "1.0"), fault=None):
    return (orgs, namespaces, fault, code, cc)


def cases():
    """[(name, {(ns, coll, key): vp tree name} or None for no key table, with a collection table, [tx(...)])]"""
    pub = [(CC, 1, 1)]
    return [
        # row 1: 255 where the dispatcher says 25; the checks before them keep their codes
        ("name_and_version_checks", None, False, [tx([0, 1], pub, OTHERR, fault="cc_name_mismatch"), tx([0, 1], pub, OTHERR, fault="empty_cc_version"),
                                                  tx([0, 1], pub, ob.BAD_RWSET, fault="bad_rwset"), tx([0, 1], pub, V)]),
        # rows 2-4
        ("writes_lscc", None, False, [tx([0, 1], pub + [("lscc", 0, 1)], BAD), tx([0, 1], pub + [("lscc", 2, 0)], V)]),
        ("writes_non_invokable", None, False, [tx([0, 1], pub + [("vscc", 0, 1)], BAD), tx([0, 1], pub + [("escc", 0, 1)], BAD),
                                               tx([0, 1], pub + [("cscc", 0, 1)], BAD),
                                               tx([0, 1], [(CC, 1, 1, [("c1", 0, ["m"], 0)]), ("escc", 0, 0, [("x", 0, ["h"], 0)])], BAD)]),
        ("invokes_vscc_or_escc", None, False, [tx([0, 1, 2, 3], [("vscc", 1, 1)], BAD, cc=("vscc", "1.0")),
                                               tx([0, 1, 2, 3], [("escc", 1, 0)], BAD, cc=("escc", "1.0"))]),
        # row 6: only the invoked namespace, no version check
        ("invokes_qscc_or_cscc", None, False, [tx([0], [("qscc", 1, 1), (STRICT, 0, 1)], V, cc=("qscc", "9.9")),
                                               tx([], [("qscc", 1, 0)], F, cc=("qscc", "1.0")),
                                               tx([3], [("cscc", 0, 1), ("lscc", 0, 1)], V, cc=("cscc", "0")),
                                               tx([3], [("cscc", 0, 1)], OTHERR, cc=("cscc", ""))]),
        # row 7: in order, the first failing namespace decides
        ("undefined_then_failing", None, False, [tx([0, 1], pub + [(GHOST, 0, 1), (STRICT, 0, 1)], NV)]),
        ("failing_then_undefined", None, False, [tx([0, 1], pub + [(STRICT, 0, 1), (GHOST, 0, 1)], F)]),
        ("invoked_fails_first", None, False, [tx([0], pub + [(GHOST, 0, 1)], F), tx([0, 1], pub + [(OTHER, 0, 1)], V),
                                              tx([0, 1], pub + [("qscc", 0, 1)], V), tx([], [(OTHER, 0, 1)], F, cc=(OTHER, "2.0"))]),
        # row 8: the invoked chaincode's lscc version, before its policy
        ("version_mismatch", None, False, [tx([0, 1], pub, EXP, cc=(CC, "2.0")), tx([0], pub, EXP, cc=(CC, "0.9")),
                                           tx([0, 1], pub, EXP, cc=(CC, "1.0.0"), fault="unknown_endorser"),
                                           tx([0, 1], pub, NV, fault="unknown_endorser"),
                                           tx([0, 1], [(NOVER, 1, 1)], NV, cc=(NOVER, "1.0")),
                                           tx([0, 1], [(GHOST, 1, 1)], NV, cc=(GHOST, "1.0")),
                                           tx([0, 1], pub + [(OTHER, 0, 1)], V, cc=(CC, "1.0"))]),
        # row 9: a namespace's own writes; a private write checks its key's parameter, else the chaincode policy, never a collection's
        ("private_write_with_and_without_parameter", {(CC, "org2coll", kh("p1")): "vp_org1"}, False,
         [tx([0], [(CC, 0, 0, [("org2coll", ["p1"], 0, 0)])], V), tx([1], [(CC, 0, 0, [("org2coll", ["p1"], 0, 0)])], F),
          tx([0], [(CC, 0, 0, [("org2coll", ["p2"], 0, 0)])], F), tx([1, 2], [(CC, 0, 0, [("org2coll", ["p2"], 0, 0)])], V)]),
        ("collection_table_not_used", None, True, [tx([1], [(CC, 0, 0, [("org2coll", 1, 0, 0)])], F), tx([0, 3], [(CC, 0, 0, [("strictcoll", 1, 0, 0)])], V)]),
        ("undefined_collection_with_key_table", {(CC, "", "k1"): "vp_org1"}, True,
         [tx([0, 1], [(CC, 0, 0, [("ghostcoll", ["g"], 0, 0)])], NV), tx([0], [(CC, 0, ["k1"])], V)]),
        ("own_writes_per_namespace", {(OTHER, "", "o1"): "vp_3of4"}, False,
         [tx([0, 1], [(CC, 0, ["a"]), (OTHER, 0, ["o1"])], F), tx([0, 1, 2], [(CC, 0, ["a"]), (OTHER, 0, ["o1"])], V),
          tx([0, 1], [(CC, 0, ["a"]), (OTHER, 0, ["o2"])], V)]),
        # row 10: an lscc invocation, with dependents on its metadata writes and a duplicate tx id in the block
        ("lscc_in_block", {(OTHER, "", "unused"): "vp_org1"}, False,
         [tx([0, 1], [("lscc", 0, 1), (CC, 0, 0, [], ["d1"])], NV, cc=("lscc", "1.0")), tx([0, 1], [(CC, 0, ["d1"])], NV),
          tx([0, 1], pub, NV), tx([0, 1], pub, ob.DUPLICATE_TXID, fault="dup_txid"), tx([0], pub, F),
          tx([0, 1], pub, ob.BAD_CREATOR_SIGNATURE, fault="bad_creator_sig")]),
        # row 10 for an lscc invocation the device stops at 254 before its lscc check: the block is marked all the same
        ("lscc_with_a_creator_outside_the_table", None, False,
         [tx([0, 1], [("lscc", 0, 1)], NV, cc=("lscc", "1.0"), fault="unknown_creator"), tx([0, 1], pub, NV), tx([0], pub, F)]),
        ("lscc_reading_more_namespaces_than_recorded", None, False,
         [tx([0, 1], [("lscc", 0, 1)] + [("ns%d" % k, 1, 0) for k in range(9)], NV, cc=("lscc", "1.0")), tx([0, 1], pub, NV)]),
        ("more_namespaces_than_recorded", None, False, [tx([0, 1], pub + [("ns%d" % k, 1, 0) for k in range(8)], NV), tx([0, 1], pub, V)]),
        ("lscc_stopped_before_validation", None, False,
         [tx([0, 1], [("lscc", 0, 1)], ob.BAD_CREATOR_SIGNATURE, cc=("lscc", "1.0"), fault="bad_creator_sig"), tx([0, 1], pub, V)]),
    ]


def key_table(case):
    """(vp nodes, {(ns, coll, key bytes): root}) of a case with a key table, or None"""
    if case[1] is None:
        return None
    nodes, r = klcases.vp_forest()
    return nodes, {(ns, coll, key if isinstance(key, bytes) else key.encode()): r[v] for (ns, coll, key), v in case[1].items()}


def materialize(case, seed=131):
    """-> (net, block, info, codes)"""
    import nodeou
    txs = case[3]
    net = nodeou.network(4)
    faults = {t: x[2] for t, x in enumerate(txs) if x[2]}
    blk, info = blockgen.build_block(net, len(txs), 3, faults, seed=seed, endorsers=lambda t: [net.org_peers[o][0] for o in txs[t][0]],
                                     namespaces=lambda t: txs[t][1], chaincode=lambda t: txs[t][4])
    return net, blk, info, [x[3] for x in txs]
