"""Test infrastructure (not product code): the private-data collection policy cases (fabgpu_collection_policies) that the host build
and the device are both held to, with every expected code written out.

One channel (nodeou.network(4)), one node array holding every tree below, one namespace table and one collection table of 200+
entries: the pairs the cases use plus the implicit collections of 20 more chaincodes x 10 orgs, as a peer with that many chaincodes
would install.
"""
import functools

from oracle import blockval as ob
from tools import blockgen
from tools import fabricpb as pb
import nodeou

V, F, NV = ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.NOT_VALIDATED
CC, OTHER, LIFECYCLE = blockgen.CHAINCODE, "othercc", "_lifecycle"

# trees of the node array, by name: the chaincode's 2 of 4 peers, a stricter and a looser n-of, each org's OR('OrgN.peer'), and the
# stock MAJORITY LifecycleEndorsement (ImplicitMeta over the orgs' Endorsement policies)
_TREES = [("cc", nodeou.n_of(2, [nodeou.signed_by(o) for o in range(4)])), ("strict", nodeou.n_of(3, [nodeou.signed_by(o) for o in range(4)])),
          ("loose", nodeou.n_of(1, [nodeou.signed_by(o) for o in range(4)]))] + \
         [("org%d" % (o + 1), nodeou.n_of(1, [nodeou.signed_by(o)])) for o in range(4)] + [("lifecycle", nodeou.stock_endorsement(4)[1])]


@functools.lru_cache(maxsize=None)
def forest():
    """-> (nodes, {tree name: root})"""
    nodes, roots = nodeou.forest([t for _, t in _TREES])
    return nodes, {name: r for (name, _), r in zip(_TREES, roots)}


def principals(use_bits):
    """(principal names, bits or None): role principals 'OrgN.peer' with bits, or the MSP ids matched as ROLE MEMBER without"""
    net = nodeou.network(4)
    pr = [nodeou.role("Org%dMSP" % (o + 1), "peer") for o in range(4)]
    if use_bits:
        return [nodeou.principal_name(p) for p in pr], nodeou.principal_bits(net, pr)
    return ["Org%dMSP" % (o + 1) for o in range(4)], None


def namespace_policies():
    _, r = forest()
    return {CC: r["cc"], OTHER: r["loose"], LIFECYCLE: r["lifecycle"]}


def collection_table():
    """{(namespace, collection): root}: 220+ entries"""
    _, r = forest()
    t = {(CC, "strictcoll"): r["strict"], (CC, "loosecoll"): r["loose"], (CC, "org1coll"): r["org1"], (CC, "org2coll"): r["org2"],
         (CC, "shared"): r["org1"], (OTHER, "shared"): r["org2"], (OTHER, "org2coll"): r["org2"],
         (CC, "staticcoll"): r["cc"]}                                        # a static collection without a policy: its chaincode's root
    for o in range(4):
        t[(LIFECYCLE, "_implicit_org_Org%dMSP" % (o + 1))] = r["org%d" % (o + 1)]
    for k in range(9):
        t[(CC, "c%d" % k)] = r["loose"]
    for k in range(20):
        for o in range(10):
            t[("cc%02d" % k, "_implicit_org_Org%dMSP" % (o + 1))] = r["org%d" % (1 + o % 4)]
    return t


def _coll(name, writes=1, md=0, reads=0):
    return (name, writes, md, reads)


def cases():
    """[(name, invoked chaincode, [(endorsing orgs, namespaces, code with the table, code without)])]; namespaces as blockgen.tx_rwset
    takes them.  Each endorsing org signs with its first peer."""
    pub = [(CC, 1, 1)]
    only = lambda *colls: [(CC, 1, 0, list(colls))]
    return [
        ("public_only", CC, [([0, 1], pub, V, V), ([0], pub, F, F), ([2, 3], pub, V, V)]),
        ("collection_stricter", CC, [([0, 1], only(_coll("strictcoll")), F, V), ([0, 1, 2], only(_coll("strictcoll")), V, V)]),
        ("collection_looser", CC, [([0], only(_coll("loosecoll")), V, F), ([], only(_coll("loosecoll")), F, F)]),
        ("lifecycle_approval", LIFECYCLE, [([0], [(LIFECYCLE, 0, 0, [_coll("_implicit_org_Org1MSP")])], V, F),
                                           ([1], [(LIFECYCLE, 0, 0, [_coll("_implicit_org_Org1MSP")])], F, F),
                                           ([0, 1, 2], [(LIFECYCLE, 0, 0, [_coll("_implicit_org_Org1MSP")])], V, V)]),
        ("public_and_collection", CC, [([0, 1], [(CC, 1, 1, [_coll("org1coll")])], V, V), ([1, 2], [(CC, 1, 1, [_coll("org1coll")])], F, V),
                                       ([0], [(CC, 1, 1, [_coll("org1coll")])], F, F)]),
        ("two_collections_one_namespace", CC, [([0], only(_coll("org1coll"), _coll("org2coll")), F, F),
                                               ([0, 1], only(_coll("org1coll"), _coll("org2coll")), V, V),
                                               ([1, 2], only(_coll("org1coll"), _coll("org2coll")), F, V)]),
        ("same_collection_two_namespaces", CC, [([0], only(_coll("shared")), V, F), ([1], only(_coll("shared")), F, F),
                                                ([0, 1], [(CC, 1, 1), (OTHER, 0, 0, [_coll("shared")])], V, V),
                                                ([0, 2], [(CC, 1, 1), (OTHER, 0, 0, [_coll("shared")])], F, V),
                                                ([1], [(CC, 1, 0, [_coll("shared")]), (OTHER, 0, 0, [_coll("shared")])], F, F),
                                                ([0, 1], [(CC, 1, 0, [_coll("shared")]), (OTHER, 0, 0, [_coll("shared")])], V, V)]),
        ("metadata_writes_count", CC, [([0, 1], only(_coll("strictcoll", 0, 1)), F, V), ([0, 1, 2], only(_coll("strictcoll", 0, 1)), V, V)]),
        ("hashed_reads_do_not_count", CC, [([0, 1], only(_coll("strictcoll", 0, 0, 2)), V, V), ([0], only(_coll("loosecoll", 0, 0, 2)), F, F),
                                           ([0], [(CC, 1, 0), (OTHER, 0, 0, [_coll("shared", 0, 0, 1)])], F, F)]),
        ("collection_in_second_namespace", CC, [([1], [(CC, 1, 0), (OTHER, 0, 0, [_coll("org2coll")])], F, F),
                                                ([0, 1], [(CC, 1, 0), (OTHER, 0, 0, [_coll("org2coll")])], V, V),
                                                ([0, 2], [(CC, 1, 0), (OTHER, 0, 0, [_coll("org2coll")])], F, V)]),
        ("collection_without_a_name", CC, [([0, 1], only(_coll(None)), V, V), ([0], only(_coll(None)), F, F), ([0, 1], only(_coll("")), V, V),
                                           ([0], only(_coll("")), F, F), ([0], only(_coll(None), _coll("loosecoll")), F, F),
                                           ([0, 1], only(_coll(""), _coll("org1coll")), V, V)]),
        ("not_in_table", CC, [([0, 1], only(_coll("ghostcoll")), NV, V), ([0, 1], [(CC, 1, 1), (OTHER, 0, 0, [_coll("strictcoll")])], NV, V),
                              ([0], only(_coll("ghostcoll", 0, 0, 1)), F, F)]),
        ("more_collections_than_the_cap", CC, [([0], only(*[_coll("c%d" % k) for k in range(8)]), V, F),
                                               ([0], only(*[_coll("c%d" % k) for k in range(9)]), NV, F),
                                               ([0, 1], only(*[_coll("c%d" % k) for k in range(9)]), NV, V)]),
        ("static_collection_without_policy", CC, [([0, 1], [(CC, 1, 1, [_coll("staticcoll")])], V, V), ([0], [(CC, 1, 1, [_coll("staticcoll")])], F, F),
                                                  ([2, 3], only(_coll("staticcoll")), V, V), ([3], only(_coll("staticcoll")), F, F)]),
    ]


def _invoke(name):
    """build_block's mutate hook: the transactions invoke chaincode `name` (header extension and chaincode action) instead of mycc."""
    def mut(t, part, data):
        if part == "ChaincodeID" and name != CC:
            return data.replace(pb.f_bytes(2, CC.encode()), pb.f_bytes(2, name.encode()), 1)
        return data
    return mut


def materialize(case, seed=83):
    """-> (net, block, info, codes with the table, codes without)"""
    name, invoked, txs = case
    net = nodeou.network(4)
    blk, info = blockgen.build_block(net, len(txs), 3, {}, seed=seed, endorsers=lambda t: [net.org_peers[o][0] for o in txs[t][0]],
                                     namespaces=lambda t: txs[t][1], mutate=_invoke(invoked))
    return net, blk, info, [x[2] for x in txs], [x[3] for x in txs]
