"""Test infrastructure (not product code): the key-level endorsement policy cases (fabgpu_key_policies) that the oracle, the host build
and the device are all held to, with every expected code written out.

The channel, the configured node array, the namespace table and the collection table are collcases'.  The validation parameters are
trees of a node array of their own (the one fabgpu_key_policies takes); the key table holds each case's keys plus 10^4 filler keys of
other chaincodes.  Each endorsing org signs with its first peer.
"""
import functools

from oracle import blockval as ob
from tools import blockgen
import collcases
import nodeou

V, F, NV = ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.NOT_VALIDATED
CC, OTHER = collcases.CC, collcases.OTHER
kh = blockgen.key_hash

_VP_TREES = [("vp_org1", nodeou.n_of(1, [nodeou.signed_by(0)])), ("vp_org2", nodeou.n_of(1, [nodeou.signed_by(1)])),
             ("vp_3of4", nodeou.n_of(3, [nodeou.signed_by(o) for o in range(4)]))] + \
            [("many%d" % k, nodeou.n_of(1, [nodeou.signed_by(k % 4)])) for k in range(17)]


@functools.lru_cache(maxsize=None)
def vp_forest():
    """-> (nodes of the validation parameters, {tree name: root within them})"""
    nodes, roots = nodeou.forest([t for _, t in _VP_TREES])
    return nodes, {name: r for (name, _), r in zip(_VP_TREES, roots)}


def filler(n=10000):
    """{(ns, coll, key): tree name}: keys of other chaincodes, as a peer's table holds them"""
    return {("cc%02d" % (k % 20), "" if k % 3 else "coll", ("asset%d" % k) if k % 3 else kh("asset%d" % k)): ["vp_org1", "vp_org2", "vp_3of4"][k % 3]
            for k in range(n)}


def pub(*keys, md=()):
    """the invoked chaincode writing public keys `keys` and metadata-writing `md`"""
    return (CC, 0, list(keys), [], list(md))


def cases():
    """[(name, with a collection table, {(ns, coll, key): tree name or -2}, [(endorsing orgs, namespaces, fault, code)])]; namespaces as
    blockgen.tx_rwset takes them."""
    many = {(CC, "", "m%d" % k): "many%d" % k for k in range(17)}
    return [
        ("vp_stricter", False, {(CC, "", "a"): "vp_3of4"}, [([0, 1], [pub("a")], None, F), ([0, 1, 2], [pub("a")], None, V)]),
        ("vp_looser", False, {(CC, "", "b"): "vp_org1"}, [([0], [pub("b")], None, V), ([1], [pub("b")], None, F), ([], [pub("b")], None, F)]),
        ("vp_and_plain_key", False, {(CC, "", "b"): "vp_org1"},
         [([0], [pub("b", "x")], None, F), ([0, 1], [pub("b", "x")], None, V), ([1, 2], [pub("b", "x")], None, F)]),
        ("metadata_write_checks_the_old_vp", False, {(CC, "", "b1"): "vp_org1", (CC, "", "b2"): "vp_org1"},
         [([0], [pub(md=["b1"])], None, V), ([1, 2], [pub(md=["b2"])], None, F)]),
        ("hashed_write_with_vp", False, {(CC, "org2coll", kh("h1")): "vp_org1"},
         [([0], [(CC, 0, 0, [("org2coll", ["h1"], 0, 0)])], None, V), ([1], [(CC, 0, 0, [("org2coll", ["h1"], 0, 0)])], None, F),
          ([1], [(CC, 0, 0, [("org2coll", ["h2"], 0, 0)])], None, F), ([0, 1], [(CC, 0, 0, [("org2coll", ["h2"], 0, 0)])], None, V)]),
        ("hashed_write_with_vp_and_collection_table", True, {(CC, "org2coll", kh("h1")): "vp_org1", (CC, "ghostcoll", kh("g1")): "vp_org1"},
         [([0], [(CC, 0, 0, [("org2coll", ["h1"], 0, 0)])], None, V), ([1], [(CC, 0, 0, [("org2coll", ["h1"], 0, 0)])], None, F),
          ([1], [(CC, 0, 0, [("org2coll", ["h2"], 0, 0)])], None, V), ([0], [(CC, 0, 0, [("org2coll", ["h2"], 0, 0)])], None, F),
          ([0], [(CC, 0, 0, [("ghostcoll", ["h1"], 0, 0)])], None, NV), ([0], [(CC, 0, 0, [("ghostcoll", ["g1"], 0, 0)])], None, NV)]),
        ("read_only_invoked_namespace", False, {(OTHER, "", "o1"): "vp_org1"},
         [([0], [(CC, 1, 0), (OTHER, 0, ["o1"])], None, F), ([0, 1], [(CC, 1, 0), (OTHER, 0, ["o1"])], None, V),
          ([1, 2], [(CC, 1, 0), (OTHER, 0, ["o1"])], None, F)]),
        ("undecidable_key", False, {(CC, "", "u"): -2}, [([0, 1], [pub("u")], None, NV), ([0, 1], [pub("x")], None, V),
                                                         ([0, 1], [pub(md=["u"])], None, NV)]),
        ("more_than_16_roots", False, many, [([0, 1, 2, 3], [pub(*["m%d" % k for k in range(16)])], None, V),
                                             ([0, 1, 2], [pub(*["m%d" % k for k in range(16)])], None, F),
                                             ([0, 1, 2, 3], [pub(*["m%d" % k for k in range(17)])], None, NV)]),
        ("dependency_on_a_valid_writer", False, {}, [([0, 1], [pub(md=["d1"])], None, V), ([0, 1], [pub("d1")], None, F),
                                                    ([0, 1], [pub("other")], None, V)]),
        ("dependency_on_a_failing_writer", False, {}, [([0], [pub(md=["d2"])], None, F), ([0, 1], [pub("d2")], None, V),
                                                      ([1], [pub("d2")], None, F)]),
        ("dependency_on_a_bad_creator_signature", False, {}, [([0, 1], [pub(md=["d3"])], "bad_creator_sig", ob.BAD_CREATOR_SIGNATURE),
                                                             ([0, 1], [pub("d3")], None, NV), ([0], [pub("d3")], None, NV)]),
        ("dependency_on_a_failing_two_namespace_writer", False, {},
         [([0], [pub(md=["d4"]), (OTHER, 0, ["o2"])], None, F), ([0, 1], [pub("d4")], None, NV)]),
        ("writer_abandoned_before_dispatch", False, {},
         [([0, 1], [pub(md=["d5"])], "nonzero_epoch", ob.BAD_COMMON_HEADER), ([0, 1], [pub("d5")], None, NV),
          ([0, 1], [pub(md=["d6"])], "cc_name_mismatch", ob.INVALID_CHAINCODE), ([0, 1], [pub("d6")], None, NV)]),
        ("three_transaction_chain", False, {}, [([0], [pub(md=["c1"])], None, F), ([0, 1], [pub(md=["c1"])], None, V),
                                               ([0, 1], [pub("c1")], None, F)]),
        ("hot_key", False, {(CC, "", "hot"): "vp_org1"},
         [([0], [pub("hot", md=["hot"])], None, V), ([0, 1], [pub("hot", md=["hot"])], None, F), ([1], [pub("hot", md=["hot"])], None, F),
          ([0], [pub("hot", md=["hot"])], None, F), ([0], [pub("cold", md=["cold"])], None, F), ([0, 1], [pub("cold")], None, V)]),
        ("same_key_elsewhere_is_no_dependency", False, {},
         [([0, 1], [pub(md=["s1"])], None, V), ([0, 1], [(CC, 1, 0), (OTHER, 0, ["s1"])], None, V),
          ([0, 1], [(CC, 0, 0, [("org1coll", ["s1"], 0, 0)])], None, V), ([0, 1], [pub("s1")], None, F)]),
    ]


def key_table(case):
    """(vp nodes, {(ns, coll, key bytes): root within them or -2}) for a case: its keys plus the filler"""
    nodes, r = vp_forest()
    t = {k: v for k, v in filler().items()}
    t.update(case[2])
    return nodes, {(ns, coll, key if isinstance(key, bytes) else key.encode()): (v if v == -2 else r[v]) for (ns, coll, key), v in t.items()}


def combined(key_nodes, table):
    """the configured nodes with the validation parameters' appended, and the table's roots in that array (what the library evaluates)"""
    import numpy as np
    cfg = collcases.forest()[0]
    kn = np.array(key_nodes, np.int32).copy()
    kn[kn[:, 0] == 0, 2] += cfg.shape[0]
    return np.concatenate([cfg, kn]), {k: (v + cfg.shape[0] if v >= 0 else v) for k, v in table.items()}


def materialize(case, seed=89):
    """-> (net, block, info, codes)"""
    _, _, _, txs = case
    net = nodeou.network(4)
    faults = {t: x[2] for t, x in enumerate(txs) if x[2]}
    blk, info = blockgen.build_block(net, len(txs), 3, faults, seed=seed, endorsers=lambda t: [net.org_peers[o][0] for o in txs[t][0]],
                                     namespaces=lambda t: txs[t][1])
    return net, blk, info, [x[3] for x in txs]
