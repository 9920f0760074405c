"""Private-data collection endorsement policies (fabgpu_collection_policies) in the device block logic, run on the host build
(tests/host_sim/blockdev_coll_host.cpp runs blockdev.cuh's walk and decide_tx with a collection table), against the collection oracle
and against codes written out per case."""
import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from tools import fabricpb as pb
import collcases
import collection_oracle
import collutil
import policy_oracle


def _flags(net, info, blk, names, bits, table, ids=None, policies=None, nodes=None):
    ids = ids or net.identities()
    nodes = collcases.forest()[0] if nodes is None else nodes
    policies = collcases.namespace_policies() if policies is None else policies
    host = collutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, names, policies=policies,
                                       principal_bits=bits, collections=table)
    exp = collection_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=policies, collections=table,
                                           known=[i[0] for i in ids])
    return host.tolist(), exp.tolist()


@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
@pytest.mark.parametrize("case", collcases.cases(), ids=lambda c: c[0])
def test_collection_case_host_build(case, use_bits):
    """Every case with the table and without it, with role principals (bits) and with MSP-id matching: the oracle and the host build
    give the codes written out."""
    net, blk, info, with_table, without = collcases.materialize(case)
    names, bits = collcases.principals(use_bits)
    host, exp = _flags(net, info, blk, names, bits, collcases.collection_table())
    assert exp == with_table
    assert host == with_table
    for table in (None, {}):
        host, exp = _flags(net, info, blk, names, bits, table)
        assert exp == without
        assert host == without


def test_without_table_collection_oracle_is_policy_oracle():
    """Without a table the collection oracle is tests/policy_oracle.py's, and every case's codes are the ones the device gave before
    collection policies existed."""
    names, bits = collcases.principals(True)
    nodes = collcases.forest()[0]
    for case in collcases.cases():
        net, blk, info, _, without = collcases.materialize(case)
        ids = net.identities()
        exp = policy_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=collcases.namespace_policies(),
                                           known=[i[0] for i in ids])
        assert exp.tolist() == without, case[0]


def test_case_table_covers_the_issue():
    names = {c[0] for c in collcases.cases()}
    assert {"public_only", "collection_stricter", "collection_looser", "lifecycle_approval", "public_and_collection",
            "two_collections_one_namespace", "same_collection_two_namespaces", "metadata_writes_count", "hashed_reads_do_not_count",
            "collection_in_second_namespace", "collection_without_a_name", "not_in_table", "more_collections_than_the_cap",
            "static_collection_without_policy"} <= names
    assert len(collcases.collection_table()) >= 200
    for _, _, txs in collcases.cases():
        for _, _, a, b in txs:
            assert a in (ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.NOT_VALIDATED) and b in (ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE)
    flips = [(a, b) for _, _, txs in collcases.cases() for _, _, a, b in txs if a != b]
    assert (ob.ENDORSEMENT_POLICY_FAILURE, ob.VALID) in flips and (ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE) in flips


def test_duplicate_pair_refused_by_the_table_builder():
    """coll_table_fill, which the library's fabgpu_collection_policies uses, refuses a (namespace, collection) given twice; the same
    collection name under two namespaces, or two names under one, is no duplicate."""
    net, blk, info, with_table, _ = collcases.materialize(collcases.cases()[0])
    names, bits = collcases.principals(True)
    roots = collcases.forest()[1]

    class Twice(dict):                          # hands the binding-order key list one pair twice
        def __iter__(self):
            return iter([("mycc", "a"), ("mycc", "a")])
    with pytest.raises(ValueError):
        collutil.device_logic_flags(info["env_blob"], info["env_off"], net.identities(), net.channel, collcases.forest()[0], names,
                                    policies=collcases.namespace_policies(), principal_bits=bits,
                                    collections=Twice({("mycc", "a"): roots["cc"]}))
    ok = {("mycc", "a"): roots["cc"], ("othercc", "a"): roots["org1"], ("mycc", "ab"): roots["org2"], ("mycc", "b"): roots["loose"]}
    host, exp = _flags(net, info, blk, names, bits, ok)
    assert host == exp == with_table


def test_tx_rwset_forms():
    """The collection list form of blockgen.tx_rwset: several named collections, each with hashed writes, hashed metadata writes and
    hashed reads, and a collection without the name field; the existing forms are unchanged."""
    rw = blockgen.tx_rwset([("mycc", 1, 1, [("a", 2, 1, 3), (None, 1, 0, 0), ("", 0, 0, 1)])])
    ns = pb.parse(pb.parse(rw, ob.S_TXRWSET)["ns_rwset"][0], ob.S_NSRWSET)
    colls = [pb.parse(c, ob.S_COLLHASHED) for c in ns["collection_hashed_rwset"]]
    assert [c["collection_name"] for c in colls] == [b"a", None, b""]
    h = pb.parse(colls[0]["hashed_rwset"], ob.S_HASHEDRWSET)
    assert (len(h["hashed_writes"]), len(h["metadata_writes"]), len(h["hashed_reads"])) == (2, 1, 3)
    assert [w for _, _, w in collection_oracle.written(rw)] == [["a"]]
    old = blockgen.tx_rwset([("mycc", 2, 2, 1), ("strictcc", 0, 1)])
    ref = (pb.f_bytes(2, pb.f_bytes(1, b"mycc") + pb.f_bytes(2, blockgen.kv_rwset(2, 2, b"mycc")) +
                      pb.f_bytes(3, pb.f_bytes(1, b"collection") + pb.f_bytes(2, blockgen.hashed_rwset(1, b"mycc")))) +
           pb.f_bytes(2, pb.f_bytes(1, b"strictcc") + pb.f_bytes(2, blockgen.kv_rwset(0, 1, b"strictcc"))))
    assert old == ref


def test_wire_mutation_corpus_with_a_stricter_collection_policy():
    """The wire-mutation corpus, whose transactions write public keys and collection 'collection', with a table that gives 'collection'
    the STRICT_NAMESPACE tree (one endorsement more than the chaincode's): the host build's flags equal the collection oracle's for every
    transaction, mutated collection names included."""
    import wiremut
    net, ids, nodes, pol, blocks = wiremut.corpus()
    table = {(blockgen.CHAINCODE, "collection"): pol[blockgen.STRICT_NAMESPACE]}
    counts = {}
    for blk, info, _, before in blocks:
        host = collutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol,
                                           collections=table)
        exp = collection_oracle.validate_block(blk, ids, net.channel, nodes, net.principals, policies=pol, collections=table,
                                               known=[i[0] for i in ids])
        assert host.tolist() == exp.tolist()
        for a, b in zip(before.tolist(), exp.tolist()):
            counts[(a, b)] = counts.get((a, b), 0) + 1
    # the table moves some transactions: VALID under the chaincode policy, failing the collection's, or renamed collections handed back
    assert counts.get((ob.VALID, ob.VALID), 0) >= 1000
    assert counts.get((ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE), 0) >= 10 and counts.get((ob.VALID, ob.NOT_VALIDATED), 0) >= 1
