"""Role and identity principals (fabgpu_msp_principal_bits) and ImplicitMeta policy nodes in the device block logic, run on the host
build (tests/host_sim/blockdev_policy_host.cpp runs blockdev.cuh's decide_tx with the bits), against the policy oracle and against codes written out per
case."""
import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from util import pkg
import blockutil
import nodeou
import policy_oracle
import policyutil

CASES = nodeou.policy_cases()


def _both(net, info, blk, nodes, names, bits, pol, ids=None):
    ids = ids or net.identities()
    host = policyutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, names, policies=pol, principal_bits=bits)
    exp = policy_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=pol, known=[i[0] for i in ids])
    return host.tolist(), exp.tolist()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_policy_case_host_build(case):
    net, blk, info, nodes, names, bits, pol, expected = nodeou.materialize(case)
    host, exp = _both(net, info, blk, nodes, names, bits, pol)
    assert exp == expected
    assert host == expected


def test_case_table_covers_the_issue():
    names = {c[0] for c in CASES}
    assert {"stock_majority_2_orgs", "stock_majority_3_orgs", "stock_majority_4_orgs", "role_peer_vs_client", "admin", "orderer", "identity",
            "principal_in_second_word", "implicit_any", "implicit_all", "implicit_no_sub_policies", "implicit_org_without_sub_policy",
            "implicit_nested_any_of_majority", "same_role_twice_implicit_all", "same_role_twice_n_of_2",
            "namespaces_implicit_and_signature_roots"} <= names
    wide = [c for c in CASES if c[0] == "principal_in_second_word"][0]
    assert len(wide[3]) > 32 and wide[2][0][2][0] == ("signed_by", 37)


def test_principal_bits_follow_the_msp_rules():
    """The bits the test MSP hands the device: NodeOU roles, admin by OU or by list (the listed one without Validate()), IDENTITY across
    both serializations of one certificate."""
    net = nodeou.network(4)
    pr = [nodeou.role("Org1MSP", r) for r in nodeou.ROLES] + [nodeou.identity_principal(net.peers[0])]
    b = dict(zip([i.serialized for i in net.msp_table], nodeou.principal_bits(net, pr).tolist()))
    row = lambda i: [k for k, x in zip(["member", "peer", "client", "admin", "orderer", "identity"], b[i.serialized]) if x]
    assert row(net.peers[0]) == row(net.peers_alt[0]) == ["member", "peer", "identity"]
    assert row(net.org_peers[0][1]) == ["member", "peer"]
    assert row(net.clients[0]) == ["member", "client"]
    assert row(net.admins[0]) == ["member", "admin"]
    assert row(net.admins_listed[0]) == ["admin"]
    assert row(net.orderers[0]) == ["member", "orderer"]
    assert row(net.peers[1]) == row(net.invalid_cert) == []


def test_pack_principal_bits_layout():
    b = pkg().binding
    bits = np.zeros((3, 70), bool)
    bits[0, 0] = bits[0, 31] = bits[1, 32] = bits[2, 69] = True
    w = b.pack_principal_bits(bits)
    assert w.dtype == np.uint32 and w.shape == (3, 3)
    assert w.tolist() == [[1 | (1 << 31), 0, 0], [0, 1, 0], [0, 0, 1 << 5]]
    assert b.pack_principal_bits(np.zeros((4, 0), bool)).shape == (4, 0)


def test_without_bits_policy_oracle_equals_oracle():
    """No bits and only NOutOf / SignedBy nodes: the extended oracle is oracle/blockval's, fault for fault."""
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    n = 3 * len(blockgen.FAULTS) + 4
    blk, info = blockgen.build_block(net, n, 3, blockutil.fault_map(n), seed=11)
    nodes, pol = net.policies_for(3)
    known = [i[0] for i in ids]
    exp = ob.validate_block(blk, ids, net.channel, nodes, net.principals, policies=pol, known=known)
    assert policy_oracle.validate_block(blk, ids, net.channel, nodes, net.principals, policies=pol, known=known).tolist() == exp.tolist()
    assert blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol).tolist() == exp.tolist()
    assert len(set(exp.tolist())) >= 10


def test_fault_classes_under_stock_policy_with_bits():
    """Every fault class of blockgen under the stock MAJORITY-of-peer policy with bits: the host build equals the policy oracle; two
    encodings of one peer count once, 21 endorsements from all four orgs satisfy it."""
    net = blockgen.Network()
    n = 3 * len(blockgen.FAULTS) + 4
    faults = blockutil.fault_map(n)
    blk, info = blockgen.build_block(net, n, 3, faults, seed=11)
    pr, tree = nodeou.stock_endorsement(4)
    nodes, _ = nodeou.forest([tree])
    bits = nodeou.member_roles_for(net, pr)
    names = [nodeou.principal_name(p) for p in pr]
    host, exp = _both(net, info, blk, nodes, names, bits, {blockgen.CHAINCODE: 0, blockgen.STRICT_NAMESPACE: 0}, blockutil.identities_of(net))
    assert host == exp
    byf = {f: exp[t] for t, f in faults.items()}
    assert byf["same_cert_two_encodings"] == ob.ENDORSEMENT_POLICY_FAILURE and byf["many_endorsements"] == ob.VALID
    assert byf["writes_unknown_namespace"] == ob.NOT_VALIDATED and exp.count(ob.VALID) >= n // 2


def test_wire_mutation_corpus_under_stock_policy_with_bits():
    """The wire-mutation corpus under the stock policy with bits: the host build's flags equal the policy oracle's for every
    transaction."""
    import wiremut
    net, ids, _, pol, blocks = wiremut.corpus()
    pr, tree = nodeou.stock_endorsement(4)
    nodes, _ = nodeou.forest([tree])
    bits = nodeou.member_roles_for(net, pr)
    names = [nodeou.principal_name(p) for p in pr]
    roots = {ns: 0 for ns in pol}
    n_valid = 0
    for blk, info, _, _ in blocks:
        host, exp = _both(net, info, blk, nodes, names, bits, roots, ids)
        assert host == exp
        n_valid += exp.count(ob.VALID)
    assert n_valid >= 400


def test_clearing_bits_restores_member_matching():
    """A client endorsing under principal 'Org1MSP' passes by MSP id; with bits naming it a non-peer it fails; with the bits removed
    (n_ids = 0) it passes again."""
    net = nodeou.network(4)
    blk, info = blockgen.build_block(net, 2, 3, {}, seed=5, endorsers=lambda t: [net.clients[0]])
    ids = net.identities()
    nodes, _ = nodeou.forest([nodeou.n_of(1, [nodeou.signed_by(0)])])
    bits = nodeou.principal_bits(net, [nodeou.role("Org1MSP", "peer")])
    flags = lambda b: policyutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, ["Org1MSP"], principal_bits=b).tolist()
    assert flags(None) == [0, 0] and flags(bits) == [10, 10]
    assert flags(np.zeros((0, 1), bool)) == [0, 0]
