"""The v1.3 mode (fabgpu_channel_capability(FABGPU_CAP_V1_3): the v1.4 validator with the builtin v13 VSCC) in the device block logic,
run on the host build (tests/host_sim/blockdev_v13_host.cpp), against the v1.3 oracle and against codes written out per case."""
import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
import collcases
import keylevel_oracle
import klcases
import test_key_policies
import v13_oracle
import v13cases
import v13util


def _run(case, use_bits):
    net, blk, info, codes = v13cases.materialize(case)
    names, bits = collcases.principals(use_bits)
    kt = v13cases.key_table(case)
    colls = collcases.collection_table() if case[2] else None
    ids = net.identities()
    host = v13util.device_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names, policies=v13cases.policies(),
                                versions=v13cases.versions(), principal_bits=bits, collections=colls, key_calls=[(True,) + kt] if kt else ())
    nodes, vps = klcases.combined(*kt) if kt else (collcases.forest()[0], None)
    exp = v13_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=v13cases.policies(), versions=v13cases.versions(),
                                    collections=colls, vps=vps, known=[i[0] for i in ids])
    return host.tolist(), exp.tolist(), codes


@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
@pytest.mark.parametrize("case", v13cases.cases(), ids=lambda c: c[0])
def test_v13_case_host_build(case, use_bits):
    """Every case: the oracle and the host build give the codes written out."""
    host, exp, codes = _run(case, use_bits)
    assert exp == codes
    assert host == codes


def test_case_table_covers_every_row():
    names = {c[0] for c in v13cases.cases()}
    assert {"name_and_version_checks", "writes_lscc", "writes_non_invokable", "invokes_vscc_or_escc", "invokes_qscc_or_cscc",
            "undefined_then_failing", "failing_then_undefined", "version_mismatch", "private_write_with_and_without_parameter",
            "lscc_in_block", "collection_table_not_used", "own_writes_per_namespace", "lscc_with_a_creator_outside_the_table",
            "lscc_reading_more_namespaces_than_recorded"} <= names


def test_refusals_of_the_capability_calls():
    """The library's argument checks (capability.hpp, shared with the host build): a capability other than V2_0 / V1_3, a version count
    that is not the table's or decreasing version offsets, and in v1.3 mode a namespace table -- or, without one, node 0 -- reaching an
    ImplicitMeta node.  v2.0 mode takes any table."""
    import ctypes
    from blockutil import _p
    L = v13util.v13_lib()
    for f in (L.cap_check_capability, L.cap_check_namespace_table, L.cap_check_versions):
        f.restype = ctypes.c_char_p
    nodes, r = collcases.forest()
    nd = np.ascontiguousarray(nodes, np.int32)
    sig = np.array([r["cc"], r["loose"]], np.int32)
    meta = np.array([r["cc"], r["lifecycle"]], np.int32)
    none = np.zeros(1, np.int32)
    for cap in (2, -1, 13):
        assert b"FABGPU_CAP_V2_0 or FABGPU_CAP_V1_3" in L.cap_check_capability(cap, _p(nd), nd.shape[0], _p(sig), 2)
    assert L.cap_check_capability(1, _p(nd), nd.shape[0], _p(sig), 2) is None
    assert L.cap_check_capability(0, _p(nd), nd.shape[0], _p(meta), 2) is None
    assert b"ImplicitMeta" in L.cap_check_capability(1, _p(nd), nd.shape[0], _p(meta), 2)
    assert L.cap_check_namespace_table(0, _p(nd), nd.shape[0], _p(meta), 2) is None
    assert b"ImplicitMeta" in L.cap_check_namespace_table(1, _p(nd), nd.shape[0], _p(meta), 2)
    assert L.cap_check_namespace_table(1, _p(nd), nd.shape[0], _p(sig), 2) is None
    # an empty table makes node 0 every namespace's policy: refused in v1.3 mode when node 0 is ImplicitMeta
    implicit_first = np.ascontiguousarray(np.concatenate([[[2, 1, 1, 1]], [[1, 0, 0, 0]]]), np.int32)
    assert b"ImplicitMeta" in L.cap_check_namespace_table(1, _p(implicit_first), 2, _p(none), 0)
    assert b"ImplicitMeta" in L.cap_check_capability(1, _p(implicit_first), 2, _p(none), 0)
    assert L.cap_check_namespace_table(1, _p(nd), nd.shape[0], _p(none), 0) is None
    off = np.array([0, 3, 6], np.uint32)
    assert L.cap_check_versions(_p(off), 2, 2) is None
    assert b"do not match" in L.cap_check_versions(_p(off), 2, 3)
    assert b"decrease" in L.cap_check_versions(_p(np.array([0, 3, 2], np.uint32)), 2, 2)


def test_v20_mode_of_the_same_build_is_unchanged():
    """The same build in v2.0 mode gives the key-level oracle's flags on the v1.3 cases: 25 for a name mismatch, writes to lscc pass."""
    names, bits = collcases.principals(True)
    for case in v13cases.cases():
        if case[2] or "lscc" in case[0] or case[0] in ("invokes_vscc_or_escc", "invokes_qscc_or_cscc", "more_namespaces_than_recorded"):
            continue
        net, blk, info, _ = v13cases.materialize(case)
        ids = net.identities()
        kt = v13cases.key_table(case)
        host = v13util.device_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names, mode=v13util.MODE_V20,
                                    policies=v13cases.policies(), versions=v13cases.versions(), principal_bits=bits, key_calls=[(True,) + kt] if kt else ())
        nodes, vps = klcases.combined(*kt) if kt else (collcases.forest()[0], None)
        exp = keylevel_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=v13cases.policies(), vps=vps,
                                             known=[i[0] for i in ids])
        assert host.tolist() == exp.tolist(), case[0]


def _v13_policies():
    """collcases' namespace table without _lifecycle, whose policy is ImplicitMeta (refused in v1.3 mode)"""
    return {k: v for k, v in collcases.namespace_policies().items() if k != collcases.LIFECYCLE}


def test_collection_and_key_cases_in_v13_mode():
    """collcases and klcases, with their tables, in v1.3 mode: the host build equals the v1.3 oracle on every transaction."""
    names, bits = collcases.principals(True)
    pol, ver = _v13_policies(), {collcases.CC: "1.0", collcases.OTHER: "1.0"}
    moved = 0
    for case in collcases.cases():
        net, blk, info, with_table, _ = collcases.materialize(case)
        ids = net.identities()
        host = v13util.device_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names, policies=pol, versions=ver,
                                    principal_bits=bits, collections=collcases.collection_table())
        exp = v13_oracle.validate_block(blk, ids, net.channel, collcases.forest()[0], names, bits=bits, policies=pol, versions=ver,
                                        collections=collcases.collection_table(), known=[i[0] for i in ids])
        assert host.tolist() == exp.tolist(), case[0]
        moved += sum(a != b for a, b in zip(exp.tolist(), with_table))
    assert moved >= 3
    for case in klcases.cases():
        net, blk, info, codes = klcases.materialize(case)
        ids = net.identities()
        kn, table = klcases.key_table(case)
        colls = collcases.collection_table() if case[1] else None
        host = v13util.device_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names, policies=pol, versions=ver,
                                    principal_bits=bits, collections=colls, key_calls=[(True, kn, table)])
        nodes, vps = klcases.combined(kn, table)
        exp = v13_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=pol, versions=ver, collections=colls, vps=vps,
                                        known=[i[0] for i in ids])
        assert host.tolist() == exp.tolist(), case[0]


def test_wire_mutation_corpus_in_v13_mode():
    """The wire-mutation corpus in v1.3 mode, without and with a key table: host build == v1.3 oracle on every transaction."""
    import wiremut
    net, ids, nodes, pol, blocks = wiremut.corpus()
    ver = {n: "1.0" for n in pol}
    kn, r = klcases.vp_forest()
    table = test_key_policies.corpus_key_table(kn, r)
    kn_nodes = np.array(kn, np.int32).copy()
    kn_nodes[kn_nodes[:, 0] == 0, 2] += nodes.shape[0]
    all_nodes = np.concatenate([np.asarray(nodes, np.int32).reshape(-1, 4), kn_nodes])
    vps = {k: (v + nodes.shape[0] if v >= 0 else v) for k, v in table.items()}
    changed = 0
    for blk, info, _, before in blocks:
        for calls, nd, vp in (((), nodes, None), ([(True, kn, table)], all_nodes, vps)):
            host = v13util.device_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol, versions=ver,
                                        key_calls=calls)
            exp = v13_oracle.validate_block(blk, ids, net.channel, nd, net.principals, policies=pol, versions=ver, vps=vp, known=[i[0] for i in ids])
            assert host.tolist() == exp.tolist()
            changed += sum(a != b for a, b in zip(before.tolist(), exp.tolist()))
    assert changed >= 5


def random_block(seed, n_tx=40):
    """A seeded block of v1.3 traffic: invoked chaincodes and versions, system namespaces written, lscc invocations, faults."""
    import nodeou
    rng = np.random.default_rng(seed)
    net = nodeou.network(4)
    ccs = [(v13cases.CC, "1.0"), (v13cases.CC, "2.0"), (v13cases.OTHER, "2.0"), ("qscc", "1.0"), ("escc", "1.0"), (v13cases.GHOST, "1.0"),
           (v13cases.NOVER, "1.0")] + ([("lscc", "1.0")] if seed % 2 else [])
    extra = [(v13cases.STRICT, 0, 1), (v13cases.OTHER, 0, 1), ("lscc", 0, 1), ("lscc", 1, 0), ("cscc", 0, 1), ("qscc", 0, 1), (v13cases.GHOST, 0, 1)]
    plan = []
    for t in range(n_tx):
        cc = ccs[rng.integers(len(ccs))] if rng.random() < 0.5 else (v13cases.CC, "1.0")
        nss = [(cc[0], 1, ["k%d" % rng.integers(4)], [], ["k%d" % rng.integers(4)] if rng.random() < 0.2 else [])]
        nss += [extra[i] for i in rng.choice(len(extra), rng.integers(0, 3), replace=False)]
        orgs = sorted(rng.choice(4, rng.integers(1, 5), replace=False).tolist())
        plan.append((orgs, nss, cc))
    faults = {t: f for t, f in zip(rng.choice(n_tx, 4, replace=False).tolist(), ["bad_creator_sig", "cc_name_mismatch", "dup_txid", "unknown_endorser"])
              if t > 0}
    blk, info = blockgen.build_block(net, n_tx, 3, faults, seed=seed, endorsers=lambda t: [net.org_peers[o][0] for o in plan[t][0]],
                                     namespaces=lambda t: plan[t][1], chaincode=lambda t: plan[t][2])
    return net, blk, info


@pytest.mark.parametrize("seed", range(6))
def test_seeded_random_blocks(seed):
    names, bits = collcases.principals(seed % 2 == 0)
    net, blk, info = random_block(seed)
    ids = net.identities()
    kn, r = klcases.vp_forest()
    table = {(v13cases.CC, "", b"k1"): r["vp_org1"], (v13cases.CC, "", b"k2"): -2}
    for calls, (nodes, vps) in (((), (collcases.forest()[0], None)), ([(True, kn, table)], klcases.combined(kn, table))):
        host = v13util.device_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names, policies=v13cases.policies(),
                                    versions=v13cases.versions(), principal_bits=bits, key_calls=calls)
        exp = v13_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=v13cases.policies(), versions=v13cases.versions(),
                                        vps=vps, known=[i[0] for i in ids])
        assert host.tolist() == exp.tolist()
        assert len(set(exp.tolist())) >= 4


def test_tx_rwset_and_chaincode_forms():
    """blockgen: the invoked chaincode's name and version reach the header extension and the chaincode action; the default is unchanged."""
    import nodeou
    net = nodeou.network(4)
    a, _ = blockgen.build_block(net, 2, 2, seed=5)
    b, _ = blockgen.build_block(net, 2, 2, seed=5, chaincode=lambda t: (blockgen.CHAINCODE, "1.0"))
    assert a == b
    c, info = blockgen.build_block(net, 1, 2, seed=5, chaincode=lambda t: ("lscc", "7"), namespaces=lambda t: [("lscc", 0, 1)])
    env = info["env_blob"]
    assert bytes(v13_oracle._action_version(env)) == b"7"
    import collection_oracle
    assert collection_oracle._results(env)[0] == "lscc"
