"""Key-level endorsement policies (fabgpu_key_policies) in the device block logic, run on the host build
(tests/host_sim/blockdev_keylevel_host.cpp runs blockdev.cuh's walk, decide_tx and kl_resolve_tx with the library's KeyPolicyTable),
against the key-level oracle and against codes written out per case."""
import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from tools import fabricpb as pb
import collcases
import keylevel_oracle
import klcases
import klutil

HINT = 32          # write records per transaction: every case fits (more_than_16_roots writes 17 keys in one transaction)


def _flags(case, use_bits, calls=None, hint=HINT, out=None):
    net, blk, info, codes = klcases.materialize(case)
    names, bits = collcases.principals(use_bits)
    kn, table = klcases.key_table(case)
    calls = [(True, kn, table)] if calls is None else calls
    colls = collcases.collection_table() if case[1] else None
    ids = net.identities()
    host = klutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names,
                                     policies=collcases.namespace_policies(), principal_bits=bits, collections=colls, key_calls=calls,
                                     writes_hint=hint, out=out)
    return net, blk, ids, names, bits, colls, host.tolist(), codes


def _oracle(blk, ids, net, names, bits, colls, kn, table):
    nodes, vps = klcases.combined(kn, table)
    return keylevel_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=collcases.namespace_policies(),
                                          collections=colls, vps=vps, known=[i[0] for i in ids]).tolist()


@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
@pytest.mark.parametrize("case", klcases.cases(), ids=lambda c: c[0])
def test_key_policy_case_host_build(case, use_bits):
    """Every case with its key table (and 10^4 filler keys): the oracle and the host build give the codes written out."""
    net, blk, ids, names, bits, colls, host, codes = _flags(case, use_bits)
    kn, table = klcases.key_table(case)
    assert _oracle(blk, ids, net, names, bits, colls, kn, table) == codes
    assert host == codes


def test_case_table_covers_the_issue():
    names = {c[0] for c in klcases.cases()}
    assert {"vp_stricter", "vp_looser", "vp_and_plain_key", "metadata_write_checks_the_old_vp", "hashed_write_with_vp",
            "hashed_write_with_vp_and_collection_table", "read_only_invoked_namespace", "undecidable_key", "more_than_16_roots",
            "dependency_on_a_valid_writer", "dependency_on_a_failing_writer", "dependency_on_a_bad_creator_signature",
            "dependency_on_a_failing_two_namespace_writer", "writer_abandoned_before_dispatch", "three_transaction_chain",
            "same_key_elsewhere_is_no_dependency", "hot_key"} <= names


def test_write_record_overflow_at_a_small_hint():
    """More write records than T x hint: every transaction that reaches the policy stage is 254, the others keep their codes; a hint
    that fits gives the written codes."""
    case = [c for c in klcases.cases() if c[0] == "dependency_on_a_bad_creator_signature"][0]
    out = {}
    *_, host, codes = _flags(case, True, hint=0, out=out)
    assert out["records"] > 0
    assert host == [ob.BAD_CREATOR_SIGNATURE, ob.NOT_VALIDATED, ob.NOT_VALIDATED]
    case = [c for c in klcases.cases() if c[0] == "more_than_16_roots"][0]
    *_, host, codes = _flags(case, True, hint=8)                  # 49 writes, 24 records
    assert host == [ob.NOT_VALIDATED] * 3
    *_, host, codes = _flags(case, True, hint=17)
    assert host == codes


def test_update_remove_and_undecidable_change_flags():
    """The table's lifecycle on the host mirror: install, update a key's parameter, remove it (the chaincode policy applies again), mark
    it -2; removing an absent key does nothing; each state gives the oracle's codes."""
    case = ("lifecycle", False, {}, [([0], [klcases.pub("b")], None, None), ([1], [klcases.pub("b")], None, None),
                                      ([0, 1], [klcases.pub("b")], None, None)])
    kn, r = klcases.vp_forest()
    b = (klcases.CC, "", b"b")
    steps = [([(True, kn, {b: r["vp_org1"]})], [ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.VALID]),
             ([(True, kn, {b: r["vp_org1"]}), (False, kn, {b: r["vp_org2"]})], [ob.ENDORSEMENT_POLICY_FAILURE, ob.VALID, ob.VALID]),
             ([(True, kn, {b: r["vp_org1"]}), (False, [], {b: -1, (klcases.CC, "", b"absent"): -1})],
              [ob.ENDORSEMENT_POLICY_FAILURE, ob.ENDORSEMENT_POLICY_FAILURE, ob.VALID]),
             ([(True, kn, {b: r["vp_org1"]}), (False, [], {b: -2})], [ob.NOT_VALIDATED] * 3),
             ([(True, kn, {b: -2}), (False, [], {b: -1}), (False, kn, {b: r["vp_3of4"]})], [ob.ENDORSEMENT_POLICY_FAILURE] * 3)]
    for calls, want in steps:
        net, blk, ids, names, bits, colls, host, _ = _flags(case, True, calls=calls)
        assert host == want, calls
    # the oracle agrees on the final state of each step (the update's nodes land after the earlier calls' nodes)
    net, blk, ids, names, bits, colls, host, _ = _flags(case, True, calls=steps[1][0])
    assert _oracle(blk, ids, net, names, bits, colls, kn, {b: r["vp_org2"]}) == host


def test_update_keeps_the_table_at_most_half_full_and_changes_only_what_it_names():
    kn, r = klcases.vp_forest()
    kt = klutil.KeyTable(collcases.forest()[0].shape[0], 4)
    kt.apply(True, kn, {("cc", "", b"k%d" % i): r["vp_org1"] for i in range(1000)})
    s = kt.stats()
    assert s["live"] == 1000 and 2 * 1000 <= s["size"] and s["dirty"] == -1
    kt.apply(False, kn, {("cc", "", b"k%d" % i): r["vp_org2"] for i in range(10)})
    assert kt.stats()["dirty"] == 10 and kt.stats()["size"] == s["size"]
    kt.apply(False, kn, {("cc", "", b"n%d" % i): r["vp_org2"] for i in range(5000)})          # past half full: rebuilt
    s2 = kt.stats()
    assert s2["live"] == 6000 and s2["size"] >= 12000 and s2["dirty"] == -1
    kt.apply(False, [], {("cc", "", b"n%d" % i): -1 for i in range(5000)})
    assert kt.stats()["live"] == 1000


REFUSALS = [
    ("decreasing offsets", "offsets decrease"),
    ("node type", "node type"),
    ("child out of range", "children out of range"),
    ("root out of range", "root out of range"),
    ("cycle", "deeper than the device evaluates, or cyclic"),
    ("too deep", "deeper than the device evaluates, or cyclic"),
    ("principal out of range", "principal index out of range"),
    ("duplicate", "given twice"),
    ("removal in a replace", r"removal \(-1\) in a replacing call"),
]


def refusal_args(what):
    """(replace, nodes, table or raw arrays) for one refusal; raw arrays are (nodes, ns, coll, key offsets tweak)"""
    ok = [(1, 0, 0, 0)]
    deep = [(0, 1, i + 1, 1) for i in range(13)] + [(1, 0, 0, 0)]
    return {
        "node type": (True, [(2, 1, 0, 0)], {("cc", "", b"k"): 0}),
        "child out of range": (True, [(0, 1, 1, 1)], {("cc", "", b"k"): 0}),
        "root out of range": (True, ok, {("cc", "", b"k"): 1}),
        "cycle": (True, [(0, 1, 0, 1)], {("cc", "", b"k"): 0}),
        "too deep": (True, deep, {("cc", "", b"k"): 0}),
        "principal out of range": (True, [(1, 4, 0, 0)], {("cc", "", b"k"): 0}),
        "removal in a replace": (True, ok, {("cc", "", b"k"): -1}),
        "below -2": (True, ok, {("cc", "", b"k"): -3}),
    }[what]


@pytest.mark.parametrize("what,text", [x for x in REFUSALS if x[0] not in ("decreasing offsets", "duplicate")])
def test_refusals_keep_the_table(what, text):
    kn, r = klcases.vp_forest()
    kt = klutil.KeyTable(collcases.forest()[0].shape[0], 4)
    kt.apply(True, kn, {("cc", "", b"a"): r["vp_org1"]})
    before = kt.stats()
    replace, nodes, table = refusal_args(what)
    with pytest.raises(ValueError, match=text):
        kt.apply(replace, nodes, table)
    assert kt.stats() == before


def test_refusals_with_raw_arrays():
    """decreasing offsets, a duplicate triple, an update without a table, NULL arrays"""
    import ctypes
    from blockutil import _p
    L = klutil.kl_lib()
    kt = klutil.KeyTable(10, 4)
    nd, n_nodes, nb, no, cb, co, kb, ko, roots, n = klutil.key_table_args([(1, 0, 0, 0)], {("cc", "", b"a"): 0, ("cc", "", b"b"): 0})
    assert L.kl_apply(kt.h, 0, 10, 4, _p(nd), n_nodes, _p(nb), _p(no), _p(cb), _p(co), _p(kb), _p(ko), _p(roots), n) == b"no key policy table installed"
    bad = ko.copy(); bad[1] = 5; bad[2] = 2
    assert b"offsets decrease" in L.kl_apply(kt.h, 1, 10, 4, _p(nd), n_nodes, _p(nb), _p(no), _p(cb), _p(co), _p(kb), _p(bad), _p(roots), n)
    dup = kb.copy(); dup[1] = dup[0]
    assert b"given twice" in L.kl_apply(kt.h, 1, 10, 4, _p(nd), n_nodes, _p(nb), _p(no), _p(cb), _p(co), _p(dup), _p(ko), _p(roots), n)
    assert b"arrays missing" in L.kl_apply(kt.h, 1, 10, 4, _p(nd), n_nodes, None, _p(no), _p(cb), _p(co), _p(kb), _p(ko), _p(roots), n)
    assert not kt.stats()["installed"]
    assert L.kl_apply(kt.h, 1, 10, 4, _p(nd), n_nodes, _p(nb), _p(no), _p(cb), _p(co), _p(kb), _p(ko), _p(roots), n) is None
    assert kt.stats()["live"] == 2
    assert L.kl_apply(kt.h, 1, 10, 4, _p(nd), 0, _p(nb), _p(no), _p(cb), _p(co), _p(kb), _p(ko), _p(roots), 0) is None
    assert not kt.stats()["installed"]


def test_tx_rwset_named_forms():
    """Named public write keys, public metadata writes and hashed metadata writes; the existing forms are unchanged."""
    rw = blockgen.tx_rwset([("mycc", 1, ["a", "b"], [("c1", ["h"], ["m"], 1)], ["md"])])
    ws = keylevel_oracle.writes(rw)
    assert ws == [(b"mycc", b"", b"a", False), (b"mycc", b"", b"b", False), (b"mycc", b"", b"md", True),
                  (b"mycc", b"c1", blockgen.key_hash("h"), False), (b"mycc", b"c1", blockgen.key_hash("m"), True)]
    assert blockgen.tx_rwset([("mycc", 2, 2, 1)]) == pb.f_bytes(2, pb.f_bytes(1, b"mycc") + pb.f_bytes(2, blockgen.kv_rwset(2, 2, b"mycc")) +
                                                             pb.f_bytes(3, pb.f_bytes(1, b"collection") + pb.f_bytes(2, blockgen.hashed_rwset(1, b"mycc"))))
    assert blockgen.tx_rwset([("mycc", 1, 1, [("a", 2, 1, 3)])]) == \
        pb.f_bytes(2, pb.f_bytes(1, b"mycc") + pb.f_bytes(2, blockgen.kv_rwset(1, 1, b"mycc")) +
                   pb.f_bytes(3, pb.f_bytes(1, b"a") + pb.f_bytes(2, blockgen.collection_hashed_rwset(2, 1, 3, b"mycc/a"))))


def corpus_key_table(kn, r):
    """VPs on the keys blockgen writes by default (public mycc-w0 / -w1 / -m0, the wire corpus's collection key hashes), some -2"""
    import hashlib
    t = {("mycc", "", b"mycc-w%d" % i): r["vp_org1" if i else "vp_3of4"] for i in range(2)}
    t[("mycc", "collection", hashlib.sha256(b"mycc-hw0").digest())] = r["vp_org2"]
    t[("mycc", "strictcoll", hashlib.sha256(b"mycc/strictcoll-hw0").digest())] = r["vp_org1"]
    t[("strictcc", "", b"strictcc-w0")] = -2
    return t


def test_collection_cases_with_a_key_table():
    """collcases once more with a key table covering their keys: the host build equals the key-level oracle on every transaction."""
    kn, r = klcases.vp_forest()
    table = corpus_key_table(kn, r)
    names, bits = collcases.principals(True)
    nodes, vps = klcases.combined(kn, table)
    moved = 0
    for case in collcases.cases():
        net, blk, info, with_table, _ = collcases.materialize(case)
        ids = net.identities()
        host = klutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names,
                                         policies=collcases.namespace_policies(), principal_bits=bits, collections=collcases.collection_table(),
                                         key_calls=[(True, kn, table)], writes_hint=HINT)
        exp = keylevel_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=collcases.namespace_policies(),
                                             collections=collcases.collection_table(), vps=vps, known=[i[0] for i in ids])
        assert host.tolist() == exp.tolist(), case[0]
        moved += sum(a != b for a, b in zip(exp.tolist(), with_table))
    assert moved >= 3


def test_wire_mutation_corpus_with_a_key_table():
    """The wire-mutation corpus with a key table on its keys: the host build's flags equal the key-level oracle's for every transaction."""
    import wiremut
    net, ids, nodes, pol, blocks = wiremut.corpus()
    kn, r = klcases.vp_forest()
    table = corpus_key_table(kn, r)
    kn_nodes = np.array(kn, np.int32).copy()
    kn_nodes[kn_nodes[:, 0] == 0, 2] += nodes.shape[0]
    all_nodes = np.concatenate([np.asarray(nodes, np.int32).reshape(-1, 4), kn_nodes])
    vps = {k: (v + nodes.shape[0] if v >= 0 else v) for k, v in table.items()}
    counts = {}
    for blk, info, _, before in blocks:
        host = klutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol,
                                         key_calls=[(True, kn, table)], writes_hint=HINT)
        exp = keylevel_oracle.validate_block(blk, ids, net.channel, all_nodes, net.principals, policies=pol, vps=vps, known=[i[0] for i in ids])
        assert host.tolist() == exp.tolist()
        for a, b in zip(before.tolist(), exp.tolist()):
            counts[(a, b)] = counts.get((a, b), 0) + 1
    assert sum(v for (a, b), v in counts.items() if a != b) >= 10
