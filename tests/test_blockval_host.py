"""The device-side block logic (fabric-mod_b200/csrc/blockdev.cuh: walk, dispatcher checks, gates, decisions), compiled for the host,
against the oracle's restatement of the reference's validator (oracle/blockval.py), on the CPU: every fault class of
tools/blockgen.py, per-chaincode policies, policy-evaluator semantics, de-duplication, duplicates, structural corner cases."""
import functools
import os
import random

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from tools import fabricpb as pb
import blockutil
import wiremut


# ---- the device-side implementation of the same logic (blockdev.cuh), executed on the host ---------------------------------
def _envs(blk):
    envs = pb.parse(pb.parse(blk, ob.S_BLOCK)["data"] or b"", ob.S_BLOCKDATA)["data"]
    off = np.zeros(len(envs) + 1, np.uint32)
    off[1:] = np.cumsum([len(e) for e in envs])
    return b"".join(envs), off


def _known(ids):
    return [i[0] for i in ids]


def test_device_logic_fault_classes_match_oracle():
    net = blockgen.Network()
    n = 3 * len(blockgen.FAULTS) + 4
    faults = blockutil.fault_map(n)
    assert set(faults.values()) == set(blockgen.FAULTS)
    blk, info = blockgen.build_block(net, n, 3, faults, seed=11, nthreads=2)
    ids = blockutil.identities_of(net)
    for k in (2, 3, 4):
        exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(k), net.principals, known=_known(ids))
        got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, net.policy_n_of(k), net.principals)
        assert got.tolist() == exp.tolist(), k
    nodes = np.array([(0, 2, 1, 2), (1, 0, 0, 0), (0, 1, 3, 2), (1, 1, 0, 0), (1, 2, 0, 0)], np.int32)
    exp = ob.validate_block(blk, ids, net.channel, nodes, net.principals, known=_known(ids))
    assert blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals).tolist() == exp.tolist()
    exp3 = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    assert exp3[[t for t, f in faults.items() if f == "dup_txid"][0]] == ob.DUPLICATE_TXID
    for t in range(n):
        if t not in faults:
            assert exp3[t] == ob.VALID, t


def test_device_logic_per_chaincode_policies():
    """One policy per namespace (plugindispatcher/dispatcher.go:166-221): writes to a second chaincode bring its policy in, reads do
    not; namespaces / identities the device table lacks -> NOT_VALIDATED; signers de-duplicate on Mspid + certificate."""
    net = blockgen.Network()
    n = 3 * len(blockgen.FAULTS) + 4
    faults = blockutil.fault_map(n)
    blk, info = blockgen.build_block(net, n, 3, faults, seed=11, nthreads=2)
    ids = blockutil.identities_of(net)
    for k in (2, 3):
        nodes, pol = net.policies_for(k)
        exp = ob.validate_block(blk, ids, net.channel, nodes, net.principals, policies=pol, known=_known(ids))
        got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol)
        assert got.tolist() == exp.tolist(), k
        byf = {f: int(exp[t]) for t, f in faults.items()}
        assert byf["reads_strict_namespace"] == ob.VALID and byf["writes_unknown_namespace"] == ob.NOT_VALIDATED
        assert byf["unknown_endorser"] == ob.NOT_VALIDATED and byf["unknown_creator"] == ob.NOT_VALIDATED and byf["many_endorsements"] == ob.VALID
        assert byf["writes_strict_namespace"] == (ob.ENDORSEMENT_POLICY_FAILURE if k == 3 else ob.VALID)      # 3 endorsements: 4-of-4 fails, 3-of-4 holds
        assert byf["same_cert_two_encodings"] == (ob.ENDORSEMENT_POLICY_FAILURE if k == 3 else ob.VALID)
        assert {ob.BAD_HEADER_EXTENSION, ob.BAD_RESPONSE_PAYLOAD, ob.BAD_RWSET, ob.ILLEGAL_WRITESET, ob.INVALID_CHAINCODE} <= set(exp.tolist())
    # the reference itself (every identity known to the MSP, no device in the picture) gives a verdict where the device abstains:
    # an unknown creator is a BAD_CREATOR_SIGNATURE there
    ref = ob.validate_block(blk, ids, net.channel, nodes, net.principals, policies=pol)
    t = [t for t, f in faults.items() if f == "unknown_creator"][0]
    assert ref[t] == ob.BAD_CREATOR_SIGNATURE and exp[t] == ob.NOT_VALIDATED


def test_policy_thresholds_and_dedup():
    # common/policies/policy_test.go:255-288 (two identical SignedData => one identity) and cauthdsl N-out-of semantics
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    blk, info = blockgen.build_block(net, 12, 3, {3: "dup_endorser", 5: "bad_endorsement_sig", 7: "same_cert_two_encodings"}, seed=3, nthreads=2)
    for k, expect_fail in ((2, []), (3, [3, 5, 7]), (4, list(range(12)))):
        exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(k), net.principals, known=_known(ids))
        got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, net.policy_n_of(k), net.principals)
        assert got.tolist() == exp.tolist()
        assert [t for t in range(12) if exp[t] == ob.ENDORSEMENT_POLICY_FAILURE] == expect_fail


def test_device_logic_structural_corner_cases():
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    blk, _ = blockgen.build_block(net, 6, 3, {}, seed=5, nthreads=2)
    envs = pb.parse(pb.parse(blk, ob.S_BLOCK)["data"], ob.S_BLOCKDATA)["data"]
    good = envs[0]
    variants = [good, b"", b"\x0a\x05abc", pb.f_uint(1, 5), good + pb.f_bytes(9, b"unknown field is skipped"), pb.f_bytes(1, b""),
                envs[1][: len(envs[1]) // 2], pb.f_bytes(2, b"sig-only"), envs[2], envs[3]]
    blk2 = pb.block(9, variants)
    exp = ob.validate_block(blk2, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    assert exp[0] == ob.VALID and exp[4] == ob.DUPLICATE_TXID       # same transaction + an unknown field: parses, same tx id
    assert exp[1] == ob.BAD_COMMON_HEADER and exp[5] == ob.BAD_COMMON_HEADER
    blob, off = _envs(blk2)
    assert blockutil.device_logic_flags(blob, off, ids, net.channel, net.policy_n_of(3), net.principals).tolist() == exp.tolist()
    assert blockutil.device_logic_flags(b"", np.zeros(1, np.uint32), ids, net.channel, net.policy_n_of(3), net.principals).tolist() == []


def test_device_der_gate_matches_host_gate_fuzz():
    import random
    from oracle import goasn1, p256
    from util import pkg
    b = pkg().binding
    rnd = random.Random(77)
    seeds = [goasn1.marshal_ecdsa_signature(rnd.getrandbits(256), rnd.getrandbits(255)) for _ in range(30)]
    seeds += [goasn1.marshal_ecdsa_signature(rnd.getrandbits(8 * k), rnd.getrandbits(8 * j)) for k in (1, 31, 33, 40) for j in (1, 31, 32, 33)]
    seeds += [goasn1.marshal_ecdsa_signature(5, p256.HALF_N), goasn1.marshal_ecdsa_signature(5, p256.HALF_N + 1), goasn1.marshal_ecdsa_signature(-5, 7),
              goasn1.marshal_ecdsa_signature(0, 7), goasn1.marshal_ecdsa_signature(7, 0), b"", b"\x30\x00"]
    n = 0
    for sd in seeds:
        for it in range(120):
            m = bytearray(sd)
            if it:
                for _ in range(rnd.choice((1, 1, 2, 3))):
                    op = rnd.random()
                    if op < 0.6 and m:
                        m[rnd.randrange(len(m))] = rnd.getrandbits(8)
                    elif op < 0.8 and m:
                        del m[rnd.randrange(len(m))]
                    else:
                        m.insert(rnd.randrange(len(m) + 1), rnd.getrandbits(8))
            sig = bytes(m)
            st, r, s = b.gate_signature(sig)
            ok, r2, s2, dst = blockutil.device_gate(sig)
            assert ok == (st == b.ST_VALID), sig.hex()
            if sig:
                assert dst == st, sig.hex()                     # same status code as the host gate, error kinds included
            if ok:
                assert (r, s) == (r2, s2)
            n += 1
    assert n > 5000


def test_identity_groups_follow_the_certificate_not_the_bytes():
    """binding.identity_groups (what fabgpu_msp_identity_groups is fed): Mspid + certificate digest, as the reference's IdentityIdentifier
    (common/policies/policy.go:380-386, msp/identities.go:55-76) -- and the same partition as the oracle's identity_id."""
    from util import pkg
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    g = pkg().binding.identity_groups(ids)
    n_peers = len(net.peers)
    first_alt = len(ids) - n_peers
    for k in range(n_peers):
        assert g[k] == g[first_alt + k]                         # CRLF re-encoding of peer k's certificate: same identity
    assert len(set(g.tolist())) == len(ids) - n_peers
    oracle_ids = [ob.identity_id(i[0], i[1]) for i in ids]
    for a in range(len(ids)):
        for b in range(len(ids)):
            assert (g[a] == g[b]) == (oracle_ids[a] == oracle_ids[b])
    # the same certificate under ANOTHER MSP id is another identity; unparsable id_bytes fall back to the bytes themselves
    other = [(pb.serialized_identity("OtherMSP", net.peers[0].cert_pem), "OtherMSP", net.peers[0].xy, True),
             (pb.serialized_identity("Org1MSP", b"not a pem"), "Org1MSP", net.peers[0].xy, True),
             (pb.serialized_identity("Org1MSP", b"not a pem"), "Org1MSP", net.peers[0].xy, True)]
    g2 = pkg().binding.identity_groups(ids + other)
    assert g2[len(ids)] not in g2[: len(ids)].tolist() and g2[len(ids) + 1] == g2[len(ids) + 2] != g2[len(ids)]


def test_device_logic_with_hundreds_of_client_identities():
    """An MSP of 300 client certificates (plus peers): the identity lookup (sample_hash + msp_find of blockdev.cuh) must keep finding every
    identity when the table is large and the certificates share header, MSP id and PEM footer -- flags equal the oracle's on a block with
    every fault class, and the lookup's hash puts (almost) every identity into its own bucket."""
    net = blockgen.Network(n_orgs=4, n_clients=300, seed=0xC11E)
    n = 3 * len(blockgen.FAULTS) + 40
    faults = blockutil.fault_map(n)
    blk, info = blockgen.build_block(net, n, 3, faults, seed=29, nthreads=2)
    ids = blockutil.identities_of(net)
    assert len(ids) > 300
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, net.policy_n_of(3), net.principals)
    assert got.tolist() == exp.tolist()
    assert int((exp == ob.VALID).sum()) > 40
    # the same hash, restated: FNV-style over 16 head + 32 middle + 32 pre-footer + 24 tail bytes
    M = (1 << 64) - 1

    def h(p):
        x = 1469598103934665603 ^ len(p)
        idx = list(range(min(16, len(p))))
        if len(p) >= 160:
            idx += list(range(len(p) // 2 - 16, len(p) // 2 + 16)) + list(range(len(p) - 72, len(p) - 40))
        idx += list(range(len(p) - min(24, len(p)), len(p)))
        for i in idx:
            x = ((x ^ p[i]) * 1099511628211) & M
        return x or 1
    hashes = {h(i[0]) for i in ids}
    assert len(hashes) == len(ids)                      # head + tail alone gave one value per MSP id


# ---- wire-level fuzzing of the block parser (tests/wiremut.py) -----------------------------------------------------------------
def test_wire_mutation_corpus_matches_oracle():
    """Every mutation kind at every message level of a transaction: the device logic's flag equals the oracle's for every transaction,
    and every kind changes some verdict (no kind passes without reaching a check)."""
    net, ids, nodes, pol, blocks = wiremut.corpus()
    seen, changed = set(), set()
    for blk, info, labels, exp in blocks:
        got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol)
        bad = [(t, labels[t], int(exp[t]), int(got[t])) for t in range(len(exp)) if got[t] != exp[t]]
        assert not bad, bad[:10]
        for t, lab in enumerate(labels):
            if lab is None:
                assert exp[t] == ob.VALID
                continue
            seen.add(lab)
            if exp[t] != ob.VALID:
                changed.add(lab[1])
    assert sum(lab is not None for b in blocks for lab in b[2]) >= 3000          # mutated transactions
    assert seen == {(p, k) for p in wiremut.TX_PARTS for k in wiremut.KINDS if k != "chdr_int" or p == "ChannelHeader"}
    assert changed == set(wiremut.KINDS)


def _one_tx():
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    blk, _ = blockgen.build_block(net, 1, 3, {}, seed=5, nthreads=2)
    env = pb.parse(pb.parse(blk, ob.S_BLOCK)["data"], ob.S_BLOCKDATA)["data"][0]
    e = pb.parse(env, ob.S_ENVELOPE)
    return net, ids, env, e["payload"], e["signature"]


def _flags_both(net, ids, envs):
    blk = pb.block(1, envs)
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    blob, off = _envs(blk)
    return exp.tolist(), blockutil.device_logic_flags(blob, off, ids, net.channel, net.policy_n_of(3), net.principals).tolist()


def test_field_number_2_pow_32_plus_2_is_an_unknown_field():
    net, ids, env, _, _ = _one_tx()
    assert _flags_both(net, ids, [env + pb.f_bytes((1 << 32) + 2, b"xyz")]) == ([ob.VALID], [ob.VALID])


def test_aliased_signature_field_does_not_replace_the_signature():
    net, ids, _, payload, sig = _one_tx()
    env = pb.f_bytes(1, payload) + pb.f_bytes(2, b"\x30\x06\x02\x01\x01\x02\x01\x01") + pb.f_bytes((1 << 32) + 2, sig)
    assert _flags_both(net, ids, [env]) == ([ob.BAD_CREATOR_SIGNATURE], [ob.BAD_CREATOR_SIGNATURE])


def test_field_number_2_pow_29_plus_2_is_an_unknown_field():
    net, ids, env, payload, sig = _one_tx()
    assert _flags_both(net, ids, [env + pb.f_bytes((1 << 29) + 2, b"xyz")]) == ([ob.VALID], [ob.VALID])
    env2 = pb.f_bytes(1, payload) + pb.f_bytes(2, b"\x30\x06\x02\x01\x01\x02\x01\x01") + pb.f_bytes((1 << 29) + 2, sig)
    assert _flags_both(net, ids, [env2]) == ([ob.BAD_CREATOR_SIGNATURE], [ob.BAD_CREATOR_SIGNATURE])


@pytest.mark.parametrize("value,code", [(3 + (1 << 32), ob.VALID), (3 + (1 << 63), ob.VALID), ((1 << 64) - 1, ob.BAD_COMMON_HEADER),
                                        ((1 << 32) - 3, ob.BAD_COMMON_HEADER), (2 + (1 << 32), ob.UNSUPPORTED_TX_PAYLOAD)])
def test_channel_header_type_is_an_int32(value, code):
    """ChannelHeader.type is an int32: the decoder keeps the varint's low 32 bits (3 + 2^32 is an endorser transaction, -1 sent
    as a 10-byte varint is -1)."""
    net = blockgen.Network()
    ids = blockutil.identities_of(net)

    def mut(t, part, b):
        if part != "ChannelHeader":
            return b
        return b"".join(wiremut.enc(*f) for f in wiremut.split(b) if f[0] != 1) + pb.f_uint(1, value)
    blk, info = blockgen.build_block(net, 2, 3, {}, seed=5, nthreads=2, mutate=mut)
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, net.policy_n_of(3), net.principals)
    assert exp.tolist() == [code, code] and got.tolist() == exp.tolist()


def test_epoch_2_pow_64_minus_1_is_a_bad_header():
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    mut = lambda t, part, b: b + pb.f_uint(6, (1 << 64) - 1) if part == "ChannelHeader" else b
    blk, info = blockgen.build_block(net, 1, 3, {}, seed=5, nthreads=2, mutate=mut)
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, net.policy_n_of(3), net.principals)
    assert exp.tolist() == got.tolist() == [ob.BAD_COMMON_HEADER]


def _oracle_split(blk):
    try:
        return pb.parse(pb.parse(blk, ob.S_BLOCK)["data"] or b"", ob.S_BLOCKDATA)["data"]
    except pb.PbError:
        return None


def test_split_block_matches_oracle_fuzz():
    """split_block (blockval.cpp) finds the same envelopes as the oracle's Block / BlockData parse, or fails where it fails, under every
    mutation kind of the Block and of its BlockData."""
    mutants = wiremut.block_mutants()
    failed = 0
    for i, (kind, m) in enumerate(mutants):
        exp = _oracle_split(m)
        assert blockutil.split_block(m) == exp, (kind, i, m.hex())
        failed += exp is None
    assert len(mutants) >= 900 and 0 < failed < len(mutants)


def test_split_block_aliased_data_field():
    """A Block field numbered 2^32 + 2 is not Block.data: the envelopes are those of the real data field."""
    net = blockgen.Network()
    blk, _ = blockgen.build_block(net, 3, 3, {}, seed=5, nthreads=2)
    other, _ = blockgen.build_block(net, 2, 3, {}, seed=6, nthreads=2)
    other_data = pb.parse(other, ob.S_BLOCK)["data"]
    for forged in (blk + pb.f_bytes((1 << 32) + 2, other_data), pb.f_bytes((1 << 32) + 2, other_data) + blk):
        assert blockutil.split_block(forged) == _oracle_split(forged) == _oracle_split(blk)
        assert len(_oracle_split(forged)) == 3


def test_job_overflow_writes_dead_records():
    """More than BD_ENDS_HINT endorsements per transaction on average: the endorsement-job arrays fill up and the transactions that do not
    fit go to the CPU validator (NOT_VALIDATED).  The arrays start out as garbage (what the previous block or cudaMalloc left), so every
    slot the walk hands out must get a record: a live job or a dead one.  Transactions that fit are exact."""
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    n = 12
    faults = {t: "many_endorsements" for t in range(n) if t % 4 != 1}       # 21 endorsements each, 3 for every fourth transaction
    blk, info = blockgen.build_block(net, n, 3, faults, seed=9, nthreads=2)
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    assert (exp == ob.VALID).all()
    for hint in (16, 8, 3):
        got, stale = blockutil.device_logic_run(info["env_blob"], info["env_off"], ids, net.channel, net.policy_n_of(3), net.principals,
                                                ends_hint=hint, poison=True)
        assert stale == 0, hint
        e_cap, used, fits = n * hint, 0, []
        for t in range(n):                                   # the host build hands out job slots in transaction order
            k = 21 if t in faults else 3
            fits.append(used + k <= e_cap)
            used += k
        assert not all(fits) and any(fits)
        for t in range(n):
            assert got[t] == (exp[t] if fits[t] else ob.NOT_VALIDATED), (hint, t)


def _edge_flags(net, n_tx, nodes, policies, **shape):
    ids = blockutil.identities_of(net)
    blk, info = blockgen.build_block(net, n_tx, 3, {}, seed=19, nthreads=2, **shape)
    exp = ob.validate_block(blk, ids, net.channel, nodes, net.principals, policies=policies, known=_known(ids))
    got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=policies)
    return exp.tolist(), got.tolist()


@pytest.mark.parametrize("case", blockutil.capacity_edge_cases(), ids=lambda c: c[0])
def test_capacity_edges(case):
    """BD_MAX_NS_SEEN, BD_MAX_NS and BD_MAX_SIGNERS: exact at the limit, NOT_VALIDATED one past it (the CPU validator decides)."""
    name, net, n_tx, nodes, pol, shape, at, past = case
    exp, got = _edge_flags(net, n_tx, nodes, pol, **shape)
    assert exp[at] == exp[past] == ob.VALID
    assert got[at] == ob.VALID and got[past] == ob.NOT_VALIDATED
    assert [g for i, g in enumerate(got) if i != past] == [e for i, e in enumerate(exp) if i != past]


def _chain(depth):
    """NOutOf(1) nested `depth` times over SignedBy(Org1MSP): the SignedBy node sits at depth `depth`."""
    return np.array([(0, 1, i + 1, 1) for i in range(depth)] + [(1, 0, 0, 0)], np.int32)


def test_policy_depth_limit():
    """eval_policy evaluates trees BD_MAX_POLICY_DEPTH (12) deep exactly; one level deeper it would fail where the reference accepts,
    which is why fabgpu_msp_configure refuses such trees (tests/test_gpu_block.py)."""
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    blk, info = blockgen.build_block(net, 8, 3, {}, seed=5, nthreads=2)
    for depth, device_exact in ((0, True), (12, True), (13, False)):
        exp = ob.validate_block(blk, ids, net.channel, _chain(depth), net.principals, known=_known(ids))
        got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, _chain(depth), net.principals)
        assert (exp == ob.VALID).sum() >= 6
        assert (got.tolist() == exp.tolist()) == device_exact, depth


def test_block_parser_memory_safety_under_sanitizers(tmp_path):
    """split_block, walk_tx, resolve_job and decide_tx built with -fsanitize=address,undefined and run as a separate process over the
    mutation corpus, the Block-level mutants, the capacity edges and job-array overflow (small job arrays): no sanitizer report."""
    import struct
    import subprocess
    from util import ROOT
    d = os.path.join(ROOT, "tests", "host_sim")
    exe = str(tmp_path / "blockdev_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-o", exe, os.path.join(d, "blockdev_asan.cpp"), os.path.join(ROOT, "fabric-mod_b200", "csrc", "blockval.cpp")])
    net, ids, _, _, blocks = wiremut.corpus()
    u32 = lambda v: struct.pack("<I", v)
    lb = lambda b: u32(len(b)) + bytes(b)
    nodes = np.ascontiguousarray(net.policy_n_of(2), np.int32)
    head = u32(len(ids)) + b"".join(lb(i[0]) + lb(i[1].encode()) + bytes([1 if i[3] else 0]) for i in ids)
    head += u32(nodes.shape[0]) + nodes.tobytes() + u32(len(net.principals)) + b"".join(lb(p.encode()) for p in net.principals) + lb(net.channel.encode())
    items = [(16, b[0]) for b in blocks] + [(1, b[0]) for b in blocks[:2]] + [(16, m) for _, m in wiremut.block_mutants()]
    for case in blockutil.capacity_edge_cases():
        items.append((16, blockgen.build_block(case[1], case[2], 3, {}, seed=19, nthreads=2, **case[5])[0]))
    overflow, _ = blockgen.build_block(net, 12, 3, {t: "many_endorsements" for t in range(12) if t % 4 != 1}, seed=9, nthreads=2)
    items += [(16, overflow), (3, overflow)]
    corpus = tmp_path / "corpus.bin"
    corpus.write_bytes(head + u32(len(items)) + b"".join(u32(h) + lb(b) for h, b in items))
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    run = subprocess.run([exe, str(corpus)], capture_output=True, text=True, env=env, timeout=600)
    assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
    parsed = sum(_oracle_split(b) is not None for _, b in items)
    assert run.stdout.split()[:4] == ["blocks", str(len(items)), "parsed", str(parsed)], run.stdout
    assert int(run.stdout.split()[5]) > 3000


@pytest.mark.parametrize("field,v,last,code", wiremut.TEN_BYTE_CASES)
def test_ten_byte_varint_last_byte(field, v, last, code):
    """golang/protobuf's decodeVarint takes a 10th byte only when it is 0 or 1; a larger one overflows and the ChannelHeader does not
    unmarshal.  epoch = 0 with a 10th byte of 2 is a bad header, not epoch 0."""
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    blk, info = wiremut.ten_byte_block(net, field, v, last)
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=_known(ids))
    got = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, net.policy_n_of(3), net.principals)
    assert exp.tolist() == [code, code] and got.tolist() == exp.tolist()


@pytest.mark.parametrize("last", [0, 1, 2, 0x7F])
def test_ten_byte_varint_in_block_and_envelope(last):
    """The same rule for the lengths and values split_block and the envelope walk read: an unknown varint field whose 10th byte is
    0 or 1 is skipped; a larger 10th byte makes the Block (split_block) or the Envelope (INVALID_OTHER_REASON) fail to parse."""
    net, ids, env, _, _ = _one_tx()
    extra = wiremut.uvarint(9 << 3) + wiremut.ten_byte_varint(5, last)
    exp_code = ob.VALID if last < 2 else ob.INVALID_OTHER_REASON
    assert _flags_both(net, ids, [env + extra]) == ([exp_code], [exp_code])
    blk = pb.block(1, [env]) + extra
    assert blockutil.split_block(blk) == _oracle_split(blk) == (None if last >= 2 else [env])
    blk = pb.block(1, [env]) + wiremut.uvarint(9 << 3 | 2) + wiremut.ten_byte_varint(8, last) + b"x" * 8          # a length in 10 bytes
    assert blockutil.split_block(blk) == _oracle_split(blk) == (None if last else [env])          # 1: bit 63 of the length
