"""GPU: device SHA-256 and the block-level pre-pass (fabgpu_validate_block) against hashlib and the oracle's block validator."""
import hashlib
import random

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from tools import fabricpb as pb
from util import pkg
import blockutil

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    yield c
    c.close()


def test_sha256_segments_vs_hashlib(ctx):
    rnd = random.Random(9)
    buf = bytes(rnd.getrandbits(8) for _ in range(20000))
    jobs, exp = [], []
    lens = [0, 1, 3, 4, 5, 31, 32, 33, 54, 55, 56, 57, 63, 64, 65, 119, 120, 127, 128, 129, 1000, 4097]
    for la in lens:
        for lb in (0, 1, 7, 64, 333):
            for lc in (0, 5):
                oa, ob_, oc = rnd.randrange(0, 9000), rnd.randrange(0, 9000), rnd.randrange(0, 9000)
                jobs.append((oa, ob_, oc, la, lb, lc))
                exp.append(hashlib.sha256(buf[oa:oa + la] + buf[ob_:ob_ + lb] + buf[oc:oc + lc]).digest())
    got = ctx.sha256_segments(buf, np.array(jobs, np.uint32))
    assert [bytes(g) for g in got] == exp


def _configure(ctx, net, n):
    ctx.msp_configure(blockutil.identities_of(net), net.policy_n_of(n), net.principals, net.channel)


def _oracle(blk, net, nodes, policies=None):
    """The oracle's flags for a device that holds exactly net.msp_table (identities outside it -> NOT_VALIDATED)."""
    ids = blockutil.identities_of(net)
    return ob.validate_block(blk, ids, net.channel, nodes, net.principals, policies=policies, known=[i[0] for i in ids])


def test_block_fault_classes_match_oracle(ctx):
    net = blockgen.Network()
    faults = blockutil.fault_map(70)
    blk, _ = blockgen.build_block(net, 70, 3, faults, seed=11)
    exp = _oracle(blk, net, net.policy_n_of(3))
    _configure(ctx, net, 3)
    got = ctx.validate_block(blk)
    assert got.tolist() == exp.tolist()
    assert len(set(exp.tolist())) >= 10
    # other thresholds / nested policy reuse the same block
    for n in (2, 4):
        _configure(ctx, net, n)
        assert ctx.validate_block(blk).tolist() == _oracle(blk, net, net.policy_n_of(n)).tolist()


def test_block_per_chaincode_policies_and_dispatcher_checks(ctx):
    """Every fault class incl. the plugin dispatcher's (dispatcher.go:102-221) with a policy PER NAMESPACE: a transaction that writes to
    a second chaincode is held to that chaincode's policy too; one that only reads it is not; an unknown namespace or identity -> 254;
    21 endorsements (both encodings of every certificate) de-duplicate to four signers."""
    net = blockgen.Network()
    n = 3 * len(blockgen.FAULTS) + 4
    faults = blockutil.fault_map(n)
    assert set(faults.values()) == set(blockgen.FAULTS)
    blk, info = blockgen.build_block(net, n, 3, faults, seed=11)
    nodes, pol = net.policies_for(3)
    exp = _oracle(blk, net, nodes, pol)
    ctx.msp_configure(blockutil.identities_of(net), nodes, net.principals, net.channel, policies=pol)
    assert ctx.validate_block(blk).tolist() == exp.tolist()
    assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp.tolist()
    byf = {f: int(exp[t]) for t, f in faults.items()}
    assert byf["writes_strict_namespace"] == ob.ENDORSEMENT_POLICY_FAILURE and byf["reads_strict_namespace"] == ob.VALID
    assert byf["writes_unknown_namespace"] == ob.NOT_VALIDATED and byf["unknown_endorser"] == ob.NOT_VALIDATED and byf["unknown_creator"] == ob.NOT_VALIDATED
    assert byf["same_cert_two_encodings"] == ob.ENDORSEMENT_POLICY_FAILURE and byf["many_endorsements"] == ob.VALID
    assert {ob.BAD_HEADER_EXTENSION, ob.BAD_RESPONSE_PAYLOAD, ob.BAD_RWSET, ob.ILLEGAL_WRITESET, ob.INVALID_CHAINCODE, ob.INVALID_OTHER_REASON} <= set(exp.tolist())


def test_block_2000_tx_mixed_and_pinned_buffer(ctx):
    net = blockgen.Network(n_orgs=4, n_clients=3)
    rnd = random.Random(4)
    faults = {t: rnd.choice(blockgen.FAULTS) for t in rnd.sample(range(1, 2000), 240)}
    blk, binfo = blockgen.build_block(net, 2000, 3, faults, seed=13)
    exp = _oracle(blk, net, net.policy_n_of(3))
    _configure(ctx, net, 3)
    assert ctx.validate_block(blk).tolist() == exp.tolist()
    assert ctx.validate_envelopes(binfo["env_blob"], binfo["env_off"]).tolist() == exp.tolist()      # Block.Data.Data form
    pinned = ctx.block_buffer(len(blk))
    pinned[:] = np.frombuffer(blk, np.uint8)
    assert ctx.validate_block(pinned).tolist() == exp.tolist()
    assert 1700 < int((exp == ob.VALID).sum()) < 1850


def test_config3_block_replay_10k_tx(ctx):
    # BASELINE.json configs[2]: 10 k synthetic txs x 3 endorsements, 3-of-4 policy: 40 000 verifications, every flag VALID
    net = blockgen.Network()
    blk, info = blockgen.build_block(net, 10000, 3, {}, seed=17)
    assert info["n_sigs"] == 40000
    _configure(ctx, net, 3)
    pinned = ctx.block_buffer(len(blk))
    pinned[:] = np.frombuffer(blk, np.uint8)
    got = ctx.validate_block(pinned)
    assert got.shape[0] == 10000 and (got == ob.VALID).all()
    exp = _oracle(blk, net, net.policy_n_of(3))
    assert (exp == ob.VALID).all()
    # one flipped byte inside one endorsement signature flips exactly that transaction
    b = bytearray(blk)
    marker = net.peers[1].serialized
    pos = blk.index(marker, len(blk) // 2) + len(marker) + 10
    b[pos] ^= 0x20
    got2 = ctx.validate_block(bytes(b))
    exp2 = _oracle(bytes(b), net, net.policy_n_of(3))
    assert got2.tolist() == exp2.tolist() and int((got2 != ob.VALID).sum()) == 1


def test_block_survives_key_table_eviction():
    """Identity tables recycled by unrelated registrations between fabgpu_msp_configure and a block: still exact."""
    import os
    from tools import workload
    os.environ["FABGPU_KEY_SLOTS"] = "8"
    try:
        c = pkg().binding.Context(max_batch=4096)
    finally:
        del os.environ["FABGPU_KEY_SLOTS"]
    net = blockgen.Network()
    faults = blockutil.fault_map(60)
    blk, binfo = blockgen.build_block(net, 60, 3, faults, seed=23)
    exp = _oracle(blk, net, net.policy_n_of(3))
    c.msp_configure(blockutil.identities_of(net), net.policy_n_of(3), net.principals, net.channel)
    assert c.validate_envelopes(binfo["env_blob"], binfo["env_off"]).tolist() == exp.tolist()
    other = workload.Workload(64, 8, seed=99)
    assert (c.keys_register(other.keys_xy) >= 0).all()          # evicts every identity's table
    assert c.validate_envelopes(binfo["env_blob"], binfo["env_off"]).tolist() == exp.tolist()
    c.keys_register(other.keys_xy)
    assert c.validate_block(blk).tolist() == exp.tolist()       # serialized-Block entry point after another eviction
    c.close()


def test_two_blocks_in_flight(ctx):
    """fabgpu_validate_*_async / fabgpu_validate_wait: two different blocks on the two slots at once, several rounds, both entry
    forms; each slot returns the oracle's flags for ITS block (separate device buffers, counters and pinned staging per slot)."""
    net = blockgen.Network(n_orgs=4, n_clients=3)
    ids = blockutil.identities_of(net)
    _configure(ctx, net, 3)
    blocks = []
    for k, (ntx, nfault, seed) in enumerate([(900, 120, 31), (333, 60, 32)]):
        rnd = random.Random(seed)
        faults = {t: rnd.choice(blockgen.FAULTS) for t in rnd.sample(range(1, ntx), nfault)}
        blk, info = blockgen.build_block(net, ntx, 3, faults, seed=seed)
        exp = _oracle(blk, net, net.policy_n_of(3))
        blob = np.frombuffer(info["env_blob"], np.uint8)
        pinned = ctx.block_buffer(blob.shape[0], slot=k)
        pinned[:] = blob
        blocks.append((blk, pinned, info["env_off"], exp))
    binding = pkg().binding
    for rnd_i in range(4):
        order = (0, 1) if rnd_i % 2 == 0 else (1, 0)
        caps = {}
        for sl in order:
            blk, pinned, eoff, _ = blocks[sl]
            caps[sl] = ctx.validate_envelopes_async(sl, pinned, eoff) if rnd_i < 2 else ctx.validate_block_async(sl, blk)
        with pytest.raises(binding.FabGpuError):                              # a slot holds one block at a time
            ctx.validate_envelopes_async(0, blocks[0][1], blocks[0][2])
        for sl in order:
            got = ctx.validate_wait(sl, caps[sl])
            assert got.tolist() == blocks[sl][3].tolist(), (rnd_i, sl)
    with pytest.raises(binding.FabGpuError):                                  # nothing in flight
        ctx.validate_wait(1, 16)
    # the blocking calls still work afterwards, and an empty envelope list goes through both halves
    assert ctx.validate_envelopes(blocks[1][1], blocks[1][2]).tolist() == blocks[1][3].tolist()
    assert ctx.validate_envelopes_async(1, np.zeros(1, np.uint8), np.zeros(1, np.uint32)) == 0
    assert ctx.validate_wait(1, 1).shape[0] == 0


# ---- wire-level fuzzing: the host-side tests/test_blockval_host.py corpus on the device -----------------------------------------
def test_wire_mutation_corpus_all_entry_points(ctx):
    """Every block of the mutation corpus (3 080 mutated transactions, every mutation kind at every message level) through the envelope form,
    the serialized-Block form (split_block), a pinned buffer and the two async slots: the flags equal the oracle's and the host
    build's, byte for byte."""
    import wiremut
    net, ids, nodes, pol, blocks = wiremut.corpus()
    ctx.msp_configure(ids, nodes, net.principals, net.channel, policies=pol)
    for k, (blk, info, labels, exp) in enumerate(blocks):
        host = blockutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol)
        assert host.tolist() == exp.tolist()
        assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp.tolist(), k
        assert ctx.validate_block(blk).tolist() == exp.tolist(), k
        if k % 2 == 0:
            pinned = ctx.block_buffer(len(blk))
            pinned[:] = np.frombuffer(blk, np.uint8)
            assert ctx.validate_block(pinned).tolist() == exp.tolist(), k
    for (b0, i0, _, e0), (b1, i1, _, e1) in zip(blocks[0::2], blocks[1::2]):
        n0 = ctx.validate_envelopes_async(0, i0["env_blob"], i0["env_off"])
        n1 = ctx.validate_block_async(1, b1)
        assert ctx.validate_wait(1, n1).tolist() == e1.tolist()
        assert ctx.validate_wait(0, n0).tolist() == e0.tolist()


def test_block_with_aliased_data_field(ctx):
    """A Block field numbered 2^32 + 2 carrying other envelopes is an unknown field, not Block.data."""
    net = blockgen.Network()
    blk, _ = blockgen.build_block(net, 30, 3, {}, seed=41)
    other, _ = blockgen.build_block(net, 5, 3, {2: "bad_creator_sig"}, seed=42)
    forged = blk + pb.f_bytes((1 << 32) + 2, pb.parse(other, ob.S_BLOCK)["data"])
    exp = _oracle(forged, net, net.policy_n_of(3))
    assert exp.tolist() == _oracle(blk, net, net.policy_n_of(3)).tolist() and len(exp) == 30
    _configure(ctx, net, 3)
    assert ctx.validate_block(forged).tolist() == exp.tolist()


def test_job_overflow_after_a_larger_block():
    """A block that needs more endorsement jobs than the job arrays hold, first on fresh device memory, then on a slot whose arrays
    hold a larger block's jobs: every flag is the oracle's or NOT_VALIDATED, only the few transactions that do not fit get the latter,
    and the slot validates the larger block exactly afterwards.  The flags cannot show whether the walk wrote dead records into the
    slots it gave up (a stale record belongs to no transaction of this block); test_job_overflow_writes_dead_records in
    tests/test_blockval_host.py checks that on the host build, with the job arrays filled with garbage."""
    c = pkg().binding.Context(max_batch=8192)
    try:
        net = blockgen.Network()
        n = 12
        small, _ = blockgen.build_block(net, n, 3, {t: "many_endorsements" for t in range(n) if t % 4 != 1}, seed=9)   # 198 jobs, room for 192
        exp = _oracle(small, net, net.policy_n_of(3))
        assert (exp == ob.VALID).all()
        big, _ = blockgen.build_block(net, 3000, 3, blockutil.fault_map(3000), seed=43)
        exp_big = _oracle(big, net, net.policy_n_of(3))
        _configure(c, net, 3)

        def check(got):
            assert all(g in (e, ob.NOT_VALIDATED) for g, e in zip(got.tolist(), exp.tolist())), got
            assert 1 <= int((got == ob.NOT_VALIDATED).sum()) <= 2
        for slot in (0, 1):
            check(c.validate_wait(slot, c.validate_block_async(slot, small)))
            assert c.validate_wait(slot, c.validate_block_async(slot, big)).tolist() == exp_big.tolist()
            check(c.validate_wait(slot, c.validate_block_async(slot, small)))
        assert c.validate_block(big).tolist() == exp_big.tolist()           # and nothing stale is left behind
    finally:
        c.close()


@pytest.mark.parametrize("case", blockutil.capacity_edge_cases(), ids=lambda c: c[0])
def test_capacity_edges(ctx, case):
    """BD_MAX_NS_SEEN, BD_MAX_NS, BD_MAX_SIGNERS on the device: exact at the limit, NOT_VALIDATED one past it."""
    name, net, n_tx, nodes, pol, shape, at, past = case
    blk, _ = blockgen.build_block(net, n_tx, 3, {}, seed=19, **shape)
    exp = _oracle(blk, net, nodes, pol)
    ctx.msp_configure(blockutil.identities_of(net), nodes, net.principals, net.channel, policies=pol)
    got = ctx.validate_block(blk).tolist()
    assert exp[at] == exp[past] == ob.VALID and got[past] == ob.NOT_VALIDATED
    assert [g for i, g in enumerate(got) if i != past] == [e for i, e in enumerate(exp.tolist()) if i != past]


def _chain(depth):
    return np.array([(0, 1, i + 1, 1) for i in range(depth)] + [(1, 0, 0, 0)], np.int32)


def test_msp_configure_refuses_policies_it_cannot_evaluate(ctx):
    """Deeper than BD_MAX_POLICY_DEPTH, cyclic, or a SignedBy principal out of range: FABGPU_E_ARG (the caller validates on the CPU),
    also when the tree is one of several namespace policies.  At the depth limit the flags are exact."""
    binding = pkg().binding
    net = blockgen.Network()
    ids = blockutil.identities_of(net)
    a = net.policy_n_of(3)
    refused = [_chain(13), np.array([(0, 1, 1, 1), (0, 1, 0, 1)], np.int32), np.array([(0, 1, 1, 1), (0, 1, 1, 1)], np.int32),
               np.array([(0, 1, 1, 1), (1, 4, 0, 0)], np.int32), np.array([(1, -1, 0, 0)], np.int32)]
    for nodes in refused:
        with pytest.raises(binding.FabGpuError) as e:
            ctx.msp_configure(ids, nodes, net.principals, net.channel)
        assert e.value.code == binding.E_ARG
    deep = _chain(13).copy(); deep[:-1, 2] += a.shape[0]
    with pytest.raises(binding.FabGpuError) as e:
        ctx.msp_configure(ids, np.concatenate([a, deep]), net.principals, net.channel, policies={blockgen.CHAINCODE: 0, "deepcc": int(a.shape[0])})
    assert e.value.code == binding.E_ARG
    blk, _ = blockgen.build_block(net, 20, 3, blockutil.fault_map(20), seed=44)
    ctx.msp_configure(ids, _chain(12), net.principals, net.channel)
    exp = _oracle(blk, net, _chain(12))
    assert ctx.validate_block(blk).tolist() == exp.tolist() and (exp == ob.VALID).sum() >= 10


def test_ten_byte_varint_last_byte(ctx):
    """A varint's 10th byte may only be 0 or 1 (golang/protobuf's decodeVarint): ChannelHeader.type and epoch written in 10 bytes,
    and an unknown Block field whose 10-byte varint overflows (the Block does not parse)."""
    import wiremut
    net = blockgen.Network()
    _configure(ctx, net, 3)
    for field, v, last, code in wiremut.TEN_BYTE_CASES:
        blk, _ = wiremut.ten_byte_block(net, field, v, last)
        exp = _oracle(blk, net, net.policy_n_of(3))
        assert exp.tolist() == [code, code] and ctx.validate_block(blk).tolist() == exp.tolist(), (field, last)
    blk, _ = blockgen.build_block(net, 3, 3, {}, seed=5)
    for last in (0, 1):
        assert ctx.validate_block(blk + wiremut.uvarint(9 << 3) + wiremut.ten_byte_varint(5, last)).tolist() == _oracle(blk, net, net.policy_n_of(3)).tolist()
    with pytest.raises(pkg().binding.FabGpuError) as e:
        ctx.validate_block(blk + wiremut.uvarint(9 << 3) + wiremut.ten_byte_varint(5, 2))
    assert e.value.code == pkg().binding.E_ARG
