"""GPU: identity admission (fabgpu_msp_identities_add) and the unknown-identity listing (fabgpu_block_unknown_identities) in the device
block validator -- a peer loop with three blocks in flight that lists each finished block's unknown identities and admits them, held to
the sequence oracle; principal bits, de-duplication groups and invalid identities; growth with the small tier on and off and a
window-pool recycle; every refusal; reconfiguration; two contexts of one table group; and a context that never admits."""
import copy
import ctypes
import os

import numpy as np
import pytest

from tools import blockgen
from util import pkg
import identity_oracle as io
import v13_oracle

pytestmark = pytest.mark.gpu

CAP = 3


def _ids(idents):
    return [(i.serialized, i.mspid, i.xy, i.valid) for i in idents]


def _block(net, creators, seed, faults=None, endorsers=None):
    """a block whose transaction t is created by creators[t]"""
    n2 = copy.copy(net)
    n2.clients = list(creators)
    return blockgen.build_block(n2, len(creators), CAP, faults or {}, seed=seed, endorsers=endorsers)


def _submit(ctx, slot, info):
    ctx.validate_envelopes_async(slot, info["env_blob"], info["env_off"])


def _oracle(net, blk, everyone, known, policies=None):
    return io.flags(blk, _ids(everyone), known, net.channel, net.policy_n_of(CAP), net.principals, policies=policies).tolist()


def _listed(ctx, slot, info, known):
    """the device's listing of the slot's finished block, checked against the listing oracle"""
    got = ctx.block_unknown_identities(slot)
    assert got == io.listing(io.envelopes(info), known)
    return got


@pytest.mark.parametrize("cap", ["v20", "v13"])
def test_peer_loop_three_in_flight(cap):
    """4 orgs, 300 clients, 50 of them configured; 20 blocks of 500 transactions, about a tenth of each block's creators new.  Each
    iteration submits block k+2, waits for k, lists and admits what the list returned.  Every block's flags are the sequence oracle's
    in the channel's validator mode (V2_0, or V1_3 with the chaincode's lscc version): blocks in flight when an identity was admitted
    keep their 254s."""
    P = pkg().binding
    v13 = cap == "v13"
    pol, ver = {blockgen.CHAINCODE: 0}, {blockgen.CHAINCODE: "1.0"}
    net = blockgen.Network(n_orgs=4, n_clients=300, seed=0xAD17)
    configured = net.peers + net.clients[:50] + [net.invalid_cert] + net.peers_alt
    by_ser = {i.serialized: i for i in net.peers + net.clients + [net.invalid_cert] + net.peers_alt + [net.unknown]}
    ctx = P.Context(max_batch=8192)
    ctx.msp_configure(_ids(configured), net.policy_n_of(CAP), net.principals, net.channel, policies=pol if v13 else None)
    if v13:
        ctx.namespace_versions(ver)
        ctx.channel_capability(P.CAP_V1_3)
    known = {i.serialized for i in configured}
    rng = np.random.default_rng(5)
    fresh = list(net.clients[50:])
    blocks, known_at, seen = [], [], list(net.clients[:50])
    for k in range(20):
        creators = [seen[int(rng.integers(len(seen)))] for _ in range(500)]
        for t in rng.choice(500, 50, replace=False):
            if fresh:
                creators[int(t)] = fresh.pop(0)
        seen += [c for c in creators if c not in seen]
        faults = {int(t): "unknown_endorser" for t in rng.choice(500, 5, replace=False)}
        blocks.append(_block(net, creators, seed=100 + k, faults=faults))
    everyone = list(by_ser.values())
    slot = lambda j: j % 3
    for j in range(2):
        known_at.append(set(known)); _submit(ctx, slot(j), blocks[j][1])
    admitted = []
    for k in range(20):
        if k + 2 < 20:
            known_at.append(set(known)); _submit(ctx, slot(k + 2), blocks[k + 2][1])
        flags = ctx.validate_wait(slot(k), 600).tolist()
        blk, info = blocks[k]
        if v13:
            exp = v13_oracle.validate_block(blk, _ids(everyone), net.channel, net.policy_n_of(CAP), net.principals, policies=pol, versions=ver,
                                            known=list(known_at[k])).tolist()
        else:
            exp = _oracle(net, blk, everyone, known_at[k])
        assert flags == exp, "block %d" % k
        assert exp.count(0) > 100                       # the oracle decides a good part of each block in either mode
        listed = _listed(ctx, slot(k), info, known_at[k])
        new = [by_ser[s] for s, _ in listed if s not in known]
        if new:
            # group ids over the whole table in its order (configured, then admitted), so that earlier ids stay what they were
            ctx.msp_identities_add(_ids(new), groups=P.identity_groups(_ids(configured + admitted + new))[-len(new):])
            admitted += new
            known |= {i.serialized for i in new}
    assert len(admitted) > 200
    ctx.close()


def _base(P, net, configured, bits=None):
    ctx = P.Context(max_batch=8192)
    ctx.msp_configure(_ids(configured), net.policy_n_of(CAP), net.principals, net.channel)
    if bits is not None:
        ctx.msp_principal_bits(bits)
    return ctx


def _member_bits(net, idents):
    """principal bits that restate MSP-id member matching"""
    return np.array([[i.mspid == p and i.valid for p in net.principals] for i in idents], bool).reshape(len(idents), len(net.principals))


def test_admitted_endorser_satisfies_its_principal_with_bits():
    """Principal bits installed: an admitted peer endorser satisfies OrgN.peer; admitted with no bits it satisfies nothing."""
    P = pkg().binding
    net = blockgen.Network(n_orgs=4, n_clients=4, seed=0xB175)
    configured = net.peers + net.clients
    everyone = configured + [net.unknown]
    faults = {t: "unknown_endorser" for t in range(0, 40, 2)}
    blk, info = _block(net, net.clients * 10, seed=3, faults=faults)
    known = {i.serialized for i in configured}
    for good in (True, False):
        ctx = _base(P, net, configured, _member_bits(net, configured))
        _submit(ctx, 0, info)
        before = ctx.validate_wait(0, 64).tolist()
        assert before == _oracle(net, blk, everyone, known)
        assert ctx.block_unknown_identities(0) == [(net.unknown.serialized, 0)]
        bits = _member_bits(net, [net.unknown]) if good else np.zeros((1, len(net.principals)), bool)
        ctx.msp_identities_add(_ids([net.unknown]), groups=[len(configured) + 7], bits=bits)
        _submit(ctx, 1, info)
        after = ctx.validate_wait(1, 64).tolist()
        exp = _oracle(net, blk, everyone, known | {net.unknown.serialized})
        if good:
            assert after == exp and after != before
        else:
            assert all(a == (10 if e == 0 and t in faults else e) for t, (a, e) in enumerate(zip(after, exp)))
            assert any(after[t] == 10 for t in faults)
        ctx.close()


def test_admitted_reserialisation_joins_its_group():
    """An admitted second serialization of a configured peer, in that peer's group, is de-duplicated as the oracle says."""
    P = pkg().binding
    net = blockgen.Network(n_orgs=4, n_clients=2, seed=0x6209)
    configured = net.peers + net.clients
    faults = {t: "same_cert_two_encodings" for t in range(40)}
    blk, info = _block(net, net.clients * 20, seed=8, faults=faults)
    ctx = _base(P, net, configured)
    groups = P.identity_groups(_ids(configured + net.peers_alt))
    _submit(ctx, 0, info)
    ctx.validate_wait(0, 64)
    listed = ctx.block_unknown_identities(0)
    assert {s for s, _ in listed} <= {i.serialized for i in net.peers_alt} and listed
    ctx.msp_identities_add(_ids(net.peers_alt), groups=groups[len(configured):])
    _submit(ctx, 1, info)
    got = ctx.validate_wait(1, 64).tolist()
    assert got == _oracle(net, blk, configured + net.peers_alt, {i.serialized for i in configured + net.peers_alt})
    ctx.close()


def test_admitted_invalid_identity_is_a_bad_creator():
    P = pkg().binding
    net = blockgen.Network(n_orgs=4, n_clients=3, seed=0x1A7)
    configured = net.peers + net.clients[:1]
    revoked = blockgen.Identity(net.clients[2].mspid, net.clients[2].priv_index, net.clients[2].xy, net.clients[2].cert_pem, valid=False)
    blk, info = _block(net, [net.clients[0], revoked, net.clients[1]] * 4, seed=2)
    ctx = _base(P, net, configured)
    ctx.msp_identities_add(_ids([revoked, net.clients[1]]), groups=[100, 101])
    got = ctx.validate_block(blk).tolist()
    assert got == _oracle(net, blk, configured + [revoked, net.clients[1]], {i.serialized for i in configured + [revoked, net.clients[1]]})
    assert got[1] == 4 and got[0] == 0 and got[2] == 0
    ctx.close()


@pytest.mark.parametrize("small", [True, False], ids=["small_tier", "generic"])
def test_growth_with_blocks_in_flight(small):
    """5 000 identities in 50 calls with blocks in flight: later blocks decide them; with the small tier on each admitted key gets a
    small table, with it off they go through the generic kernel."""
    P = pkg().binding
    net = blockgen.Network(n_orgs=4, n_clients=5000, seed=0x5000)
    configured = net.peers + net.clients[:10]
    old = os.environ.get("FABGPU_SMALL_SLOTS")
    if not small:
        os.environ["FABGPU_SMALL_SLOTS"] = "0"
    try:
        ctx = _base(P, net, configured)
    finally:
        if old is None:
            os.environ.pop("FABGPU_SMALL_SLOTS", None)
        else:
            os.environ["FABGPU_SMALL_SLOTS"] = old
    small0 = ctx.key_table_stats()["small"]
    rng = np.random.default_rng(1)
    blk, info = _block(net, [net.clients[int(c)] for c in rng.integers(0, 5000, 400)], seed=6)
    known = {i.serialized for i in configured}
    everyone = net.peers + net.clients
    groups = P.identity_groups(_ids(configured + net.clients[10:]))
    for c in range(50):
        slot = c % 3
        if c >= 3:
            ctx.validate_wait(slot, 512)
        _submit(ctx, slot, info)
        batch = net.clients[10 + 100 * c:10 + 100 * (c + 1)]
        lo = len(configured) + 100 * c
        ctx.msp_identities_add(_ids(batch), groups=groups[lo:lo + len(batch)])
    for slot in range(3):
        ctx.validate_wait(slot, 512)
    known |= {i.serialized for i in net.clients}
    _submit(ctx, 0, info)
    assert ctx.validate_wait(0, 512).tolist() == _oracle(net, blk, everyone, known)
    assert ctx.block_unknown_identities(0) == []
    grown = ctx.key_table_stats()["small"] - small0
    assert (grown >= 4990) if small else grown == 0
    ctx.close()


def test_window_pool_recycle_reissues_each_tier():
    """An MSP that fits the window pool, plus admitted clients: after the pool recycles the peers' window tables, the next submit
    re-issues the peers window tables and the clients small ones -- no small table is built for a peer."""
    P = pkg().binding
    old = os.environ.get("FABGPU_KEY_SLOTS")
    os.environ["FABGPU_KEY_SLOTS"] = "16"
    try:
        net = blockgen.Network(n_orgs=4, n_clients=40, seed=0x7EC1)
        ctx = _base(P, net, net.peers + net.clients[:4])
    finally:
        if old is None:
            os.environ.pop("FABGPU_KEY_SLOTS", None)
        else:
            os.environ["FABGPU_KEY_SLOTS"] = old
    assert ctx.key_slot_capacity() == 16
    ctx.msp_identities_add(_ids(net.clients[4:24]), groups=list(range(100, 120)))
    small = ctx.key_table_stats()["small"]
    other = np.frombuffer(b"".join(net.clients[k].xy for k in range(24, 40)), np.uint8).reshape(-1, 64)
    ctx.keys_register(other)                              # 16 other keys: every window table changes hands
    blk, info = _block(net, net.clients[:24], seed=12)
    got = ctx.validate_block(blk).tolist()
    assert got == _oracle(net, blk, net.peers + net.clients, {i.serialized for i in net.peers + net.clients[:24]})
    assert ctx.key_table_stats()["small"] == small
    ctx.close()


def test_refusals_change_nothing():
    """Every refusal is FABGPU_E_ARG and the next block's flags are unchanged."""
    P = pkg().binding
    L = P.lib()
    net = blockgen.Network(n_orgs=4, n_clients=3, seed=0x4EF)
    configured = net.peers + net.clients[:2]
    blk, info = _block(net, net.clients * 4, seed=1)
    fresh = P.Context(max_batch=1024)
    with pytest.raises(P.FabGpuError) as e:
        fresh.msp_identities_add(_ids([net.clients[2]]))   # no configured table
    assert e.value.code == P.E_ARG
    fresh.close()
    ctx = _base(P, net, configured)
    exp = ctx.validate_block(blk).tolist()
    c2 = net.clients[2]
    cases = [
        dict(identities=_ids([c2])),                                        # a group table is installed: groups required
        dict(identities=_ids([c2, c2]), groups=[1, 1]),                     # given twice
        dict(identities=_ids([c2, net.clients[0]]), groups=[1, 2]),         # held already
        dict(identities=_ids([c2]), groups=[-1]),                           # negative group
        dict(identities=_ids([c2]), groups=[1], bits=np.ones((1, 4), bool)),   # no bits installed
        dict(identities=[(b"", "Org1MSP", c2.xy, True)], groups=[1]),       # empty identity
    ]
    for kw in cases:
        with pytest.raises(P.FabGpuError) as e:
            ctx.msp_identities_add(**kw)
        assert e.value.code == P.E_ARG, kw
    blob = np.frombuffer(c2.serialized, np.uint8).copy()
    off = np.array([0, len(c2.serialized)], np.uint32)
    bad_off = np.array([len(c2.serialized), 0], np.uint32)
    mb = np.frombuffer(b"Org1MSP", np.uint8).copy(); mo = np.array([0, 7], np.uint32)
    keys = np.frombuffer(c2.xy, np.uint8).copy(); valid = np.ones(1, np.uint8); g = np.ones(1, np.int32)
    p = P._p
    for args in [(p(blob), p(off), p(mb), p(mo), p(keys), p(valid), p(g), None, -1),
                 (None, p(off), p(mb), p(mo), p(keys), p(valid), p(g), None, 1),
                 (p(blob), p(bad_off), p(mb), p(mo), p(keys), p(valid), p(g), None, 1)]:
        assert L.fabgpu_msp_identities_add(ctx._h, *args[:8], ctypes.c_int(args[8])) == P.E_ARG
    n = ctypes.c_size_t(0)
    assert L.fabgpu_block_unknown_identities(ctx._h, ctypes.c_int(2), None, ctypes.c_size_t(0), ctypes.byref(n)) == P.E_ARG   # no finished block
    assert L.fabgpu_block_unknown_identities(ctx._h, ctypes.c_int(0), None, ctypes.c_size_t(0), None) == P.E_ARG              # NULL count
    assert ctx.validate_block(blk).tolist() == exp
    assert [s for s, _ in ctx.block_unknown_identities(0)] == [c2.serialized]
    ctx.close()


def test_configure_after_adds_resets_the_table():
    P = pkg().binding
    net = blockgen.Network(n_orgs=4, n_clients=3, seed=0xC0F)
    configured = net.peers + net.clients[:1]
    blk, info = _block(net, net.clients * 4, seed=4)
    ctx = _base(P, net, configured)
    before = ctx.validate_block(blk).tolist()
    ctx.msp_identities_add(_ids(net.clients[1:]), groups=[50, 51])
    assert ctx.validate_block(blk).tolist() == _oracle(net, blk, net.peers + net.clients, {i.serialized for i in net.peers + net.clients})
    ctx.msp_configure(_ids(configured), net.policy_n_of(CAP), net.principals, net.channel)
    assert ctx.validate_block(blk).tolist() == before
    assert [s for s, _ in ctx.block_unknown_identities(0)] == [i.serialized for i in net.clients[1:]]
    ctx.close()


def test_shared_contexts_admit_independently():
    P = pkg().binding
    net = blockgen.Network(n_orgs=4, n_clients=4, seed=0x5A4E)
    configured = net.peers + net.clients[:1]
    blk, info = _block(net, net.clients * 4, seed=9)
    a = _base(P, net, configured)
    b = P.Context(max_batch=8192, share_tables_with=a)
    b.msp_configure(_ids(configured), net.policy_n_of(CAP), net.principals, net.channel)
    before = b.validate_block(blk).tolist()
    a.msp_identities_add(_ids(net.clients[1:]), groups=[60, 61, 62])
    assert a.validate_block(blk).tolist() == _oracle(net, blk, net.peers + net.clients, {i.serialized for i in net.peers + net.clients})
    assert b.validate_block(blk).tolist() == before == _oracle(net, blk, net.peers + net.clients, {i.serialized for i in configured})
    b.close()
    a.close()


# Launches of one block whose signers all own window tables, without key-level or v1.3 stages: block_walk_kernel, block_resolve_kernel
# and two sha256_segments_kernel for the creators, block_resolve_kernel and sha256_segments_kernel for the endorsements, the key-table
# verify path (ecdsa_prep_kernel + ecdsa_verify_cached_kernel), block_decide_kernel -- what the block path launched before admission.
BLOCK_LAUNCHES = 9


def test_a_context_that_never_admits_launches_as_before():
    """A context where admission is never touched launches BLOCK_LAUNCHES per block, block after block, with the oracle's flags; so does
    one that admitted an identity whose key owns a window table (the ordering adds waits and events, no launch).  (An admitted key in
    the small tier adds the small-table verify launch, as it would had it been configured.)"""
    P = pkg().binding
    net = blockgen.Network(n_orgs=4, n_clients=3, seed=0x9A9)
    configured = net.peers + net.clients
    blk, info = _block(net, net.clients * 10, seed=10)
    plain, admitting = _base(P, net, configured), _base(P, net, configured)
    admitting.msp_identities_add(_ids(net.peers_alt[:1]), groups=P.identity_groups(_ids(configured + net.peers_alt[:1]))[-1:])
    exp = _oracle(net, blk, configured, {i.serialized for i in configured})
    deltas = []
    for ctx in (plain, admitting):
        for _ in range(3):
            n0 = ctx.launch_count()
            assert ctx.validate_block(blk).tolist() == exp
            deltas.append(ctx.launch_count() - n0)
    assert deltas == [BLOCK_LAUNCHES] * 6, deltas
    plain.close()
    admitting.close()
