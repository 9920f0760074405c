"""GPU: role and identity principals (fabgpu_msp_principal_bits) and ImplicitMeta policy nodes in the device block validator, through
every entry point, against the policy oracle, the host build and codes written out per case; and the configurations
fabgpu_msp_configure / fabgpu_msp_principal_bits refuse."""
import random

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from util import pkg
import blockutil
import nodeou
import policy_oracle
import policyutil

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    yield c
    c.close()


def _configure(ctx, ids, nodes, names, channel, bits, pol=None):
    ctx.msp_configure(ids, nodes, names, channel, policies=pol)
    if bits is not None:
        ctx.msp_principal_bits(bits)


@pytest.mark.parametrize("case", nodeou.policy_cases(), ids=lambda c: c[0])
def test_policy_case_on_device(ctx, case):
    net, blk, info, nodes, names, bits, pol, expected = nodeou.materialize(case)
    _configure(ctx, net.identities(), nodes, names, net.channel, bits, pol)
    assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == expected
    assert ctx.validate_block(blk).tolist() == expected


def _stock_block(net, n_tx, seed):
    """n_tx transactions whose endorser sets cycle through majorities, minorities, duplicates, second encodings and non-peers."""
    P, n = net.org_peers, net.n_orgs
    rnd = random.Random(seed)

    def ends(t):
        k = rnd.randrange(1, n + 1)
        orgs = rnd.sample(range(n), k)
        kind = t % 5
        if kind == 0:
            return [P[o][rnd.randrange(2)] for o in orgs]
        if kind == 1:
            return [P[o][0] for o in orgs] + [P[orgs[0]][0]]
        if kind == 2:
            return [net.peers_alt[o] for o in orgs] + [net.peers[orgs[0]]]
        if kind == 3:
            return [rnd.choice([net.clients[o], net.admins[o], net.orderers[o], net.admins_listed[o]]) for o in orgs]
        return [P[o][0] for o in orgs[:-1]] + [net.clients[orgs[-1]]]
    return blockgen.build_block(net, n_tx, 3, {}, seed=seed, endorsers=ends)


def test_stock_policy_every_entry_point(ctx):
    """The stock MAJORITY-of-peer policy with bits through validate_envelopes, validate_block, a pinned buffer and two async slots."""
    net = nodeou.network(4)
    ids = net.identities()
    pr, tree = nodeou.stock_endorsement(4)
    nodes, _ = nodeou.forest([tree])
    names = [nodeou.principal_name(p) for p in pr]
    bits = nodeou.principal_bits(net, pr)
    blocks = []
    for seed, n_tx in ((71, 700), (72, 333)):
        blk, info = _stock_block(net, n_tx, seed)
        exp = policy_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, known=[i[0] for i in ids])
        host = policyutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, names, principal_bits=bits)
        assert host.tolist() == exp.tolist()
        assert 0.2 < float((exp == ob.VALID).mean()) < 0.8 and set(exp.tolist()) == {ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE}
        blocks.append((blk, info, exp))
    _configure(ctx, ids, nodes, names, net.channel, bits)
    for k, (blk, info, exp) in enumerate(blocks):
        assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp.tolist()
        assert ctx.validate_block(blk).tolist() == exp.tolist()
        pinned = ctx.block_buffer(len(blk), slot=k)
        pinned[:] = np.frombuffer(blk, np.uint8)
        assert ctx.validate_block(pinned).tolist() == exp.tolist()
    for rnd_i in range(2):
        (b0, i0, e0), (b1, i1, e1) = blocks
        n0 = ctx.validate_envelopes_async(0, i0["env_blob"], i0["env_off"])
        n1 = ctx.validate_block_async(1, b1)
        assert ctx.validate_wait(1, n1).tolist() == e1.tolist()
        assert ctx.validate_wait(0, n0).tolist() == e0.tolist()


def test_small_tier_msp_with_bits():
    """An MSP of a few hundred identities, more than the window-table pool holds (small tables), with bits installed."""
    c = pkg().binding.Context(max_batch=8192)
    try:
        net = nodeou.NodeOUNetwork(n_orgs=4, clients_per_org=80, seed=0x5A11)
        ids = net.identities()
        assert len(ids) > c.key_slot_capacity()
        pr, tree = nodeou.stock_endorsement(4)
        nodes, _ = nodeou.forest([tree])
        names = [nodeou.principal_name(p) for p in pr]
        bits = nodeou.principal_bits(net, pr)
        blk, info = _stock_block(net, 600, 73)
        exp = policy_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, known=[i[0] for i in ids])
        assert set(exp.tolist()) == {ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE}
        _configure(c, ids, nodes, names, net.channel, bits)
        assert c.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp.tolist()
        assert c.validate_block(blk).tolist() == exp.tolist()
    finally:
        c.close()


def test_wire_mutation_corpus_stock_policy_with_bits(ctx):
    """The wire-mutation corpus under the stock policy with bits: the device equals the policy oracle and the host build."""
    import wiremut
    net, ids, _, pol, blocks = wiremut.corpus()
    pr, tree = nodeou.stock_endorsement(4)
    nodes, _ = nodeou.forest([tree])
    bits = nodeou.member_roles_for(net, pr)
    names = [nodeou.principal_name(p) for p in pr]
    roots = {ns: 0 for ns in pol}
    _configure(ctx, ids, nodes, names, net.channel, bits, roots)
    exps = []
    for k, (blk, info, _, _) in enumerate(blocks):
        exp = policy_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=roots, known=[i[0] for i in ids])
        exps.append(exp)
        assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp.tolist(), k
        assert ctx.validate_block(blk).tolist() == exp.tolist(), k
    for (b0, i0, _, _), e0, (b1, _, _, _), e1 in zip(blocks[0::2], exps[0::2], blocks[1::2], exps[1::2]):
        n0 = ctx.validate_envelopes_async(0, i0["env_blob"], i0["env_off"])
        n1 = ctx.validate_block_async(1, b1)
        assert ctx.validate_wait(1, n1).tolist() == e1.tolist()
        assert ctx.validate_wait(0, n0).tolist() == e0.tolist()


def _contrast_setup():
    """A client of Org1 endorsing under principal 0; member matching accepts it, the bits of 'Org1MSP.peer' do not."""
    net = nodeou.network(4)
    blk, info = blockgen.build_block(net, 3, 3, {}, seed=5, endorsers=lambda t: [net.clients[0]])
    nodes, _ = nodeou.forest([nodeou.n_of(1, [nodeou.signed_by(0)])])
    bits = nodeou.principal_bits(net, [nodeou.role("Org1MSP", "peer")])
    return net, blk, nodes, bits


def test_refusals_keep_the_previous_configuration(ctx):
    """ImplicitMeta below NOutOf, a threshold NewImplicitMetaPolicy cannot produce, node types 3 and -1, and bits of the wrong shape:
    FABGPU_E_ARG with a message, and the configuration installed before keeps deciding."""
    binding = pkg().binding
    net, blk, nodes, bits = _contrast_setup()
    ids = net.identities()
    _configure(ctx, ids, nodes, ["Org1MSP"], net.channel, bits)
    assert ctx.validate_block(blk).tolist() == [10, 10, 10]
    S, NOF, IM = 1, 0, 2
    refused = [np.array([(NOF, 1, 1, 1), (IM, 1, 2, 1), (S, 0, 0, 0)], np.int32),          # ImplicitMeta under NOutOf
               np.array([(IM, 2, 1, 1), (S, 0, 0, 0)], np.int32),                           # threshold above the children
               np.array([(IM, 0, 1, 1), (S, 0, 0, 0)], np.int32),                           # threshold 0 with a child
               np.array([(IM, -1, 0, 0)], np.int32),                                        # negative threshold
               np.array([(IM, 1, 0, 0)], np.int32),                                         # threshold 1 over nothing
               np.array([(3, 0, 0, 0)], np.int32), np.array([(-1, 0, 0, 0)], np.int32),
               np.array([(NOF, 1, 1, 1), (3, 0, 0, 0)], np.int32),
               np.array([(IM, 1, 1, 1), (IM, 1, 0, 1)], np.int32)]                          # a cycle through ImplicitMeta
    for bad in refused:
        with pytest.raises(binding.FabGpuError) as e:
            ctx.msp_configure(ids, bad, ["Org1MSP"], net.channel)
        assert e.value.code == binding.E_ARG, bad.tolist()
        assert binding.lib().fabgpu_last_error(ctx._h), bad.tolist()
        assert ctx.validate_block(blk).tolist() == [10, 10, 10], bad.tolist()
    for shape in ((len(ids) - 1, 1), (len(ids) + 1, 1), (len(ids), 2), (len(ids), 33)):
        with pytest.raises(binding.FabGpuError) as e:
            ctx.msp_principal_bits(np.ones(shape, bool))
        assert e.value.code == binding.E_ARG, shape
        assert ctx.validate_block(blk).tolist() == [10, 10, 10], shape
    # ImplicitMeta below ImplicitMeta, at the root of a namespace, and depth counted through it: accepted
    ok = nodeou.forest([nodeou.implicit_meta("ANY", [nodeou.implicit_meta("ALL", [nodeou.n_of(1, [nodeou.signed_by(0)])])])])[0]
    _configure(ctx, ids, ok, ["Org1MSP"], net.channel, None)
    assert ctx.validate_block(blk).tolist() == [0, 0, 0]
    chain = lambda depth: np.array([(IM, 1, i + 1, 1) for i in range(depth)] + [(S, 0, 0, 0)], np.int32)
    with pytest.raises(binding.FabGpuError) as e:
        ctx.msp_configure(ids, chain(13), ["Org1MSP"], net.channel)
    assert e.value.code == binding.E_ARG
    _configure(ctx, ids, chain(12), ["Org1MSP"], net.channel, None)
    assert ctx.validate_block(blk).tolist() == [0, 0, 0]


def test_bits_lifecycle(ctx):
    """Member matching, then bits, then fabgpu_msp_configure again (member matching is back), then bits removed with n_ids = 0."""
    net, blk, nodes, bits = _contrast_setup()
    ids = net.identities()
    _configure(ctx, ids, nodes, ["Org1MSP"], net.channel, None)
    assert ctx.validate_block(blk).tolist() == [0, 0, 0]
    ctx.msp_principal_bits(bits)
    assert ctx.validate_block(blk).tolist() == [10, 10, 10]
    ctx.msp_configure(ids, nodes, ["Org1MSP"], net.channel)
    assert ctx.validate_block(blk).tolist() == [0, 0, 0]
    ctx.msp_principal_bits(bits)
    assert ctx.validate_block(blk).tolist() == [10, 10, 10]
    ctx.msp_principal_bits(None)
    assert ctx.validate_block(blk).tolist() == [0, 0, 0]
