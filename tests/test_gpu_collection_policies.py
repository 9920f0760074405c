"""GPU: private-data collection endorsement policies (fabgpu_collection_policies) in the device block validator, through
validate_envelopes, validate_block and two async slots, against the collection oracle, the host build and codes written out per case;
the table's lifecycle; and the tables fabgpu_collection_policies refuses."""
import ctypes

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from util import pkg
import collcases
import collection_oracle
import collutil

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    yield c
    c.close()


def _configure(ctx, ids, names, channel, bits, table):
    ctx.msp_configure(ids, collcases.forest()[0], names, channel, policies=collcases.namespace_policies())
    if bits is not None:
        ctx.msp_principal_bits(bits)
    ctx.collection_policies(table)


@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
def test_collection_cases_on_device(ctx, use_bits):
    """Every case, with the table and without it, through validate_envelopes and validate_block, and the cases' blocks in pairs on two
    async slots; the host build and the oracle give the same codes."""
    names, bits = collcases.principals(use_bits)
    mats = [collcases.materialize(c) for c in collcases.cases()]
    net = mats[0][0]
    ids = net.identities()
    nodes, table = collcases.forest()[0], collcases.collection_table()
    for tab, col in ((table, 3), (None, 4)):
        _configure(ctx, ids, names, net.channel, bits, tab)
        for case, m in zip(collcases.cases(), mats):
            _, blk, info = m[:3]
            exp = m[col]
            assert collection_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=collcases.namespace_policies(),
                                                    collections=tab, known=[i[0] for i in ids]).tolist() == exp, case[0]
            assert collutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, names,
                                               policies=collcases.namespace_policies(), principal_bits=bits, collections=tab).tolist() == exp, case[0]
            assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp, case[0]
            assert ctx.validate_block(blk).tolist() == exp, case[0]
        for a, b in zip(mats[0::2], mats[1::2]):
            n0 = ctx.validate_envelopes_async(0, a[2]["env_blob"], a[2]["env_off"])
            n1 = ctx.validate_block_async(1, b[1])
            assert ctx.validate_wait(1, n1).tolist() == b[col]
            assert ctx.validate_wait(0, n0).tolist() == a[col]


def _lifecycle_block():
    case = [c for c in collcases.cases() if c[0] == "lifecycle_approval"][0]
    return collcases.materialize(case)


def test_table_lifecycle(ctx):
    """Install, remove with n = 0, install again; fabgpu_msp_configure clears the table; the flags follow."""
    net, blk, info, with_table, without = _lifecycle_block()
    names, bits = collcases.principals(True)
    ids = net.identities()
    assert with_table != without
    _configure(ctx, ids, names, net.channel, bits, None)
    assert ctx.validate_block(blk).tolist() == without
    ctx.collection_policies(collcases.collection_table())
    assert ctx.validate_block(blk).tolist() == with_table
    ctx.collection_policies({})
    assert ctx.validate_block(blk).tolist() == without
    ctx.collection_policies(collcases.collection_table())
    assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == with_table
    ctx.msp_configure(ids, collcases.forest()[0], names, net.channel, policies=collcases.namespace_policies())
    ctx.msp_principal_bits(bits)
    assert ctx.validate_block(blk).tolist() == without
    ctx.collection_policies(collcases.collection_table())
    assert ctx.validate_block(blk).tolist() == with_table
    ctx.collection_policies(None)
    assert ctx.validate_block(blk).tolist() == without


def _raw(ctx, pairs, roots, null=None):
    """fabgpu_collection_policies on exactly these (namespace, collection) pairs (the binding would sort and de-duplicate them);
    null names one array to pass as NULL."""
    b = pkg().binding
    nb, no = b._blob([n.encode() for n, _ in pairs])
    cb, co = b._blob([c.encode() for _, c in pairs])
    r = np.array(roots or [0], np.int32)
    args = {"ns_blob": nb, "ns_off": no, "coll_blob": cb, "coll_off": co, "coll_root": r}
    ptr = [None if k == null else b._p(a) for k, a in args.items()]
    return b.lib().fabgpu_collection_policies(ctx._h, *ptr, ctypes.c_int(len(pairs)))


def test_refusals_keep_the_previous_table(ctx):
    """NULL arrays with n > 0, a root outside [0, n_nodes), an empty collection name, decreasing offsets and a duplicate pair:
    FABGPU_E_ARG with a message, and the table installed before keeps deciding."""
    binding = pkg().binding
    net, blk, info, with_table, without = _lifecycle_block()
    names, bits = collcases.principals(True)
    ids = net.identities()
    _configure(ctx, ids, names, net.channel, bits, collcases.collection_table())
    assert ctx.validate_block(blk).tolist() == with_table
    n_nodes = collcases.forest()[0].shape[0]
    org1 = collcases.forest()[1]["org1"]
    refused = [dict(pairs=[("mycc", "a")], roots=[0], null=k) for k in ("ns_blob", "ns_off", "coll_blob", "coll_off", "coll_root")]
    refused += [dict(pairs=[("mycc", "a")], roots=[-1]), dict(pairs=[("mycc", "a")], roots=[n_nodes]),
                dict(pairs=[("mycc", "a"), ("mycc", "")], roots=[0, 0]),
                dict(pairs=[("_lifecycle", "_implicit_org_Org1MSP"), ("mycc", "b"), ("_lifecycle", "_implicit_org_Org1MSP")], roots=[org1, 0, org1])]
    for bad in refused:
        assert _raw(ctx, **bad) == binding.E_ARG, bad
        assert binding.lib().fabgpu_last_error(ctx._h), bad
        assert ctx.validate_block(blk).tolist() == with_table, bad
    # decreasing offsets
    nb, no = binding._blob([b"_lifecycle", b"mycc"])
    cb, co = binding._blob([b"x", b"y"])
    no = np.array([0, 10, 4], np.uint32)
    r = np.zeros(2, np.int32)
    assert binding.lib().fabgpu_collection_policies(ctx._h, binding._p(nb), binding._p(no), binding._p(cb), binding._p(co),
                                                    binding._p(r), ctypes.c_int(2)) == binding.E_ARG
    assert ctx.validate_block(blk).tolist() == with_table
    # the same collection under two namespaces and two collections of one namespace are no duplicates
    assert _raw(ctx, [("_lifecycle", "_implicit_org_Org1MSP"), ("mycc", "_implicit_org_Org1MSP"), ("_lifecycle", "_implicit_org_Org2MSP")],
                [org1, 0, 0]) == binding.OK
    assert ctx.validate_block(blk).tolist() == with_table
    assert _raw(ctx, [], []) == binding.OK
    assert ctx.validate_block(blk).tolist() == without


def test_wire_mutation_corpus_with_a_stricter_collection_policy(ctx):
    """The wire-mutation corpus with 'collection' under the STRICT_NAMESPACE tree: device, host build and collection oracle agree on every
    transaction, through both entry points and two async slots."""
    import wiremut
    net, ids, nodes, pol, blocks = wiremut.corpus()
    table = {(blockgen.CHAINCODE, "collection"): pol[blockgen.STRICT_NAMESPACE]}
    ctx.msp_configure(ids, nodes, net.principals, net.channel, policies=pol)
    ctx.collection_policies(table)
    exps = []
    for k, (blk, info, _, before) in enumerate(blocks):
        exp = collection_oracle.validate_block(blk, ids, net.channel, nodes, net.principals, policies=pol, collections=table,
                                               known=[i[0] for i in ids])
        exps.append(exp)
        host = collutil.device_logic_flags(info["env_blob"], info["env_off"], ids, net.channel, nodes, net.principals, policies=pol,
                                           collections=table)
        assert host.tolist() == exp.tolist(), k
        assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp.tolist(), k
        assert ctx.validate_block(blk).tolist() == exp.tolist(), k
    assert sum(int(((b[3] == ob.VALID) & (e == ob.ENDORSEMENT_POLICY_FAILURE)).sum()) for b, e in zip(blocks, exps)) >= 10
    for (b0, i0, _, _), e0, (b1, _, _, _), e1 in zip(blocks[0::2], exps[0::2], blocks[1::2], exps[1::2]):
        n0 = ctx.validate_envelopes_async(0, i0["env_blob"], i0["env_off"])
        n1 = ctx.validate_block_async(1, b1)
        assert ctx.validate_wait(1, n1).tolist() == e1.tolist()
        assert ctx.validate_wait(0, n0).tolist() == e0.tolist()
    ctx.collection_policies(None)
    for blk, _, _, before in blocks[:2]:
        assert ctx.validate_block(blk).tolist() == before.tolist()
