"""GPU: key-level endorsement policies (fabgpu_key_policies / _update) in the device block validator, through validate_envelopes,
validate_block and two async slots, against the key-level oracle, the host build and codes written out per case; write-record overflow
and the growth after it; the table's lifecycle; the calls the library refuses; and seeded blocks with dependency chains."""
import numpy as np
import pytest

from oracle import blockval as ob
from util import pkg
import collcases
import keylevel_oracle
import klcases
import klutil
import nodeou

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    _grown(c)                                  # sized for the 17-write transactions of more_than_16_roots
    yield c
    c.close()


def _configure(ctx, ids, names, channel, bits, colls=None):
    ctx.msp_configure(ids, collcases.forest()[0], names, channel, policies=collcases.namespace_policies())
    if bits is not None:
        ctx.msp_principal_bits(bits)
    ctx.collection_policies(colls)


def _case(name):
    return [c for c in klcases.cases() if c[0] == name][0]


def _grown(c):
    """c after a block with 17 writes per transaction: the write records are sized for every block below"""
    case = _case("more_than_16_roots")
    net, blk, info, codes = klcases.materialize(case)
    names, bits = collcases.principals(True)
    _configure(c, net.identities(), names, net.channel, bits)
    kn, table = klcases.key_table(case)
    c.key_policies(kn, table)
    first = c.validate_block(blk).tolist()
    assert c.validate_block(blk).tolist() == codes
    return first, codes


def test_write_record_overflow_then_growth():
    """On a context of its own (the record sizing only grows): a block with more writes than T x 8 records is 254 at the policy stage;
    the library then sizes the records for it, and the same block gets the written codes."""
    c = pkg().binding.Context(max_batch=8192)
    try:
        first, codes = _grown(c)
        assert first == [ob.NOT_VALIDATED] * 3 and codes != first
    finally:
        c.close()


def test_collection_cases_and_wire_corpus_with_a_key_table():
    """collcases (with their collection table and role principals) and the wire-mutation corpus (MSP-id principals), each with a key
    table on their keys, through validate_block and validate_envelopes: every flag is the key-level oracle's."""
    import wiremut
    import test_key_policies
    c = pkg().binding.Context(max_batch=8192)
    try:
        _grown(c)
        kn, r = klcases.vp_forest()
        table = test_key_policies.corpus_key_table(kn, r)
        names, bits = collcases.principals(True)
        nodes, vps = klcases.combined(kn, table)
        for case in collcases.cases():
            net, blk, info, _, _ = collcases.materialize(case)
            ids = net.identities()
            _configure(c, ids, names, net.channel, bits, collcases.collection_table())
            c.key_policies(kn, table)
            exp = keylevel_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=collcases.namespace_policies(),
                                                 collections=collcases.collection_table(), vps=vps, known=[i[0] for i in ids]).tolist()
            assert c.validate_block(blk).tolist() == exp, case[0]
            assert c.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp, case[0]
        net, ids, wnodes, pol, blocks = wiremut.corpus()
        c.msp_configure(ids, wnodes, net.principals, net.channel, policies=pol)
        c.key_policies(kn, table)
        knn = np.array(kn, np.int32).copy()
        knn[knn[:, 0] == 0, 2] += wnodes.shape[0]
        all_nodes = np.concatenate([np.asarray(wnodes, np.int32).reshape(-1, 4), knn])
        wvps = {k: (v + wnodes.shape[0] if v >= 0 else v) for k, v in table.items()}
        n = 0
        for blk, info, _, _ in blocks:
            exp = keylevel_oracle.validate_block(blk, ids, net.channel, all_nodes, net.principals, policies=pol, vps=wvps,
                                                 known=[i[0] for i in ids]).tolist()
            assert c.validate_block(blk).tolist() == exp
            assert c.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp
            n += len(exp)
        assert n > 1000
    finally:
        c.close()


@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
def test_key_policy_cases_on_device(ctx, use_bits):
    """Every case through validate_envelopes and validate_block, and the cases' blocks in pairs on two async slots; the host build and
    the oracle give the same codes."""
    names, bits = collcases.principals(use_bits)
    mats = [(c,) + klcases.materialize(c) for c in klcases.cases()]
    ids = mats[0][1].identities()
    channel = mats[0][1].channel
    for case, net, blk, info, codes in mats:
        colls = collcases.collection_table() if case[1] else None
        _configure(ctx, ids, names, channel, bits, colls)
        kn, table = klcases.key_table(case)
        ctx.key_policies(kn, table)
        nodes, vps = klcases.combined(kn, table)
        assert keylevel_oracle.validate_block(blk, ids, channel, nodes, names, bits=bits, policies=collcases.namespace_policies(),
                                              collections=colls, vps=vps, known=[i[0] for i in ids]).tolist() == codes, case[0]
        assert klutil.device_logic_flags(info["env_blob"], info["env_off"], ids, channel, collcases.forest()[0], names,
                                         policies=collcases.namespace_policies(), principal_bits=bits, collections=colls,
                                         key_calls=[(True, kn, table)], writes_hint=32).tolist() == codes, case[0]
        assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == codes, case[0]
        assert ctx.validate_block(blk).tolist() == codes, case[0]
    # two slots at once: cases without a collection table, under one key table holding every such case's keys
    _configure(ctx, ids, names, channel, bits)
    kn, r = klcases.vp_forest()
    merged = {}
    plain = [m for m in mats if not m[0][1]]
    for m in plain:
        merged.update(klcases.key_table(m[0])[1])
    ctx.key_policies(kn, merged)
    for a, b in zip(plain[0::2], plain[1::2]):
        n0 = ctx.validate_envelopes_async(0, a[3]["env_blob"], a[3]["env_off"])
        n1 = ctx.validate_block_async(1, b[2])
        assert ctx.validate_wait(1, n1).tolist() == b[4], b[0][0]
        assert ctx.validate_wait(0, n0).tolist() == a[4], a[0][0]


def test_table_lifecycle(ctx):
    """Install, update, remove an entry, mark it -2, remove the table; fabgpu_msp_configure clears it; the flags follow."""
    case = ("lifecycle", False, {}, [([0], [klcases.pub("b")], None, None), ([1], [klcases.pub("b")], None, None),
                                      ([0, 1], [klcases.pub("b")], None, None)])
    net, blk, info, _ = klcases.materialize(case)
    names, bits = collcases.principals(True)
    ids = net.identities()
    kn, r = klcases.vp_forest()
    b = (klcases.CC, "", b"b")
    V, F, NV = ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.NOT_VALIDATED
    _configure(ctx, ids, names, net.channel, bits)
    plain = ctx.validate_block(blk).tolist()
    assert plain == [F, F, V]
    ctx.key_policies(kn, {b: r["vp_org1"]})
    assert ctx.validate_block(blk).tolist() == [V, F, V]
    ctx.key_policies_update(kn, {b: r["vp_org2"]})
    assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == [F, V, V]
    ctx.key_policies_update([], {b: -1, (klcases.CC, "", b"absent"): -1})
    assert ctx.validate_block(blk).tolist() == plain
    ctx.key_policies_update([], {b: -2})
    assert ctx.validate_block(blk).tolist() == [NV] * 3
    ctx.key_policies([], {})
    assert ctx.validate_block(blk).tolist() == plain
    ctx.key_policies(kn, {b: r["vp_org1"]})
    ctx.msp_configure(ids, collcases.forest()[0], names, net.channel, policies=collcases.namespace_policies())
    ctx.msp_principal_bits(bits)
    assert ctx.validate_block(blk).tolist() == plain
    with pytest.raises(pkg().binding.FabGpuError):
        ctx.key_policies_update(kn, {b: r["vp_org1"]})                   # cleared: nothing to update


def test_refusals_keep_the_previous_table(ctx):
    """Every argument the library refuses: FABGPU_E_ARG with a message, and the installed table still decides."""
    from test_key_policies import REFUSALS, refusal_args
    case = _case("vp_looser")
    net, blk, info, codes = klcases.materialize(case)
    names, bits = collcases.principals(True)
    _configure(ctx, net.identities(), names, net.channel, bits)
    kn, table = klcases.key_table(case)
    ctx.key_policies(kn, table)
    B = pkg().binding
    for what, text in REFUSALS + [("below -2", "root out of range")]:
        if what in ("decreasing offsets", "duplicate"):
            nd, n_nodes, nb, no, cb, co, kb, ko, roots, n = klutil.key_table_args([(1, 0, 0, 0)], {("cc", "", b"a"): 0, ("cc", "", b"b"): 0})
            if what == "decreasing offsets":
                ko = ko.copy(); ko[1] = 5; ko[2] = 2
            else:
                kb = kb.copy(); kb[1] = kb[0]
            import ctypes
            rc = B.lib().fabgpu_key_policies(ctx._h, B._p(nd), ctypes.c_int(n_nodes), B._p(nb), B._p(no), B._p(cb), B._p(co), B._p(kb), B._p(ko),
                                             B._p(roots), ctypes.c_int(n))
            assert rc != 0 and text.encode() in B.lib().fabgpu_last_error(ctx._h), what
        else:
            replace, nodes, tab = refusal_args(what)
            with pytest.raises(B.FabGpuError):
                (ctx.key_policies if replace else ctx.key_policies_update)(nodes, tab)
        assert ctx.validate_block(blk).tolist() == codes, what


def _seeded(seed, n_tx=10000, n_keys=400):
    """A block of n_tx transactions over a pool of keys, endorsed by random org subsets, with dependencies built in: 1 % of the
    transactions metadata-write a random pool key, every 25th starts a chain (it and the next three write and metadata-write one chain
    key), and 2 % write and metadata-write one hot key.  A 10^5-entry table with VPs on half the pool and on the hot key."""
    rng = np.random.default_rng(seed)
    net = nodeou.network(4)
    pool = ["k%d" % i for i in range(n_keys)]
    txs = []
    for t in range(n_tx):
        ks = list(rng.choice(pool, size=int(rng.integers(1, 4)), replace=False))
        md = [str(rng.choice(pool))] if rng.random() < 0.01 else []
        if t % 25 < 4:
            ks.append("chain%d" % (t // 25)); md.append("chain%d" % (t // 25))
        if rng.random() < 0.02:
            ks.append("hot"); md.append("hot")
        orgs = sorted(set(rng.choice(4, size=int(rng.integers(1, 4)), replace=True).tolist()))
        txs.append((orgs, [klcases.pub(*ks, md=md)]))
    from tools import blockgen
    blk, info = blockgen.build_block(net, n_tx, 3, {}, seed=seed, endorsers=lambda t: [net.org_peers[o][0] for o in txs[t][0]],
                                     namespaces=lambda t: txs[t][1])
    kn, r = klcases.vp_forest()
    table = {k: r[v] for k, v in klcases.filler(100000 - n_keys // 2).items()}
    for i, k in enumerate(pool[: n_keys // 2]):
        table[(klcases.CC, "", k.encode())] = [r["vp_org1"], r["vp_org2"], r["vp_3of4"], -2][i % 4] if i % 9 else -2
    table[(klcases.CC, "", b"hot")] = r["vp_org1"]
    return net, blk, info, kn, table


@pytest.mark.parametrize("seed", [1])
def test_seeded_blocks_against_the_oracle(ctx, seed):
    net, blk, info, kn, table = _seeded(seed)
    names, bits = collcases.principals(True)
    ids = net.identities()
    _configure(ctx, ids, names, net.channel, bits)
    ctx.key_policies(kn, table)
    nodes, vps = klcases.combined(kn, table)
    exp = keylevel_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=collcases.namespace_policies(), vps=vps,
                                         known=[i[0] for i in ids]).tolist()
    got = ctx.validate_block(blk).tolist()
    assert got == exp
    assert got == ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist()
    assert {ob.VALID, ob.ENDORSEMENT_POLICY_FAILURE, ob.NOT_VALIDATED} <= set(got)
