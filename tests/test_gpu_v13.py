"""GPU: the v1.3 mode (fabgpu_channel_capability(FABGPU_CAP_V1_3): the v1.4 validator with the builtin v13 VSCC) in the device block
validator, through validate_block, validate_envelopes and two async slots, against the v1.3 oracle and the codes written out per case;
switching back to v2.0; fabgpu_msp_configure resetting the mode; and the calls the library refuses."""
import ctypes

import numpy as np
import pytest

from oracle import blockval as ob
from util import pkg
from blockutil import _blob, _p
import collcases
import keylevel_oracle
import klcases
import v13_oracle
import v13cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    yield c
    c.close()


def _configure(ctx, net, names, bits, case, colls=False, cap=1):
    B = pkg().binding
    ctx.msp_configure(net.identities(), collcases.forest()[0], names, net.channel, policies=v13cases.policies())
    if bits is not None:
        ctx.msp_principal_bits(bits)
    ctx.collection_policies(collcases.collection_table() if colls else None)
    kt = v13cases.key_table(case) if case is not None else None
    if kt:
        ctx.key_policies(*kt)
    ctx.namespace_versions(v13cases.versions())
    ctx.channel_capability(B.CAP_V1_3 if cap else B.CAP_V2_0)
    return kt


def _three_ways(ctx, blk, info):
    B = pkg().binding
    a = ctx.validate_block(blk).tolist()
    b = ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist()
    ctx.validate_block_async(1, blk)
    ctx.validate_envelopes_async(2, info["env_blob"], info["env_off"])
    c = ctx.validate_wait(1, len(a) + 16).tolist()
    d = ctx.validate_wait(2, len(a) + 16).tolist()
    assert a == b == c == d
    assert B.SLOTS >= 3
    return a


@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
def test_v13_cases_on_the_device(ctx, use_bits):
    """Every case: device == oracle == the codes written out, on every entry point."""
    names, bits = collcases.principals(use_bits)
    for case in v13cases.cases():
        net, blk, info, codes = v13cases.materialize(case)
        kt = _configure(ctx, net, names, bits, case, colls=case[2])
        ids = net.identities()
        nodes, vps = klcases.combined(*kt) if kt else (collcases.forest()[0], None)
        exp = v13_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=v13cases.policies(), versions=v13cases.versions(),
                                        collections=collcases.collection_table() if case[2] else None, vps=vps, known=[i[0] for i in ids]).tolist()
        assert exp == codes, case[0]
        assert _three_ways(ctx, blk, info) == codes, case[0]


def test_collection_key_and_wire_corpora_in_v13_mode(ctx):
    """collcases and klcases with their tables, and the wire-mutation corpus, in v1.3 mode: device == v1.3 oracle."""
    import wiremut
    names, bits = collcases.principals(True)
    pol = {k: v for k, v in collcases.namespace_policies().items() if k != collcases.LIFECYCLE}
    ver = {collcases.CC: "1.0", collcases.OTHER: "1.0"}
    B = pkg().binding
    for case in collcases.cases():
        net, blk, info, _, _ = collcases.materialize(case)
        ids = net.identities()
        ctx.msp_configure(ids, collcases.forest()[0], names, net.channel, policies=pol)
        ctx.msp_principal_bits(bits)
        ctx.collection_policies(collcases.collection_table())
        ctx.namespace_versions(ver)
        ctx.channel_capability(B.CAP_V1_3)
        exp = v13_oracle.validate_block(blk, ids, net.channel, collcases.forest()[0], names, bits=bits, policies=pol, versions=ver,
                                        collections=collcases.collection_table(), known=[i[0] for i in ids]).tolist()
        assert _three_ways(ctx, blk, info) == exp, case[0]
    for case in klcases.cases():
        if case[0] == "more_than_16_roots":
            continue                                  # 17 writes per transaction: past the default write-record sizing of a fresh context
        net, blk, info, _ = klcases.materialize(case)
        ids = net.identities()
        kn, table = klcases.key_table(case)
        colls = collcases.collection_table() if case[1] else None
        ctx.msp_configure(ids, collcases.forest()[0], names, net.channel, policies=pol)
        ctx.msp_principal_bits(bits)
        ctx.collection_policies(colls)
        ctx.key_policies(kn, table)
        ctx.namespace_versions(ver)
        ctx.channel_capability(B.CAP_V1_3)
        nodes, vps = klcases.combined(kn, table)
        exp = v13_oracle.validate_block(blk, ids, net.channel, nodes, names, bits=bits, policies=pol, versions=ver, collections=colls, vps=vps,
                                        known=[i[0] for i in ids]).tolist()
        assert _three_ways(ctx, blk, info) == exp, case[0]
    net, ids, nodes, wpol, blocks = wiremut.corpus()
    wver = {n: "1.0" for n in wpol}
    ctx.msp_configure(ids, nodes, net.principals, net.channel, policies=wpol)
    ctx.namespace_versions(wver)
    ctx.channel_capability(B.CAP_V1_3)
    for blk, info, _, _ in blocks:
        exp = v13_oracle.validate_block(blk, ids, net.channel, nodes, net.principals, policies=wpol, versions=wver, known=[i[0] for i in ids]).tolist()
        assert ctx.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == exp


def test_seeded_random_blocks_on_the_device(ctx):
    import test_v13_host
    names, bits = collcases.principals(True)
    for seed in range(6):
        net, blk, info = test_v13_host.random_block(seed, n_tx=200)
        ids = net.identities()
        _configure(ctx, net, names, bits, None)
        exp = v13_oracle.validate_block(blk, ids, net.channel, collcases.forest()[0], names, bits=bits, policies=v13cases.policies(),
                                        versions=v13cases.versions(), known=[i[0] for i in ids]).tolist()
        assert _three_ways(ctx, blk, info) == exp


def test_switching_back_to_v20_and_configure_resets(ctx):
    """v1.3 -> v2.0 gives the v2.0 oracle's flags again; fabgpu_msp_configure puts a v1.3 context back into v2.0 mode."""
    B = pkg().binding
    names, bits = collcases.principals(True)
    case = [c for c in v13cases.cases() if c[0] == "version_mismatch"][0]
    net, blk, info, codes = v13cases.materialize(case)
    ids = net.identities()
    v20 = keylevel_oracle.validate_block(blk, ids, net.channel, collcases.forest()[0], names, bits=bits, policies=v13cases.policies(),
                                         known=[i[0] for i in ids]).tolist()
    assert v20 != codes
    _configure(ctx, net, names, bits, case)
    assert ctx.validate_block(blk).tolist() == codes
    ctx.channel_capability(B.CAP_V2_0)
    assert ctx.validate_block(blk).tolist() == v20
    ctx.channel_capability(B.CAP_V1_3)
    assert ctx.validate_block(blk).tolist() == codes
    ctx.msp_configure(ids, collcases.forest()[0], names, net.channel, policies=v13cases.policies())
    ctx.msp_principal_bits(bits)
    assert ctx.validate_block(blk).tolist() == v20


def test_refusals(ctx):
    """A capability other than V2_0 / V1_3, a version count that is not the table's, and ImplicitMeta roots in v1.3 mode are refused
    with FABGPU_E_ARG, and the previous state is kept."""
    B = pkg().binding
    L = B.lib()
    names, bits = collcases.principals(True)
    case = [c for c in v13cases.cases() if c[0] == "version_mismatch"][0]
    net, blk, info, codes = v13cases.materialize(case)
    _configure(ctx, net, names, bits, case)
    for cap in (2, -1, 13):
        with pytest.raises(B.FabGpuError):
            ctx.channel_capability(cap)
    vb, vo = _blob([b"1.0"] * 3)
    assert L.fabgpu_namespace_versions(ctx._h, _p(vb), _p(vo), ctypes.c_int(3)) == -3
    assert ctx.validate_block(blk).tolist() == codes                     # mode and versions kept
    # _lifecycle's policy is ImplicitMeta: no namespace table holding it in v1.3 mode ...
    pol = dict(v13cases.policies()); pol[collcases.LIFECYCLE] = collcases.forest()[1]["lifecycle"]
    nb, no = _blob([n.encode() for n in sorted(pol)])
    roots = np.array([pol[n] for n in sorted(pol)], np.int32)
    assert L.fabgpu_namespace_policies(ctx._h, _p(nb), _p(no), _p(roots), ctypes.c_int(len(pol))) == -3
    assert ctx.validate_block(blk).tolist() == codes                     # the previous table kept
    # ... and no v1.3 mode while such a table is installed
    ctx.channel_capability(B.CAP_V2_0)
    assert L.fabgpu_namespace_policies(ctx._h, _p(nb), _p(no), _p(roots), ctypes.c_int(len(pol))) == 0
    with pytest.raises(B.FabGpuError):
        ctx.channel_capability(B.CAP_V1_3)
    ids = net.identities()
    v20 = keylevel_oracle.validate_block(blk, ids, net.channel, collcases.forest()[0], names, bits=bits, policies=pol,
                                         known=[i[0] for i in ids]).tolist()
    assert ctx.validate_block(blk).tolist() == v20                       # still v2.0
