"""GPU: the private-data check (fabgpu_validate_pvtdata) -- every case through validate_block and validate_envelopes in both validator
modes, with and without the MVCC stage before it; seeded blocks submitted three slots deep against pvt_oracle; and the refusals."""
import ctypes

import numpy as np
import pytest

from tools import blockgen
from util import pkg
import pvt_oracle as po
import pvtcases

pytestmark = pytest.mark.gpu

POLICIES = {pvtcases.CC: 0, pvtcases.OTHER: 0}


@pytest.fixture(scope="module")
def net():
    return blockgen.Network()


@pytest.fixture(scope="module")
def ctx(net):
    c = pkg().binding.Context(max_batch=8192)
    _configure(c, net, pkg().binding.CAP_V2_0)
    yield c
    c.close()


def _configure(c, net, cap):
    c.msp_configure([(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table], net.policy_n_of(3), net.principals, net.channel, policies=POLICIES)
    c.namespace_versions({pvtcases.CC: "1.0"})
    c.channel_capability(cap)


def _block(net, rwsets, seed):
    """a signed block whose transaction t carries rwsets[t]; None: a config-update transaction (the walk never reaches its results)"""
    faults = {t: "config_update_type" for t, rw in enumerate(rwsets) if rw is None}
    hook = lambda t, part, b: rwsets[t] if part == "TxReadWriteSet" and rwsets[t] is not None else b
    return blockgen.build_block(net, len(rwsets), 3, faults, seed=seed, mutate=hook)


@pytest.mark.parametrize("mvcc", [False, True], ids=["alone", "after_mvcc"])
@pytest.mark.parametrize("entry", ["block", "envelopes"])
@pytest.mark.parametrize("mode", ["v20", "v13"])
def test_cases_on_the_device(ctx, net, entry, mode, mvcc):
    """Every case gives its written-out codes with the case's flags, and pvt_oracle's with the device's own flags; a second call gives
    the same answer"""
    B = pkg().binding
    _configure(ctx, net, B.CAP_V1_3 if mode == "v13" else B.CAP_V2_0)
    try:
        for k, (name, txs, flags, pvt, status, verdict) in enumerate(pvtcases.cases()):
            rwsets = pvtcases.rwsets_of(txs, pvt)
            blk, info = _block(net, rwsets, seed=41 + k)
            dev = ctx.validate_block(blk) if entry == "block" else ctx.validate_envelopes(info["env_blob"], info["env_off"])
            if mvcc:
                ctx.state_versions([], 1, capacity=64)
                dev = ctx.validate_mvcc(0, 1, dev)
            assert ctx.validate_pvtdata(0, flags, pvt) == (verdict, status), name
            assert ctx.validate_pvtdata(0, flags, pvt) == (verdict, status), name
            assert ctx.validate_pvtdata(0, dev.tolist(), pvt) == po.validate(rwsets, dev.tolist(), pvt), name
    finally:
        _configure(ctx, net, B.CAP_V2_0)
        ctx.state_versions([], 0)


def test_seeded_blocks_three_slots_deep(ctx, net):
    """Seeded blocks submitted three slots deep; block k's check runs after its wait while k+1 and k+2 are in flight, with the device's
    flags and with the case's; each answer equals pvt_oracle's"""
    S = pkg().binding.SLOTS
    blocks = []
    for b in range(9):
        txs, flags, pvt = pvtcases.seeded(700 + b, 60 + 7 * b)
        rwsets = pvtcases.rwsets_of(txs, pvt)
        blk, _ = _block(net, rwsets, seed=900 + b)
        blocks.append((rwsets, flags, pvt, blk))
    codes = []
    for k in range(min(S, len(blocks))):
        ctx.validate_block_async(k % S, blocks[k][3])
    for k, (rwsets, flags, pvt, _) in enumerate(blocks):
        slot = k % S
        dev = ctx.validate_wait(slot, 256).tolist()
        for fl in (dev, flags):
            got = ctx.validate_pvtdata(slot, fl, pvt)
            assert got == po.validate(rwsets, fl, pvt), k
            codes += [s[0] for s in got[1].values()]
        if k + S < len(blocks):
            ctx.validate_block_async(slot, blocks[k + S][3])
    assert all(codes.count(c) > 0 for c in (po.OK, po.MISMATCH, po.SKIP, po.UNDET))


def test_refusals(ctx, net):
    B = pkg().binding
    _, txs, flags, pvt, status, verdict = pvtcases.cases()[0]
    rwsets = pvtcases.rwsets_of(txs, pvt)
    blk, _ = _block(net, rwsets, seed=5)
    S = B.SLOTS
    ctx.validate_block_async(1 % S, blk)                     # in flight: no finished block on that slot
    with pytest.raises(B.FabGpuError, match="no finished block"):
        ctx.validate_pvtdata(1 % S, flags, pvt)
    ctx.validate_wait(1 % S, 16)
    assert ctx.validate_pvtdata(1 % S, flags, pvt) == (verdict, status)
    ctx.validate_block(blk)
    with pytest.raises(B.FabGpuError, match="transaction count"):
        ctx.validate_pvtdata(0, flags + [0], pvt)
    with pytest.raises(B.FabGpuError, match="below the block"):
        ctx.validate_pvtdata(0, flags, {5: pvt[0]})
    lib, h = B.lib(), ctx._h
    fl = np.array(flags, np.uint8)
    blob = np.frombuffer(pvt[0] + pvt[0], np.uint8).copy()
    st = np.zeros(6, np.int32)
    out = np.zeros(4, np.int32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    call = lambda off, seq, n_pvt, status=st: lib.fabgpu_validate_pvtdata(h, 0, p(fl), ctypes.c_size_t(1), p(blob), p(off), p(seq),
                                                                          ctypes.c_size_t(n_pvt), p(status) if status is not None else None, p(out))
    two = np.array([0, len(pvt[0]), 2 * len(pvt[0])], np.uint32)
    assert call(two, np.array([0, 0], np.uint32), 2) == B.E_ARG                          # a seq given twice
    assert "twice" in B.lib().fabgpu_last_error(h).decode()
    assert call(np.array([len(pvt[0]), 0], np.uint32), np.array([0], np.uint32), 1) == B.E_ARG   # offsets decrease
    assert call(two, np.array([0], np.uint32), 1, status=None) == B.E_ARG                # NULL status with entries
    assert call(two[:2], np.array([0], np.uint32), 1) == 0 and tuple(out) == verdict
    ctx.validate_block_async(0, blk)                          # a new submit ends the previous block's calls
    with pytest.raises(B.FabGpuError, match="no finished block"):
        ctx.validate_pvtdata(0, flags, pvt)
    ctx.validate_wait(0, 16)
    assert ctx.validate_pvtdata(0, flags, {}) == ((0, -1, -1, -1), {})
