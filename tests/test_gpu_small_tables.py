"""GPU: the small-table tier (signed 8-bit windows, fabgpu_keys_register_small; ecdsa_verify_small_kernel) against the oracle, through
every entry point that takes key handles.  Same bar as the other tiers: bit-exact."""
import os

import numpy as np
import pytest

from oracle import bccsp_sw as o
from oracle import blockval as ob
from oracle import fast
from tools import blockgen, workload
from util import mask_bits, pkg
import blockutil
import vectors

pytestmark = pytest.mark.gpu

R = 1 << 256


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=1 << 15)
    yield c
    c.close()


def _fill(ctx, slot, w, key_slots):
    hb = ctx.host_buffers(slot)
    for name, arr in (("qx", w.qx()), ("qy", w.qy()), ("e", w.digest), ("r", w.r), ("s", w.s)):
        hb[name][: w.n] = arr
    ctx.host_key_slots(slot)[: w.n] = key_slots
    return hb


def test_small_tables_through_the_keyed_entry_points(ctx):
    w = workload.Workload(16384, 96, seed=141)
    w.tamper_r(0.05)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    hs = ctx.keys_register_small(w.keys_xy)
    assert (hs <= -2).all() and len(set(hs.tolist())) == 96
    assert (ctx.keys_register_small(w.keys_xy) == hs).all()        # second lookup hits the cache
    assert ctx.key_table_stats()["small"] >= 96
    # every signature through its key's small table
    hb = _fill(ctx, 0, w, hs[w.key_idx])
    ctx.verify_p256_keyed(0, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all() and not hb["offcurve"][: w.n // 32].any()
    assert (ctx.host_key_slots(0)[: w.n] <= -2).all()              # handles were replaced by live device codes
    # three classes interleaved: window table / small table / no table
    big = ctx.keys_register(w.keys_xy[:32])
    mix = np.where(w.key_idx % 3 == 0, hs[w.key_idx], -1).astype(np.int32)
    sel = (w.key_idx % 3 == 1) & (w.key_idx < 32)
    mix[sel] = big[w.key_idx[sel]]
    assert (mix >= 0).sum() > 1000 and (mix == -1).sum() > 1000 and (mix <= -2).sum() > 1000
    hb = _fill(ctx, 1, w, mix)
    ctx.verify_p256_keyed(1, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all()
    # small + none only (no window table in the batch), ragged n
    hb = _fill(ctx, 2, w, np.where(w.key_idx % 2 == 0, hs[w.key_idx], -1))
    ctx.verify_p256_keyed(2, 5001)
    assert (mask_bits(hb["mask"], 5001) == mask_bits(exp, 5001)).all()


def _fill_soa(ctx, slot, soa, key_slots):
    hb = ctx.host_buffers(slot)
    for name, arr in zip(("qx", "qy", "e", "r", "s"), soa):
        hb[name][: arr.shape[0]] = arr
    ctx.host_key_slots(slot)[: len(key_slots)] = key_slots
    return hb


def _mismatches(cases, mix, hb):
    bits = mask_bits(hb["mask"], len(mix["valid"])).astype(bool)
    return [c["name"] for c, p in zip(cases, mix["pos"]) if bits[p] != mix["valid"][p]] + \
        ["honest row %d" % i for i in np.flatnonzero(bits != mix["valid"]) if i not in mix["pos"]][:4]


def test_chain_collisions_through_the_small_table_kernels(ctx):
    """The small-table order's chain cases (vectors.chain_cases: a doubling or an infinity at every signed window of the key, at the
    library's widths) interleaved with honest signatures: first with every handle small (ecdsa_verify_small_kernel over the whole
    batch), then in one batch of window-table, small-table and no-table handles together with the key-table and generic orders'
    cases (compact_classes_kernel, then ecdsa_verify_indexed_kernel and the indexed form of the small kernel)."""
    b = pkg().binding
    widths = b.build_info() + (b.Context.small_table_info()[0],)
    cases = vectors.chain_cases(*widths, orders=("small",))
    mix = vectors.mix_with_workload(cases, seed=0x5A11)
    hs = ctx.keys_register_small(mix["keys_xy"])
    assert (hs <= -2).all()
    hb = _fill_soa(ctx, 0, mix["soa"], hs[mix["kidx"]])
    ctx.verify_p256_keyed(0, len(mix["valid"]))
    bad = _mismatches(cases, mix, hb)
    assert not bad, bad[:8]
    cases = vectors.chain_cases(*widths, orders=("small", "jac", "generic"))
    mix = vectors.mix_with_workload(cases, seed=0x5A12)
    big, small = ctx.keys_register(mix["keys_xy"]), ctx.keys_register_small(mix["keys_xy"])
    assert (big >= 0).all() and (small <= -2).all()
    kidx = mix["kidx"]
    code = np.select([kidx % 3 == 0, kidx % 3 == 1], [small[kidx], big[kidx]], -1).astype(np.int32)
    handles = {"small": small, "jac": big, "generic": None}             # each case through the kernel of its own order
    for c, p in zip(cases, mix["pos"]):
        h = handles[c["order"]]
        code[p] = -1 if h is None else h[kidx[p]]
    assert (code >= 0).sum() > 100 and (code == -1).sum() > 100 and (code <= -2).sum() > 100
    hb = _fill_soa(ctx, 1, mix["soa"], code)
    ctx.verify_p256_keyed(1, len(mix["valid"]))
    bad = _mismatches(cases, mix, hb)
    assert not bad, bad[:8]


def test_small_tables_device_resident(ctx):
    import torch
    w = workload.Workload(8192, 40, seed=143)
    w.tamper_r(0.1)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    codes = ctx.small_raw_codes(ctx.keys_register_small(w.keys_xy))
    assert (codes <= -2).all()
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(a).to(dev) for a in (w.qx(), w.qy(), w.digest, w.r, w.s)]
    ks = torch.from_numpy(codes[w.key_idx]).to(dev)
    mask = torch.zeros(w.n // 32, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev)
    ctx.verify_p256_device_keyed(2, ks.data_ptr(), 0, 0, t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(), w.n, mask.data_ptr(), 0, st.cuda_stream)
    st.synchronize()
    assert (mask.cpu().numpy().view(np.uint32) == exp).all()


def test_edge_vectors_and_off_curve_keys_through_small_tables():
    """FABGPU_SMALL_MIN_USES=1: every key of a bccsp-level call gets a small table at first sight, including keys that are not curve
    points (their table says so: status ERR_OFF_CURVE, as from the generic kernel)."""
    os.environ["FABGPU_SMALL_MIN_USES"] = "1"
    try:
        csp = pkg().bccsp.GPUCSP(max_batch=8192)
    finally:
        del os.environ["FABGPU_SMALL_MIN_USES"]
    cases = vectors.build()
    keys = [csp.KeyImport((c["qx"] % R, c["qy"] % R)) for c in cases]
    for _ in range(2):                                             # second round: tables already there
        st = csp.VerifyBatch(keys, list(range(len(cases))), [c["digest"] for c in cases], [c["sig"] for c in cases])
        for c, got in zip(cases, st):
            assert int(got) == vectors.expected_status(c), c["name"]
    assert any(vectors.expected_status(c) == o.ERR_OFF_CURVE for c in cases)
    stats = csp.ctx.key_table_stats()
    assert stats["small"] > 10 and stats["big"] == 0
    w = workload.Workload(6000, 300, seed=153)
    w.tamper_r(0.2)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)
    assert (csp.ctx.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off) == exp).all()
    assert csp.ctx.key_table_stats()["small"] >= stats["small"] + 300
    csp.close()


def test_a_key_earns_its_small_table_after_min_uses_signatures():
    os.environ["FABGPU_SMALL_MIN_USES"] = "4"
    try:
        c = pkg().binding.Context(max_batch=4096)                  # 4 signatures seen earn a small table (default 32), 256 in one call a window table
    finally:
        del os.environ["FABGPU_SMALL_MIN_USES"]
    w = workload.Workload(600, 300, seed=157)                      # two signatures per key and call
    w.tamper_r(0.1)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)
    uses = np.bincount(w.key_idx, minlength=300)
    built = []
    for _ in range(4):
        assert (c.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off) == exp).all()
        built.append(c.key_table_stats()["small"])
    assert built[0] == int((uses >= 4).sum())                      # only keys with >= 4 signatures in the first call
    assert built[-1] == int((uses > 0).sum()) and built == sorted(built)
    assert c.key_table_stats()["big"] == 0
    c.close()


def test_small_table_recycling_and_stale_handles():
    os.environ["FABGPU_SMALL_SLOTS"] = "16"
    try:
        c = pkg().binding.Context(max_batch=4096)
    finally:
        del os.environ["FABGPU_SMALL_SLOTS"]
    assert c.small_slot_capacity() == 16
    w = workload.Workload(4096, 24, seed=161)
    w.tamper_r(0.1)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    h1 = c.keys_register_small(w.keys_xy[:16])
    assert (h1 <= -2).all()
    h2 = c.keys_register_small(w.keys_xy[16:24])                   # pool full: the least recently used tables go
    assert (h2 <= -2).all() and c.key_table_stats()["small_recycled"] >= 8
    handles = np.concatenate([h1, h2])                             # some of h1 are stale now
    hb = _fill(c, 0, w, handles[w.key_idx])
    c.verify_p256_keyed(0, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all()                  # stale handles fell back to the generic arithmetic
    live = c.host_key_slots(0)[: w.n]
    assert (live == -1).sum() > 0 and (live <= -2).sum() > 0
    h3 = c.keys_register_small(w.keys_xy)                          # 24 keys, 16 tables: the rest stay -1
    assert int((h3 == -1).sum()) == 8
    hb = _fill(c, 1, w, h3[w.key_idx])
    c.verify_p256_keyed(1, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all()
    c.close()


def test_block_prepass_with_more_identities_than_window_tables():
    """fabgpu_msp_configure with more identities than window-table slots: the identities live in the small tier; flags equal the
    oracle's, before and after the small tables were recycled by unrelated registrations."""
    os.environ["FABGPU_KEY_SLOTS"] = "4"
    os.environ["FABGPU_SMALL_SLOTS"] = "64"
    try:
        c = pkg().binding.Context(max_batch=4096)
    finally:
        del os.environ["FABGPU_KEY_SLOTS"]; del os.environ["FABGPU_SMALL_SLOTS"]
    net = blockgen.Network(n_orgs=4, n_clients=3)
    ids = blockutil.identities_of(net)
    assert 4 < len(ids) <= 64
    faults = blockutil.fault_map(70)
    blk, binfo = blockgen.build_block(net, 70, 3, faults, seed=171)
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=[i[0] for i in ids])
    c.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    st = c.key_table_stats()
    assert st["big"] == 0 and 4 < st["small"] <= len(ids)           # one table per distinct key
    assert c.validate_block(blk).tolist() == exp.tolist()
    assert c.validate_envelopes(binfo["env_blob"], binfo["env_off"]).tolist() == exp.tolist()
    other = workload.Workload(128, 64, seed=173)
    assert (c.keys_register_small(other.keys_xy) <= -2).all()      # recycles the identities' tables
    assert c.validate_block(blk).tolist() == exp.tolist()
    # the busy identities (the four endorsing peers) registered for window tables BEFORE the MSP is configured keep them; the rest go small
    peer_keys = np.stack([np.frombuffer(p.xy, np.uint8) for p in net.peers])
    assert (c.keys_register(peer_keys) >= 0).all()
    c.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    st = c.key_table_stats()
    assert st["big"] == 4
    assert c.validate_block(blk).tolist() == exp.tolist()
    assert c.validate_envelopes(binfo["env_blob"], binfo["env_off"]).tolist() == exp.tolist()
    assert (c.keys_register(other.keys_xy[:4]) >= 0).all()         # evicts the peers' window tables: their identities fall back to small ones
    assert c.validate_block(blk).tolist() == exp.tolist()
    c.close()


def test_config5_shape_through_small_tables_full_size():
    """BASELINE.json configs[4]'s size (262 144 signatures, 5 % tampered r) with every key in the small tier (8 192 keys, 32 signatures
    each): statuses equal the C oracle's bit for bit, plus the size-independent properties -- no tampered signature accepted, every
    untouched one accepted."""
    n = 1 << 18
    w = workload.Workload(n, 8192, seed=workload.DEFAULT_SEED + 21, nthreads=os.cpu_count())
    picked = w.tamper_r(0.05)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=os.cpu_count())
    assert int((exp != o.VALID).sum()) == len(picked) and 12000 < len(picked) < 14500
    os.environ["FABGPU_SMALL_MIN_USES"] = "1"
    try:
        c = pkg().binding.Context(max_batch=n)
    finally:
        del os.environ["FABGPU_SMALL_MIN_USES"]
    st = c.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off)     # every key earns its small table at first sight
    assert (st == exp).all()
    stats = c.key_table_stats()
    assert stats["small"] == 8192 and stats["big"] == 0
    hs = c.keys_register_small(w.keys_xy)
    hb = _fill(c, 0, w, hs[w.key_idx])
    c.verify_p256_keyed(0, n)
    bits = mask_bits(hb["mask"], n)
    assert (hb["mask"][: n // 32] == fast.valid_mask(exp)).all()
    assert int(bits.sum()) == n - len(picked) and bits[picked].sum() == 0
    c.close()
