"""GPU parity tests proper: the CUDA path, called through the C ABI, against the oracle.
Integer work: the bar is bit-exact."""
import json
import os
import random

import numpy as np
import pytest

from oracle import bccsp_sw as o
from oracle import fast, goasn1, p256
from tools import workload
from util import be32, from_be, mask_bits, pkg
import vectors

pytestmark = pytest.mark.gpu

R = 1 << 256


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=1 << 17)
    yield c
    c.close()


@pytest.fixture(scope="module")
def csp():
    c = pkg().bccsp.GPUCSP(max_batch=4096)
    yield c
    c.close()


def _ints(arr):
    return [from_be(row) for row in arr]


# ---------------------------------------------------------------------------------------------------------
# device tables vs the oracle's scalar multiplication (the field primitives: tests/test_gpu_field.py)
# ---------------------------------------------------------------------------------------------------------
def _table_picks(w, rnd):
    """(window, digit) samples that hit the corners of the two-level build: digits below 2^(w/2) (low table only), multiples of
    2^(w/2) (high table only), chunk boundaries (64 entries per thread), the last entry, the top window's largest useful digit."""
    per = (1 << w) - 1
    nwin = (256 + w - 1) // w
    half = 1 << (w // 2)
    top = min(per, (1 << (256 - w * (nwin - 1))) - 1)
    picks = [(0, 1), (0, per), (nwin - 1, 1), (nwin - 1, top), (1, half - 1), (1, half), (1, half + 1), (2, 3 * half), (0, 64), (0, 65),
             (3, per - 62), (3, per - 63), (nwin - 2, per - 1), (1, 2 * half - 1)]
    picks += [(rnd.randrange(nwin), rnd.randrange(1, per + 1)) for _ in range(20)]
    return [(j, min(d, top) if j == nwin - 1 else d) for j, d in picks]


def _check_entries(ent, picks, w, base):
    rinv = pow(R, -1, p256.P)
    for (j, d), row in zip(picks, ent):
        x = sum(int(row[i]) << (32 * i) for i in range(8)) * rinv % p256.P
        y = sum(int(row[8 + i]) << (32 * i) for i in range(8)) * rinv % p256.P
        assert (x, y) == p256.scalar_mult((d << (w * j)) % p256.N, base), (j, d)


def test_fixed_base_table(ctx):
    """Sampled entries of the device-built generator table == oracle scalar multiplication (entry (j, d) = d * 2^(w j) * G)."""
    wg, _ = pkg().binding.build_info()
    picks = _table_picks(wg, random.Random(3))
    ent = ctx.test_table_entries(-1, [j for j, _ in picks], [d for _, d in picks])
    _check_entries(ent, picks, wg, (p256.GX, p256.GY))


def test_key_table_entries(ctx):
    """The same for a per-key table (fabgpu_keys_register): entry (j, d) = d * 2^(w j) * Q."""
    _, wq = pkg().binding.build_info()
    w = workload.Workload(32, 2, seed=91)
    slots = ctx.keys_register(w.keys_xy) & 0xFFF
    for k in range(2):
        q = (from_be(w.keys_xy[k, :32]), from_be(w.keys_xy[k, 32:]))
        picks = _table_picks(wq, random.Random(4 + k))
        ent = ctx.test_table_entries(int(slots[k]), [j for j, _ in picks], [d for _, d in picks])
        _check_entries(ent, picks, wq, q)


# ---------------------------------------------------------------------------------------------------------
# leaf: pre-gated SoA -> bitmask
# ---------------------------------------------------------------------------------------------------------
def test_config1_1024_tuples(ctx):
    w = workload.Workload(1024, 16, seed=workload.DEFAULT_SEED)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)
    mask, off = ctx.verify_p256_host(w.qx(), w.qy(), w.digest, w.r, w.s)
    assert (mask == fast.valid_mask(exp)).all() and (mask == 0xFFFFFFFF).all() and not off.any()


def test_ragged_sizes_and_empty(ctx):
    w = workload.Workload(300, 4, seed=11)
    w.tamper_r(0.2)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=4)
    bits = (exp == o.VALID).astype(np.uint8)
    for n in (0, 1, 31, 32, 33, 127, 128, 129, 300):
        mask, off = ctx.verify_p256_host(w.qx()[:n], w.qy()[:n], w.digest[:n], w.r[:n], w.s[:n])
        assert mask.shape[0] == (n + 31) // 32
        assert (mask_bits(mask, n) == bits[:n]).all(), n
        if n % 32:
            assert int(mask[-1]) >> (n % 32) == 0       # padding bits are zero


def test_config2_64k_all_valid(ctx):
    # BASELINE.json configs[1]: 64k-signature batch, K = 64 keys, bitmask equals bccsp/sw (oracle: all ones)
    w = workload.Workload(65536, 64, seed=workload.DEFAULT_SEED + 2)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=os.cpu_count())
    mask, off = ctx.verify_p256_host(w.qx(), w.qy(), w.digest, w.r, w.s)
    assert (mask == fast.valid_mask(exp)).all()
    assert (mask == 0xFFFFFFFF).all()


def test_config5_tampered_mask_exact(ctx):
    # BASELINE.json configs[4] on one GPU at reduced size: 5 % tampered r, exact-match bitmask, no false accept
    w = workload.Workload(32768, 64, seed=workload.DEFAULT_SEED + 5)
    picked = w.tamper_r(0.05)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=os.cpu_count())
    mask, off = ctx.verify_p256_host(w.qx(), w.qy(), w.digest, w.r, w.s)
    assert (mask == fast.valid_mask(exp)).all()
    bits = mask_bits(mask, w.n)
    assert bits[picked].sum() == 0 and 1200 < len(picked) < 2100


def test_config4_one_million_signatures_full_size():
    """BASELINE.json configs[3] / [4] at FULL size on whatever GPUs the box has: 1 048 576 signatures, 256 keys, 5 % tampered r,
    through the bccsp-level call (raw DER in, status bytes out; key tables built on first sight) and through the pre-gated SoA
    leaf (bitmask out).  Exact equality with the C oracle, plus the size-independent properties: no tampered signature is
    accepted, every untouched one is, and the number of set mask bits is N minus the number tampered."""
    import torch
    n = 1 << 20
    w = workload.Workload(n, 256, seed=workload.DEFAULT_SEED + 4, nthreads=os.cpu_count())
    picked = w.tamper_r(0.05)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=os.cpu_count())
    assert int((exp != o.VALID).sum()) == len(picked) and 50000 < len(picked) < 55000
    ndev = min(torch.cuda.device_count(), 8)
    c = pkg().binding.Context(max_batch=n, device_ids=list(range(ndev)))
    st = c.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off)
    assert (st == exp).all()
    mask, off = c.verify_p256_host(w.qx(), w.qy(), w.digest, w.r, w.s)
    bits = mask_bits(mask, n)
    assert not off.any() and (mask == fast.valid_mask(exp)).all()
    assert int(bits.sum()) == n - len(picked) and bits[picked].sum() == 0
    c.close()


def test_async_slots_and_pinned_buffers(ctx):
    w = workload.Workload(4096, 8, seed=21)
    w.tamper_r(0.1)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    half = 2048
    for slot, sl in ((0, slice(0, half)), (1, slice(half, 4096))):
        hb = ctx.host_buffers(slot)
        for name, arr in (("qx", w.qx()), ("qy", w.qy()), ("e", w.digest), ("r", w.r), ("s", w.s)):
            hb[name][:half] = arr[sl]
        ctx.verify_p256_async(slot, half)
    ctx.wait(0); ctx.wait(1)
    got = np.concatenate([ctx.host_buffers(0)["mask"][:half // 32], ctx.host_buffers(1)["mask"][:half // 32]])
    assert (got == exp).all()


def test_x509_golden_fixtures(csp):
    fix = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "x509_fixtures.json")))
    keys, kidx, digs, sigs, exp = [], [], [], [], []
    for i, x in enumerate(fix):
        keys.append(csp.KeyImport((int(x["qx"], 16), int(x["qy"], 16))))
        kidx.append(i); digs.append(bytes.fromhex(x["digest"])); sigs.append(bytes.fromhex(x["sig_der"]))
        exp.append({"VALID": o.VALID, "ERR_HIGH_S": o.ERR_HIGH_S}[x["expect"]])
    st = csp.VerifyBatch(keys, kidx, digs, sigs)
    assert list(st) == exp
    # msp/cert_test.go:70-97: after s -> N - s the 31 high-S signatures verify
    sigs2 = [goasn1.marshal_ecdsa_signature(int(x["r"], 16), p256.N - int(x["s"], 16)) if x["expect"] == "ERR_HIGH_S" else s
             for x, s in zip(fix, sigs)]
    assert set(csp.VerifyBatch(keys, kidx, digs, sigs2)) == {o.VALID}


def test_constructed_edge_cases(csp):
    cases = vectors.build()
    keys = [csp.KeyImport((c["qx"] % R, c["qy"] % R)) for c in cases]
    st = csp.VerifyBatch(keys, list(range(len(cases))), [c["digest"] for c in cases], [c["sig"] for c in cases])
    for c, got in zip(cases, st):
        assert int(got) == vectors.expected_status(c), c["name"]


def _chain_cases(orders=vectors.CHAIN_ORDERS):
    """vectors.chain_cases at the library's window widths."""
    b = pkg().binding
    return vectors.chain_cases(*b.build_info(), b.Context.small_table_info()[0], orders=orders)


def _fill_soa(ctx, slot, soa, key_slots):
    hb = ctx.host_buffers(slot)
    for name, arr in zip(("qx", "qy", "e", "r", "s"), soa):
        hb[name][: arr.shape[0]] = arr
    ctx.host_key_slots(slot)[: len(key_slots)] = key_slots
    return hb


def _chain_mismatches(cases, mix, bits):
    assert bits.shape == mix["valid"].shape
    bad = [c["name"] for c, p in zip(cases, mix["pos"]) if bits[p] != mix["valid"][p]]
    return bad + ["honest row %d" % i for i in np.flatnonzero(bits != mix["valid"]) if i not in set(mix["pos"].tolist())][:4]


def test_chain_collisions_through_the_generic_kernel(ctx):
    """ecdsa_verify_kernel (Booth u2 Q, then the G windows ascending): a doubling, a mid-chain infinity and a final infinity at every
    G window (vectors.chain_cases), plus the other kernels' chain cases as further adversarial inputs, interleaved with honest
    signatures at rows that are not warp aligned."""
    cases = _chain_cases()
    mix = vectors.mix_with_workload(cases)
    mask, off = ctx.verify_p256_host(*mix["soa"])
    bad = _chain_mismatches(cases, mix, mask_bits(mask, len(mix["valid"])).astype(bool))
    assert not bad and not off.any(), bad[:8]


def test_nil_key_empty_digest_statuses(csp):
    k = csp.KeyImport((p256.GX, p256.GY))
    good = goasn1.marshal_ecdsa_signature(5, 7)
    st = csp.VerifyBatch([k, None], [0, 1, 0, 0, -1], [b"\x01" * 32, b"\x01" * 32, b"", b"\x01" * 32, b"\x01" * 32], [good, good, good, b"", good])
    assert list(st) == [o.INVALID, o.ERR_NIL_KEY, o.ERR_EMPTY_DIGEST, o.ERR_EMPTY_SIG, o.ERR_NIL_KEY]


# ---------------------------------------------------------------------------------------------------------
# bccsp / msp interface behaviour (reads like bccsp/sw/ecdsa_test.go, bccsp/sw/impl_test.go, msp/msp_test.go)
# ---------------------------------------------------------------------------------------------------------
def test_verify_error_strings_match_reference(csp):
    d = 0x1F2E3D4C
    k = csp.KeyImport(p256.scalar_mult(d, (p256.GX, p256.GY)))
    msg = b"hello world"                                   # bccsp/sw/ecdsa_test.go:47-56 uses the message as digest
    r, s = p256.ecdsa_sign_lows(d, msg, 0xABCDEF)
    sigma = goasn1.marshal_ecdsa_signature(r, s)
    ok = o.P256PublicKey(k.x, k.y)
    for key, sig, dig in ((k, sigma, msg), (k, None, msg), (k, b"", msg), (k, sigma, b""), (None, sigma, msg),
                          (k, goasn1.marshal_ecdsa_signature(r, p256.HALF_N + 1), msg), (k, goasn1.marshal_ecdsa_signature(-1, 1), msg),
                          (k, goasn1.marshal_ecdsa_signature(1, 0), msg), (k, sigma[1:], msg), (k, sigma, msg[1:]),
                          (k, goasn1.marshal_ecdsa_signature(p256.N, s), msg)):
        got = csp.Verify(key, sig, dig, None)
        exp = o.csp_verify(ok if key is not None else None, sig, dig)
        assert got[0] == exp[0]
        if exp[1] is None:
            assert got[1] is None
        elif "asn1:" in exp[1]:
            assert got[1].startswith("Failed verifing with opts [<nil>]: Failed unmashalling signature [failed unmashalling signature [asn1: ")
        else:
            assert got[1] == exp[1]
    assert csp.Verify(k, sigma, msg, None) == (True, None)
    valid, err = csp.Verify(k, goasn1.marshal_ecdsa_signature(r, p256.HALF_N + 1), msg, None)
    assert not valid and "Invalid S. Must be smaller than half the order [" in err
    assert "Unsupported 'VerifyKey' provided [" in csp.Verify(object(), sigma, msg, None)[1]


def test_identity_verify(csp):
    # msp/msp_test.go:494-625 TestSignAndVerify / _Failures / OtherHash / longMessage
    d = 0x5EED5EED5EED
    pk = csp.KeyImport(p256.scalar_mult(d, (p256.GX, p256.GY)))
    import hashlib
    for fam, h in ((pkg().bccsp.SHA2, hashlib.sha256), (pkg().bccsp.SHA3, hashlib.sha3_256)):
        ident = pkg().bccsp.Identity(csp, pk, fam)
        for msg in (b"foo", b"x" * 100000):
            r, s = p256.ecdsa_sign_lows(d, h(msg).digest(), 0x1234567 + len(msg))
            sig = goasn1.marshal_ecdsa_signature(r, s)
            assert ident.Verify(msg, sig) is None
            assert ident.Verify(msg[1:], sig) == "The signature is invalid"
            assert ident.Verify(msg, sig[1:]).startswith("could not determine the validity of the signature: Failed verifing with opts")
            assert o.identity_verify(o.P256PublicKey(pk.x, pk.y), msg, sig, fam) is None


def test_fault_injection_never_reports_invalid(ctx):
    w = workload.Workload(64, 2, seed=3)
    b = pkg().binding
    os.environ["FABGPU_FAULT_INJECT"] = "1"
    try:
        with pytest.raises(b.FabGpuError) as ei:
            ctx.verify_p256_host(w.qx(), w.qy(), w.digest, w.r, w.s)
        assert ei.value.code == b.E_INJECTED
    finally:
        del os.environ["FABGPU_FAULT_INJECT"]
    mask, _ = ctx.verify_p256_host(w.qx(), w.qy(), w.digest, w.r, w.s)
    assert (mask == 0xFFFFFFFF).all()


def test_device_resident_entry_with_torch_stream(ctx):
    import torch
    w = workload.Workload(8192, 16, seed=31)
    w.tamper_r(0.07)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(a).to(dev) for a in (w.qx(), w.qy(), w.digest, w.r, w.s)]
    mask = torch.zeros(w.n // 32, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev)
    ctx.verify_p256_device(*[x.data_ptr() for x in t], w.n, mask.data_ptr(), 0, st.cuda_stream)
    st.synchronize()
    assert (mask.cpu().numpy().view(np.uint32) == exp).all()


# ---------------------------------------------------------------------------------------------------------
# per-key fixed-base tables (fabgpu_keys_register + the _keyed entry points)
# ---------------------------------------------------------------------------------------------------------
def _fill(ctx, slot, w, key_slots):
    hb = ctx.host_buffers(slot)
    for name, arr in (("qx", w.qx()), ("qy", w.qy()), ("e", w.digest), ("r", w.r), ("s", w.s)):
        hb[name][: w.n] = arr
    ctx.host_key_slots(slot)[: w.n] = key_slots
    return hb


def test_key_tables_all_cached_and_mixed(ctx):
    w = workload.Workload(16384, 32, seed=41)
    w.tamper_r(0.05)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    slots = ctx.keys_register(w.keys_xy)
    assert (slots >= 0).all() and len(set(slots.tolist())) == 32
    assert (ctx.keys_register(w.keys_xy) == slots).all()           # second lookup hits the cache
    hb = _fill(ctx, 0, w, slots[w.key_idx])
    ctx.verify_p256_keyed(0, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all() and not hb["offcurve"][: w.n // 32].any()
    # mixed batch: signatures of odd keys take the generic kernel
    hb = _fill(ctx, 1, w, np.where(w.key_idx % 2 == 0, slots[w.key_idx], -1))
    ctx.verify_p256_keyed(1, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all()
    # no key cached at all through the keyed entry point
    hb = _fill(ctx, 0, w, np.full(w.n, -1, np.int32))
    ctx.verify_p256_keyed(0, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all()
    # ragged n
    hb = _fill(ctx, 0, w, slots[w.key_idx])
    ctx.verify_p256_keyed(0, 1000)
    assert (mask_bits(hb["mask"], 1000) == mask_bits(exp, 1000)).all()


def test_key_tables_device_resident(ctx):
    import torch
    w = workload.Workload(8192, 8, seed=43)
    w.tamper_r(0.1)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    slots = ctx.keys_register(w.keys_xy)
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(a).to(dev) for a in (w.qx(), w.qy(), w.digest, w.r, w.s)]
    ks = torch.from_numpy((slots & 0xFFF)[w.key_idx]).to(dev)      # raw slot indices for the device-resident API
    mask = torch.zeros(w.n // 32, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev)
    ctx.verify_p256_device_keyed(True, ks.data_ptr(), 0, 0, t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(), w.n, mask.data_ptr(), 0, st.cuda_stream)
    st.synchronize()
    assert (mask.cpu().numpy().view(np.uint32) == exp).all()


def test_key_table_eviction_and_off_curve_keys():
    os.environ["FABGPU_KEY_SLOTS"] = "4"
    try:
        c = pkg().binding.Context(max_batch=4096)
    finally:
        del os.environ["FABGPU_KEY_SLOTS"]
    assert c.key_slot_capacity() == 4
    w = workload.Workload(2048, 6, seed=47)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    s1 = c.keys_register(w.keys_xy[:4])
    assert sorted(s1.tolist()) == [0, 1, 2, 3]
    s2 = c.keys_register(w.keys_xy[2:6])                  # keys 2,3 stay; 4,5 evict the two least recently used (0,1)
    assert (s2[:2] == s1[2:4]).all() and sorted((s2[2:] & 0xFFF).tolist()) == sorted(s1[:2].tolist())
    assert (s2[2:] >> 12 == 1).all()                      # recycled slots carry a new generation
    # handles of the evicted keys 0 and 1 are stale now: the keyed entry point must fall back to the generic kernel for
    # them (correct answers), never read the tables that now belong to keys 4 and 5
    stale = np.concatenate([s1[:2], s2])                  # handles for keys 0..5, the first two stale
    hb = _fill(c, 0, w, stale[w.key_idx])
    c.verify_p256_keyed(0, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all()
    assert (c.host_key_slots(0)[: w.n][w.key_idx < 2] == -1).all()
    all6 = c.keys_register(w.keys_xy)                     # six keys, four slots: two stay generic
    assert int((all6 < 0).sum()) == 2
    hb = _fill(c, 0, w, all6[w.key_idx])
    c.verify_p256_keyed(0, w.n)
    assert (hb["mask"][: w.n // 32] == exp).all()
    bad = w.keys_xy[:1].copy(); bad[0, 63] ^= 1           # not a curve point: no table
    assert c.keys_register(bad)[0] == -1
    c.close()


def test_bccsp_batch_with_forced_key_tables():
    """Every key registered (FABGPU_KEY_MIN_USES=1): statuses must equal the generic path's and the oracle's."""
    os.environ["FABGPU_KEY_MIN_USES"] = "1"
    try:
        csp2 = pkg().bccsp.GPUCSP(max_batch=4096)
    finally:
        del os.environ["FABGPU_KEY_MIN_USES"]
    cases = vectors.build()
    keys = [csp2.KeyImport((c["qx"] % R, c["qy"] % R)) for c in cases]
    st = csp2.VerifyBatch(keys, list(range(len(cases))), [c["digest"] for c in cases], [c["sig"] for c in cases])
    for c, got in zip(cases, st):
        assert int(got) == vectors.expected_status(c), c["name"]
    w = workload.Workload(3000, 5, seed=53)
    w.tamper_r(0.2)
    exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)
    assert (csp2.ctx.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off) == exp).all()
    csp2.close()


def test_bccsp_batch_large_call_is_chunked_over_the_slots():
    """A blocking fabgpu_bccsp_verify_batch call of >= 24576 signatures is cut into one chunk per slot (offset tables windowed,
    blobs rebased on the device): statuses must equal the oracle's across the chunk boundaries, with damaged DER, empty
    signatures / digests and nil keys sprinkled in, and while another thread's async batch occupies a slot (single-slot path)."""
    c = pkg().binding.Context(max_batch=1 << 16)
    w = workload.Workload(40003, 7, seed=77)
    w.tamper_r(0.07)
    rnd = random.Random(5)
    sigs = bytearray(w.sigs.tobytes())
    for i in rnd.sample(range(w.n), 900):                    # damage one byte of the DER header / integer headers / body
        o_ = int(w.sig_off[i]); ln = int(w.sig_off[i + 1]) - o_
        sigs[o_ + rnd.choice([0, 1, 2, 3, 4, ln - 1, rnd.randrange(ln)])] ^= 1 << rnd.randrange(8)
    sigs = np.frombuffer(bytes(sigs), np.uint8)
    kidx = w.key_idx.copy()
    kidx[rnd.sample(range(w.n), 50)] = -1                    # nil keys
    kidx[rnd.sample(range(w.n), 50)] = 7                     # not a key of the table
    exp = fast.verify_batch(w.keys_xy, kidx, w.digest, w.dig_off(), sigs, w.sig_off, nthreads=os.cpu_count())
    assert len(set(exp.tolist())) >= 6
    got = c.bccsp_verify_batch(w.keys_xy, kidx, w.digest, w.dig_off(), sigs, w.sig_off)
    assert (got == exp).all()
    # a slot is taken by an async batch: the blocking call must still be exact (it then goes through slot 0 alone)
    small = workload.Workload(2000, 2, seed=78)
    nn = c.bccsp_verify_batch_async(2, small.keys_xy, small.key_idx, small.digest, small.dig_off(), small.sigs, small.sig_off)
    assert (c.bccsp_verify_batch(w.keys_xy, kidx, w.digest, w.dig_off(), sigs, w.sig_off) == exp).all()
    assert (c.bccsp_verify_batch_wait(2, nn) == 0).all()
    c.close()


def test_bccsp_batch_async_two_slots_in_flight():
    """fabgpu_bccsp_verify_batch_async / _wait: two different batches in flight on the two slots, several rounds; each
    slot's statuses must equal the oracle's for ITS batch (no cross-talk between the slots' buffers), in either gate mode."""
    c = pkg().binding.Context(max_batch=8192)
    ws = []
    for k, (n, keys, seed) in enumerate([(5000, 3, 71), (3777, 400, 72)]):       # second batch: most keys below the table threshold
        w = workload.Workload(n, keys, seed=seed)
        w.tamper_r(0.1 + 0.2 * k)
        exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)
        ws.append((w, exp))
    for host_gates in ("0", "1"):
        os.environ["FABGPU_BCCSP_HOST_GATES"] = host_gates
        try:
            for rnd in range(3):
                order = (0, 1) if rnd % 2 == 0 else (1, 0)
                ns = {}
                for sl in order:
                    w = ws[sl][0]
                    ns[sl] = c.bccsp_verify_batch_async(sl, w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off)
                with pytest.raises(pkg().binding.FabGpuError):                  # a slot holds one batch at a time
                    w = ws[0][0]
                    c.bccsp_verify_batch_async(0, w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off)
                for sl in order:
                    got = c.bccsp_verify_batch_wait(sl, ns[sl])
                    assert (got == ws[sl][1]).all(), (host_gates, rnd, sl)
            with pytest.raises(pkg().binding.FabGpuError):                      # nothing in flight
                c.bccsp_verify_batch_wait(0, 1)
        finally:
            del os.environ["FABGPU_BCCSP_HOST_GATES"]
    # the blocking call still works after async use, and an empty batch goes through both halves
    w, exp = ws[0]
    assert (c.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off) == exp).all()
    n0 = c.bccsp_verify_batch_async(1, w.keys_xy, np.zeros(0, np.int32), np.zeros(0, np.uint8), np.zeros(1, np.uint32), np.zeros(0, np.uint8), np.zeros(1, np.uint32))
    assert n0 == 0 and c.bccsp_verify_batch_wait(1, 0).shape[0] == 0
    c.close()


@pytest.mark.parametrize("variant", ["jac", "ba", "ba2", "l2", "l4"])
def test_key_table_kernel_variants_are_bit_exact(variant):
    """Every key-table kernel shape that was built and measured (DESIGN.md section 4.1; FABGPU_CACHED_KERNEL) gives the oracle's bits:
    5 % tampered batch of ragged size through the keyed leaf, and the adversarial vectors through the bccsp-level call with every key
    tabled (u1 = 0, u1 G = +-u2 Q, x(R) >= n, zero digits ...)."""
    os.environ["FABGPU_CACHED_KERNEL"] = variant
    os.environ["FABGPU_KEY_MIN_USES"] = "1"
    try:
        c = pkg().binding.Context(max_batch=1 << 15)
    finally:
        del os.environ["FABGPU_CACHED_KERNEL"]
        del os.environ["FABGPU_KEY_MIN_USES"]
    try:
        _check_key_table_variant(c, variant)
    finally:
        c.close()                       # a failing variant must not leave its tables on the device for the next one


def _check_key_table_variant(c, variant):
    w = workload.Workload(20000 + 7, 16, seed=workload.DEFAULT_SEED + 21)
    w.tamper_r(0.05)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=os.cpu_count()))
    handles = c.keys_register(w.keys_xy)
    assert (handles >= 0).all()
    hb = _fill(c, 0, w, handles[w.key_idx])
    c.verify_p256_keyed(0, w.n)
    assert (hb["mask"][: exp.shape[0]] == exp).all()
    cases = [cs for cs in vectors.build() if len(cs["sig"]) and cs["qx"] < p256.P and cs["qy"] < p256.P]
    keys = np.stack([np.concatenate([be32(cs["qx"]), be32(cs["qy"])]) for cs in cases])
    digs, sigs = [cs["digest"] for cs in cases], [cs["sig"] for cs in cases]
    doff = np.zeros(len(cases) + 1, np.uint32); doff[1:] = np.cumsum([len(d) for d in digs])
    soff = np.zeros(len(cases) + 1, np.uint32); soff[1:] = np.cumsum([len(x) for x in sigs])
    st = c.bccsp_verify_batch(keys, np.arange(len(cases), dtype=np.int32), np.frombuffer(b"".join(digs), np.uint8), doff, np.frombuffer(b"".join(sigs), np.uint8), soff)
    for cs, got in zip(cases, st):
        assert int(got) == vectors.expected_status(cs), (variant, cs["name"])
    # the chain-collision cases of this kernel's own addition order (a doubling or an infinity at every step that can collide, the
    # lane combines and the batch-affine tail included) and of the Jacobian chain, interleaved with honest signatures so that every
    # CTA mixes both, through the keyed leaf.  One window table per distinct key: all of them fit, nothing is evicted.
    own = {"jac": ("jac",), "ba": ("ba", "jac"), "ba2": ("ba", "jac"), "l2": ("l2", "jac"), "l4": ("l4", "jac")}[variant]
    cases = _chain_cases(own)
    mix = vectors.mix_with_workload(cases)
    handles = c.keys_register(mix["keys_xy"])
    assert (handles >= 0).all() and mix["keys_xy"].shape[0] < c.key_slot_capacity()
    n = len(mix["valid"])
    hb = _fill_soa(c, 1, mix["soa"], handles[mix["kidx"]])
    c.verify_p256_keyed(1, n)
    bad = _chain_mismatches(cases, mix, mask_bits(hb["mask"], n).astype(bool))
    assert not bad, (variant, bad[:8])


def test_bccsp_batch_inplace_pinned_buffers_match_the_copying_form():
    """fabgpu_bccsp_batch_buffers + fabgpu_bccsp_verify_batch_inplace_async: the batch is written straight into the slot's pinned
    buffers; statuses must equal the staging form's and the oracle's, slot after slot, including a ragged adversarial tail."""
    from tools import parity_workload as pw
    c = pkg().binding.Context(max_batch=8192)
    sh = pw.Shard(0, 1, 6000, 12, nthreads=8)                        # 5 % tampered r + the tests/vectors.py tail (ragged digests, bad DER)
    exp = pw.oracle_status(sh, 8)
    ref = c.bccsp_verify_batch(*sh.args())
    assert (ref == exp).all()
    for slot in range(pkg().binding.SLOTS):
        K, n = c.bccsp_fill_batch_buffers(slot, *sh.args())
        assert n == sh.n
        c.bccsp_verify_batch_inplace_async(slot, K, n)
    for slot in range(pkg().binding.SLOTS):
        got = c.bccsp_verify_batch_wait(slot, sh.n)
        assert (got == exp).all(), slot
    # resubmitting a slot reuses the bytes it holds; an oversized batch is refused
    c.bccsp_verify_batch_inplace_async(0, K, 100)
    assert (c.bccsp_verify_batch_wait(0, 100) == exp[:100]).all()
    with pytest.raises(pkg().binding.FabGpuError):
        c.bccsp_verify_batch_inplace_async(1, K, 1 << 20)
    c.close()


# ---------------------------------------------------------------------------------------------------------
# one context driving several GPUs (what the Go provider does: Devices: [0..7] in core.yaml)
# ---------------------------------------------------------------------------------------------------------
def test_multi_device_context_splits_batch():
    import torch
    ndev = min(torch.cuda.device_count(), 4)
    # On a 1-GPU box the context is given device 0 twice: two device entries (own streams, tables and buffers), so the split /
    # per-device launch / mask reassembly logic runs exactly as it does over distinct GPUs.
    ids = list(range(ndev)) if ndev >= 2 else [0, 0]
    ndev = len(ids)
    c = pkg().binding.Context(max_batch=1 << 17, device_ids=ids)
    assert c.device_count() == ndev
    # BASELINE.json configs[4] shape at reduced size: 5 % tampered r, exact-match bitmask (generic kernel, then key tables)
    w = workload.Workload(100000 + 77, 64, seed=workload.DEFAULT_SEED + 5)        # ragged: not a multiple of 32 * ndev
    w.tamper_r(0.05)
    exp = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=os.cpu_count()))
    mask, off = c.verify_p256_host(w.qx(), w.qy(), w.digest, w.r, w.s)
    assert (mask == exp).all() and not off.any()
    handles = c.keys_register(w.keys_xy)                                          # tables on every device of the context
    assert (handles >= 0).all()
    hb = _fill(c, 1, w, handles[w.key_idx])
    c.verify_p256_keyed(1, w.n)
    assert (hb["mask"][: exp.shape[0]] == exp).all()
    st = c.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off)
    assert (fast.valid_mask(st) == exp).all()
    c.close()
