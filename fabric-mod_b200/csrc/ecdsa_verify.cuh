// One ECDSA-P256 verification, written once for device (the product) and host (tests/host_sim).
//
// Restates, for the GPU, what the reference reaches at bccsp/sw/ecdsa.go:56 -- Go 1.14 crypto/ecdsa.Verify:
//   r,s in [1,n-1]  ->  w = s^-1 mod n  ->  u1 = e*w, u2 = r*w  ->  R = u1*G + u2*Q  ->  R != inf and R.x mod n == r.
// The DER parse, positivity and low-S gates (bccsp/utils/ecdsa.go:43-92, bccsp/sw/ecdsa.go:42-54) run before these
// functions -- in bccsp_gate_kernel / block_resolve_kernel (blockdev.cuh) or on host threads (bccsp_host.cpp); the
// functions below still enforce the range checks r, s in [1, n-1] themselves.
//
// Scalar multiplication layout (GPU-first, not Go's CombinedMult):
//   u1*G : fixed-base, FAB_WG-bit unsigned windows over a precomputed affine table in HBM/L2
//          (ceil(256/FAB_WG) mixed additions, no doublings);
//   u2*Q : keys with a table (ecdsa_verify_one_cached): FAB_WQ-bit unsigned windows over the key's own table;
//          keys without (ecdsa_verify_one): signed 5-bit Booth windows, 16-entry Jacobian table of 1Q..16Q per signature.
// The window chains accumulate in XYZZ coordinates (p256_point.cuh), the generic kernel in Jacobian ones.
// The final comparison avoids the field inversion: R.x == r' * R.ZZ (Jacobian: r' * R.Z^2) for r' in {r, r+n (if < p)}.
#pragma once
#include "p256_point.cuh"
#include "p256_modinv.cuh"

#ifndef FAB_WG
#define FAB_WG 22                     // window bits of the fixed-base table of G: 12 windows x 4 194 303 points = 3.2 GB per
#endif                                // device, 12 mixed additions for u1*G (wider windows: fewer additions for more memory)
#ifndef FAB_WQ
#define FAB_WQ 16                     // window bits of the per-key tables: 16 windows x 65 535 points = 64 MiB per key,
#endif                                // 16 mixed additions for u2*Q
#ifndef FAB_CACHED_INLINE
#define FAB_CACHED_INLINE 1              // the key-table kernel expands the field multiplications of its point addition in place
                                      // (one copy, ~34 KB of code): no argument moves for 8 calls per addition
#endif
#define FAB_Q_WINDOWS ((256 + FAB_WQ - 1) / FAB_WQ)
#define FAB_Q_ENTRIES ((1 << FAB_WQ) - 1)
#ifndef FAB_JAC_NEXT_PREFETCH
#define FAB_JAC_NEXT_PREFETCH 1      // request the next window's table entry from the L2 during the current addition
#endif
#ifndef FAB_JAC_L2PREFETCH
#define FAB_JAC_L2PREFETCH 0
#endif
#ifndef FAB_SAFEGCD
#define FAB_SAFEGCD 1
#endif
#define FAB_G_WINDOWS ((256 + FAB_WG - 1) / FAB_WG)
#define FAB_G_ENTRIES ((1 << FAB_WG) - 1)

namespace fabgpu {

enum : uint32_t { V_INVALID = 0u, V_VALID = 1u, V_OFFCURVE = 2u };

// 6-bit Booth window -> (negative?, |digit| in 0..16)
FAB_HD void booth5(uint32_t w6, uint32_t& neg, uint32_t& mag)
{
    neg = w6 >> 5;
    const uint32_t d = neg ? (63u - w6) : w6;
    mag = (d >> 1) + (d & 1u);
}

// out = (k+1)*Q for k = 0..15 (Jacobian)
FAB_HD void build_q_table(jac* tab, const aff& q)
{
    tab[0] = jac_from_aff(q);
    tab[1] = jac_double(tab[0]);
    for (int k = 2; k < 16; k++) tab[k] = jac_add_aff(tab[k - 1], q);
}

// u2 * Q by signed 5-bit windows.  k9 holds u2 << 28 in 9 limbs so that the current 6-bit Booth window
// (bits 5i+4 .. 5i-1 of u2) is always the top 6 bits; it is shifted left by 5 per window (no dynamic limb index).
FAB_HD jac scalar_mul_var(const u256& k, const jac* tab)
{
    uint32_t k9[9];
    k9[0] = k.v[0] << 28;
#pragma unroll
    for (int i = 1; i < 8; i++) k9[i] = (k.v[i] << 28) | (k.v[i - 1] >> 4);
    k9[8] = k.v[7] >> 4;
    jac r = jac_infinity();
    for (int i = 51; i >= 0; i--) {
        if (i != 51) {
            for (int d = 0; d < 5; d++) r = jac_double(r);
        }
        uint32_t neg, mag;
        booth5(k9[8] >> 26, neg, mag);
#pragma unroll
        for (int j = 8; j > 0; j--) k9[j] = (k9[j] << 5) | (k9[j - 1] >> 27);
        k9[0] <<= 5;
        if (mag) {
            jac t = tab[mag - 1];
            if (neg) t.Y = fe_neg(t.Y);
            r = jac_add(r, t);
        }
    }
    return r;
}

// Hint the table entry the NEXT window will need into the cache while the current addition runs (no register cost).
FAB_HD void prefetch_entry(const aff* p)
{
#if defined(__CUDA_ARCH__) && defined(FAB_PREFETCH)   /* opt-in: measured neutral-to-negative (L2 hit rates are already high) */
    asm volatile("prefetch.global.L2 [%0];" :: "l"(p));
#else
    (void)p;
#endif
}

// The window chains' table gathers go through here: one register copy made of four 128-bit loads on the read-only path.  Handed a
// reference into global memory instead, the expanded addition loads each limb where it uses it: 16 scalar loads per point, each a
// divergent request of its own, since every lane of a warp gathers a different random point.  Tables are cudaMalloc'ed arrays of
// 64-byte points (16-byte aligned) that no kernel writes while a verification reads them.
FAB_HD aff load_aff_nc(const aff* p)
{
#if defined(__CUDA_ARCH__)
    const uint4* q = reinterpret_cast<const uint4*>(p);
    const uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
    aff r;
    r.x = u256_const(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w);
    r.y = u256_const(c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w);
    return r;
#else
    return *p;
#endif
}

// r += u1 * G using the fixed-base table gtab[window][digit-1] (affine, Montgomery form)
FAB_HD jac add_fixed_base(jac r, const u256& k, const aff* gtab)
{
    uint32_t kk[8];
#pragma unroll
    for (int i = 0; i < 8; i++) kk[i] = k.v[i];
    for (int j = 0; j < FAB_G_WINDOWS; j++) {
        const uint32_t d = kk[0] & (uint32_t)FAB_G_ENTRIES;
#pragma unroll
        for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> FAB_WG) | (kk[i + 1] << (32 - FAB_WG));
        kk[7] >>= FAB_WG;
        const uint32_t dn = kk[0] & (uint32_t)FAB_G_ENTRIES;
        if (dn && j + 1 < FAB_G_WINDOWS) prefetch_entry(gtab + (size_t)(j + 1) * FAB_G_ENTRIES + (dn - 1));
        if (d) r = jac_add_aff(r, load_aff_nc(gtab + (size_t)j * FAB_G_ENTRIES + (d - 1)));
    }
    return r;
}

// x = X / zz of a finite point: valid iff x mod n == r, i.e. X == r' * zz for r' in {r, r + n (only when r + n < p)}.
FAB_HD uint32_t x_check(const u256& X, const u256& zz, const u256& r)
{
    const u256 n = sc_n();
    if (u256_eq(fe_mul(fe_to_mont(r), zz), X)) return V_VALID;
    if (u256_lt(r, p_minus_n())) {                    // x mod n == r also when x = r + n < p
        u256 rn; uint32_t c = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const uint32_t a = r.v[i], b = n.v[i];
            const uint32_t t = a + b; const uint32_t c1 = t < a;
            const uint32_t t2 = t + c; const uint32_t c2 = t2 < t;
            rn.v[i] = t2; c = c1 | c2;
        }
        if (u256_eq(fe_mul(fe_to_mont(rn), zz), X)) return V_VALID;
    }
    return V_INVALID;
}

// Accept iff acc != infinity (Go: x == 0 && y == 0 -> false) and acc.x mod n == r, without leaving the projective coordinates.
FAB_HD uint32_t final_check(const jac& acc, const u256& r)
{
    if (jac_is_infinity(acc)) return V_INVALID;
    return x_check(acc.X, fe_sqr(acc.Z), r);
}
FAB_HD uint32_t final_check(const xyzz& acc, const u256& r)
{
    if (u256_is_zero(acc.ZZ)) return V_INVALID;
    return x_check(acc.X, acc.ZZ, r);
}

// All five inputs are plain 256-bit integers (e already formed by hashToInt: leftmost 32 digest bytes, left-padded).
FAB_HD uint32_t ecdsa_verify_one(const u256& qx, const u256& qy, const u256& e, const u256& r, const u256& s, const aff* gtab)
{
    const u256 n = sc_n();
    const u256 p = fe_p();
    // Go: r.Sign() <= 0 || s.Sign() <= 0 -> false ; r >= N || s >= N -> false
    if (u256_is_zero(r) || u256_is_zero(s) || !u256_lt(r, n) || !u256_lt(s, n)) return V_INVALID;
    // Q must be a curve point: Go's Verify does not check, so off-curve keys are outside the restated domain
    // and are reported separately (the host routes them to the CPU provider).
    if (!u256_lt(qx, p) || !u256_lt(qy, p)) return V_OFFCURVE;
    aff q; q.x = fe_to_mont(qx); q.y = fe_to_mont(qy);
    if (!aff_on_curve(q)) return V_OFFCURVE;

#if FAB_SAFEGCD
    const u256 w = sc_inv_to_mont_safegcd(s);         // s^-1 * 2^256 mod n (division steps, p256_modinv.cuh)
#else
    const u256 w = sc_inv_to_mont(s);                 // s^-1 * 2^256 mod n (Fermat)
#endif
    const u256 u1 = sc_mul(sc_reduce_once(e), w);     // e*w mod n, plain
    const u256 u2 = sc_mul(r, w);                     // r*w mod n, plain

    jac tab[16];
    build_q_table(tab, q);
    jac acc = scalar_mul_var(u2, tab);
    acc = add_fixed_base(acc, u1, gtab);
    return final_check(acc, r);
}

// u1 = e*w mod n, u2 = r*w mod n (plain) from w = s^-1 * 2^256 mod n.  For r, s in [1, n-1] u2 is never 0 (n is prime).
FAB_HD void ecdsa_u1u2(const u256& e, const u256& r, const u256& w, u256& u1, u256& u2)
{
    u1 = sc_mul(sc_reduce_once(e), w);
    u2 = sc_mul(r, w);
}

// The two scalars of a chain held in registers: scalar(0) = u1, scalar(1) = u2.
struct ChainScalars {
    u256 u1, u2;
    FAB_HD u256 operator()(int t) const { return t ? u2 : u1; }
};

// The point of a verification when the public key has a precomputed window table (fabgpu_keys_register): from the scalars u1, u2,
// R = u1*G + u2*Q with u2*Q fixed-base too -- FAB_G_WINDOWS + FAB_Q_WINDOWS mixed additions in total, no doublings, no per-signature
// table.  The caller checks R against r (final_check).  The key was checked to be a curve point when its table was built.
// ecdsa_verify_cached_kernel runs this on the scalars ecdsa_prep_kernel computed, read from memory where the chain needs them
// (Scalars: a functor, scalar(t) for t = 0, 1); ecdsa_verify_one_cached below is the whole verification for one signature.
template <class Scalars> FAB_HD xyzz ecdsa_chain_cached(const aff* qtab, const Scalars& scalar, const aff* gtab)
{
    // One loop over both tables -- 12 windows of u1 in the generator's table, then 16 windows of u2 in the key's table -- so that
    // the kernel holds a single copy of the point addition (expanded in place when FAB_CACHED_INLINE).
    xyzz acc = xyzz_infinity();
#if defined(__CUDA_ARCH__) && FAB_JAC_L2PREFETCH
    // every table entry this signature will gather, requested from the L2 up front (the tables are HBM-resident: 3.2 GB + 64 MiB per key)
#pragma unroll 1
    for (int t = 0; t < 2; t++) {
        uint32_t kk[8];
        const u256 k = scalar(t);
#pragma unroll
        for (int i = 0; i < 8; i++) kk[i] = k.v[i];
        const aff* tab = t ? qtab : gtab;
        const uint32_t wbits = t ? FAB_WQ : FAB_WG, entries = (1u << wbits) - 1u;
        const int windows = t ? FAB_Q_WINDOWS : FAB_G_WINDOWS;
#pragma unroll 1
        for (int j = 0; j < windows; j++) {
            const uint32_t d = kk[0] & entries;
#pragma unroll
            for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> wbits) | (kk[i + 1] << (32u - wbits));
            kk[7] >>= wbits;
            if (d) asm volatile("prefetch.global.L2 [%0];" :: "l"(tab + (size_t)j * entries + (d - 1)));
        }
    }
#endif
    // cur: this window's entry (nullptr for a zero digit).  Each pass forms the NEXT window's entry address once, for its prefetch and
    // as the next pass's gather address.
    const uint32_t d0 = scalar(0).v[0] & (uint32_t)FAB_G_ENTRIES, dq0 = scalar(1).v[0] & (uint32_t)FAB_Q_ENTRIES;
    const aff* cur = d0 ? gtab + (d0 - 1) : nullptr;
#pragma unroll 1
    for (int t = 0; t < 2; t++) {
        uint32_t kk[8];
        const u256 k = scalar(t);
#pragma unroll
        for (int i = 0; i < 8; i++) kk[i] = k.v[i];
        const aff* tab = t ? qtab : gtab;
        const uint32_t wbits = t ? FAB_WQ : FAB_WG, entries = (1u << wbits) - 1u;
        const int windows = t ? FAB_Q_WINDOWS : FAB_G_WINDOWS;
#pragma unroll 1
        for (int j = 0; j < windows; j++) {
#pragma unroll
            for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> wbits) | (kk[i + 1] << (32u - wbits));
            kk[7] >>= wbits;
            // the entry of the next window (or the first window of the key's table)
            const aff* nx = nullptr;
            if (j + 1 < windows) { const uint32_t dn = kk[0] & entries; if (dn) nx = tab + (size_t)(j + 1) * entries + (dn - 1); }
            else if (t == 0 && dq0) nx = qtab + (dq0 - 1);
#if defined(__CUDA_ARCH__) && FAB_JAC_NEXT_PREFETCH
            // requested from the L2 while this addition runs: the tables are HBM-resident, so without it one DRAM round trip per
            // addition is exposed
            if (nx) asm volatile("prefetch.global.L2 [%0];" :: "l"(nx));
#endif
            if (cur) acc = xyzz_add_aff_t<FAB_CACHED_INLINE != 0>(acc, load_aff_nc(cur));
            cur = nx;
        }
    }
    return acc;
}

// One signature through a key's window table, scalars included (one inversion of its own).
FAB_HD uint32_t ecdsa_verify_one_cached(const aff* qtab, const u256& e, const u256& r, const u256& s, const aff* gtab)
{
    const u256 n = sc_n();
    if (u256_is_zero(r) || u256_is_zero(s) || !u256_lt(r, n) || !u256_lt(s, n)) return V_INVALID;
#if FAB_SAFEGCD
    const u256 w = sc_inv_to_mont_safegcd(s);
#else
    const u256 w = sc_inv_to_mont(s);
#endif
    ChainScalars sc;
    ecdsa_u1u2(e, r, w, sc.u1, sc.u2);
    return final_check(ecdsa_chain_cached(qtab, sc, gtab), r);
}

// ---- small key tables: the tier between "never seen" and a 64 MiB window table --------------------------------------------------
// A key that recurs but not often enough to earn the big table (client / creator certificates: thousands of identities, a few
// signatures per block each) gets FAB_S_WINDOWS windows of SIGNED FAB_WS-bit digits: entry (j, d) = d * 2^(FAB_WS j) * Q for
// d = 1 .. 2^(FAB_WS-1); a negative digit is the same entry with Y negated.  u2*Q = at most FAB_S_WINDOWS mixed additions and no
// doublings, against 255 doublings + 52 additions of the generic kernel.  Windows cover >= 257 bits, so the carry of the signed
// recoding is always absorbed by the last window.  Each halving of the window count buys what the additions it removes cost, so
// the width is set by memory (tests/test_host_sim.py checks the 5-, 6- and 7-bit builds on the host):
//   FAB_WS   windows   table
//     5        52       52 KiB
//     6        43       86 KiB
//     7        37      148 KiB
//     8        33      264 KiB     <- default: 16 384 tables are 4.4 GB of an H100's 80 GB
#ifndef FAB_WS
#define FAB_WS 8
#endif
#define FAB_S_WINDOWS ((257 + FAB_WS - 1) / FAB_WS)
#define FAB_S_HALF (1 << (FAB_WS - 1))
#define FAB_S_POINTS (FAB_S_WINDOWS * FAB_S_HALF)
#define FAB_S_SEG 32                  /* entries normalised per shared inversion when a window is built (bounds the builder's frame) */

// r += k * Q through Q's small table: signed FAB_WS-bit digits, least significant window first, the carry of a negative digit
// moves into the next window (k < 2^256 and the windows cover 258 bits: the last one absorbs it).
FAB_HD jac add_small_table(jac acc, const u256& k, const aff* stab)
{
    uint32_t kk[8];
#pragma unroll
    for (int i = 0; i < 8; i++) kk[i] = k.v[i];
    uint32_t carry = 0;
#pragma unroll 1
    for (int j = 0; j < FAB_S_WINDOWS; j++) {
        uint32_t d = (kk[0] & ((1u << FAB_WS) - 1u)) + carry;
#pragma unroll
        for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> FAB_WS) | (kk[i + 1] << (32 - FAB_WS));
        kk[7] >>= FAB_WS;
        const bool neg = d > (uint32_t)FAB_S_HALF;
        if (neg) d = (1u << FAB_WS) - d;
        carry = neg ? 1u : 0u;
        if (d) {
            aff pt = load_aff_nc(stab + (size_t)j * FAB_S_HALF + (d - 1));
            if (neg) pt.y = fe_neg(pt.y);
            acc = jac_add_aff(acc, pt);
        }
    }
    return acc;
}

// Same verification with a small table.  An all-zero first entry marks a key that is not a curve point (small_bases_kernel wrote it).
// One loop over both tables, like ecdsa_verify_one_cached (a single expanded copy of the point addition): 12 unsigned windows of u1 in
// the generator's table, then FAB_S_WINDOWS signed windows of u2 in the key's.
FAB_HD uint32_t ecdsa_verify_one_small(const aff* stab, const u256& e, const u256& r, const u256& s, const aff* gtab)
{
    const u256 n = sc_n();
    if (u256_is_zero(r) || u256_is_zero(s) || !u256_lt(r, n) || !u256_lt(s, n)) return V_INVALID;
    {
        const aff first = stab[0];
        if (u256_is_zero(first.x) && u256_is_zero(first.y)) return V_OFFCURVE;
    }
#if FAB_SAFEGCD
    const u256 w = sc_inv_to_mont_safegcd(s);
#else
    const u256 w = sc_inv_to_mont(s);
#endif
    const u256 u1 = sc_mul(sc_reduce_once(e), w);
    const u256 u2 = sc_mul(r, w);
    xyzz acc = xyzz_infinity();
#pragma unroll 1
    for (int t = 0; t < 2; t++) {
        uint32_t kk[8];
#pragma unroll
        for (int i = 0; i < 8; i++) kk[i] = t ? u2.v[i] : u1.v[i];
        const aff* tab = t ? stab : gtab;
        const uint32_t wbits = t ? FAB_WS : FAB_WG, dmask = (1u << wbits) - 1u;
        const uint32_t stride = t ? (uint32_t)FAB_S_HALF : (uint32_t)FAB_G_ENTRIES;
        const uint32_t half = t ? (uint32_t)FAB_S_HALF : 0xffffffffu;          // the generator's digits are unsigned: never "negative"
        const int windows = t ? FAB_S_WINDOWS : FAB_G_WINDOWS;
        uint32_t carry = 0;
#pragma unroll 1
        for (int j = 0; j < windows; j++) {
            uint32_t d = (kk[0] & dmask) + carry;
#pragma unroll
            for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> wbits) | (kk[i + 1] << (32u - wbits));
            kk[7] >>= wbits;
            const bool neg = d > half;
            if (neg) d = (1u << wbits) - d;
            carry = neg ? 1u : 0u;
            if (d) {
                aff pt = load_aff_nc(tab + (size_t)j * stride + (d - 1));
                if (neg) pt.y = fe_neg(pt.y);
                acc = xyzz_add_aff_t<FAB_CACHED_INLINE != 0>(acc, pt);
            }
        }
    }
    return final_check(acc, r);
}

// Stage 1 of a small table, ONE thread per key: bases[j] = 2^(FAB_WS j) * Q (affine) for every window -- one chain of
// FAB_WS * (FAB_S_WINDOWS - 1) = 256 doublings, the Z's removed by one shared inversion.  Returns false (and writes nothing) when
// (x, y) is not a curve point.
FAB_HD bool small_bases(const u256& x, const u256& y, aff* bases)
{
    const u256 p = fe_p();
    if (!u256_lt(x, p) || !u256_lt(y, p)) return false;
    aff q; q.x = fe_to_mont(x); q.y = fe_to_mont(y);
    if (!aff_on_curve(q)) return false;
    u256 zs[FAB_S_WINDOWS], ps[FAB_S_WINDOWS];
    jac t = jac_from_aff(q);
    u256 run = fe_one();
    for (int j = 0; j < FAB_S_WINDOWS; j++) {
        if (j) for (int b = 0; b < FAB_WS; b++) t = jac_double(t);
        bases[j].x = t.X; bases[j].y = t.Y;
        zs[j] = t.Z;
        run = fe_mul(run, t.Z);
        ps[j] = run;
    }
    u256 inv = fe_inv_safegcd(run);                 // a point of odd prime order never doubles to infinity: run != 0
    for (int j = FAB_S_WINDOWS - 1; j >= 0; j--) {
        const u256 zi = (j > 0) ? fe_mul(inv, ps[j - 1]) : inv;
        if (j > 0) inv = fe_mul(inv, zs[j]);
        const u256 zi2 = fe_sqr(zi);
        bases[j].x = fe_mul(bases[j].x, zi2);
        bases[j].y = fe_mul(bases[j].y, fe_mul(zi2, zi));
    }
    return true;
}

// Stage 2, one thread per (key, window): out[d-1] = d * base for d = 1 .. FAB_S_HALF -- one chain of mixed additions, brought to
// affine FAB_S_SEG entries at a time (one shared division-step inversion per segment; the scratch lives in the thread's frame).
FAB_HD void small_window(const aff& base, aff* out)
{
    u256 zs[FAB_S_SEG], ps[FAB_S_SEG];
    jac t = jac_from_aff(base);
    for (int d0 = 1; d0 <= FAB_S_HALF; d0 += FAB_S_SEG) {
        const int cnt = (FAB_S_HALF - d0 + 1 < FAB_S_SEG) ? (FAB_S_HALF - d0 + 1) : FAB_S_SEG;
        u256 run = fe_one();
        for (int k = 0; k < cnt; k++) {
            if (d0 + k > 1) t = jac_add_aff(t, base);    // d = 2 takes the doubling branch of the complete addition
            out[d0 + k - 1].x = t.X; out[d0 + k - 1].y = t.Y;
            zs[k] = t.Z;
            run = fe_mul(run, t.Z);
            ps[k] = run;
        }
        u256 inv = fe_inv_safegcd(run);
        for (int k = cnt - 1; k >= 0; k--) {
            const u256 zi = (k > 0) ? fe_mul(inv, ps[k - 1]) : inv;
            if (k > 0) inv = fe_mul(inv, zs[k]);
            const u256 zi2 = fe_sqr(zi);
            out[d0 + k - 1].x = fe_mul(out[d0 + k - 1].x, zi2);
            out[d0 + k - 1].y = fe_mul(out[d0 + k - 1].y, fe_mul(zi2, zi));
        }
    }
}

// Fixed-base table entry (window j, digit d in 1..FAB_G_ENTRIES) = d * 2^(FAB_WG*j) * G, affine Montgomery.
FAB_HD aff table_entry(const aff& g, int wbits, int j, uint32_t d)
{
    jac acc = jac_infinity();
    // scalar = d << (wbits*j): MSB-first double-and-add over d's bits, then wbits*j doublings
    for (int b = wbits - 1; b >= 0; b--) {
        acc = jac_double(acc);
        if ((d >> b) & 1u) acc = jac_add_aff(acc, g);
    }
    for (int t = 0; t < wbits * j; t++) acc = jac_double(acc);
    return jac_to_aff(acc);
}
// out[d-1] = d * 2^shift * q for d = 1..count, built by ONE thread: chain of mixed additions from the affine base
// 2^shift q, then one shared inversion for the whole chain (Montgomery's trick).  zs / ps: scratch of `count` elements each.
FAB_HD void build_multiples(const aff& q, int shift, int count, aff* out, u256* zs, u256* ps)
{
    jac b = jac_from_aff(q);
    for (int t = 0; t < shift; t++) b = jac_double(b);
    const aff base = jac_to_aff(b);
    jac t = jac_from_aff(base);
    u256 run = fe_one();
    for (int d = 1; d <= count; d++) {
        if (d > 1) t = jac_add_aff(t, base);
        out[d - 1].x = t.X; out[d - 1].y = t.Y;
        zs[d - 1] = t.Z;
        run = fe_mul(run, t.Z);
        ps[d - 1] = run;                       // z_1 * ... * z_d
    }
    u256 inv = fe_inv(run);
    for (int d = count; d >= 1; d--) {
        const u256 zi = (d > 1) ? fe_mul(inv, ps[d - 2]) : inv;      // 1 / z_d
        if (d > 1) inv = fe_mul(inv, zs[d - 1]);
        const u256 zi2 = fe_sqr(zi);
        out[d - 1].x = fe_mul(out[d - 1].x, zi2);
        out[d - 1].y = fe_mul(out[d - 1].y, fe_mul(zi2, zi));
    }
}

// Window j of a key's table in one go (small windows): out[d-1] = d * 2^(FAB_WQ*j) * q, d = 1..FAB_Q_ENTRIES.
FAB_HD void build_key_window(const aff& q, int j, aff* out, u256* zs, u256* ps)
{
    build_multiples(q, FAB_WQ * j, FAB_Q_ENTRIES, out, zs, ps);
}

// Wide windows (>= 14 bits) are built in two levels: with h = w / 2, entry x = hi * 2^h + lo of window j is
//   hi * (2^h B_j) + lo * B_j,   B_j = 2^(w j) P,
// i.e. ONE mixed addition of two points from two small tables (2^h - 1 multiples each, built by build_multiples).
// A thread produces FAB_TAB_CHUNK consecutive entries and shares one inversion among them.  Used for the per-key
// tables (P = Q) and for the generator's table (P = G).
#ifndef FAB_Q_TWO_LEVEL
#define FAB_Q_TWO_LEVEL ((FAB_WQ >= 14) && (FAB_WQ % 2 == 0))
#endif
#ifndef FAB_G_TWO_LEVEL
#define FAB_G_TWO_LEVEL ((FAB_WG >= 14) && (FAB_WG % 2 == 0))
#endif
#define FAB_TAB_CHUNK 64
// lo[d-1] = d B_j, hi[d-1] = d 2^half B_j (affine); writes out[x-1] for x in [x0, x0 + count), count <= FAB_TAB_CHUNK
FAB_HD void build_window_chunk(const aff* lo, const aff* hi, int half, uint32_t x0, int count, aff* out)
{
    u256 zs[FAB_TAB_CHUNK], ps[FAB_TAB_CHUNK];
    const uint32_t lomask = (1u << half) - 1u;
    u256 run = fe_one();
    for (int k = 0; k < count; k++) {
        const uint32_t x = x0 + (uint32_t)k, h = x >> half, l = x & lomask;
        jac p;
        if (h == 0) p = jac_from_aff(lo[l - 1]);
        else if (l == 0) p = jac_from_aff(hi[h - 1]);
        else p = jac_add_aff(jac_from_aff(hi[h - 1]), lo[l - 1]);
        out[x - 1].x = p.X; out[x - 1].y = p.Y;
        zs[k] = p.Z;
        run = fe_mul(run, p.Z);
        ps[k] = run;
    }
    u256 inv = fe_inv(run);
    for (int k = count - 1; k >= 0; k--) {
        const u256 zi = (k > 0) ? fe_mul(inv, ps[k - 1]) : inv;
        if (k > 0) inv = fe_mul(inv, zs[k]);
        const u256 zi2 = fe_sqr(zi);
        const uint32_t x = x0 + (uint32_t)k;
        out[x - 1].x = fe_mul(out[x - 1].x, zi2);
        out[x - 1].y = fe_mul(out[x - 1].y, fe_mul(zi2, zi));
    }
}

FAB_HD aff g_table_entry(int j, uint32_t d)
{
    aff g; g.x = fe_gx_mont(); g.y = fe_gy_mont();
    return table_entry(g, FAB_WG, j, d);
}

}  // namespace fabgpu
