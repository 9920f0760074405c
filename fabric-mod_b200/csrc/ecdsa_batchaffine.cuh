// Batch-affine accumulation for the key-table verification path: the GPU restatement of the sum
//   R = sum_j T_G[j][u1_j] + sum_j T_Q[j][u2_j]
// that ecdsa_verify_one_cached (ecdsa_verify.cuh) computes with 28 XYZZ mixed additions of 10 field multiplications each.
// (What it replaces in the reference: the CombinedMult behind Go's ecdsa.Verify at bccsp/sw/ecdsa.go:56.)
//
// Every operand is an AFFINE table entry, so the additions can be affine too -- lambda = (y2 - y1)/(x2 - x1), 1M + 1S + 1M -- if the
// division is shared: the 28 leaves are summed as a binary tree, all additions of one tree level are independent, and
// Montgomery's trick turns their denominators into 3 multiplications each plus ONE inversion per level.  The inversion itself
// is shared by a whole CTA: every thread (= one signature) hands the product of its level's denominators to an exchange buffer
// in shared memory, the lanes of one warp run the same trick over FAB_BA_THREADS / 32 of them each and pay for a single
// division-step inversion (p256_modinv.cuh), and every thread reads its own quotient back.  s^-1 mod n goes through the same
// exchange (modulus n).  Per signature: ~6 multiplications per addition instead of 11, ~1/8 of an inversion instead of one.
//
// Tree shape: the leaves are [G windows (padded to a multiple of 4)] ++ [Q windows (padded to a multiple of 4)]; level 1 adds
// leaves (2k, 2k+1), level 2 adds level-1 results (2k, 2k+1), and the results of level 2 (FAB_BA_NP / 4 points) are summed with
// the complete Jacobian mixed addition inside level 2's backward pass.  Pairs never straddle the G / Q boundary, and two
// partial sums of disjoint windows of one reduced scalar k < n can neither be equal nor opposite (a P = +-b P with 0 < a + b < n
// and a != b is impossible in a group of prime order n), so x2 = x1 cannot occur inside the affine levels; the crafted
// u1 G = +-u2 Q cases meet only in the Jacobian tail, whose group law is complete.  A zero denominator is still detected and
// sends that one signature through ecdsa_verify_one_cached.  Zero digits (no table entry) travel as "infinity" flags.
//
// Everything below the CTA exchange is plain per-thread code, compiled for the host as well (tests/host_sim).
#pragma once
#include "ecdsa_verify.cuh"

namespace fabgpu {

#define FAB_BA_NGP (((FAB_G_WINDOWS + 3) / 4) * 4)
#define FAB_BA_NQP (((FAB_Q_WINDOWS + 3) / 4) * 4)
#define FAB_BA_NP (FAB_BA_NGP + FAB_BA_NQP)        // leaves (28 with 22-bit G windows and 16-bit key windows)
#define FAB_BA_N1 (FAB_BA_NP / 2)                  // additions of level 1 (14)
#define FAB_BA_N2 (FAB_BA_NP / 4)                  // additions of level 2 (7) = points summed by the Jacobian tail
#define FAB_BA_INF 0xffffffffu                     // "digit 0": this leaf is the point at infinity
static_assert(FAB_BA_N1 <= 32, "infinity flags are kept in 32-bit masks");

// Per-thread scratch of the two levels (local memory on the device: dynamically indexed, 1 344 bytes with 28 leaves).
struct BaScratch {
    u256 pre[FAB_BA_N1];        // prefix products of the current level's denominators
    aff pts[FAB_BA_N1];         // results of level 1
};

// Leaf table indices of one signature: dig[k * stride] = entry index into the G table (k < FAB_BA_NGP) or into the key's own
// table (k >= FAB_BA_NGP), FAB_BA_INF for a zero digit or a padding leaf.
FAB_HD void ba_digits(const u256& u1, const u256& u2, uint32_t* dig, int stride)
{
    uint32_t kk[8];
#pragma unroll
    for (int i = 0; i < 8; i++) kk[i] = u1.v[i];
#pragma unroll
    for (int j = 0; j < FAB_BA_NGP; j++) {
        uint32_t idx = FAB_BA_INF;
        if (j < FAB_G_WINDOWS) {
            const uint32_t d = kk[0] & (uint32_t)FAB_G_ENTRIES;
#pragma unroll
            for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> FAB_WG) | (kk[i + 1] << (32 - FAB_WG));
            kk[7] >>= FAB_WG;
            if (d) idx = (uint32_t)j * (uint32_t)FAB_G_ENTRIES + (d - 1u);
        }
        dig[j * stride] = idx;
    }
#pragma unroll
    for (int i = 0; i < 8; i++) kk[i] = u2.v[i];
#pragma unroll
    for (int j = 0; j < FAB_BA_NQP; j++) {
        uint32_t idx = FAB_BA_INF;
        if (j < FAB_Q_WINDOWS) {
            const uint32_t d = kk[0] & (uint32_t)FAB_Q_ENTRIES;
#pragma unroll
            for (int i = 0; i < 7; i++) kk[i] = (kk[i] >> FAB_WQ) | (kk[i + 1] << (32 - FAB_WQ));
            kk[7] >>= FAB_WQ;
            if (d) idx = (uint32_t)j * (uint32_t)FAB_Q_ENTRIES + (d - 1u);
        }
        dig[(FAB_BA_NGP + j) * stride] = idx;
    }
}

// Ask the L2 for every table entry of a signature as soon as its digits exist (no register cost).  The forward pass has one
// multiplication per two gathers: without this, each of its 14 iterations waits out a DRAM round trip (ncu: long_scoreboard 25 % of
// all warp time); with the lines already on their way only the first wait is a DRAM latency, the rest are L2 hits.
#ifndef FAB_BA_L2PREFETCH
#define FAB_BA_L2PREFETCH 0             // off: the extra requests compete with the gathers (measured slower with it on)
#endif
FAB_HD void ba_prefetch_leaves(const uint32_t* dig, int stride, const aff* gtab, const aff* qtab)
{
#if defined(__CUDA_ARCH__) && FAB_BA_L2PREFETCH
    for (int leaf = 0; leaf < FAB_BA_NP; leaf++) {
        const uint32_t idx = dig[leaf * stride];
        if (idx != FAB_BA_INF) asm volatile("prefetch.global.L2 [%0];" :: "l"((leaf < FAB_BA_NGP ? gtab : qtab) + idx));
    }
#else
    (void)dig; (void)stride; (void)gtab; (void)qtab;
#endif
}

// Operand `leaf` of a level: first = a table entry named by the digit array, otherwise a level-1 result.  (Runtime flags, not
// template parameters: the kernel holds ONE copy of each pass and loops over the levels -- the first version, with a copy per
// level and per modulus, was 212 KB of code.)
FAB_HD const aff* ba_operand(bool first, int leaf, const aff* gtab, const aff* qtab, const uint32_t* dig, int stride, const aff* pts,
                             uint32_t infmask, bool& inf)
{
    if (first) {
        const uint32_t idx = dig[leaf * stride];
        inf = idx == FAB_BA_INF;
        return (leaf < FAB_BA_NGP ? gtab : qtab) + (inf ? 0u : idx);
    }
    inf = (infmask >> leaf) & 1u;
    return pts + leaf;
}

#ifndef FAB_BA_PREFETCH
#define FAB_BA_PREFETCH 0             // 1: request the operands of the next addition before the multiplications of the current one.  Off: the
#endif                                // extra live registers spill, which measured slower
#if FAB_BA_PREFETCH
// Forward pass of one level: pre[k] = d_0 ... d_k with d_k = x(2k+1) - x(2k) (1 where an operand is infinity); returns the product
// of all n denominators.  exc is set when two finite operands share their x (see the header: cannot happen for reduced scalars).
// The operands of addition k+1 are loaded before the multiplication of addition k is issued (software pipelining: the table
// gathers are DRAM / L2 round trips, and with ~3 warps per scheduler nothing else would cover them).
FAB_HD u256 ba_forward(bool first, int n, const aff* gtab, const aff* qtab, const uint32_t* dig, int stride, const aff* pts,
                       uint32_t infmask, u256* pre, uint32_t& exc)
{
    u256 c = fe_one();
    bool fa, fb;
    const aff* pa = ba_operand(first, 0, gtab, qtab, dig, stride, pts, infmask, fa);
    const aff* pb = ba_operand(first, 1, gtab, qtab, dig, stride, pts, infmask, fb);
    u256 xa = pa->x, xb = pb->x;
    for (int k = 0; k < n; k++) {
        bool nfa = false, nfb = false;
        u256 nxa = xa, nxb = xb;
        if (k + 1 < n) {
            const aff* na = ba_operand(first, 2 * k + 2, gtab, qtab, dig, stride, pts, infmask, nfa);
            const aff* nb = ba_operand(first, 2 * k + 3, gtab, qtab, dig, stride, pts, infmask, nfb);
            nxa = na->x; nxb = nb->x;
        }
        u256 dx = fe_sub(xb, xa);
        const bool z = u256_is_zero(dx);
        if (fa || fb) dx = fe_one();
        else if (z) { exc = 1u; dx = fe_one(); }
        c = (k == 0) ? dx : fe_mul(c, dx);
        pre[k] = c;
        xa = nxa; xb = nxb; fa = nfa; fb = nfb;
    }
    return c;
}

// Backward pass: inv = (d_0 ... d_{n-1})^-1.  Walks k = n-1 .. 0, peels 1/d_k off the running inverse, finishes the affine
// addition and either stores the result (out[k], infinity flags returned) or, on the last level, adds it to the Jacobian
// accumulator.  Same pipelining: the operands of addition k-1 are requested before the five multiplications of addition k.
FAB_HD uint32_t ba_backward(bool first, bool last, int n, u256 inv, const aff* gtab, const aff* qtab, const uint32_t* dig, int stride,
                            const aff* pts, uint32_t infmask, const u256* pre, aff* out, jac& acc)
{
    uint32_t outmask = 0;
    bool fa, fb;
    aff a, b;
    {
        const aff* pa = ba_operand(first, 2 * n - 2, gtab, qtab, dig, stride, pts, infmask, fa);
        const aff* pb = ba_operand(first, 2 * n - 1, gtab, qtab, dig, stride, pts, infmask, fb);
        a = *pa; b = *pb;
    }
    for (int k = n - 1; k >= 0; k--) {
        bool nfa = false, nfb = false;
        aff na = a, nb = b;
        if (k > 0) {
            const aff* pa = ba_operand(first, 2 * k - 2, gtab, qtab, dig, stride, pts, infmask, nfa);
            const aff* pb = ba_operand(first, 2 * k - 1, gtab, qtab, dig, stride, pts, infmask, nfb);
            na = *pa; nb = *pb;
        }
        u256 dx = fe_sub(b.x, a.x);
        if (fa || fb || u256_is_zero(dx)) dx = fe_one();
        u256 di;                                            // 1 / d_k
        if (k > 0) {
            u256 nx;
            fe_mul2(inv, pre[k - 1], inv, dx, di, nx);
            inv = nx;
        } else di = inv;
        const u256 lam = fe_mul(fe_sub(b.y, a.y), di);
        aff s;
        s.x = fe_sub(fe_sub(fe_sqr(lam), a.x), b.x);
        s.y = fe_sub(fe_mul(lam, fe_sub(a.x, s.x)), a.y);
        if (fa) s = b;
        else if (fb) s = a;
        const bool finf = fa && fb;
        if (last) {
            if (!finf) acc = jac_add_aff(acc, s);
        } else {
            out[k] = s;
            outmask |= (finf ? 1u : 0u) << k;
        }
        a = na; b = nb; fa = nfa; fb = nfb;
    }
    return outmask;
}

#else
FAB_HD u256 ba_forward(bool first, int n, const aff* gtab, const aff* qtab, const uint32_t* dig, int stride, const aff* pts,
                       uint32_t infmask, u256* pre, uint32_t& exc)
{
    u256 c = fe_one();
    for (int k = 0; k < n; k++) {
        bool fa, fb;
        const aff* pa = ba_operand(first, 2 * k, gtab, qtab, dig, stride, pts, infmask, fa);
        const aff* pb = ba_operand(first, 2 * k + 1, gtab, qtab, dig, stride, pts, infmask, fb);
        u256 dx = fe_sub(pb->x, pa->x);
        const bool z = u256_is_zero(dx);
        if (fa || fb) dx = fe_one();
        else if (z) { exc = 1u; dx = fe_one(); }
        c = (k == 0) ? dx : fe_mul(c, dx);
        pre[k] = c;
    }
    return c;
}

FAB_HD uint32_t ba_backward(bool first, bool last, int n, u256 inv, const aff* gtab, const aff* qtab, const uint32_t* dig, int stride,
                            const aff* pts, uint32_t infmask, const u256* pre, aff* out, jac& acc)
{
    uint32_t outmask = 0;
    for (int k = n - 1; k >= 0; k--) {
        bool fa, fb;
        const aff* pa = ba_operand(first, 2 * k, gtab, qtab, dig, stride, pts, infmask, fa);
        const aff* pb = ba_operand(first, 2 * k + 1, gtab, qtab, dig, stride, pts, infmask, fb);
        const aff a = *pa, b = *pb;
        u256 dx = fe_sub(b.x, a.x);
        if (fa || fb || u256_is_zero(dx)) dx = fe_one();
        u256 di;                                            // 1 / d_k
        if (k > 0) {
            u256 nx;
            fe_mul2(inv, pre[k - 1], inv, dx, di, nx);
            inv = nx;
        } else di = inv;
        const u256 lam = fe_mul(fe_sub(b.y, a.y), di);
        aff s;
        s.x = fe_sub(fe_sub(fe_sqr(lam), a.x), b.x);
        s.y = fe_sub(fe_mul(lam, fe_sub(a.x, s.x)), a.y);
        if (fa) s = b;
        else if (fb) s = a;
        const bool finf = fa && fb;
        if (last) {
            if (!finf) acc = jac_add_aff(acc, s);
        } else {
            out[k] = s;
            outmask |= (finf ? 1u : 0u) << k;
        }
    }
    return outmask;
}

#endif

// Montgomery's trick over V values held in a strided array (one lane of the CTA's inverter warp; on the host: one call per
// group).  modn: values are plain scalars s in [1, n-1] and the results are s^-1 R mod n (the Montgomery form sc_mul wants);
// otherwise values are field elements a R and the results a^-1 R.  Element j, limb l lives at [j * vstride + l * lstride];
// val[] is replaced by the inverses, tmp[] is scratch of the same shape.
FAB_HD void ba_inverse_lane(bool modn, uint32_t* val, uint32_t* tmp, int V, int vstride, int lstride)
{
    u256 c;
#pragma unroll
    for (int l = 0; l < 8; l++) c.v[l] = val[l * lstride];
    for (int j = 1; j < V; j++) {
#pragma unroll
        for (int l = 0; l < 8; l++) tmp[(j - 1) * vstride + l * lstride] = c.v[l];      // prefix j-1
        u256 v;
#pragma unroll
        for (int l = 0; l < 8; l++) v.v[l] = val[j * vstride + l * lstride];
        c = modn ? sc_mul(c, v) : fe_mul(c, v);
    }
    // modn:  c = s_0 ... s_{V-1} R^-(V-1); its plain inverse times R (one product with R^2) is what the peeling below needs.
    // field: c = a_0 ... a_{V-1} R; the plain inverse of that residue is (a_0 ...)^-1 R^-1, one product with R^3 restores a^-1 R.
    const u256 r3p = u256_const(0x0000000au, 0xfffffffdu, 0xfffffff7u, 0xffffffedu, 0xfffffffcu, 0x00000005u, 0x00000001u, 0x00000018u);
    u256 inv = inv_safegcd_rt(c, modn ? 0 : 1);
    inv = modn ? sc_mul(inv, sc_r2()) : fe_mul(inv, r3p);
    for (int j = V - 1; j >= 1; j--) {
        u256 p, v;
#pragma unroll
        for (int l = 0; l < 8; l++) { p.v[l] = tmp[(j - 1) * vstride + l * lstride]; v.v[l] = val[j * vstride + l * lstride]; }
        const u256 o = modn ? sc_mul(inv, p) : fe_mul(inv, p);
        inv = modn ? sc_mul(inv, v) : fe_mul(inv, v);
#pragma unroll
        for (int l = 0; l < 8; l++) val[j * vstride + l * lstride] = o.v[l];
    }
#pragma unroll
    for (int l = 0; l < 8; l++) val[l * lstride] = inv.v[l];
}

// Montgomery's trick over the TWO values of one thread (ecdsa_verify_ba2_kernel: a thread carries two signatures and shares
// each inversion between them -- no exchange through shared memory, no barrier).  Same domains as ba_inverse_lane.
FAB_HD void ba_inverse_pair(bool modn, u256& a, u256& b)
{
    const u256 r3p = u256_const(0x0000000au, 0xfffffffdu, 0xfffffff7u, 0xffffffedu, 0xfffffffcu, 0x00000005u, 0x00000001u, 0x00000018u);
    const u256 c = modn ? sc_mul(a, b) : fe_mul(a, b);
    u256 inv = inv_safegcd_rt(c, modn ? 0 : 1);
    inv = modn ? sc_mul(inv, sc_r2()) : fe_mul(inv, r3p);
    const u256 ia = modn ? sc_mul(inv, b) : fe_mul(inv, b);
    const u256 ib = modn ? sc_mul(inv, a) : fe_mul(inv, a);
    a = ia; b = ib;
}

// r, s in [1, n-1] (Go: r.Sign() <= 0 || s.Sign() <= 0 -> false; r >= N || s >= N -> false)
FAB_HD bool ba_range_ok(const u256& r, const u256& s)
{
    const u256 n = sc_n();
    return !(u256_is_zero(r) || u256_is_zero(s) || !u256_lt(r, n) || !u256_lt(s, n));
}

// Stage between the exchanges, per signature: w = s^-1 R mod n  ->  u1 = e w, u2 = r w  ->  leaf indices.
FAB_HD void ba_scalars(const u256& e, const u256& r, const u256& w, uint32_t* dig, int stride)
{
    u256 u1, u2;
    ecdsa_u1u2(e, r, w, u1, u2);
    ba_digits(u1, u2, dig, stride);
}

}  // namespace fabgpu
