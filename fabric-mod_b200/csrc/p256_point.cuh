// P-256 group law in Jacobian coordinates over the Montgomery field of p256_fe.cuh, and the XYZZ mixed addition of the window chains.
// Infinity is Z == 0 (XYZZ: ZZ == 0).  All routines are complete: P = Q, P = -Q and infinity operands are handled, because
// the reference's verifier (Go crypto/elliptic CombinedMult behind bccsp/sw/ecdsa.go:56) is complete and the
// bitmask must match it on adversarial inputs too (SURVEY.md A.5 items 6-7).
#pragma once
#include "p256_fe.cuh"

namespace fabgpu {

struct jac { u256 X, Y, Z; };     // Jacobian, Montgomery form
struct aff { u256 x, y; };        // affine, Montgomery form (never infinity)

FAB_HD jac jac_infinity() { jac r; r.X = fe_one(); r.Y = fe_one(); r.Z = u256_zero(); return r; }
FAB_HD bool jac_is_infinity(const jac& p) { return u256_is_zero(p.Z); }
FAB_HD jac jac_from_aff(const aff& a) { jac r; r.X = a.x; r.Y = a.y; r.Z = fe_one(); return r; }
FAB_HD jac jac_neg(const jac& p) { jac r = p; r.Y = fe_neg(p.Y); return r; }

// Doubling, a = -3: 4M + 4S + 12 additive ops.  Same quantities as dbl-2001-b (alpha = 3(X-delta)(X+delta),
// X3 = alpha^2 - 8 beta, Y3 = alpha(4 beta - X3) - 8 gamma^2, Z3 = 2 Y Z) but Z3 is a product instead of
// (Y+Z)^2 - gamma - delta and the multiples of beta/gamma reuse 2*gamma: the additive ops run on the alu pipe, which
// ncu shows is the busier one, so trading one squaring for a multiplication and four fewer add/sub is a net win.
// Infinity in -> infinity out (Z3 = 2*Y1*Z1 = 0).
FAB_HD jac jac_double(const jac& p)
{
    const u256 delta = fe_sqr(p.Z);
    const u256 gamma = fe_sqr(p.Y);
    const u256 gamma2 = fe_dbl(gamma);                       // 2 Y^2
    const u256 beta4 = fe_dbl(fe_mul(p.X, gamma2));          // 4 X Y^2
    const u256 t2 = fe_mul(fe_sub(p.X, delta), fe_add(p.X, delta));
    const u256 alpha = fe_add(fe_dbl(t2), t2);
    jac r;
    r.X = fe_sub(fe_sqr(alpha), fe_dbl(beta4));
    r.Z = fe_dbl(fe_mul(p.Y, p.Z));
    const u256 g8 = fe_dbl(fe_sqr(gamma2));                  // 2 * (2 Y^2)^2 = 8 Y^4
    r.Y = fe_sub(fe_mul(alpha, fe_sub(beta4, r.X)), g8);
    return r;
}

// Addition (add-1998-cmo-2 shape): 12M + 4S + 7 additive ops, with the exceptional cases resolved explicitly.
FAB_HD jac jac_add(const jac& p, const jac& q)
{
    if (jac_is_infinity(p)) return q;
    if (jac_is_infinity(q)) return p;
    const u256 z1z1 = fe_sqr(p.Z);
    const u256 z2z2 = fe_sqr(q.Z);
    const u256 u1 = fe_mul(p.X, z2z2);
    const u256 u2 = fe_mul(q.X, z1z1);
    const u256 s1 = fe_mul(fe_mul(p.Y, q.Z), z2z2);
    const u256 s2 = fe_mul(fe_mul(q.Y, p.Z), z1z1);
    const u256 h = fe_sub(u2, u1);
    const u256 rr = fe_sub(s2, s1);
    if (u256_is_zero(h)) {
        if (u256_is_zero(rr)) return jac_double(p);   // same point
        return jac_infinity();                         // opposite points
    }
    const u256 hh = fe_sqr(h);
    const u256 hhh = fe_mul(h, hh);
    const u256 v = fe_mul(u1, hh);
    jac r;
    r.X = fe_sub(fe_sub(fe_sqr(rr), hhh), fe_dbl(v));
    r.Y = fe_sub(fe_mul(rr, fe_sub(v, r.X)), fe_mul(s1, hhh));
    r.Z = fe_mul(fe_mul(p.Z, q.Z), h);
    return r;
}

// The two exceptional cases of an addition whose H = 0: same point -> doubling, opposite points -> infinity.  Out of line:
// never taken on honest inputs, and the doubling must not be expanded into the caller's loop body.  Arguments by value: a
// reference would need the caller's accumulator in local memory wherever this call can happen, i.e. a store of it on every pass
// of a verify kernel's window loop; by value it is copied out only when the call is taken.
#if defined(__CUDA_ARCH__)
__device__ __noinline__
#else
inline
#endif
jac jac_add_h_zero(jac p, u256 rr)
{
    if (u256_is_zero(rr)) return jac_double(p);
    return jac_infinity();
}

// Mixed addition (madd-2004-hmv shape, Z2 = 1): 8M + 3S + 7 additive ops.  Independent products are issued in pairs
// (fe_mul2) so that one warp keeps both integer pipes busier.  INL: field multiplications expanded in place (fe_mul_t).
template <bool INL> FAB_HD jac jac_add_aff_t(const jac& p, const aff& q)
{
    if (jac_is_infinity(p)) return jac_from_aff(q);
    const u256 z1z1 = fe_sqr_t<INL>(p.Z);
    u256 u2, yz;
    fe_mul2_t<INL>(q.x, z1z1, q.y, p.Z, u2, yz);          // U2 = X2 Z1^2 ; Y2 Z1
    const u256 s2 = fe_mul_t<INL>(yz, z1z1);
    const u256 h = fe_sub(u2, p.X);
    const u256 rr = fe_sub(s2, p.Y);
    if (u256_is_zero(h)) return jac_add_h_zero(p, rr);
    const u256 hh = fe_sqr_t<INL>(h);
    u256 hhh, v;
    fe_mul2_t<INL>(h, hh, p.X, hh, hhh, v);               // H^3 ; V = X1 H^2
    jac r;
    r.X = fe_sub(fe_sub(fe_sqr_t<INL>(rr), hhh), fe_dbl(v));
    u256 t, yh;
    fe_mul2_t<INL>(rr, fe_sub(v, r.X), p.Y, hhh, t, yh);  // r (V - X3) ; Y1 H^3
    r.Y = fe_sub(t, yh);
    r.Z = fe_mul_t<INL>(p.Z, h);
    return r;
}
FAB_HD jac jac_add_aff(const jac& p, const aff& q) { return jac_add_aff_t<false>(p, q); }

// XYZZ coordinates for the window chains, which only ever add affine table points into one accumulator: x = X / ZZ, y = Y / ZZZ,
// ZZ^3 = ZZZ^2.  Infinity is ZZ == 0.  A mixed addition needs no Z1^2, and its products sit four levels deep instead of seven.
struct xyzz { u256 X, Y, ZZ, ZZZ; };     // Montgomery form

FAB_HD xyzz xyzz_infinity() { xyzz r; r.X = fe_one(); r.Y = fe_one(); r.ZZ = u256_zero(); r.ZZZ = u256_zero(); return r; }

// The P = 0 cases of xyzz_add_aff_t: the accumulator is q itself (R = 0) -> 2q, or -q -> infinity.  Out of line and by value for
// the reasons given at jac_add_h_zero; it needs only q, so the accumulator is not copied out at all.
#if defined(__CUDA_ARCH__)
__device__ __noinline__
#else
inline
#endif
xyzz xyzz_add_p_zero(aff q, u256 rr)
{
    if (!u256_is_zero(rr)) return xyzz_infinity();
    const jac d = jac_double(jac_from_aff(q));
    xyzz r;
    r.X = d.X; r.Y = d.Y;
    r.ZZ = fe_sqr(d.Z);
    r.ZZZ = fe_mul(r.ZZ, d.Z);
    return r;
}

// Mixed addition (madd-2008-s, Z2 = 1): 8M + 2S + 7 additive ops.  INL: field multiplications expanded in place (fe_mul_t).
// The ZZ3 / ZZZ3 pair goes last: issued before the Y3 pair, it cost the key-table kernel a local frame and 1 % of its time.
template <bool INL> FAB_HD xyzz xyzz_add_aff_t(const xyzz& p, const aff& q)
{
    if (u256_is_zero(p.ZZ)) { xyzz r; r.X = q.x; r.Y = q.y; r.ZZ = fe_one(); r.ZZZ = fe_one(); return r; }
    u256 u2, s2;
    fe_mul2_t<INL>(q.x, p.ZZ, q.y, p.ZZZ, u2, s2);          // U2 = x2 ZZ1 ; S2 = y2 ZZZ1
    const u256 pe = fe_sub(u2, p.X);
    const u256 rr = fe_sub(s2, p.Y);
    if (u256_is_zero(pe)) return xyzz_add_p_zero(q, rr);
    const u256 pp = fe_sqr_t<INL>(pe);
    const u256 r2 = fe_sqr_t<INL>(rr);
    u256 ppp, qq;
    fe_mul2_t<INL>(pe, pp, p.X, pp, ppp, qq);               // PPP = P PP ; Q = X1 PP
    xyzz r;
    r.X = fe_sub(fe_sub(r2, ppp), fe_dbl(qq));
    u256 t, yp;
    fe_mul2_t<INL>(rr, fe_sub(qq, r.X), p.Y, ppp, t, yp);   // R (Q - X3) ; Y1 PPP
    r.Y = fe_sub(t, yp);
    fe_mul2_t<INL>(p.ZZ, pp, p.ZZZ, ppp, r.ZZ, r.ZZZ);      // ZZ3 = ZZ1 PP ; ZZZ3 = ZZZ1 PPP
    return r;
}

// y^2 == x^3 - 3x + b  (x, y already in Montgomery form and < p)
FAB_HD bool aff_on_curve(const aff& a)
{
    const u256 x2 = fe_sqr(a.x);
    const u256 x3 = fe_mul(x2, a.x);
    const u256 x_3 = fe_add(fe_dbl(a.x), a.x);
    const u256 rhs = fe_add(fe_sub(x3, x_3), fe_b_mont());
    return u256_eq(fe_sqr(a.y), rhs);
}

// Jacobian -> affine (one field inversion); only used when building tables. p must not be infinity.
FAB_HD aff jac_to_aff(const jac& p)
{
    const u256 zi = fe_inv(p.Z);
    const u256 zi2 = fe_sqr(zi);
    aff r;
    r.x = fe_mul(p.X, zi2);
    r.y = fe_mul(p.Y, fe_mul(zi2, zi));
    return r;
}

}  // namespace fabgpu
