// Unit-test hook over the field and scalar primitives: ONE op table for the device (fieldop_kernel behind fabgpu_test_fieldop) and
// the host build (tests/host_sim: hostsim_fieldop), so that an op code names the same routine on both.  tests/test_gpu_field.py
// and tests/test_host_sim.py check every op against Python integers.  Not on any verify path.
#pragma once
#include "ecdsa_verify.cuh"

namespace fabgpu {

// R = 2^256.  "mont" operands are a R mod p; "plain" operands are integers.
enum : int {
    FOP_FE_MUL = 0,                 // fe_mul: a b R^-1 mod p
    FOP_FE_ADD = 1,                 // fe_add: a + b mod p
    FOP_FE_SUB = 2,                 // fe_sub: a - b mod p
    FOP_SC_MUL = 3,                 // sc_mul: a b R^-1 mod n
    FOP_FE_INV = 4,                 // fe_inv (Fermat): a^-1 R^2 mod p, i.e. Montgomery in and out
    FOP_SC_INV_TO_MONT = 5,         // sc_inv_to_mont (Fermat): a^-1 R mod n
    FOP_SC_INV_TO_MONT_SAFEGCD = 6, // sc_inv_to_mont_safegcd: a^-1 R mod n by division steps
    FOP_FE_SQR = 7,                 // fe_sqr: a^2 R^-1 mod p
    FOP_FE_INV_SAFEGCD = 8,         // fe_inv_safegcd: a^-1 R^2 mod p by division steps
    FOP_INV_RT_N = 9,               // inv_safegcd_rt(a, 0): plain a^-1 mod n (the shared inversion of the batch-affine kernels)
    FOP_INV_RT_P = 10,              // inv_safegcd_rt(a, 1): plain a^-1 mod p
    FOP_FE_MUL2_FIRST = 11,         // fe_mul2, first output: a b R^-1, with (a + b) a in the second slot
    FOP_FE_MUL2_SECOND = 12,        // fe_mul2, second output: a b R^-1, with (a + b) b in the first slot
    FOP_FE_MUL_INL = 13,            // fe_mul_t<true> (expanded in place on the device)
    FOP_FE_SQR_INL = 14,            // fe_sqr_t<true>
    FOP_FE_MUL2_INL_FIRST = 15,     // fe_mul2_t<true>, first output (as FOP_FE_MUL2_FIRST)
    FOP_FE_MUL2_INL_SECOND = 16,    // fe_mul2_t<true>, second output (as FOP_FE_MUL2_SECOND)
    FOP_COUNT = 17
};

FAB_HD u256 fieldop(int op, const u256& a, const u256& b)
{
    u256 r0 = u256_zero(), r1 = u256_zero();
    switch (op) {
        case FOP_FE_MUL: return fe_mul(a, b);
        case FOP_FE_ADD: return fe_add(a, b);
        case FOP_FE_SUB: return fe_sub(a, b);
        case FOP_SC_MUL: return sc_mul(a, b);
        case FOP_FE_INV: return fe_inv(a);
        case FOP_SC_INV_TO_MONT: return sc_inv_to_mont(a);
        case FOP_SC_INV_TO_MONT_SAFEGCD: return sc_inv_to_mont_safegcd(a);
        case FOP_FE_SQR: return fe_sqr(a);
        case FOP_FE_INV_SAFEGCD: return fe_inv_safegcd(a);
        case FOP_INV_RT_N: return inv_safegcd_rt(a, 0);
        case FOP_INV_RT_P: return inv_safegcd_rt(a, 1);
        case FOP_FE_MUL2_FIRST: fe_mul2(a, b, fe_add(a, b), a, r0, r1); return r0;
        case FOP_FE_MUL2_SECOND: fe_mul2(fe_add(a, b), b, a, b, r0, r1); return r1;
        case FOP_FE_MUL_INL: return fe_mul_t<true>(a, b);
        case FOP_FE_SQR_INL: return fe_sqr_t<true>(a);
        case FOP_FE_MUL2_INL_FIRST: fe_mul2_t<true>(a, b, fe_add(a, b), a, r0, r1); return r0;
        case FOP_FE_MUL2_INL_SECOND: fe_mul2_t<true>(fe_add(a, b), b, a, b, r0, r1); return r1;
        default: return r0;             // callers reject op outside [0, FOP_COUNT)
    }
}

}  // namespace fabgpu
