// glibc's binary32 expf on the device, bit for bit: the exp the reference's compiled f32 code calls (PMF's sigmoid,
// MTER's BPR weight).
#pragma once
#include <stdint.h>

namespace b200 {

// glibc's expf (the binary32 exp the reference's sigmoid calls): x / ln2 * 32 = k + r with |r| <= 1/2,
// exp(x) = 2^(k/32) * 2^(r/32), 2^(r/32) by a cubic.  Every value in [-6, 6] is reproduced bit for bit (checked against
// libm exhaustively on the device and host); the arguments here never leave that range.
// EXPF_TAB[i] = bits(2^(i/32)) - (i << 47): adding k << 47 to entry k % 32 gives bits(2^(k/32)).
static __device__ const uint64_t EXPF_TAB[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull,
};

__device__ __forceinline__ float pmf_expf(float x)
{
    constexpr double INV_LN2_N = 0x1.71547652b82fep+0 * 32, SHIFT = 0x1.8p+52;
    constexpr double C0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32, C1 = 0x1.ebfce50fac4f3p-3 / 32 / 32,
                     C2 = 0x1.62e42ff0c52d6p-1 / 32;
    const double z = __dmul_rn(INV_LN2_N, (double)x);
    double kd = __dadd_rn(z, SHIFT);
    const uint64_t ki = (uint64_t)__double_as_longlong(kd);
    kd = __dsub_rn(kd, SHIFT);
    const double r = __dsub_rn(z, kd);
    const double s = __longlong_as_double((long long)(EXPF_TAB[ki % 32] + (ki << 47)));
    const double p = __dadd_rn(__dmul_rn(C0, r), C1);
    const double r2 = __dmul_rn(r, r);
    double y = __dadd_rn(__dmul_rn(C2, r), 1.0);
    y = __dadd_rn(__dmul_rn(p, r2), y);
    return __double2float_rn(__dmul_rn(y, s));
}

// pmf_expf over the whole binary32 range, with glibc's two range checks: above log(2^128) the result overflows to +inf,
// below log(2^-150) it underflows to 0; in between (subnormal results included) glibc evaluates the same formula.  NaN
// propagates through the formula.
__device__ __forceinline__ float glibc_expf(float x)
{
    if (x > 0x1.62e42ep6f) return __int_as_float(0x7f800000);
    if (x < -0x1.9fe368p6f) return 0.0f;
    return pmf_expf(x);
}

}  // namespace b200
