// Per-point scalar multiplication and the radix-2 transform over curve points that turns the powers of tau of a
// Powers-of-Tau file into its Lagrange bases (ptau.cu: `powersoftau prepare phase2`), for G1 (Fq) and G2 (Fq2).
//
// A scalar is recoded into its non-adjacent form (signed binary digits, at most one in two non-zero, a third of them
// on average) and applied to an AFFINE point by mixed additions of +P or -P.  The "table" is P itself: a 4-bit window
// of XYZZ multiples would need full additions (14 products against the mixed addition's 10) and, in G2, 2 KB of table
// per thread that cannot stay in registers.  So the transform keeps its points affine between stages: every stage reads
// affine points, writes XYZZ, and the caller converts them back with one batched inversion (xyzz_to_affine_batch).
//
// Inverse transform of size n = 2^k, natural order in and out (decimation in time):
//   load    X[i] = n^-1 * T[bitrev_k(i)]
//   stage s = 1..k, m = 2^(s-1): for every group g and j < m, with a = X[2mg + j], b = X[2mg + j + m], t = w_{2m}^-j b:
//           X[2mg + j] = a + t,  X[2mg + j + m] = a - t   (j = 0: t = b, no multiplication)
// so X[i] = n^-1 sum_j omega^(-ij) T[j].  The twiddle table holds omega_N^-j (standard form) for the largest domain N;
// the stage of half-size m reads it with stride N / 2m.
//
// Compiles under ZKE_FF_EMULATE with g++ like ec.cuh (tests/test_ec_ntt_emulation.py runs the per-thread bodies).
#pragma once
#include "ec.cuh"
#include <cstddef>

namespace zke {
namespace dev {

// k (8 words, standard form, k < 2^255) -> non-adjacent form as two masks: bit i of pos / neg is digit i = +1 / -1.
// With h = 3k, digit i = h_{i+1} - k_{i+1}: sum_i (h_{i+1} - k_{i+1}) 2^i = (3k - k) / 2 = k.
__device__ __forceinline__ void naf_recode(const uint32_t* k, uint32_t* pos, uint32_t* neg) {
    uint32_t h[8], p[8], q[8];
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { const uint64_t t = (uint64_t)k[i] * 3 + c; h[i] = (uint32_t)t; c = t >> 32; }
#pragma unroll
    for (int i = 0; i < 8; ++i) { p[i] = h[i] & ~k[i]; q[i] = ~h[i] & k[i]; }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        pos[i] = (p[i] >> 1) | (i < 7 ? p[i + 1] << 31 : 0u);
        neg[i] = (q[i] >> 1) | (i < 7 ? q[i + 1] << 31 : 0u);
    }
}

// k * P for an affine P and a scalar k < 2^255 in standard form
template <class F>
__device__ __forceinline__ XYZZ<F> mul_naf(const Affine<F>& p, const uint32_t* k) {
    uint32_t pos[8], neg[8];
    naf_recode(k, pos, neg);
    XYZZ<F> acc = XYZZ<F>::inf();
    if (p.is_inf()) return acc;
    // the digits from the top, the masks shifted left one bit per step: the loop body has one call site of each formula
    // and no indexed register array.  Leading zero digits cost a test each (doubling infinity returns at once).
    for (int d = 0; d < 256; ++d) {
        acc.dbl();
        const bool dp = pos[7] >> 31, dn = neg[7] >> 31;
        if (dp || dn) acc.madd(p, dn);
#pragma unroll
        for (int i = 7; i > 0; --i) { pos[i] = (pos[i] << 1) | (pos[i - 1] >> 31); neg[i] = (neg[i] << 1) | (neg[i - 1] >> 31); }
        pos[0] <<= 1; neg[0] <<= 1;
    }
    return acc;
}

__device__ __forceinline__ uint32_t bit_reverse(uint32_t i, int bits) {
    uint32_t r = 0;
    for (int b = 0; b < bits; ++b) r |= ((i >> b) & 1u) << (bits - 1 - b);
    return r;
}

// Thread i of the per-point scaling: out[i] = k_i * in[rev(i)], k_i = scalars[i * stride] (8 words each; stride 0: one
// scalar for all), rev = bit reversal over rev_bits bits (0: identity).
template <class F>
__device__ __forceinline__ void scale_point_each(const uint8_t* in_affine, const uint32_t* scalars, uint32_t stride, int rev_bits, uint32_t i,
                                                 uint8_t* out_xyzz) {
    const uint32_t src = rev_bits ? bit_reverse(i, rev_bits) : i;
    const Affine<F> p = Affine<F>::load(in_affine + sizeof(Affine<F>) * (size_t)src);
    uint32_t k[8];
    for (int w = 0; w < 8; ++w) k[w] = scalars[(size_t)i * stride * 8 + w];
    mul_naf(p, k).store(out_xyzz + sizeof(XYZZ<F>) * (size_t)i);
}

// Butterfly t (< n/2) of the stage with half-size m: twiddles tw[j * tw_stride] (8 words each, omega_N^-j)
template <class F>
__device__ __forceinline__ void point_butterfly(const uint8_t* in_affine, uint32_t m, const uint32_t* tw, uint32_t tw_stride, uint32_t t,
                                                uint8_t* out_xyzz) {
    const uint32_t j = t & (m - 1), i0 = ((t - j) << 1) + j, i1 = i0 + m;
    const Affine<F> a = Affine<F>::load(in_affine + sizeof(Affine<F>) * (size_t)i0);
    const Affine<F> b = Affine<F>::load(in_affine + sizeof(Affine<F>) * (size_t)i1);
    XYZZ<F> s = j ? mul_naf(b, tw + (size_t)j * tw_stride * 8) : XYZZ<F>::from_affine(b);
    XYZZ<F> d = s;
    d.negate();
    s.madd(a, false);
    d.madd(a, false);
    s.store(out_xyzz + sizeof(XYZZ<F>) * (size_t)i0);
    d.store(out_xyzz + sizeof(XYZZ<F>) * (size_t)i1);
}

#ifndef ZKE_FF_EMULATE
template <class F>
__global__ void __launch_bounds__(128)
scale_each_kernel(const uint8_t* __restrict__ in_affine, uint32_t n, const uint32_t* __restrict__ scalars, uint32_t stride, int rev_bits,
                  uint8_t* __restrict__ out_xyzz) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) scale_point_each<F>(in_affine, scalars, stride, rev_bits, i, out_xyzz);
}

template <class F>
__global__ void __launch_bounds__(128)
point_ntt_stage_kernel(const uint8_t* __restrict__ in_affine, uint32_t half_n, uint32_t m, const uint32_t* __restrict__ tw, uint32_t tw_stride,
                       uint8_t* __restrict__ out_xyzz) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < half_n) point_butterfly<F>(in_affine, m, tw, tw_stride, t, out_xyzz);
}
#endif

}  // namespace dev
}  // namespace zke
