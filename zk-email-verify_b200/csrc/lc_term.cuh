// Evaluation of one linear-combination term {variable, coefficient word} shared by the witness kernel and the R1CS
// mat-vec (both walk LCs of the same circuit; the coefficient words are built by witness_program.cpp: coef_words).
#pragma once
#include "ff.cuh"

namespace zke {
namespace dev {

// Term word y = coefficient index (bits 0-15) | k << 16 | kind << 24 with kind 0: +1, 1: -1, 2: +2^k, 3: -2^k,
// 4: any other coefficient - there the index takes bits 0-23 (a circom-compiled key may hold more than 2^16 distinct
// coefficients; a +-2^k coefficient whose index does not fit 16 bits is simply encoded as kind 4).  Kinds 0-3 are 97.6 % of the terms of EmailVerifier (bit / byte packings, the -2ab / 4abc
// terms of the SHA-256 gadgets): they need no Montgomery product - a power of two is a shift as long as x * 2^k stays
// below 2^253 < r, which holds whenever x is the bit, byte or limb it is in these gadgets; otherwise (kind 4, or a
// shifted value that would overflow) the term falls back to (c*R) (x) x with the Montgomery-scaled coefficient table.
static const uint32_t TERM_KIND_POW2 = 2, TERM_KIND_GENERAL = 4;

__device__ __forceinline__ uint32_t bit_length(const Fr& x) {
    uint32_t top = 0, idx = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) if (x.v[i]) { top = x.v[i]; idx = i; }
    return top ? 32u * idx + 32u - __clz(top) : 0u;
}
// x << k for k < 256 (bits shifted beyond 2^256 are dropped - the caller checks bit_length first)
__device__ __forceinline__ Fr shl256(const Fr& x, uint32_t k) {
    Fr a = x;
    if (k & 128) {
#pragma unroll
        for (int i = 7; i >= 0; --i) a.v[i] = i >= 4 ? a.v[i - 4] : 0;
    }
    if (k & 64) {
#pragma unroll
        for (int i = 7; i >= 0; --i) a.v[i] = i >= 2 ? a.v[i - 2] : 0;
    }
    if (k & 32) {
#pragma unroll
        for (int i = 7; i >= 0; --i) a.v[i] = i >= 1 ? a.v[i - 1] : 0;
    }
    const uint32_t bs = k & 31;
    Fr o;
#pragma unroll
    for (int i = 7; i >= 1; --i) o.v[i] = __funnelshift_l(a.v[i - 1], a.v[i], bs);
    o.v[0] = a.v[0] << bs;
    return o;
}

struct TermVal { Fr v; bool neg; };
__device__ __forceinline__ TermVal term_value(const uint8_t* coef_r, const uint2& term, const Fr& x) {
    const uint32_t kind = term.y >> 24, k = (term.y >> 16) & 0xffu;
    TermVal t;
    t.neg = (kind & 1u) != 0 && kind < TERM_KIND_GENERAL;
    if (kind < TERM_KIND_POW2) { t.v = x; return t; }
    if (kind < TERM_KIND_GENERAL && bit_length(x) + k <= 253) { t.v = shl256(x, k); return t; }
    t.neg = false;
    t.v = Fr::load(coef_r + 32ull * (term.y & (kind == TERM_KIND_GENERAL ? 0xffffffu : 0xffffu))) * x;   // (c*R) (x) -> c*x, standard form
    return t;
}

}  // namespace dev
}  // namespace zke
