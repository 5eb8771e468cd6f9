// Device-side BN254 prime-field arithmetic for sm_90a: 8 x 32-bit limbs, Montgomery form (R = 2^256),
// carry chains written with mad.lo/hi.cc PTX (IMAD pipe).
// Memory image of an element = 32 bytes little-endian, identical to the host's U256.
//
// Role in the reference: the Fr/Fq layer of wasmcurves 0.2.0 (un-vendored; /root/reference/yarn.lock:8521-8525)
// that snarkjs' prover and circom's witness calculator run on.
#pragma once
#include <cstdint>
#ifdef ZKE_FF_EMULATE
// Host emulation of the PTX carry-chain primitives (tests/test_ff_emulation.py compiles this header with g++ and
// checks every product / square / reduction routine against Python integers).  Test infrastructure only: no
// product code path defines ZKE_FF_EMULATE.
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __constant__
struct uint4 { uint32_t x, y, z, w; };
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 r = {x, y, z, w}; return r; }
static thread_local uint32_t zke_cc = 0;   // the PTX condition-code carry bit
#else
#include <cuda_runtime.h>
#endif

namespace zke {
namespace dev {

struct FieldConsts {
    uint32_t mod[8];
    uint32_t r[8];    // 2^256 mod p  (Montgomery one)
    uint32_t r2[8];   // 2^512 mod p
    uint32_t inv;     // -p^-1 mod 2^32
    uint32_t nmod[8]; // 2^256 - p  (the modulus negated mod 2^256: fixed-operand products accumulate a*w + q*(-p))
};
// One copy per translation unit (whole-program device compilation, no -rdc): every .cu that uses field arithmetic
// instantiates ZKE_DEFINE_CONSTANT_UPLOAD(name) and the engine calls each TU's upload function once per device.
static __constant__ FieldConsts FR_C;
static __constant__ FieldConsts FQ_C;
#ifndef ZKE_FF_EMULATE
#define ZKE_DEFINE_CONSTANT_UPLOAD(fn)                                                          \
    cudaError_t fn(const ::zke::dev::FieldConsts* fr, const ::zke::dev::FieldConsts* fq) {       \
        cudaError_t e = cudaMemcpyToSymbol(::zke::dev::FR_C, fr, sizeof(::zke::dev::FieldConsts)); \
        if (e != cudaSuccess) return e;                                                          \
        return cudaMemcpyToSymbol(::zke::dev::FQ_C, fq, sizeof(::zke::dev::FieldConsts));          \
    }
#endif

struct FrTag { static __device__ __forceinline__ const FieldConsts& C() { return FR_C; } };
struct FqTag { static __device__ __forceinline__ const FieldConsts& C() { return FQ_C; } };

// ---- carry-chain primitives --------------------------------------------------------------------
#ifndef ZKE_FF_EMULATE
__device__ __forceinline__ uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
// 32 x 32 -> 64 multiply(-accumulate) on an aligned register pair (lo, hi).  Each mad.lo(.cc) / madc.hi(.cc) pair is
// fused by ptxas into ONE 64-bit IMAD.WIDE(.X) - the unit all cost figures in DESIGN.md count.
__device__ __forceinline__ void pair_mul(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {            // {hi,lo} = a*b
    asm volatile("mul.lo.u32 %0, %2, %3; mul.hi.u32 %1, %2, %3;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ void pair_mad_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {         // {hi,lo} += a*b ; CC out
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ void pair_madc_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {        // {hi,lo} += a*b + CC ; CC out
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ void pair_madc_cc_from(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t slo, uint32_t shi) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b), "r"(slo), "r"(shi));
}
__device__ __forceinline__ void pair_mad_cc_lo(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {      // lo += lo(a*b) ; hi = hi(a*b) + CC ; CC out
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, 0;" : "+r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ void pair_madc_cc_lo(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {     // same with CC in
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, 0;" : "+r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ void pair_madc_cc_new(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {    // {hi,lo} = a*b + CC ; CC out (always 0)
    asm volatile("madc.lo.cc.u32 %0, %2, %3, 0; madc.hi.cc.u32 %1, %2, %3, 0;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ void pair_madc_last(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {      // {hi,lo} = a*b + CC ; no CC out
    asm volatile("madc.lo.cc.u32 %0, %2, %3, 0; madc.hi.u32 %1, %2, %3, 0;" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
__device__ __forceinline__ uint32_t mad_lo(uint32_t a, uint32_t b, uint32_t c) { return a * b + c; }                 // low word of a*b + c
__device__ __forceinline__ uint32_t madc_lo(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }   // + CC
#else
static inline uint32_t zke_add3(uint32_t a, uint32_t b, uint32_t c, bool set) { uint64_t s = (uint64_t)a + b + c; if (set) zke_cc = (uint32_t)(s >> 32); return (uint32_t)s; }
static inline uint32_t add_cc(uint32_t a, uint32_t b) { return zke_add3(a, b, 0, true); }
static inline uint32_t addc_cc(uint32_t a, uint32_t b) { return zke_add3(a, b, zke_cc, true); }
static inline uint32_t addc(uint32_t a, uint32_t b) { return zke_add3(a, b, zke_cc, false); }
static inline uint32_t zke_sub3(uint32_t a, uint32_t b, uint32_t borrow, bool set) {   // PTX: CC = 1 means "no borrow" is NOT used; sub.cc sets CC.CF to the borrow
    uint64_t d = (uint64_t)a - b - borrow; if (set) zke_cc = (uint32_t)((d >> 32) & 1); return (uint32_t)d; }
static inline uint32_t sub_cc(uint32_t a, uint32_t b) { return zke_sub3(a, b, 0, true); }
static inline uint32_t subc_cc(uint32_t a, uint32_t b) { return zke_sub3(a, b, zke_cc, true); }
static inline uint32_t subc(uint32_t a, uint32_t b) { return zke_sub3(a, b, zke_cc, false); }
static inline uint32_t zke_lo(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a * b); }
static inline uint32_t zke_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
static inline void pair_mul(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = zke_lo(a, b); hi = zke_hi(a, b); }
static inline void pair_mad_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = zke_add3(zke_lo(a, b), lo, 0, true); hi = zke_add3(zke_hi(a, b), hi, zke_cc, true); }
static inline void pair_madc_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = zke_add3(zke_lo(a, b), lo, zke_cc, true); hi = zke_add3(zke_hi(a, b), hi, zke_cc, true); }
static inline void pair_madc_cc_from(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b, uint32_t slo, uint32_t shi) { lo = zke_add3(zke_lo(a, b), slo, zke_cc, true); hi = zke_add3(zke_hi(a, b), shi, zke_cc, true); }
static inline void pair_mad_cc_lo(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = zke_add3(zke_lo(a, b), lo, 0, true); hi = zke_add3(zke_hi(a, b), 0, zke_cc, true); }
static inline void pair_madc_cc_lo(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = zke_add3(zke_lo(a, b), lo, zke_cc, true); hi = zke_add3(zke_hi(a, b), 0, zke_cc, true); }
static inline void pair_madc_cc_new(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = zke_add3(zke_lo(a, b), 0, zke_cc, true); hi = zke_add3(zke_hi(a, b), 0, zke_cc, true); }
static inline void pair_madc_last(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = zke_add3(zke_lo(a, b), 0, zke_cc, true); hi = zke_add3(zke_hi(a, b), 0, zke_cc, false); }
static inline uint32_t mad_lo(uint32_t a, uint32_t b, uint32_t c) { return a * b + c; }
static inline uint32_t madc_lo(uint32_t a, uint32_t b, uint32_t c) { return a * b + c + zke_cc; }
#endif

template <class Tag>
struct Fp {
    uint32_t v[8];

    static __device__ __forceinline__ Fp zero() { Fp r; for (int i = 0; i < 8; ++i) r.v[i] = 0; return r; }
    static __device__ __forceinline__ Fp one() { Fp r; for (int i = 0; i < 8; ++i) r.v[i] = Tag::C().r[i]; return r; }
    static __device__ __forceinline__ Fp r2() { Fp r; for (int i = 0; i < 8; ++i) r.v[i] = Tag::C().r2[i]; return r; }
    static __device__ __forceinline__ Fp load(const void* p) {  // 32-byte aligned global / shared address
        Fp r;
        const uint4* q = reinterpret_cast<const uint4*>(p);
        uint4 a = q[0], b = q[1];
        r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
        return r;
    }
    __device__ __forceinline__ void store(void* p) const {
        uint4* q = reinterpret_cast<uint4*>(p);
        q[0] = make_uint4(v[0], v[1], v[2], v[3]);
        q[1] = make_uint4(v[4], v[5], v[6], v[7]);
    }
    __device__ __forceinline__ bool is_zero() const { return (v[0] | v[1] | v[2] | v[3] | v[4] | v[5] | v[6] | v[7]) == 0; }
    __device__ __forceinline__ bool operator==(const Fp& o) const {
        uint32_t d = 0;
        for (int i = 0; i < 8; ++i) d |= v[i] ^ o.v[i];
        return d == 0;
    }
    __device__ __forceinline__ bool operator!=(const Fp& o) const { return !(*this == o); }

    // r = a - p if a >= p (a < 2p)
    __device__ __forceinline__ void reduce_once() {
        const FieldConsts& C = Tag::C();
        uint32_t t[8];
        t[0] = sub_cc(v[0], C.mod[0]);
#pragma unroll
        for (int i = 1; i < 8; ++i) t[i] = subc_cc(v[i], C.mod[i]);
        uint32_t borrow = subc(0, 0);  // 0xffffffff if a < p
        if (borrow == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = t[i];
        }
    }

    friend __device__ __forceinline__ Fp operator+(const Fp& a, const Fp& b) {
        Fp r;
        r.v[0] = add_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < 8; ++i) r.v[i] = addc_cc(a.v[i], b.v[i]);
        // p < 2^254: no carry out of 256 bits
        r.reduce_once();
        return r;
    }
    friend __device__ __forceinline__ Fp operator-(const Fp& a, const Fp& b) {
        const FieldConsts& C = Tag::C();
        Fp r;
        r.v[0] = sub_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < 8; ++i) r.v[i] = subc_cc(a.v[i], b.v[i]);
        uint32_t borrow = subc(0, 0);
        if (borrow) {
            r.v[0] = add_cc(r.v[0], C.mod[0]);
#pragma unroll
            for (int i = 1; i < 7; ++i) r.v[i] = addc_cc(r.v[i], C.mod[i]);
            r.v[7] = addc(r.v[7], C.mod[7]);
        }
        return r;
    }
    __device__ __forceinline__ Fp neg() const { return is_zero() ? *this : (zero() - *this); }
    __device__ __forceinline__ Fp dbl() const { return *this + *this; }

    // ---- Montgomery product a*b/2^256 mod p -------------------------------------------------------------------
    // Even/odd accumulator formulation: a running total is kept as two interleaved vectors, `even` (limb k at
    // position k) and `odd` (limb k at position k + 1), so that every 32x32 product (lo, hi) lands on an ALIGNED
    // register pair of one of them and is one IMAD.WIDE (pair_* primitives above).
    //
    // Two formulations are provided:
    //   mul_cios  - operand scanning with the reduction interleaved row by row: 64 + 72 = 136 IMAD.WIDE, smallest
    //               register footprint;
    //   mul_sos   - separated: a 512-bit product by one level of Karatsuba (3 x 16 = 48 IMAD.WIDE plus ~60 adds on
    //               the otherwise idle ALU pipe) followed by redc_wide (72): 120 IMAD.WIDE; the square uses the
    //               symmetric half product (36 + 72 = 108).  The kernels of this library are bound by the IMAD pipe
    //               (DESIGN.md section 5), so fewer IMAD.WIDE per product is what raises their throughput.
    // Both return the same fully reduced value (tests/test_ff_emulation.py checks them against each other and
    // against Python integers); ZKE_FP_MUL_CIOS selects the interleaved one at compile time.
    static __device__ __forceinline__ void mul_n(uint32_t* acc, const uint32_t* a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < 8; j += 2) pair_mul(acc[j], acc[j + 1], a[j], bi);
    }
    // acc[0..8) += a[0,2,4,6] * bi (pairs), carry chained; the final carry is left in CC
    static __device__ __forceinline__ void cmad_n(uint32_t* acc, const uint32_t* a, uint32_t bi) {
        pair_mad_cc(acc[0], acc[1], a[0], bi);
#pragma unroll
        for (int j = 2; j < 8; j += 2) pair_madc_cc(acc[j], acc[j + 1], a[j], bi);
    }
    // odd[j], odd[j+1] = a[j] * bi + odd[j+2], odd[j+3] (+ incoming carry): multiply-accumulate and shift down two limbs
    static __device__ __forceinline__ void madc_n_rshift(uint32_t* odd, const uint32_t* a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < 6; j += 2) pair_madc_cc_from(odd[j], odd[j + 1], a[j], bi, odd[j + 2], odd[j + 3]);
        pair_madc_last(odd[6], odd[7], a[6], bi);
    }
    template <bool FIRST>
    static __device__ __forceinline__ void mad_n_redc(uint32_t* even, uint32_t* odd, const uint32_t* a, uint32_t bi) {
        const FieldConsts& C = Tag::C();
        if (FIRST) {
            mul_n(odd, a + 1, bi);
            mul_n(even, a, bi);
        } else {
            even[0] = add_cc(even[0], odd[1]);
            madc_n_rshift(odd, a + 1, bi);
            cmad_n(even, a, bi);
            odd[7] = addc(odd[7], 0);
        }
        const uint32_t mi = even[0] * C.inv;
        cmad_n(odd, C.mod + 1, mi);
        cmad_n(even, C.mod, mi);
        odd[7] = addc(odd[7], 0);
    }
    static __device__ __forceinline__ Fp mul_cios(const Fp& a, const Fp& b) {
        uint32_t even[8], odd[8];
        mad_n_redc<true>(even, odd, a.v, b.v[0]);
        mad_n_redc<false>(odd, even, a.v, b.v[1]);
#pragma unroll
        for (int i = 2; i < 8; i += 2) {
            mad_n_redc<false>(even, odd, a.v, b.v[i]);
            mad_n_redc<false>(odd, even, a.v, b.v[i + 1]);
        }
        // merge: result limb k = even[k] + odd[k + 1]
        Fp r;
        r.v[0] = add_cc(even[0], odd[1]);
#pragma unroll
        for (int k = 1; k < 7; ++k) r.v[k] = addc_cc(even[k], odd[k + 1]);
        r.v[7] = addc(even[7], 0);
        r.reduce_once();
        return r;
    }

    // ---- interleaved square: a^2 = sum_i a_i B^i (a_i B^i + 2 a_{>i}), i.e. row i only multiplies a_i with limb i of a
    // and the limbs above i of 2a - 36 instead of 64 multiply IMAD.WIDE (the 72 of the reduction rows stay).  2a < 2^255
    // fits 8 limbs because p < 2^254; limb i + 1 of 2 a_{>i} is limb i + 1 of 2a with the bit shifted in from a_i
    // cleared.  Pairs below the row index are skipped at compile time (the shifted vector still takes its carry).
    template <int I>
    static __device__ __forceinline__ uint32_t sqr_limb(const uint32_t* a, const uint32_t* a2, int j) {
        return j == I ? a[j] : (j == I + 1 ? (a2[j] & ~1u) : a2[j]);
    }
    template <int I, int J>
    static __device__ __forceinline__ void sqr_shifted_pair(uint32_t* odd, const uint32_t* a, const uint32_t* a2, uint32_t bi) {
        if constexpr (J + 1 >= I) pair_madc_cc_from(odd[J], odd[J + 1], sqr_limb<I>(a, a2, J + 1), bi, odd[J + 2], odd[J + 3]);
        else { odd[J] = addc_cc(odd[J + 2], 0); odd[J + 1] = addc_cc(odd[J + 3], 0); }
    }
    template <int I, int J>
    static __device__ __forceinline__ void sqr_unshifted_pair(uint32_t* even, const uint32_t* a, const uint32_t* a2, uint32_t bi) {
        constexpr int FIRST_J = (I + 1) & ~1;     // the first pair at or above the row index starts the carry chain
        if constexpr (J >= I) {
            if constexpr (J > FIRST_J) pair_madc_cc(even[J], even[J + 1], sqr_limb<I>(a, a2, J), bi);
            else pair_mad_cc(even[J], even[J + 1], sqr_limb<I>(a, a2, J), bi);
        }
    }
    template <int I, bool FIRST>
    static __device__ __forceinline__ void sqr_n_redc(uint32_t* even, uint32_t* odd, const uint32_t* a, const uint32_t* a2) {
        const FieldConsts& C = Tag::C();
        const uint32_t bi = a[I];
        if (FIRST) {
#pragma unroll
            for (int j = 0; j < 8; j += 2) pair_mul(odd[j], odd[j + 1], sqr_limb<I>(a, a2, j + 1), bi);
#pragma unroll
            for (int j = 0; j < 8; j += 2) pair_mul(even[j], even[j + 1], sqr_limb<I>(a, a2, j), bi);
        } else {
            // The pairs are expanded at compile time (template pair index, not an unrolled loop): left to the unroller,
            // the compute_90a front end keeps the first loop rolled and moves even / odd / a / a2 to local memory.
            even[0] = add_cc(even[0], odd[1]);
            // shifted vector: pair t takes multiplicand limb 2t + 1
            sqr_shifted_pair<I, 0>(odd, a, a2, bi);
            sqr_shifted_pair<I, 2>(odd, a, a2, bi);
            sqr_shifted_pair<I, 4>(odd, a, a2, bi);
            pair_madc_last(odd[6], odd[7], sqr_limb<I>(a, a2, 7), bi);     // limb 7 >= I always
            // unshifted vector: pair t takes multiplicand limb 2t; pairs below the row index are untouched
            sqr_unshifted_pair<I, 0>(even, a, a2, bi);
            sqr_unshifted_pair<I, 2>(even, a, a2, bi);
            sqr_unshifted_pair<I, 4>(even, a, a2, bi);
            sqr_unshifted_pair<I, 6>(even, a, a2, bi);
            if constexpr (I <= 6) odd[7] = addc(odd[7], 0);               // some unshifted pair was added
        }
        const uint32_t mi = even[0] * C.inv;
        cmad_n(odd, C.mod + 1, mi);
        cmad_n(even, C.mod, mi);
        odd[7] = addc(odd[7], 0);
    }
    static __device__ __forceinline__ Fp sqr_cios(const Fp& x) {
        uint32_t a2[8], even[8], odd[8];
        const uint32_t* a = x.v;
        a2[0] = a[0] << 1;
#pragma unroll
        for (int j = 1; j < 8; ++j) a2[j] = (a[j] << 1) | (a[j - 1] >> 31);
        sqr_n_redc<0, true>(even, odd, a, a2);
        sqr_n_redc<1, false>(odd, even, a, a2);
        sqr_n_redc<2, false>(even, odd, a, a2);
        sqr_n_redc<3, false>(odd, even, a, a2);
        sqr_n_redc<4, false>(even, odd, a, a2);
        sqr_n_redc<5, false>(odd, even, a, a2);
        sqr_n_redc<6, false>(even, odd, a, a2);
        sqr_n_redc<7, false>(odd, even, a, a2);
        Fp r;
        r.v[0] = add_cc(even[0], odd[1]);
#pragma unroll
        for (int k = 1; k < 7; ++k) r.v[k] = addc_cc(even[k], odd[k + 1]);
        r.v[7] = addc(even[7], 0);
        r.reduce_once();
        return r;
    }

    // (a*b + c*d) / 2^256 mod p in ONE interleaved pass: every row adds both partial products before its reduction row,
    // so the sum costs 64 + 64 + 72 = 200 IMAD.WIDE instead of 2 x 136 and needs no wide intermediate.  Operands must
    // be fully reduced (< p < 2^254): three 30-bit top-limb products then still fit the top accumulator limb.
    // Used where the curve formulas have a difference of two products (Y3 = R (Q - X3) - Y1 PPP).
    template <bool FIRST>
    static __device__ __forceinline__ void mad2_n_redc(uint32_t* even, uint32_t* odd, const uint32_t* a, uint32_t bi,
                                                       const uint32_t* c, uint32_t di) {
        const FieldConsts& C = Tag::C();
        if (FIRST) {
            mul_n(odd, a + 1, bi);
            mul_n(even, a, bi);
        } else {
            even[0] = add_cc(even[0], odd[1]);
            madc_n_rshift(odd, a + 1, bi);
            cmad_n(even, a, bi);
            odd[7] = addc(odd[7], 0);
        }
        cmad_n(odd, c + 1, di);
        cmad_n(even, c, di);
        odd[7] = addc(odd[7], 0);
        const uint32_t mi = even[0] * C.inv;
        cmad_n(odd, C.mod + 1, mi);
        cmad_n(even, C.mod, mi);
        odd[7] = addc(odd[7], 0);
    }
    static __device__ __forceinline__ Fp mul_add2(const Fp& a, const Fp& b, const Fp& c, const Fp& d) {
        uint32_t even[8], odd[8];
        mad2_n_redc<true>(even, odd, a.v, b.v[0], c.v, d.v[0]);
        mad2_n_redc<false>(odd, even, a.v, b.v[1], c.v, d.v[1]);
#pragma unroll
        for (int i = 2; i < 8; i += 2) {
            mad2_n_redc<false>(even, odd, a.v, b.v[i], c.v, d.v[i]);
            mad2_n_redc<false>(odd, even, a.v, b.v[i + 1], c.v, d.v[i + 1]);
        }
        Fp r;
        r.v[0] = add_cc(even[0], odd[1]);
#pragma unroll
        for (int k = 1; k < 7; ++k) r.v[k] = addc_cc(even[k], odd[k + 1]);
        r.v[7] = addc(even[7], 0);
        r.reduce_once();      // (ab + cd + m p) / R < p (2p / R + 1) < 1.4 p
        return r;
    }
    // a*b - c*d (Montgomery), via the negated second factor
    static __device__ __forceinline__ Fp mul_sub2(const Fp& a, const Fp& b, const Fp& c, const Fp& d) { return mul_add2(a, b, c.neg(), d); }

    // One reduction row (a "multiplication by 1" row of the interleaved product): the running total loses its lowest
    // limb (made zero by adding mi * p) and is implicitly divided by 2^32; the roles of the two vectors swap.
    template <bool FIRST>
    static __device__ __forceinline__ void redc_row(uint32_t* even, uint32_t* odd) {
        const FieldConsts& C = Tag::C();
        if (FIRST) {
            const uint32_t mi = even[0] * C.inv;
            mul_n(odd, C.mod + 1, mi);
            cmad_n(even, C.mod, mi);
            odd[7] = addc(odd[7], 0);
        } else {
            const uint32_t mi = (even[0] + odd[1]) * C.inv;
            even[0] = add_cc(even[0], odd[1]);
            madc_n_rshift(odd, C.mod + 1, mi);
            cmad_n(even, C.mod, mi);
            odd[7] = addc(odd[7], 0);
        }
    }
    // Montgomery reduction of a 16-limb value T < p * 2^256: T / 2^256 mod p = T_hi + redc(T_lo), fully reduced
    static __device__ __forceinline__ Fp redc_wide(const uint32_t* T) {
        uint32_t even[8], odd[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) even[i] = T[i];
        redc_row<true>(even, odd);
        redc_row<false>(odd, even);
#pragma unroll
        for (int i = 2; i < 8; i += 2) {
            redc_row<false>(even, odd);
            redc_row<false>(odd, even);
        }
        Fp r;
        r.v[0] = add_cc(even[0], odd[1]);
#pragma unroll
        for (int k = 1; k < 7; ++k) r.v[k] = addc_cc(even[k], odd[k + 1]);
        r.v[7] = addc(even[7], 0);
        // redc(T_lo) <= p and T_hi < p: one conditional subtraction after the addition
        r.v[0] = add_cc(r.v[0], T[8]);
#pragma unroll
        for (int k = 1; k < 7; ++k) r.v[k] = addc_cc(r.v[k], T[8 + k]);
        r.v[7] = addc(r.v[7], T[15]);
        r.reduce_once();
        return r;
    }

    // Accumulates sum a[j] * bi * 2^(32 (pos0 + 2t)) for the N/2 given limbs into the pair vector `x`, whose limbs below
    // `ext` are defined (limbs at or above are treated as zero and get defined by this call).  Returns the new extent.
    // Fully unrolled: `ext`, `base` are compile-time values after unrolling.
    template <int CNT>
    static __device__ __forceinline__ int chain(uint32_t* x, int ext, int base, const uint32_t* a, int a0, int astep, uint32_t bi) {
        bool cc_live = false, last_full = false;   // cc_live: CC holds the carry of the previous pair of this chain
#pragma unroll
        for (int t = 0; t < CNT; ++t) {
            const int p = base + 2 * t;
            const uint32_t av = a[a0 + astep * t];
            if (p + 1 < ext) {
                if (cc_live) pair_madc_cc(x[p], x[p + 1], av, bi); else pair_mad_cc(x[p], x[p + 1], av, bi);
                last_full = true; cc_live = true;
            } else if (p < ext) {
                if (cc_live) pair_madc_cc_lo(x[p], x[p + 1], av, bi); else pair_mad_cc_lo(x[p], x[p + 1], av, bi);
                last_full = false; cc_live = false;   // hi(a*b) + carry cannot overflow: the carry out is 0
            } else {
                if (cc_live) pair_madc_cc_new(x[p], x[p + 1], av, bi); else pair_mul(x[p], x[p + 1], av, bi);
                last_full = false; cc_live = false;
            }
        }
        int new_ext = base + 2 * CNT;
        if (new_ext < ext) new_ext = ext;
        if (last_full) {
            // the chain ended inside defined limbs: its carry goes to the next limb
            const int q = base + 2 * CNT;
            if (q < ext) x[q] = addc(x[q], 0);     // bounded by the value of the full product: cannot ripple further
            else { x[q] = addc(0, 0); new_ext = q + 1; }
        }
        return new_ext;
    }
    // T[0..2N) = a[0..N) * b[0..N), N even, schoolbook on pair vectors (N^2 IMAD.WIDE)
    template <int N>
    static __device__ __forceinline__ void mul_wide(uint32_t* T, const uint32_t* a, const uint32_t* b) {
        uint32_t ev[2 * N], od[2 * N];     // od[k] sits at limb position k + 1
        int ext_ev = 0, ext_od = 0;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            if ((i & 1) == 0) {
                ext_ev = chain<N / 2>(ev, ext_ev, i, a, 0, 2, b[i]);        // a[0,2,..] * b[i] at even positions i + j
                ext_od = chain<N / 2>(od, ext_od, i, a, 1, 2, b[i]);        // a[1,3,..] * b[i] at odd positions -> od index i + j - 1
            } else {
                ext_od = chain<N / 2>(od, ext_od, i - 1, a, 0, 2, b[i]);
                ext_ev = chain<N / 2>(ev, ext_ev, i + 1, a, 1, 2, b[i]);
            }
        }
        // merge T = ev + (od << 32)
        T[0] = ev[0];
        T[1] = add_cc(ev[1], od[0]);
#pragma unroll
        for (int k = 2; k < 2 * N; ++k) {
            const uint32_t e = k < ext_ev ? ev[k] : 0, o = (k - 1) < ext_od ? od[k - 1] : 0;
            T[k] = k + 1 < 2 * N ? addc_cc(e, o) : addc(e, o);
        }
    }
    // T[0..16) = a^2 : off-diagonal products once (28), doubled, plus the diagonal (8)
    static __device__ __forceinline__ void sqr_wide(uint32_t* T, const uint32_t* a) {
        uint32_t ev[16], od[16];
        int ext_ev = 0, ext_od = 0;
        // row i: a[i] * a[j], j > i, at position i + j: same parity -> ev[i + j], else od[i + j - 1]
#define ZKE_SQR_ROW(i)                                                                                     \
        if ((7 - (i)) / 2 > 0) ext_ev = chain<(7 - (i)) / 2>(ev, ext_ev, 2 * (i) + 2, a, (i) + 2, 2, a[i]);  \
        ext_od = chain<(8 - (i)) / 2>(od, ext_od, 2 * (i), a, (i) + 1, 2, a[i]);
        // ev is undefined below index 2: treat as zero there
        ev[0] = 0; ev[1] = 0; ext_ev = 2;
        ZKE_SQR_ROW(0) ZKE_SQR_ROW(1) ZKE_SQR_ROW(2) ZKE_SQR_ROW(3) ZKE_SQR_ROW(4) ZKE_SQR_ROW(5)
        ext_od = chain<1>(od, ext_od, 12, a, 7, 2, a[6]);
#undef ZKE_SQR_ROW
        // U = ev + (od << 32); T = 2U
        uint32_t U[16];
        U[0] = 0;
        U[1] = add_cc(ev[1], od[0]);
#pragma unroll
        for (int k = 2; k < 16; ++k) {
            const uint32_t e = k < ext_ev ? ev[k] : 0, o = (k - 1) < ext_od ? od[k - 1] : 0;
            U[k] = k < 15 ? addc_cc(e, o) : addc(e, o);
        }
        T[0] = 0;
        T[1] = add_cc(U[1], U[1]);
#pragma unroll
        for (int k = 2; k < 15; ++k) T[k] = addc_cc(U[k], U[k]);
        T[15] = addc(U[15], U[15]);
        // + diagonal
        pair_mad_cc(T[0], T[1], a[0], a[0]);
#pragma unroll
        for (int i = 1; i < 8; ++i) pair_madc_cc(T[2 * i], T[2 * i + 1], a[i], a[i]);
    }
    // T[0..16) = a * b by one level of (subtractive) Karatsuba over 128-bit halves:
    //   a*b = z0 + (z0 + z2 + (a0 - a1)(b1 - b0)) 2^128 + z2 2^256,  z0 = a0 b0, z2 = a1 b1
    static __device__ __forceinline__ void mul_wide_karatsuba(uint32_t* T, const uint32_t* a, const uint32_t* b) {
        uint32_t da[4], db[4];
        // da = |a0 - a1|, db = |b1 - b0| with signs
        da[0] = sub_cc(a[0], a[4]); da[1] = subc_cc(a[1], a[5]); da[2] = subc_cc(a[2], a[6]); da[3] = subc_cc(a[3], a[7]);
        const uint32_t sa = subc(0, 0);          // 0xffffffff if a0 < a1
        db[0] = sub_cc(b[4], b[0]); db[1] = subc_cc(b[5], b[1]); db[2] = subc_cc(b[6], b[2]); db[3] = subc_cc(b[7], b[3]);
        const uint32_t sb = subc(0, 0);          // 0xffffffff if b1 < b0
        // conditional negation: (x ^ s) - s
        da[0] = sub_cc(da[0] ^ sa, sa); da[1] = subc_cc(da[1] ^ sa, sa); da[2] = subc_cc(da[2] ^ sa, sa); da[3] = subc(da[3] ^ sa, sa);
        db[0] = sub_cc(db[0] ^ sb, sb); db[1] = subc_cc(db[1] ^ sb, sb); db[2] = subc_cc(db[2] ^ sb, sb); db[3] = subc(db[3] ^ sb, sb);
        uint32_t zm[8];
        mul_wide<4>(T, a, b);            // z0 -> T[0..8)
        mul_wide<4>(T + 8, a + 4, b + 4);  // z2 -> T[8..16)
        mul_wide<4>(zm, da, db);         // |a0 - a1| |b1 - b0|
        const uint32_t neg = sa ^ sb;    // all ones: the middle product is negative
        // mid = z0 + z2 (9 limbs)
        uint32_t mid[9];
        mid[0] = add_cc(T[0], T[8]);
#pragma unroll
        for (int k = 1; k < 8; ++k) mid[k] = addc_cc(T[k], T[8 + k]);
        mid[8] = addc(0, 0);
        // mid += (zm ^ neg) - neg  ==  mid +/- zm   (two's complement over 9 limbs; the true result is non-negative)
        const uint32_t one = neg & 1u;
        mid[0] = add_cc(mid[0], one);            // +1 of the two's complement
#pragma unroll
        for (int k = 1; k < 8; ++k) mid[k] = addc_cc(mid[k], 0);
        mid[8] = addc(mid[8], 0);
        mid[0] = add_cc(mid[0], zm[0] ^ neg);
#pragma unroll
        for (int k = 1; k < 8; ++k) mid[k] = addc_cc(mid[k], zm[k] ^ neg);
        mid[8] = addc(mid[8], neg);
        // T += mid << 128
        T[4] = add_cc(T[4], mid[0]);
#pragma unroll
        for (int k = 1; k < 9; ++k) T[4 + k] = addc_cc(T[4 + k], mid[k]);
        T[13] = addc_cc(T[13], 0);
        T[14] = addc_cc(T[14], 0);
        T[15] = addc(T[15], 0);
    }
    static __device__ __forceinline__ Fp mul_sos(const Fp& a, const Fp& b) {
        uint32_t T[16];
        mul_wide_karatsuba(T, a.v, b.v);
        return redc_wide(T);
    }
    static __device__ __forceinline__ Fp mul_sos_plain(const Fp& a, const Fp& b) {   // schoolbook product + redc_wide (tests)
        uint32_t T[16];
        mul_wide<8>(T, a.v, b.v);
        return redc_wide(T);
    }
    // The separated form (mul_sos) has fewer IMAD.WIDE than mul_cios but twice the IADD3 carry chains, and with the 5
    // warps per scheduler the register budget allows those serial chains are not hidden.  The interleaved product is the default; the
    // separated routines stay for the cases that need a wide intermediate (define ZKE_FP_MUL_SOS to use them).
    friend __device__ __forceinline__ Fp operator*(const Fp& a, const Fp& b) {
#ifdef ZKE_FP_MUL_SOS
        return mul_sos(a, b);
#else
        return mul_cios(a, b);
#endif
    }
    __device__ __forceinline__ Fp sqr() const {
#ifdef ZKE_FP_SQR_SOS
        uint32_t T[16];
        sqr_wide(T, v);
        return redc_wide(T);
#elif defined(ZKE_FP_SQR_MUL)
        return mul_cios(*this, *this);
#else
        return sqr_cios(*this);
#endif
    }
    // ---- fixed-operand (Shoup / Barrett) product a * w mod p for a CONSTANT w ------------------------------------
    // w is given in standard form together with wq = floor(w * 2^256 / p) (precomputed per constant: NTT twiddles,
    // coset factors).  With q ~ floor(a * wq / 2^256) the value a*w - q*p lies in [0, 3p) and p < 2^254, so it is
    // determined by its low 256 bits: no reduction rows at all, only
    //   - the upper part of a * wq, from the 43 limb products of weight >= 2^(32*6) (the dropped ones sum to less
    //     than 2^229: q is at most one below the exact quotient digit, which the [0, 3p) range absorbs),
    //   - the low halves of a * w and q * (2^256 - p): 2 x (28 full + 8 low-word) limb products,
    // i.e. 99 IMAD.WIDE + 16 IMAD instead of the 136 IMAD.WIDE of the interleaved Montgomery product.  The result is
    // a*w mod p exactly, for ANY a < 2^256: if a is in Montgomery form (x R), so is the result (x w R) - the data of
    // the transforms stays in Montgomery form and only the constants change representation.
    // low-half accumulation row: ev[k] <-> limb k, od[k] <-> limb k + 1; adds X[j] * y for i + j <= 7 (j = 7 - i: low word)
    template <int I, bool FIRST>
    static __device__ __forceinline__ void lo_row(uint32_t* ev, uint32_t* od, const uint32_t* X, uint32_t y) {
        constexpr int PE = (I & 1) ? I + 1 : I;          // first even limb position of this row
        constexpr int JE = (I & 1) ? 1 : 0;              // and the X index that lands there
        constexpr int NE = (8 - PE) / 2;                 // full pairs into ev (positions PE, PE + 2, .., 6)
        constexpr int PO = (I & 1) ? I : I + 1;          // first odd limb position
        constexpr int JO = (I & 1) ? 0 : 1;
        constexpr int NO = (7 - PO) / 2;                 // full pairs into od (positions PO .. 5)
        if (FIRST) {
#pragma unroll
            for (int t = 0; t < NE; ++t) pair_mul(ev[PE + 2 * t], ev[PE + 2 * t + 1], X[JE + 2 * t], y);
#pragma unroll
            for (int t = 0; t < NO; ++t) pair_mul(od[PO - 1 + 2 * t], od[PO + 2 * t], X[JO + 2 * t], y);
            od[6] = X[7 - I] * y;
        } else {
#pragma unroll
            for (int t = 0; t < NE; ++t) {
                if (t == 0) pair_mad_cc(ev[PE], ev[PE + 1], X[JE], y);
                else pair_madc_cc(ev[PE + 2 * t], ev[PE + 2 * t + 1], X[JE + 2 * t], y);
            }
            // the carry out of limb 7 is dropped (arithmetic mod 2^256); a new chain starts for the odd positions
#pragma unroll
            for (int t = 0; t < NO; ++t) {
                if (t == 0) pair_mad_cc(od[PO - 1], od[PO], X[JO], y);
                else pair_madc_cc(od[PO - 1 + 2 * t], od[PO + 2 * t], X[JO + 2 * t], y);
            }
            od[6] = NO > 0 ? madc_lo(X[7 - I], y, od[6]) : mad_lo(X[7 - I], y, od[6]);
        }
    }
    static __device__ __forceinline__ Fp mul_shoup(const Fp& a_in, const uint32_t* w, const uint32_t* wq) {
        const FieldConsts& C = Tag::C();
        const uint32_t* a = a_in.v;
        // ---- q = upper half of a * wq (limb products of weight >= 6 only); local index k <-> limb 6 + k (ev), 7 + k (od)
        uint32_t hev[10], hod[10];
        int ee = 0, eo = 0;
        ee = chain<1>(hev, ee, 0, a, 6, 2, wq[0]);  eo = chain<1>(hod, eo, 0, a, 7, 2, wq[0]);
        eo = chain<1>(hod, eo, 0, a, 6, 2, wq[1]);  ee = chain<2>(hev, ee, 0, a, 5, 2, wq[1]);
        ee = chain<2>(hev, ee, 0, a, 4, 2, wq[2]);  eo = chain<2>(hod, eo, 0, a, 5, 2, wq[2]);
        eo = chain<2>(hod, eo, 0, a, 4, 2, wq[3]);  ee = chain<3>(hev, ee, 0, a, 3, 2, wq[3]);
        ee = chain<3>(hev, ee, 0, a, 2, 2, wq[4]);  eo = chain<3>(hod, eo, 0, a, 3, 2, wq[4]);
        eo = chain<3>(hod, eo, 0, a, 2, 2, wq[5]);  ee = chain<4>(hev, ee, 0, a, 1, 2, wq[5]);
        ee = chain<4>(hev, ee, 0, a, 0, 2, wq[6]);  eo = chain<4>(hod, eo, 0, a, 1, 2, wq[6]);
        eo = chain<4>(hod, eo, 0, a, 0, 2, wq[7]);  ee = chain<4>(hev, ee, 2, a, 1, 2, wq[7]);
        uint32_t q[8];
        {
            // limb 7: hev[1] + hod[0] only contributes its carry; limbs 8..15 are q
            (void)add_cc(hev[1], hod[0]);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t e = (k + 2) < ee ? hev[k + 2] : 0, o = (k + 1) < eo ? hod[k + 1] : 0;
                q[k] = k < 7 ? addc_cc(e, o) : addc(e, o);
            }
        }
        // ---- r = low 256 bits of a * w + q * (2^256 - p)
        uint32_t ev[8], od[8];
        lo_row<0, true>(ev, od, a, w[0]);
        lo_row<1, false>(ev, od, a, w[1]); lo_row<2, false>(ev, od, a, w[2]); lo_row<3, false>(ev, od, a, w[3]);
        lo_row<4, false>(ev, od, a, w[4]); lo_row<5, false>(ev, od, a, w[5]); lo_row<6, false>(ev, od, a, w[6]);
        lo_row<7, false>(ev, od, a, w[7]);
        lo_row<0, false>(ev, od, q, C.nmod[0]); lo_row<1, false>(ev, od, q, C.nmod[1]); lo_row<2, false>(ev, od, q, C.nmod[2]);
        lo_row<3, false>(ev, od, q, C.nmod[3]); lo_row<4, false>(ev, od, q, C.nmod[4]); lo_row<5, false>(ev, od, q, C.nmod[5]);
        lo_row<6, false>(ev, od, q, C.nmod[6]); lo_row<7, false>(ev, od, q, C.nmod[7]);
        Fp r;
        r.v[0] = ev[0];
        r.v[1] = add_cc(ev[1], od[0]);
#pragma unroll
        for (int k = 2; k < 7; ++k) r.v[k] = addc_cc(ev[k], od[k - 1]);
        r.v[7] = addc(ev[7], od[6]);
        r.reduce_once();
        r.reduce_once();
        return r;
    }

    __device__ __forceinline__ Fp to_mont() const { return *this * r2(); }
    __device__ __forceinline__ Fp from_mont() const {
        Fp o = zero(); o.v[0] = 1;
        return *this * o;
    }
    // Fermat inverse (Montgomery in/out); inv(0) = 0.  ~380 products - use sparingly / batch.
    __device__ Fp inv() const {
        const FieldConsts& C = Tag::C();
        uint32_t e[8];
        e[0] = sub_cc(C.mod[0], 2);
#pragma unroll
        for (int i = 1; i < 8; ++i) e[i] = subc_cc(C.mod[i], 0);
        Fp res = one(), base = *this;
        for (int w = 7; w >= 0; --w) {
            for (int bit = 31; bit >= 0; --bit) {
                res = res.sqr();
                if ((e[w] >> bit) & 1) res = res * base;
            }
        }
        return res;
    }
};

typedef Fp<FrTag> Fr;
typedef Fp<FqTag> Fq;

// Fq2 = Fq[u]/(u^2+1)
struct Fq2 {
    Fq c0, c1;
    static __device__ __forceinline__ Fq2 zero() { Fq2 r; r.c0 = Fq::zero(); r.c1 = Fq::zero(); return r; }
    static __device__ __forceinline__ Fq2 one() { Fq2 r; r.c0 = Fq::one(); r.c1 = Fq::zero(); return r; }
    static __device__ __forceinline__ Fq2 load(const void* p) { Fq2 r; r.c0 = Fq::load(p); r.c1 = Fq::load((const char*)p + 32); return r; }
    __device__ __forceinline__ void store(void* p) const { c0.store(p); c1.store((char*)p + 32); }
    __device__ __forceinline__ bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    __device__ __forceinline__ bool operator==(const Fq2& o) const { return c0 == o.c0 && c1 == o.c1; }
    friend __device__ __forceinline__ Fq2 operator+(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = a.c0 + b.c0; r.c1 = a.c1 + b.c1; return r; }
    friend __device__ __forceinline__ Fq2 operator-(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = a.c0 - b.c0; r.c1 = a.c1 - b.c1; return r; }
    // not inlined: a G2 addition holds ten of these; inlining them all makes the G2 kernels compile for minutes
    // and spill (the call costs ~20 instructions against ~600 of work)
    friend __device__ __noinline__ Fq2 operator*(const Fq2& a, const Fq2& b) {
        Fq t0 = a.c0 * b.c0, t1 = a.c1 * b.c1;
        Fq2 r;
        r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1;
        r.c0 = t0 - t1;
        return r;
    }
    __device__ __noinline__ Fq2 sqr() const {
        Fq2 r;
        Fq t = c0 * c1;
        r.c0 = (c0 + c1) * (c0 - c1);
        r.c1 = t + t;
        return r;
    }
    __device__ __forceinline__ Fq2 neg() const { Fq2 r; r.c0 = c0.neg(); r.c1 = c1.neg(); return r; }
    __device__ __forceinline__ Fq2 dbl() const { return *this + *this; }
    __device__ Fq2 inv() const {
        Fq d = (c0.sqr() + c1.sqr()).inv();
        Fq2 r; r.c0 = c0 * d; r.c1 = (c1 * d).neg();
        return r;
    }
};

// x < modulus (x is a canonical representative): the borrow out of x - p
template <class Tag>
__device__ __forceinline__ bool below_modulus(const Fp<Tag>& x) {
    const FieldConsts& C = Tag::C();
    (void)sub_cc(x.v[0], C.mod[0]);
#pragma unroll
    for (int i = 1; i < 8; ++i) (void)subc_cc(x.v[i], C.mod[i]);
    return subc(0, 0) != 0;
}
__device__ __forceinline__ bool below_modulus(const Fq2& x) { return below_modulus(x.c0) && below_modulus(x.c1); }

}  // namespace dev
}  // namespace zke
