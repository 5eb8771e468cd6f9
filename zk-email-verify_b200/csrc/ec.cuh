// Device-side short-Weierstrass (a = 0) point arithmetic for BN254 G1 (over Fq) and G2 (over Fq2).
// Accumulators use extended Jacobian "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2): a mixed addition
// costs 8M + 2S and needs no inversion.  Affine points are 2 field elements, Montgomery form; (0, 0) encodes the
// point at infinity (it is not on either curve).
//
// Role in the reference: the G1/G2 layer of wasmcurves' `multiExpAffine` (un-vendored, SURVEY section 2).
#pragma once
#include "ff.cuh"

namespace zke {
namespace dev {

// a*b - c*d: one interleaved dual product for the prime field (ff.cuh: mul_add2), two products otherwise
template <class Tag>
__device__ __forceinline__ Fp<Tag> mul_sub2(const Fp<Tag>& a, const Fp<Tag>& b, const Fp<Tag>& c, const Fp<Tag>& d) {
#ifdef ZKE_NO_DUAL_PRODUCT
    return a * b - c * d;
#else
    return Fp<Tag>::mul_sub2(a, b, c, d);
#endif
}
__device__ __forceinline__ Fq2 mul_sub2(const Fq2& a, const Fq2& b, const Fq2& c, const Fq2& d) { return a * b - c * d; }

template <class F>
struct Affine {
    F x, y;
    __device__ __forceinline__ bool is_inf() const { return x.is_zero() && y.is_zero(); }
    static __device__ __forceinline__ Affine load(const void* p) {
        Affine a; a.x = F::load(p); a.y = F::load((const char*)p + sizeof(F)); return a;
    }
    __device__ __forceinline__ void store(void* p) const { x.store(p); y.store((char*)p + sizeof(F)); }
};

template <class F>
struct XYZZ {
    F x, y, zz, zzz;
    static __device__ __forceinline__ XYZZ inf() { XYZZ r; r.x = F::zero(); r.y = F::zero(); r.zz = F::zero(); r.zzz = F::zero(); return r; }
    __device__ __forceinline__ bool is_inf() const { return zz.is_zero(); }
    static __device__ __forceinline__ XYZZ load(const void* p) {
        XYZZ r; const char* c = (const char*)p;
        r.x = F::load(c); r.y = F::load(c + sizeof(F)); r.zz = F::load(c + 2 * sizeof(F)); r.zzz = F::load(c + 3 * sizeof(F));
        return r;
    }
    __device__ __forceinline__ void store(void* p) const {
        char* c = (char*)p;
        x.store(c); y.store(c + sizeof(F)); zz.store(c + 2 * sizeof(F)); zzz.store(c + 3 * sizeof(F));
    }
    static __device__ __forceinline__ XYZZ from_affine(const Affine<F>& p) {
        if (p.is_inf()) return inf();
        XYZZ r; r.x = p.x; r.y = p.y; r.zz = F::one(); r.zzz = F::one(); return r;
    }

    // dbl-2008-s-1 (a = 0)
    __device__ __forceinline__ void dbl() {
        if (is_inf()) return;
        F U = y.dbl();
        F V = U.sqr();
        F W = U * V;
        F S = x * V;
        F X2 = x.sqr();
        F M = X2.dbl() + X2;
        F X3 = M.sqr() - S.dbl();
        F Y3 = mul_sub2(M, S - X3, W, y);
        zz = V * zz;
        zzz = W * zzz;
        x = X3; y = Y3;
    }

    // madd-2008-s: this += (+/-) affine P
    __device__ __forceinline__ void madd(const Affine<F>& p, bool negate) {
        if (p.is_inf()) return;
        F py = negate ? p.y.neg() : p.y;
        if (is_inf()) { x = p.x; y = py; zz = F::one(); zzz = F::one(); return; }
        F U2 = p.x * zz;
        F S2 = py * zzz;
        F P = U2 - x;
        F R = S2 - y;
        if (P.is_zero()) {
            if (R.is_zero()) { dbl(); return; }
            *this = inf();
            return;
        }
        F PP = P.sqr();
        F PPP = P * PP;
        F Q = x * PP;
        F X3 = R.sqr() - PPP - Q.dbl();
        F Y3 = mul_sub2(R, Q - X3, y, PPP);
        zz = zz * PP;
        zzz = zzz * PPP;
        x = X3; y = Y3;
    }

    // add-2008-s: this += o
    __device__ __forceinline__ void add(const XYZZ& o) {
        if (o.is_inf()) return;
        if (is_inf()) { *this = o; return; }
        F U1 = x * o.zz;
        F U2 = o.x * zz;
        F S1 = y * o.zzz;
        F S2 = o.y * zzz;
        F P = U2 - U1;
        F R = S2 - S1;
        if (P.is_zero()) {
            if (R.is_zero()) { dbl(); return; }
            *this = inf();
            return;
        }
        F PP = P.sqr();
        F PPP = P * PP;
        F Q = U1 * PP;
        F X3 = R.sqr() - PPP - Q.dbl();
        F Y3 = mul_sub2(R, Q - X3, S1, PPP);
        zz = zz * o.zz * PP;
        zzz = zzz * o.zzz * PPP;
        x = X3; y = Y3;
    }

    __device__ __forceinline__ void negate() { y = y.neg(); }
};

typedef Affine<Fq> G1Affine;
typedef Affine<Fq2> G2Affine;
typedef XYZZ<Fq> G1XYZZ;
typedef XYZZ<Fq2> G2XYZZ;

// [k] P for a scalar in standard form (nbits low bits), XYZZ result
template <class F>
__device__ XYZZ<F> scalar_mul(const Affine<F>& p, const uint32_t* k, int nbits) {
    XYZZ<F> acc = XYZZ<F>::inf();
    for (int i = nbits - 1; i >= 0; --i) {
        acc.dbl();
        if ((k[i >> 5] >> (i & 31)) & 1) acc.madd(p, false);
    }
    return acc;
}

// order-r subgroup membership by [r] Q == O (as pairing_host.cpp's g2_in_subgroup); Q must be on the twist.  `inline`
// for the linkage only: engine.cu and verify.cu both define it.
inline __device__ __noinline__ bool g2_in_subgroup(const G2Affine& q) {
    if (q.is_inf()) return true;
    const FieldConsts& C = FrTag::C();
    G2XYZZ acc = G2XYZZ::inf();
    for (int i = 253; i >= 0; --i) {      // r < 2^254
        acc.dbl();
        if ((C.mod[i >> 5] >> (i & 31)) & 1) acc.madd(q, false);
    }
    return acc.is_inf();
}

}  // namespace dev
}  // namespace zke
