// Device-side BN254 optimal-ate pairing for the batch Groth16 verifier (verify.cu): the Fq2-Fq6-Fq12 tower over ff.cuh's
// Fq2, a Miller loop over 6t + 2 with the twist point in homogeneous projective coordinates (no Fq2 inversion in the
// loop) whose lines can be recorded for a fixed G2 point and replayed, and the final exponentiation with a hard part
// built from cyclotomic squarings.
//
// Tower: Fq6 = Fq2[v]/(v^3 - xi), xi = 9 + u;  Fq12 = Fq6[w]/(w^2 - v) - the layout of snarkjs' vk_alphabeta_12
// (pairing_host.cpp: pairing_alphabeta).  Coefficient c[i].c[j] of an Fq12 multiplies w^(2j + i).  All values are in
// Montgomery form; the memory image of an Fq12 is its 12 Fq2 coefficients in that (i, j) order.
//
// The Miller loop value differs from pairing_host.cpp's (affine lines) by factors in proper subfields, which the final
// exponentiation removes: the reduced pairings agree exactly.  The hard part is the Fuentes-Castaneda chain that
// ffjavascript / wasmcurves use, so final_exponentiation(miller_loop(Q, P)) is the reduced pairing raised to
// 2 z (6 z^2 + 3 z + 1), z = 4965661367192848881 - the value zke_pairing_alphabeta returns.
//
// Compiles under ZKE_FF_EMULATE with g++ like ec.cuh (tests/test_pairing_emulation.py).  verify.cu and engine.cu
// (aggregate.cu) both include it: the out-of-line functions are `inline` for the linkage.
#pragma once
#include "ec.cuh"
#include <cstddef>

namespace zke {
namespace dev {

// FROB[k - 1][m] = xi^(m (p^k - 1) / 6), Montgomery form: (c w^m)^(p^k) = frob^k(c) FROB[k - 1][m] w^m
static __constant__ uint32_t FROB[3][6][2][8] = {
    {{{0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
     {{0x33144907u, 0xaf9ba696u, 0x87afb78au, 0xca6b1d73u, 0xf08a2087u, 0x11bded5eu, 0x1a1f3a7cu, 0x02f34d75u}, {0x4c492d72u, 0xa222ae23u, 0x565de15bu, 0xd00f02a4u, 0x53dfc926u, 0xdc2ff3a2u, 0xb3899551u, 0x10a75716u}},
     {{0x4563ab30u, 0xb5773b10u, 0xa9aa6454u, 0x347f91c8u, 0x242e0991u, 0x7a007127u, 0x118214ecu, 0x1956bcd8u}, {0xa0aa4757u, 0x6e849f1eu, 0x89f89141u, 0xaa1c7b6du, 0xfae0ca3au, 0xb6e713cdu, 0x4e82ebc3u, 0x26694fbbu}},
     {{0x2936b629u, 0xe4bbdd0cu, 0xe133bacbu, 0xbb30f162u, 0xf9645366u, 0x31a9d1b6u, 0xa500f8ddu, 0x253570beu}, {0x5ffe77c7u, 0xa1d77ce4u, 0x7826d1dbu, 0x07affd11u, 0xbb7edc6bu, 0x6d16bd27u, 0x85defeccu, 0x2c872002u}},
     {{0x843abe92u, 0x7361d77fu, 0x273411fbu, 0xa5bb2bd3u, 0x4b3e2399u, 0x9c941f31u, 0xbb9fd3ecu, 0x15df9cddu}, {0x4bd8c949u, 0x5dddfd15u, 0xa4445b60u, 0x62cb29a5u, 0x0c7dd2b9u, 0x37bc870au, 0x3171f0fdu, 0x24830a9du}},
     {{0x41690fe7u, 0xc970692fu, 0x27694b0bu, 0xe2403421u, 0x83c459e8u, 0x32bee66bu, 0x0ab08841u, 0x12aabcedu}, {0x40aebfa9u, 0x0d485d23u, 0xab2fcc57u, 0x05193418u, 0x8a4910f5u, 0xd3b0a40bu, 0x35d2925au, 0x2f21ebb5u}}},
    {{{0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
     {{0x00fa1bf2u, 0xca8d8005u, 0x68b39769u, 0xf0c5d614u, 0xad0d4418u, 0x0e201271u, 0xbad856e6u, 0x04290f65u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
     {{0x13e80b9cu, 0x3350c88eu, 0xdb5e56b9u, 0x7dce557cu, 0xb615564au, 0x6001b4b8u, 0x020217e0u, 0x2682e617u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
     {{0x12edefaau, 0x68c34889u, 0x72aabf4fu, 0x8d087f68u, 0x09081231u, 0x51e1a247u, 0x4729c0fau, 0x2259d6b1u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
     {{0xd782e155u, 0x71930c11u, 0xffbe3323u, 0xa6bb947cu, 0xd4741444u, 0xaa303344u, 0x26594943u, 0x2c3b3f0du}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
     {{0xc494f1abu, 0x08cfc388u, 0x8d1373d4u, 0x19b31514u, 0xcb6c0213u, 0x584e90fdu, 0xdf2f8849u, 0x09e1685bu}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}}},
    {{{0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u}, {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
     {{0x4e46d97du, 0x36531618u, 0xd4c96d9fu, 0x0af7129eu, 0xca1009b5u, 0x659da72fu, 0x83a20d23u, 0x08116d89u}, {0xc39c1939u, 0xb1df4af7u, 0x8a73bf7fu, 0x3d9f0287u, 0x8caf0ae0u, 0x9b222092u, 0xeff054a6u, 0x26684515u}},
     {{0x16ad6badu, 0xc9af22f7u, 0x4aa662b2u, 0xb311782au, 0xe248c7f4u, 0x19eeaf64u, 0xe3439f82u, 0x20273e77u}, {0xf7ce93acu, 0xacc02860u, 0x7ba76b4cu, 0x3933d581u, 0x446c8467u, 0x69e6188bu, 0x4417cc55u, 0x0a46036du}},
     {{0xaf46471eu, 0x5764af0au, 0x873e0fc1u, 0xdc50792eu, 0x881d04f6u, 0x86a673ffu, 0x3c30a74cu, 0x0b2eddb4u}, {0x787e8580u, 0x9a490f32u, 0xf04af8b1u, 0x8fd16d7fu, 0xc6027bf2u, 0x4b39888eu, 0x5b52a15du, 0x03dd2e70u}},
     {{0x7b6762dfu, 0x448a93a5u, 0x28fdeadfu, 0xbfd62df5u, 0x0e9bd47au, 0xd858f5d0u, 0x3476ec58u, 0x06b03d4du}, {0xbcc936d1u, 0x2b19daf4u, 0x56f4299fu, 0xa1a54e7au, 0x5adeaef1u, 0xb533eee0u, 0x84dda0b2u, 0x170c812bu}},
     {{0x75cf559fu, 0xe0bc4b22u, 0xc154e60fu, 0xc238b945u, 0x929a7d5eu, 0x803982a5u, 0xf7e4a37eu, 0x15ce052du}, {0xbf3799a7u, 0x2d28efbdu, 0x1ad60773u, 0x9b097e3cu, 0xaf4a535bu, 0x982d4113u, 0xe3056063u, 0x24e18991u}}}};
// b' = 3 / xi, the constant of the twist y^2 = x^3 + b' (Montgomery form)
static __constant__ uint32_t TWIST_B[2][8] = {
    {0x77b802a8u, 0x3bf938e3u, 0x3633535du, 0x020b1b27u, 0x49755260u, 0x26b7edf0u, 0x4384a86du, 0x2514c632u},
    {0xd1dcff67u, 0x38e7ecccu, 0x93ce0d3eu, 0x65f0b37du, 0x22ac00aau, 0xd749d0ddu, 0x4a688d4du, 0x0141b9ceu}};

// 6t + 2 = 0x19d797039be763ba8: the loop walks bits 63..0 of the low word with R starting at Q (the top bit)
static constexpr uint64_t ATE_LOW = 0x9d797039be763ba8ull;
// z = t, the BN parameter (final exponentiation)
static constexpr uint64_t BN_Z = 0x44e992b44a6909f1ull;
__host__ __device__ constexpr int ate_line_count() {
    int n = 64 + 2;   // one doubling line per bit, the two Frobenius-twisted additions at the end
    for (int i = 0; i < 64; ++i) n += (int)((ATE_LOW >> i) & 1);
    return n;
}
static constexpr int ATE_LINES = ate_line_count();   // 102
static constexpr int LINE_BYTES = 3 * 64;            // three Fq2 coefficients per line (see LineCoeffs)

__device__ __forceinline__ Fq2 fq2_from(const uint32_t (*c)[8]) {
    Fq2 r;
    for (int i = 0; i < 8; ++i) { r.c0.v[i] = c[0][i]; r.c1.v[i] = c[1][i]; }
    return r;
}
__device__ __forceinline__ Fq2 conj(const Fq2& a) { Fq2 r; r.c0 = a.c0; r.c1 = a.c1.neg(); return r; }
__device__ __forceinline__ Fq2 scale(const Fq2& a, const Fq& k) { Fq2 r; r.c0 = a.c0 * k; r.c1 = a.c1 * k; return r; }
__device__ __forceinline__ Fq2 mul_xi(const Fq2& a) {    // a (9 + u)
    const Fq n0 = a.c0.dbl().dbl().dbl() + a.c0, n1 = a.c1.dbl().dbl().dbl() + a.c1;
    Fq2 r; r.c0 = n0 - a.c1; r.c1 = n1 + a.c0;
    return r;
}

struct Fq6 {
    Fq2 c0, c1, c2;
    static __device__ __forceinline__ Fq6 zero() { Fq6 r; r.c0 = Fq2::zero(); r.c1 = Fq2::zero(); r.c2 = Fq2::zero(); return r; }
    static __device__ __forceinline__ Fq6 one() { Fq6 r = zero(); r.c0 = Fq2::one(); return r; }
    __device__ __forceinline__ bool operator==(const Fq6& o) const { return c0 == o.c0 && c1 == o.c1 && c2 == o.c2; }
    friend __device__ __forceinline__ Fq6 operator+(const Fq6& a, const Fq6& b) { Fq6 r; r.c0 = a.c0 + b.c0; r.c1 = a.c1 + b.c1; r.c2 = a.c2 + b.c2; return r; }
    friend __device__ __forceinline__ Fq6 operator-(const Fq6& a, const Fq6& b) { Fq6 r; r.c0 = a.c0 - b.c0; r.c1 = a.c1 - b.c1; r.c2 = a.c2 - b.c2; return r; }
    __device__ __forceinline__ Fq6 neg() const { Fq6 r; r.c0 = c0.neg(); r.c1 = c1.neg(); r.c2 = c2.neg(); return r; }
    __device__ __forceinline__ Fq6 mul_v() const { Fq6 r; r.c0 = mul_xi(c2); r.c1 = c0; r.c2 = c1; return r; }   // * v
    // Karatsuba over three coefficients: 6 Fq2 products
    friend __device__ __noinline__ Fq6 operator*(const Fq6& a, const Fq6& b) {
        const Fq2 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1, t2 = a.c2 * b.c2;
        Fq6 r;
        r.c0 = t0 + mul_xi((a.c1 + a.c2) * (b.c1 + b.c2) - t1 - t2);
        r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1 + mul_xi(t2);
        r.c2 = (a.c0 + a.c2) * (b.c0 + b.c2) - t0 - t2 + t1;
        return r;
    }
    // * (b0 + b1 v): 5 Fq2 products
    __device__ __noinline__ Fq6 mul_01(const Fq2& b0, const Fq2& b1) const {
        const Fq2 t0 = c0 * b0, t1 = c1 * b1;
        Fq6 r;
        r.c0 = t0 + mul_xi(c2 * b1);
        r.c1 = (c0 + c1) * (b0 + b1) - t0 - t1;
        r.c2 = c2 * b0 + t1;
        return r;
    }
    __device__ Fq6 inv() const {
        const Fq2 t0 = c0.sqr() - mul_xi(c1 * c2), t1 = mul_xi(c2.sqr()) - c0 * c1, t2 = c1.sqr() - c0 * c2;
        const Fq2 d = (c0 * t0 + mul_xi(c2 * t1 + c1 * t2)).inv();
        Fq6 r; r.c0 = t0 * d; r.c1 = t1 * d; r.c2 = t2 * d;
        return r;
    }
};

struct Fq12 {
    Fq6 c0, c1;
    static __device__ __forceinline__ Fq12 one() { Fq12 r; r.c0 = Fq6::one(); r.c1 = Fq6::zero(); return r; }
    __device__ __forceinline__ bool operator==(const Fq12& o) const { return c0 == o.c0 && c1 == o.c1; }
    __device__ __forceinline__ bool is_one() const { return *this == one(); }
    __device__ __forceinline__ Fq2& at(int i, int j) { Fq6& h = i ? c1 : c0; return j == 0 ? h.c0 : (j == 1 ? h.c1 : h.c2); }
    __device__ __forceinline__ const Fq2& at(int i, int j) const { const Fq6& h = i ? c1 : c0; return j == 0 ? h.c0 : (j == 1 ? h.c1 : h.c2); }
    static __device__ __forceinline__ Fq12 load(const void* p) {
        Fq12 r;
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 3; ++j) r.at(i, j) = Fq2::load((const char*)p + 64 * (3 * i + j));
        return r;
    }
    __device__ __forceinline__ void store(void* p) const {
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 3; ++j) at(i, j).store((char*)p + 64 * (3 * i + j));
    }
    friend __device__ __noinline__ Fq12 operator*(const Fq12& a, const Fq12& b) {
        const Fq6 t0 = a.c0 * b.c0, t1 = a.c1 * b.c1;
        Fq12 r;
        r.c0 = t0 + t1.mul_v();
        r.c1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1;
        return r;
    }
    // complex squaring: 2 Fq6 products
    __device__ __noinline__ Fq12 sqr() const {
        const Fq6 t = c0 * c1;
        Fq12 r;
        r.c0 = (c0 + c1) * (c0 + c1.mul_v()) - t - t.mul_v();
        r.c1 = t + t;
        return r;
    }
    __device__ __forceinline__ Fq12 conj() const { Fq12 r; r.c0 = c0; r.c1 = c1.neg(); return r; }   // = inverse on the cyclotomic subgroup
    __device__ Fq12 inv() const {
        const Fq6 t = (c0 * c0 - (c1 * c1).mul_v()).inv();
        Fq12 r; r.c0 = c0 * t; r.c1 = (c1 * t).neg();
        return r;
    }
    // x^(p^K), K = 1, 2, 3
    template <int K>
    __device__ Fq12 frobenius() const {
        Fq12 r;
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 3; ++j) {
                const Fq2 c = (K & 1) ? dev::conj(at(i, j)) : at(i, j);
                const int m = 2 * j + i;
                r.at(i, j) = m == 0 ? c : (K == 2 ? scale(c, fq2_from(FROB[1][m]).c0) : c * fq2_from(FROB[K - 1][m]));
            }
        return r;
    }
    // Granger-Scott squaring, valid for elements of the cyclotomic subgroup (after the easy part of the final
    // exponentiation): Fq12 seen as Fq4^3 with Fq4 = Fq2[s]/(s^2 - xi); 6 Fq2 squarings' worth of products
    __device__ __noinline__ Fq12 cyclotomic_sqr() const {
        const Fq2 &z0 = c0.c0, &z4 = c0.c1, &z3 = c0.c2, &z2 = c1.c0, &z1 = c1.c1, &z5 = c1.c2;
        Fq2 t0, t1, t2, t3, t4, t5, tmp;
        tmp = z0 * z1; t0 = (z0 + z1) * (mul_xi(z1) + z0) - tmp - mul_xi(tmp); t1 = tmp.dbl();
        tmp = z2 * z3; t2 = (z2 + z3) * (mul_xi(z3) + z2) - tmp - mul_xi(tmp); t3 = tmp.dbl();
        tmp = z4 * z5; t4 = (z4 + z5) * (mul_xi(z5) + z4) - tmp - mul_xi(tmp); t5 = tmp.dbl();
        Fq12 r;
        r.c0.c0 = (t0 - z0).dbl() + t0;            // 3 t0 - 2 z0
        r.c1.c1 = (t1 + z1).dbl() + t1;            // 3 t1 + 2 z1
        tmp = mul_xi(t5);
        r.c1.c0 = (z2 + tmp).dbl() + tmp;          // 3 xi t5 + 2 z2
        r.c0.c2 = (t4 - z3).dbl() + t4;            // 3 t4 - 2 z3
        r.c0.c1 = (t2 - z4).dbl() + t2;            // 3 t2 - 2 z4
        r.c1.c2 = (t3 + z5).dbl() + t3;            // 3 t3 + 2 z5
        return r;
    }
    // * (l0 + l1 w + l2 v w), the shape of a line value (coefficients at w^0, w^1, w^3)
    __device__ __noinline__ Fq12 mul_line(const Fq2& l0, const Fq2& l1, const Fq2& l2) const {
        Fq6 a; a.c0 = c0.c0 * l0; a.c1 = c0.c1 * l0; a.c2 = c0.c2 * l0;
        const Fq6 b = c1.mul_01(l1, l2);
        Fq12 r;
        r.c1 = (c0 + c1).mul_01(l0 + l1, l2) - a - b;
        r.c0 = a + b.mul_v();
        return r;
    }
};

// ---- Miller loop ----------------------------------------------------------------------------------------------------
// A line through points of the twist, evaluated at P = (xP, yP), is  c0 yP + c1 xP w + c2 v w  up to a factor in Fq2.
// The coefficients do not depend on P: they are what a precomputed line table stores (LINE_BYTES each).
struct LineCoeffs { Fq2 c0, c1, c2; };
struct G2Proj { Fq2 x, y, z; };   // homogeneous projective: x = X/Z, y = Y/Z

// R <- 2R; tangent at R (Costello-Lange-Naehrig, as in arkworks' BN doubling step), coordinates scaled by 4 to avoid halving:
// X' = 2 XY (B - F), Y' = (B + F)^2 - 12 E^2, Z' = 4 B H with B = Y^2, E = 3 b' Z^2, F = 3E, H = 2YZ;
// line = (-H, 3 X^2, E - B)
inline __device__ __noinline__ LineCoeffs dbl_step(G2Proj& r) {
    const Fq2 B = r.y.sqr(), C = r.z.sqr();
    const Fq2 E = fq2_from(TWIST_B) * (C.dbl() + C);
    const Fq2 F = E.dbl() + E;
    const Fq2 H = (r.y + r.z).sqr() - B - C;
    const Fq2 J = r.x.sqr();
    LineCoeffs l;
    l.c0 = H.neg(); l.c1 = J.dbl() + J; l.c2 = E - B;
    const Fq2 E2 = E.sqr();
    const Fq2 BF = B + F;
    r.x = (r.x * r.y).dbl() * (B - F);
    r.y = BF.sqr() - (E2.dbl() + E2).dbl().dbl();
    r.z = (B * H).dbl().dbl();
    return l;
}
// R <- R + Q (Q affine); chord through R and Q: theta = Y - qy Z, lambda = X - qx Z; line = (lambda, -theta, theta qx - lambda qy)
inline __device__ __noinline__ LineCoeffs add_step(G2Proj& r, const G2Affine& q) {
    const Fq2 theta = r.y - q.y * r.z, lambda = r.x - q.x * r.z;
    const Fq2 C = theta.sqr(), D = lambda.sqr();
    const Fq2 E = lambda * D, F = r.z * C, G = r.x * D;
    const Fq2 H = E + F - G.dbl();
    LineCoeffs l;
    l.c0 = lambda; l.c1 = theta.neg(); l.c2 = theta * q.x - lambda * q.y;
    r.x = lambda * H;
    r.y = theta * (G - H) - E * r.y;
    r.z = r.z * E;
    return l;
}
__device__ __forceinline__ Fq12 mul_line_at(const Fq12& f, const LineCoeffs& l, const G1Affine& p) {
    return f.mul_line(scale(l.c0, p.y), scale(l.c1, p.x), l.c2);
}
__device__ __forceinline__ LineCoeffs load_line(const uint8_t* lines, int k) {
    const uint8_t* s = lines + (size_t)LINE_BYTES * k;
    LineCoeffs l; l.c0 = Fq2::load(s); l.c1 = Fq2::load(s + 64); l.c2 = Fq2::load(s + 128);
    return l;
}
// pi(Q) = (conj(x) xi^((p-1)/3), conj(y) xi^((p-1)/2)) and -pi^2(Q) = (x xi^((p^2-1)/3), -y xi^((p^2-1)/2))
__device__ __forceinline__ G2Affine twist_frobenius(const G2Affine& q) {
    G2Affine r; r.x = conj(q.x) * fq2_from(FROB[0][2]); r.y = conj(q.y) * fq2_from(FROB[0][3]); return r;
}
__device__ __forceinline__ G2Affine twist_frobenius2_neg(const G2Affine& q) {
    G2Affine r; r.x = scale(q.x, fq2_from(FROB[1][2]).c0); r.y = scale(q.y, fq2_from(FROB[1][3]).c0).neg(); return r;
}

// Product of the Miller loops of up to 1 + NFIX pairs sharing one accumulator (one Fq12 squaring per step for all):
//   pair 0: (q, p), lines computed on the fly - included only if `fly`; `record` (optional) receives its ATE_LINES lines;
//   pair 1 + k: precomputed lines fixed_lines[k] of a fixed G2 point, evaluated at fixed_p[k] - skipped if null.
// A pair with a point at infinity contributes 1 (as pairing_host.cpp's miller_loop).
template <int NFIX>
__device__ Fq12 miller_loop(bool fly, const G2Affine& q, const G1Affine& p, const uint8_t* const* fixed_lines,
                            const G1Affine* fixed_p, uint8_t* record) {
    fly = fly && !q.is_inf() && !p.is_inf();
    bool use[NFIX > 0 ? NFIX : 1];
    for (int k = 0; k < NFIX; ++k) use[k] = fixed_lines[k] != nullptr && !fixed_p[k].is_inf();
    G2Proj r; r.x = q.x; r.y = q.y; r.z = Fq2::one();
    Fq12 f = Fq12::one();
    int li = 0;
    auto step = [&](const LineCoeffs& l) {
        if (fly) {
            f = mul_line_at(f, l, p);
            if (record) {
                uint8_t* d = record + (size_t)LINE_BYTES * li;
                l.c0.store(d); l.c1.store(d + 64); l.c2.store(d + 128);
            }
        }
        for (int k = 0; k < NFIX; ++k)
            if (use[k]) f = mul_line_at(f, load_line(fixed_lines[k], li), fixed_p[k]);
        ++li;
    };
    for (int i = 63; i >= 0; --i) {
        f = f.sqr();
        step(fly ? dbl_step(r) : LineCoeffs());
        if ((ATE_LOW >> i) & 1) step(fly ? add_step(r, q) : LineCoeffs());
    }
    step(fly ? add_step(r, twist_frobenius(q)) : LineCoeffs());
    step(fly ? add_step(r, twist_frobenius2_neg(q)) : LineCoeffs());
    return f;
}

// ---- final exponentiation -------------------------------------------------------------------------------------------
// x^(-z) on the cyclotomic subgroup
inline __device__ Fq12 cyclotomic_exp_neg_z(const Fq12& x) {
    Fq12 r = x;
    for (int i = 61; i >= 0; --i) {     // bit 62 is the top bit of z
        r = r.cyclotomic_sqr();
        if ((BN_Z >> i) & 1) r = r * x;
    }
    return r.conj();
}
// f^((p^12 - 1) / r) raised to 2 z (6 z^2 + 3 z + 1): easy part f^((p^6 - 1)(p^2 + 1)), then the Fuentes-Castaneda hard part
inline __device__ Fq12 final_exponentiation(const Fq12& f) {
    Fq12 m = f.conj() * f.inv();
    m = m.frobenius<2>() * m;
    const Fq12 y0 = cyclotomic_exp_neg_z(m);
    const Fq12 y1 = y0.cyclotomic_sqr();
    const Fq12 y2 = y1.cyclotomic_sqr();
    const Fq12 y3 = y2 * y1;
    const Fq12 y4 = cyclotomic_exp_neg_z(y3);
    const Fq12 y5 = y4.cyclotomic_sqr();
    const Fq12 y6 = cyclotomic_exp_neg_z(y5);
    const Fq12 y7 = y6.conj() * y4;
    const Fq12 y8 = y7 * y3.conj();
    const Fq12 y9 = y8 * y1;
    const Fq12 y10 = y8 * y4;
    const Fq12 y11 = y10 * m;
    const Fq12 y13 = y9.frobenius<1>() * y11;
    const Fq12 y14 = y8.frobenius<2>() * y13;
    const Fq12 y15 = (m.conj() * y9).frobenius<3>();
    return y15 * y14;
}

// ---- curve membership ----------------------------------------------------------------------------------------------
__device__ __forceinline__ bool g1_on_curve(const G1Affine& a) {
    if (a.is_inf()) return true;
    const Fq three = Fq::one().dbl() + Fq::one();
    return a.y.sqr() == a.x.sqr() * a.x + three;
}
__device__ __forceinline__ bool g2_on_curve(const G2Affine& a) {
    if (a.is_inf()) return true;
    return a.y.sqr() == a.x.sqr() * a.x + fq2_from(TWIST_B);
}
__device__ __forceinline__ G1Affine g1_to_affine(const G1XYZZ& a) {
    G1Affine r;
    if (a.is_inf()) { r.x = Fq::zero(); r.y = Fq::zero(); return r; }
    const Fq zzz_inv = a.zzz.inv();
    const Fq zz_inv = (a.zz * zzz_inv).sqr();   // 1/zz = zz^2 / zzz^2 (zz^3 = zzz^2)
    r.x = a.x * zz_inv; r.y = a.y * zzz_inv;
    return r;
}

}  // namespace dev
}  // namespace zke
