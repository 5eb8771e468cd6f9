// Host-side BN254 G1 / G2 arithmetic (Jacobian coordinates) for the trusted-setup tables, the last few group
// operations of a proof (r, s blinding) and the verifier.  Heavy lifting (MSM, fixed-base batches) is on the GPU.
#pragma once
#include "ff_host.hpp"

namespace zke {

struct Fq2 {
    Fq c0, c1;
    static Fq2 zero() { return Fq2{Fq::zero(), Fq::zero()}; }
    static Fq2 one() { return Fq2{Fq::one(), Fq::zero()}; }
    bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    bool operator==(const Fq2& o) const { return c0 == o.c0 && c1 == o.c1; }
    bool operator!=(const Fq2& o) const { return !(*this == o); }
    Fq2 operator+(const Fq2& o) const { return Fq2{c0 + o.c0, c1 + o.c1}; }
    Fq2 operator-(const Fq2& o) const { return Fq2{c0 - o.c0, c1 - o.c1}; }
    Fq2 operator*(const Fq2& o) const {
        Fq t0 = c0 * o.c0, t1 = c1 * o.c1;
        return Fq2{t0 - t1, (c0 + c1) * (o.c0 + o.c1) - t0 - t1};
    }
    Fq2 sqr() const { Fq t = c0 * c1; return Fq2{(c0 + c1) * (c0 - c1), t + t}; }
    Fq2 neg() const { return Fq2{c0.neg(), c1.neg()}; }
    Fq2 scale(const Fq& k) const { return Fq2{c0 * k, c1 * k}; }
    Fq2 conj() const { return Fq2{c0, c1.neg()}; }
    Fq2 mul_xi() const {  // * (9 + u)
        Fq n0 = c0 + c0; n0 = n0 + n0; n0 = n0 + n0; n0 = n0 + c0;   // 9 c0
        Fq n1 = c1 + c1; n1 = n1 + n1; n1 = n1 + n1; n1 = n1 + c1;   // 9 c1
        return Fq2{n0 - c1, n1 + c0};
    }
    Fq2 inv() const {
        Fq d = (c0.sqr() + c1.sqr()).inv();
        return Fq2{c0 * d, (c1 * d).neg()};
    }
    Fq2& operator+=(const Fq2& o) { *this = *this + o; return *this; }
    Fq2& operator-=(const Fq2& o) { *this = *this - o; return *this; }
    Fq2& operator*=(const Fq2& o) { *this = *this * o; return *this; }
};

// Affine point; infinity is encoded as (0, 0) (same image as on the device).
template <class F>
struct AffineH {
    F x, y;
    bool is_inf() const { return x.is_zero() && y.is_zero(); }
    static AffineH inf() { return AffineH{F::zero(), F::zero()}; }
};

template <class F>
struct JacobianH {
    F x, y, z;
    static JacobianH inf() { return JacobianH{F::one(), F::one(), F::zero()}; }
    static JacobianH from_affine(const AffineH<F>& p) { return p.is_inf() ? inf() : JacobianH{p.x, p.y, F::one()}; }
    bool is_inf() const { return z.is_zero(); }

    JacobianH dbl() const {
        if (is_inf()) return *this;
        F A = x.sqr(), B = y.sqr(), C = B.sqr();
        F t = (x + B).sqr() - A - C;
        F D = t + t;
        F E = A + A + A;
        F Fv = E.sqr();
        F X3 = Fv - D - D;
        F C8 = C + C; C8 = C8 + C8; C8 = C8 + C8;
        F Y3 = E * (D - X3) - C8;
        F yz = y * z;
        return JacobianH{X3, Y3, yz + yz};
    }
    JacobianH add(const JacobianH& o) const {
        if (is_inf()) return o;
        if (o.is_inf()) return *this;
        F Z1Z1 = z.sqr(), Z2Z2 = o.z.sqr();
        F U1 = x * Z2Z2, U2 = o.x * Z1Z1;
        F S1 = y * o.z * Z2Z2, S2 = o.y * z * Z1Z1;
        if (U1 == U2) return S1 == S2 ? dbl() : inf();
        F H = U2 - U1, R = S2 - S1;
        F HH = H.sqr(), HHH = H * HH, V = U1 * HH;
        F X3 = R.sqr() - HHH - V - V;
        F Y3 = R * (V - X3) - S1 * HHH;
        return JacobianH{X3, Y3, z * o.z * H};
    }
    JacobianH add_affine(const AffineH<F>& p) const { return add(from_affine(p)); }
    JacobianH neg() const { JacobianH r = *this; r.y = F::zero() - y; return r; }
    JacobianH mul(const U256& k) const {
        JacobianH r = inf();
        for (int i = 255; i >= 0; --i) {
            r = r.dbl();
            if (u256_bit(k, i)) r = r.add(*this);
        }
        return r;
    }
    AffineH<F> to_affine() const {
        if (is_inf()) return AffineH<F>::inf();
        F zi = z.inv(), zi2 = zi.sqr();
        return AffineH<F>{x * zi2, y * zi2 * zi};
    }
};

typedef AffineH<Fq> G1AffineH;
typedef AffineH<Fq2> G2AffineH;
typedef JacobianH<Fq> G1JacH;
typedef JacobianH<Fq2> G2JacH;

G1AffineH g1_generator();
G2AffineH g2_generator();
bool g1_on_curve(const G1AffineH& p);
bool g2_on_curve(const G2AffineH& p);

// Host byte format (pairing_host.cpp): 32-byte little-endian standard form; G1 = x, y; G2 = x.c0, x.c1, y.c0, y.c1;
// infinity = all zero.  put_* append to `out`.  The readers throw "<what> not reduced" on a coordinate not below q;
// whether a point must be on its curve or in its subgroup is the caller's policy.
void store_fq(uint8_t* out, const Fq& x);
void store_fr(uint8_t* out, const Fr& x);
void store_g1(uint8_t* out, const G1AffineH& p);
void store_g2(uint8_t* out, const G2AffineH& p);
void put_fr(std::vector<uint8_t>& out, const Fr& x);
void put_g1(std::vector<uint8_t>& out, const G1AffineH& p);
void put_g2(std::vector<uint8_t>& out, const G2AffineH& p);
Fq fq_at(const uint8_t* p, const char* what = "coordinate");
G1AffineH load_g1(const uint8_t* p, const char* what = "coordinate");
G2AffineH load_g2(const uint8_t* p, const char* what = "coordinate");

// Host mirror of the device accumulator (extended Jacobian, x = X/ZZ, y = Y/ZZZ); same memory image.
template <class F>
struct XyzzH {
    F x, y, zz, zzz;
    static XyzzH inf() { return XyzzH{F::zero(), F::zero(), F::zero(), F::zero()}; }
    bool is_inf() const { return zz.is_zero(); }
    void dbl() {
        if (is_inf()) return;
        F U = y + y, V = U.sqr(), W = U * V, S = x * V;
        F X2 = x.sqr(), M = X2 + X2 + X2;
        F X3 = M.sqr() - S - S;
        F Y3 = M * (S - X3) - W * y;
        zz = V * zz; zzz = W * zzz; x = X3; y = Y3;
    }
    void add(const XyzzH& o) {
        if (o.is_inf()) return;
        if (is_inf()) { *this = o; return; }
        F U1 = x * o.zz, U2 = o.x * zz, S1 = y * o.zzz, S2 = o.y * zzz;
        F P = U2 - U1, R = S2 - S1;
        if (P.is_zero()) { if (R.is_zero()) { dbl(); return; } *this = inf(); return; }
        F PP = P.sqr(), PPP = P * PP, Q = U1 * PP;
        F X3 = R.sqr() - PPP - Q - Q;
        F Y3 = R * (Q - X3) - S1 * PPP;
        zz = zz * o.zz * PP; zzz = zzz * o.zzz * PPP; x = X3; y = Y3;
    }
    AffineH<F> to_affine() const {
        if (is_inf()) return AffineH<F>::inf();
        return AffineH<F>{x * zz.inv(), y * zzz.inv()};
    }
};

// Groth16 verification (optimal ate pairing over the Fq2-Fq6-Fq12 tower); see pairing_host.cpp.
struct VerifyingKey {
    G1AffineH alpha1;
    G2AffineH beta2, gamma2, delta2;
    std::vector<G1AffineH> ic;   // nPublic + 1
};
struct Proof {
    G1AffineH a, c;
    G2AffineH b;
};
bool groth16_verify(const VerifyingKey& vk, const std::vector<U256>& publics, const Proof& pr);
// n proofs under one key with one randomised product of pairings; rnd: n non-zero scalars below 2^128
bool groth16_verify_batch(const VerifyingKey& vk, const std::vector<std::vector<U256>>& publics, const std::vector<Proof>& proofs,
                          const std::vector<U256>& rnd);
bool g2_in_subgroup(const G2AffineH& p);
// prod_i e(P_i, Q_i) == 1 (points on their curves, G2 points in the subgroup)
bool pairing_product_is_one(const std::vector<std::pair<G1AffineH, G2AffineH>>& terms);
// snarkjs vkey.json -> key (capi_json.cpp); throws on malformed JSON, unreduced coordinates or an empty IC
VerifyingKey vkey_from_json(const char* json);
void pairing_alphabeta(const G1AffineH& alpha1, const G2AffineH& beta2, U256 out[12]);   // snarkjs vk_alphabeta_12, [i][j][k] flattened

}  // namespace zke
