// Host Groth16 verifier: optimal ate pairing on BN254.
//
// Boundary: snarkjs.groth16.verify(vkey, publicSignals, proof) (/root/reference/packages/helpers/src/chunked-zkey.ts:101)
// and its Rust twin GrothBn::verify (/root/reference/packages/rust-verifier/src/verifier_utils.rs:20).  ms-scale CPU
// work (SURVEY 8(a) a18), so a compact formulation is used: Fq12 = Fq[w]/(w^12 - 18 w^6 + 82) as dense
// polynomials (w^6 = 9 + u), point arithmetic on the sextic twist in Fq2 (affine), line functions embedded as
// sparse Fq12 elements, final exponentiation by plain square-and-multiply with the exponent (p^12 - 1)/r.
#include "ec_host.hpp"
#include "aggregate_host.hpp"
#include <array>
#include <cstring>

namespace zke {

G1AffineH g1_generator() { return G1AffineH{Fq::from_u64(1), Fq::from_u64(2)}; }
G2AffineH g2_generator() {
    return G2AffineH{
        Fq2{Fq::from_dec("10857046999023057135944570762232829481370756359578518086990519993285655852781"),
            Fq::from_dec("11559732032986387107991004021392285783925812861821192530917403151452391805634")},
        Fq2{Fq::from_dec("8495653923123431417604973247489272438418190587263600148770280649306958101930"),
            Fq::from_dec("4082367875863433681332203403145435568316851327593401208105741076214120093531")}};
}
bool g1_on_curve(const G1AffineH& p) {
    if (p.is_inf()) return true;
    return p.y.sqr() == p.x.sqr() * p.x + Fq::from_u64(3);
}
static Fq2 twist_b() {
    static const Fq2 b = Fq2{Fq::from_u64(3), Fq::zero()} * Fq2{Fq::from_u64(9), Fq::one()}.inv();
    return b;
}
bool g2_on_curve(const G2AffineH& p) {
    if (p.is_inf()) return true;
    return p.y.sqr() == p.x.sqr() * p.x + twist_b();
}

void store_fq(uint8_t* out, const Fq& x) { const U256 s = x.to_u256(); memcpy(out, s.v, 32); }
void store_fr(uint8_t* out, const Fr& x) { const U256 s = x.to_u256(); memcpy(out, s.v, 32); }
void store_g1(uint8_t* out, const G1AffineH& p) { store_fq(out, p.x); store_fq(out + 32, p.y); }
void store_g2(uint8_t* out, const G2AffineH& p) { store_fq(out, p.x.c0); store_fq(out + 32, p.x.c1); store_fq(out + 64, p.y.c0); store_fq(out + 96, p.y.c1); }
void put_fr(std::vector<uint8_t>& out, const Fr& x) { out.resize(out.size() + 32); store_fr(&out[out.size() - 32], x); }
void put_g1(std::vector<uint8_t>& out, const G1AffineH& p) { out.resize(out.size() + 64); store_g1(&out[out.size() - 64], p); }
void put_g2(std::vector<uint8_t>& out, const G2AffineH& p) { out.resize(out.size() + 128); store_g2(&out[out.size() - 128], p); }

Fq fq_at(const uint8_t* p, const char* what) {
    U256 x;
    memcpy(x.v, p, 32);
    if (u256_cmp(x, fq_params().p) >= 0) throw std::runtime_error(std::string(what) + " not reduced");
    return Fq::from_u256(x);
}
G1AffineH load_g1(const uint8_t* p, const char* what) { return G1AffineH{fq_at(p, what), fq_at(p + 32, what)}; }
G2AffineH load_g2(const uint8_t* p, const char* what) {
    return G2AffineH{Fq2{fq_at(p, what), fq_at(p + 32, what)}, Fq2{fq_at(p + 64, what), fq_at(p + 96, what)}};
}

namespace {

struct F12 {
    std::array<Fq, 12> c;
    static F12 zero() { F12 r; for (auto& x : r.c) x = Fq::zero(); return r; }
    static F12 one() { F12 r = zero(); r.c[0] = Fq::one(); return r; }
    bool operator==(const F12& o) const { for (int i = 0; i < 12; ++i) if (c[i] != o.c[i]) return false; return true; }
};

F12 mul(const F12& a, const F12& b) {
    Fq t[23];
    for (auto& x : t) x = Fq::zero();
    for (int i = 0; i < 12; ++i) {
        if (a.c[i].is_zero()) continue;
        for (int j = 0; j < 12; ++j) t[i + j] += a.c[i] * b.c[j];
    }
    static const Fq k18 = Fq::from_u64(18), k82 = Fq::from_u64(82);
    for (int i = 22; i >= 12; --i) {   // w^12 = 18 w^6 - 82
        if (t[i].is_zero()) continue;
        t[i - 6] += k18 * t[i];
        t[i - 12] -= k82 * t[i];
    }
    F12 r;
    for (int i = 0; i < 12; ++i) r.c[i] = t[i];
    return r;
}

// a + b*u (Fq2) times w^k, embedded with u = w^6 - 9
void add_fq2_term(F12& f, const Fq2& v, int k) {
    Fq nine_b = v.c1 + v.c1; nine_b = nine_b + nine_b; nine_b = nine_b + nine_b; nine_b = nine_b + v.c1;
    f.c[k] += v.c0 - nine_b;
    f.c[k + 6] += v.c1;
}

// line through R (and S, or tangent at R) on the twist, evaluated at P:  -yP + (lambda xP) w + (yR - lambda xR) w^3
F12 line_eval(const Fq2& lambda, const G2AffineH& r, const G1AffineH& p) {
    F12 f = F12::zero();
    f.c[0] = p.y.neg();
    add_fq2_term(f, lambda.scale(p.x), 1);
    add_fq2_term(f, r.y - lambda * r.x, 3);
    return f;
}

Fq2 fq2_pow(const Fq2& a, const U256& e) {
    Fq2 res = Fq2::one();
    for (int i = 255; i >= 0; --i) {
        res = res.sqr();
        if (u256_bit(e, i)) res = res * a;
    }
    return res;
}

G2AffineH frobenius_twist(const G2AffineH& q) {
    // (x w^2, y w^3)^p = (conj(x) xi^((p-1)/3) w^2, conj(y) xi^((p-1)/2) w^3)
    static bool init = false;
    static Fq2 gx, gy;
    if (!init) {
        U256 pm1; U256 one = {{1, 0, 0, 0}};
        u256_sub(pm1, fq_params().p, one);
        // (p-1)/3 and (p-1)/2 by schoolbook division of a 256-bit integer by a small constant
        auto div_small = [](const U256& a, uint64_t d) {
            U256 q; u128 rem = 0;
            for (int i = 3; i >= 0; --i) { u128 cur = (rem << 64) | a.v[i]; q.v[i] = (uint64_t)(cur / d); rem = cur % d; }
            return q;
        };
        Fq2 xi{Fq::from_u64(9), Fq::one()};
        gx = fq2_pow(xi, div_small(pm1, 3));
        gy = fq2_pow(xi, div_small(pm1, 2));
        init = true;
    }
    return G2AffineH{q.x.conj() * gx, q.y.conj() * gy};
}

F12 miller_loop(const G2AffineH& q, const G1AffineH& p) {
    if (q.is_inf() || p.is_inf()) return F12::one();
    static const uint64_t ATE = 0x9d797039be763ba8ull;  // low 64 bits of 6t+2 = 0x19d797039be763ba8 (top bit implicit: R starts at Q)
    G2AffineH r = q;
    F12 f = F12::one();
    auto dbl_step = [&]() {
        Fq2 x2 = r.x.sqr();
        Fq2 lambda = (x2 + x2 + x2) * (r.y + r.y).inv();
        F12 l = line_eval(lambda, r, p);
        Fq2 x3 = lambda.sqr() - r.x - r.x;
        Fq2 y3 = lambda * (r.x - x3) - r.y;
        r = G2AffineH{x3, y3};
        return l;
    };
    auto add_step = [&](const G2AffineH& s) {
        // r == +-s cannot happen for a point of the order-r subgroup (the callers check membership); should it, the
        // line degenerates - treat it like the tangent / vertical case instead of dividing by zero
        if (s.x == r.x) {
            if (s.y == r.y) return dbl_step();
            F12 l = F12::zero();
            l.c[0] = p.x;
            add_fq2_term(l, r.x.neg(), 2);
            r = G2AffineH::inf();
            return l;
        }
        Fq2 lambda = (s.y - r.y) * (s.x - r.x).inv();
        F12 l = line_eval(lambda, r, p);
        Fq2 x3 = lambda.sqr() - r.x - s.x;
        Fq2 y3 = lambda * (r.x - x3) - r.y;
        r = G2AffineH{x3, y3};
        return l;
    };
    for (int i = 63; i >= 0; --i) {
        f = mul(mul(f, f), dbl_step());
        if ((ATE >> i) & 1) f = mul(f, add_step(q));
    }
    G2AffineH q1 = frobenius_twist(q);
    G2AffineH q2 = frobenius_twist(q1);
    q2.y = q2.y.neg();
    f = mul(f, add_step(q1));
    f = mul(f, add_step(q2));
    return f;
}

F12 final_exponentiation(const F12& f) {
    static const char* EXP_HEX =
        "2f4b6dc97020fddadf107d20bc842d43bf6369b1ff6a1c71015f3f7be2e1e30a73bb94fec0daf15466b2383a5d3ec3d15ad524d8f70c54efee1b"
        "d8c3b21377e563a09a1b705887e72eceaddea3790364a61f676baaf977870e88d5c6c8fef0781361e443ae77f5b63a2a2264487f2940a8b1ddb3"
        "d15062cd0fb2015dfc6668449aed3cc48a82d0d602d268c7daab6a41294c0cc4ebe5664568dfc50e1648a45a4a1e3a5195846a3ed011a337a020"
        "88ec80e0ebae8755cfe107acf3aafb40494e406f804216bb10cf430b0f37856b42db8dc5514724ee93dfb10826f0dd4a0364b9580291d2cd6566"
        "4814fde37ca80bb4ea44eacc5e641bbadf423f9a2cbf813b8d145da90029baee7ddadda71c7f3811c4105262945bba1668c3be69a3c230974d83"
        "561841d766f9c9d570bb7fbe04c7e8a6c3c760c0de81def35692da361102b6b9b2b918837fa97896e84abb40a4efb7e54523a486964b64ca86f1"
        "20";
    F12 res = F12::one();
    for (const char* s = EXP_HEX; *s; ++s) {
        int d = (*s >= '0' && *s <= '9') ? *s - '0' : *s - 'a' + 10;
        for (int b = 3; b >= 0; --b) {
            res = mul(res, res);
            if ((d >> b) & 1) res = mul(res, f);
        }
    }
    return res;
}

F12 pow_u256(const F12& f, const U256& e) {
    F12 res = F12::one();
    for (int i = 255; i >= 0; --i) {
        res = mul(res, res);
        if (u256_bit(e, i)) res = mul(res, f);
    }
    return res;
}

}  // namespace

// Order-r subgroup membership of a G2 point: BN254's G2 has a large cofactor, so the curve equation alone does not
// imply it (ark-groth16, the Rust twin of this verifier, rejects such points on deserialisation).
bool g2_in_subgroup(const G2AffineH& p) {
    if (p.is_inf()) return true;
    return G2JacH::from_affine(p).mul(fr_params().p).is_inf();
}

// vk_alphabeta_12 of `snarkjs zkey export verificationkey`: e(alpha_1, beta_2) as the Fq2-Fq6-Fq12 tower element
// out[i][j][k] (Fq12 = Fq6[w]/(w^2 - v), Fq6 = Fq2[v]/(v^3 - (9 + u))), in standard form.  ffjavascript / wasmcurves
// (like libff) finish the pairing with the Fuentes-Castaneda hard part, which yields the reduced pairing raised to
// 2 z (6 z^2 + 3 z + 1), z = 4965661367192848881 - reproduced here; pinned on the reference's fixture
// (/root/reference/packages/rust-verifier/tests/data/proof_of_twitter/vkey.json:43).
void pairing_alphabeta(const G1AffineH& alpha1, const G2AffineH& beta2, U256 out[12]) {
    static const U256 K = u256_from_hex("3bec47df15e307c81ea96b02d9d9e38d2e5d4e223ddedaf4");
    const F12 e = pow_u256(final_exponentiation(miller_loop(beta2, alpha1)), K);
    // dense sum c_n w^n with u = w^6 - 9  ->  tower coefficient (i, j) = (c[2j+i] + 9 c[2j+i+6]) + c[2j+i+6] u
    const Fq nine = Fq::from_u64(9);
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 3; ++j) {
            const int n = 2 * j + i;
            out[(i * 3 + j) * 2 + 0] = (e.c[n] + nine * e.c[n + 6]).to_u256();
            out[(i * 3 + j) * 2 + 1] = e.c[n + 6].to_u256();
        }
}

// GT arithmetic for the aggregate verifier (aggregate_host.hpp): values normalised like pairing_alphabeta
namespace agg {
Gt gt_one() { return Gt{F12::one().c}; }
Gt gt_mul(const Gt& a, const Gt& b) { return Gt{mul(F12{a.c}, F12{b.c}).c}; }
Gt gt_pow(const Gt& a, const U256& e) { return Gt{pow_u256(F12{a.c}, e).c}; }
Gt gt_pairing_product(const std::vector<std::pair<G1AffineH, G2AffineH>>& terms) {
    static const U256 K = u256_from_hex("3bec47df15e307c81ea96b02d9d9e38d2e5d4e223ddedaf4");
    F12 f = F12::one();
    for (auto& t : terms) f = mul(f, miller_loop(t.second, t.first));
    return Gt{pow_u256(final_exponentiation(f), K).c};
}
void gt_store(const Gt& e, uint8_t out[384]) {
    const Fq nine = Fq::from_u64(9);
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 3; ++j) {
            const int n = 2 * j + i;
            store_fq(out + 64 * (3 * i + j), e.c[n] + nine * e.c[n + 6]);
            store_fq(out + 64 * (3 * i + j) + 32, e.c[n + 6]);
        }
}
Gt gt_load(const uint8_t* in) {
    const Fq nine = Fq::from_u64(9);
    Gt e;
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 3; ++j) {
            const int n = 2 * j + i;
            const Fq a = fq_at(in + 64 * (3 * i + j)), b = fq_at(in + 64 * (3 * i + j) + 32);
            e.c[n] = a - nine * b;
            e.c[n + 6] = b;
        }
    return e;
}
}  // namespace agg

bool pairing_product_is_one(const std::vector<std::pair<G1AffineH, G2AffineH>>& terms) {
    F12 f = F12::one();
    for (auto& t : terms) f = mul(f, miller_loop(t.second, t.first));
    return final_exponentiation(f) == F12::one();
}

bool groth16_verify(const VerifyingKey& vk, const std::vector<U256>& publics, const Proof& pr) {
    if (publics.size() + 1 != vk.ic.size()) return false;
    for (auto& s : publics) if (u256_cmp(s, fr_params().p) >= 0) return false;
    if (!g1_on_curve(pr.a) || !g1_on_curve(pr.c) || !g2_on_curve(pr.b)) return false;
    if (!g1_on_curve(vk.alpha1) || !g2_on_curve(vk.beta2) || !g2_on_curve(vk.gamma2) || !g2_on_curve(vk.delta2)) return false;
    if (!g2_in_subgroup(pr.b) || !g2_in_subgroup(vk.beta2) || !g2_in_subgroup(vk.gamma2) || !g2_in_subgroup(vk.delta2)) return false;
    G1JacH vkx = G1JacH::from_affine(vk.ic[0]);
    for (size_t i = 0; i < publics.size(); ++i) {
        if (!g1_on_curve(vk.ic[i + 1])) return false;
        vkx = vkx.add(G1JacH::from_affine(vk.ic[i + 1]).mul(publics[i]));
    }
    G1AffineH neg_a = pr.a;
    neg_a.y = neg_a.y.neg();
    // e(-A, B) e(alpha, beta) e(vk_x, gamma) e(C, delta) == 1
    F12 f = miller_loop(pr.b, neg_a);
    f = mul(f, miller_loop(vk.beta2, vk.alpha1));
    f = mul(f, miller_loop(vk.gamma2, vkx.to_affine()));
    f = mul(f, miller_loop(vk.delta2, pr.c));
    return final_exponentiation(f) == F12::one();
}

// Batch verification under one key (SURVEY 8(f) rank 4; the step after the path when proofs are produced 64 at a time).
// With random 128-bit r_i the n equations e(A_i, B_i) = e(alpha, beta) e(X_i, gamma) e(C_i, delta) are checked as ONE
// product:  prod_i e(-r_i A_i, B_i) * e((sum r_i) alpha, beta) * e(sum_i r_i X_i, gamma) * e(sum_i r_i C_i, delta) == 1,
// i.e. n + 3 Miller loops and one final exponentiation instead of 4 n and n (a false proof passes with probability
// ~2^-128 over the r_i, which the prover must not know in advance).  sum_i r_i X_i only needs nPublic + 1 scalar
// multiplications: X_i = IC_0 + sum_j s_ij IC_j, so the coefficient of IC_j is sum_i r_i s_ij mod r.
// Input validation is that of groth16_verify; a malformed or off-curve proof makes the batch fail.
bool groth16_verify_batch(const VerifyingKey& vk, const std::vector<std::vector<U256>>& publics, const std::vector<Proof>& proofs,
                          const std::vector<U256>& rnd) {
    const size_t n = proofs.size();
    if (publics.size() != n || rnd.size() != n) return false;
    if (n == 0) return true;
    if (!g1_on_curve(vk.alpha1) || !g2_on_curve(vk.beta2) || !g2_on_curve(vk.gamma2) || !g2_on_curve(vk.delta2)) return false;
    if (!g2_in_subgroup(vk.beta2) || !g2_in_subgroup(vk.gamma2) || !g2_in_subgroup(vk.delta2)) return false;
    for (auto& p : vk.ic) if (!g1_on_curve(p)) return false;
    const size_t np = vk.ic.size() - 1;
    std::vector<Fr> coeff(np + 1, Fr::zero());
    G1JacH c_sum = G1JacH::inf();
    F12 f = F12::one();
    for (size_t i = 0; i < n; ++i) {
        const Proof& pr = proofs[i];
        if (publics[i].size() != np) return false;
        for (auto& sgn : publics[i]) if (u256_cmp(sgn, fr_params().p) >= 0) return false;
        if (rnd[i].is_zero() || rnd[i].v[2] != 0 || rnd[i].v[3] != 0) return false;
        if (!g1_on_curve(pr.a) || !g1_on_curve(pr.c) || !g2_on_curve(pr.b) || !g2_in_subgroup(pr.b)) return false;
        const Fr ri = Fr::from_u256(rnd[i]);
        coeff[0] = coeff[0] + ri;
        for (size_t j = 0; j < np; ++j) coeff[j + 1] = coeff[j + 1] + ri * Fr::from_u256(publics[i][j]);
        c_sum = c_sum.add(G1JacH::from_affine(pr.c).mul(rnd[i]));
        G1AffineH ra = G1JacH::from_affine(pr.a).mul(rnd[i]).to_affine();
        ra.y = ra.y.neg();
        f = mul(f, miller_loop(pr.b, ra));
    }
    G1JacH x_sum = G1JacH::inf();
    for (size_t j = 0; j <= np; ++j) x_sum = x_sum.add(G1JacH::from_affine(vk.ic[j]).mul(coeff[j].to_u256()));
    f = mul(f, miller_loop(vk.beta2, G1JacH::from_affine(vk.alpha1).mul(coeff[0].to_u256()).to_affine()));
    f = mul(f, miller_loop(vk.gamma2, x_sum.to_affine()));
    f = mul(f, miller_loop(vk.delta2, c_sum.to_affine()));
    return final_exponentiation(f) == F12::one();
}

}  // namespace zke
