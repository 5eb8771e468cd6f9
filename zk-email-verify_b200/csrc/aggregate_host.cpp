// Host verifier of a Groth16 proof aggregate (SnarkPack; DESIGN.md "Proof aggregation") and the pieces the GPU prover
// (aggregate.cu) shares with it: SHA-256 transcript, encodings, folded-key polynomials.  The pairings are those of
// pairing_host.cpp; the verifier runs 10 GT exponentiations per round, then 18 Miller loops and 10 final exponentiations.
#include "aggregate_host.hpp"
#include "../../include/zkemail_b200.h"
#include "engine.hpp"
#include <cstring>
#include <stdexcept>

namespace zke {
namespace agg {

namespace {
const char DOMAIN_TAG[] = "zkemail-snarkpack-groth16-v1";

uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
const uint32_t K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
}  // namespace

void sha256(const uint8_t* data, size_t len, uint8_t out[32]) {
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
    std::vector<uint8_t> m(data, data + len);
    m.push_back(0x80);
    while (m.size() % 64 != 56) m.push_back(0);
    for (int i = 7; i >= 0; --i) m.push_back((uint8_t)((uint64_t)len * 8 >> (8 * i)));
    for (size_t off = 0; off < m.size(); off += 64) {
        uint32_t w[64];
        for (int i = 0; i < 16; ++i)
            w[i] = (uint32_t)m[off + 4 * i] << 24 | (uint32_t)m[off + 4 * i + 1] << 16 | (uint32_t)m[off + 4 * i + 2] << 8 | m[off + 4 * i + 3];
        for (int i = 16; i < 64; ++i) {
            const uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
            const uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
            w[i] = w[i - 16] + s0 + w[i - 7] + s1;
        }
        uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], k = h[7];
        for (int i = 0; i < 64; ++i) {
            const uint32_t t1 = k + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K256[i] + w[i];
            const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
            k = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
        h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += k;
    }
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 4; ++j) out[4 * i + j] = (uint8_t)(h[i] >> (24 - 8 * j));
}

Fr challenge(const std::vector<uint8_t>& bytes) {
    uint8_t d[32];
    sha256(bytes.data(), bytes.size(), d);
    U256 x;
    memcpy(x.v, d, 32);
    while (u256_cmp(x, fr_params().p) >= 0) u256_sub(x, x, fr_params().p);
    if (x.is_zero()) throw std::runtime_error("aggregation transcript produced a zero challenge");
    return Fr::from_u256(x);
}

Fr first_challenge(const VerifyingKey& vk, size_t n, const uint8_t* com, const uint8_t* publics) {
    std::vector<uint8_t> tr(DOMAIN_TAG, DOMAIN_TAG + sizeof(DOMAIN_TAG) - 1);
    put_vkey(tr, vk);
    for (int i = 0; i < 4; ++i) tr.push_back((uint8_t)(n >> (8 * i)));
    tr.insert(tr.end(), com, com + 4 * GT_BYTES);
    if (vk.ic.size() > 1) tr.insert(tr.end(), publics, publics + 32 * n * (vk.ic.size() - 1));
    return challenge(tr);
}
Fr next_challenge(const Fr& prev, const uint8_t* msg, size_t len) {
    std::vector<uint8_t> tr;
    put_fr(tr, prev);
    tr.insert(tr.end(), msg, msg + len);
    return challenge(tr);
}

void check_count(size_t n) {
    if (n < 2 || n > MAX_PROOFS || (n & (n - 1)))
        throw std::runtime_error("the number of proofs must be a power of two from 2 to 8192, not " + std::to_string(n));
}

void put_vkey(std::vector<uint8_t>& out, const VerifyingKey& vk) {
    put_g1(out, vk.alpha1); put_g2(out, vk.beta2); put_g2(out, vk.gamma2); put_g2(out, vk.delta2);
    for (auto& p : vk.ic) put_g1(out, p);
}

G1AffineH g1_at(const uint8_t* p) {
    const G1AffineH a = load_g1(p);
    if (!g1_on_curve(a)) throw std::runtime_error("G1 point not on the curve");
    return a;
}
G2AffineH g2_at(const uint8_t* p) {
    const G2AffineH a = load_g2(p);
    if (!g2_on_curve(a)) throw std::runtime_error("G2 point not on the twist curve");
    if (!g2_in_subgroup(a)) throw std::runtime_error("G2 point not in the order-r subgroup");
    return a;
}

void fold_polys(const std::vector<Fr>& xs, const Fr& r_inv, size_t n, std::vector<Fr>& cv, std::vector<Fr>& cw) {
    const size_t k = xs.size();
    std::vector<Fr> xinv(xs);
    for (auto& x : xinv) x = x.inv();
    cv.assign(n, Fr::one());
    cw.assign(2 * n, Fr::zero());
    Fr rp = Fr::one();
    for (size_t i = 0; i < n; ++i) {
        Fr a = rp, b = Fr::one();
        for (size_t j = 0; j < k; ++j)
            if ((i >> (k - 1 - j)) & 1) { a = a * xinv[j]; b = b * xs[j]; }
        cv[i] = a;
        cw[n + i] = b;
        rp = rp * r_inv;
    }
}
std::vector<Fr> kzg_quotient(const std::vector<Fr>& c, const Fr& z) {
    std::vector<Fr> q(c.size() - 1, Fr::zero());
    Fr acc = Fr::zero();
    for (size_t i = c.size() - 1; i >= 1; --i) { acc = acc * z + c[i]; q[i - 1] = acc; }
    return q;
}
Fr poly_eval(const std::vector<Fr>& c, const Fr& z) {
    Fr acc = Fr::zero();
    for (size_t i = c.size(); i-- > 0;) acc = acc * z + c[i];
    return acc;
}

bool verify(const AggVk& avk, const VerifyingKey& vk, size_t n, const uint8_t* publics, const uint8_t* agg, size_t agg_len) {
    check_count(n);
    if (agg_len != agg_bytes(n)) throw std::runtime_error("an aggregate of " + std::to_string(n) + " proofs has " + std::to_string(agg_bytes(n)) + " bytes");
    const size_t np = vk.ic.size() - 1;
    for (const G1AffineH* p : {&avk.g, &avk.g_a, &avk.g_b, &vk.alpha1})
        if (!g1_on_curve(*p)) throw std::runtime_error("key point not on the curve");
    for (auto& p : vk.ic) if (!g1_on_curve(p)) throw std::runtime_error("vkey IC point not on the curve");
    for (const G2AffineH* p : {&avk.h, &avk.h_a, &avk.h_b, &vk.beta2, &vk.gamma2, &vk.delta2})
        if (!g2_on_curve(*p) || !g2_in_subgroup(*p)) throw std::runtime_error("key point not in G2");
    std::vector<Fr> pub(n * np);
    for (size_t i = 0; i < n * np; ++i) {
        U256 s;
        memcpy(s.v, publics + 32 * i, 32);
        if (u256_cmp(s, fr_params().p) >= 0) throw std::runtime_error("public signal not below r");
        pub[i] = Fr::from_u256(s);
    }
    const uint8_t* p = agg;
    Gt t_ab = gt_load(p), u_ab = gt_load(p + GT_BYTES), t_c = gt_load(p + 2 * GT_BYTES), u_c = gt_load(p + 3 * GT_BYTES);
    const Gt z_ab0 = gt_load(p + 4 * GT_BYTES);
    const G1AffineH z_c0 = g1_at(p + 5 * GT_BYTES);
    const Fr r = first_challenge(vk, n, p, publics);
    Fr x = r, beta = Fr::one();
    std::vector<Fr> xs;
    Gt z_ab = z_ab0;
    G1JacH z_c = G1JacH::from_affine(z_c0);
    p += HEAD_BYTES;
    for (unsigned j = 0; j < log2_exact(n); ++j, p += ROUND_BYTES) {
        Gt m[ROUND_GT];
        for (int k = 0; k < ROUND_GT; ++k) m[k] = gt_load(p + GT_BYTES * k);
        const G1AffineH zcl = g1_at(p + ROUND_GT * GT_BYTES), zcr = g1_at(p + ROUND_GT * GT_BYTES + G1_BYTES);
        x = next_challenge(x, p, ROUND_BYTES);
        xs.push_back(x);
        const Fr xi = x.inv();
        const U256 xe = x.to_u256(), xie = xi.to_u256();
        Gt* acc[5] = {&z_ab, &t_ab, &u_ab, &t_c, &u_c};
        for (int k = 0; k < 5; ++k) *acc[k] = gt_mul(*acc[k], gt_mul(gt_pow(m[2 * k], xe), gt_pow(m[2 * k + 1], xie)));
        z_c = z_c.add(G1JacH::from_affine(zcl).mul(xe)).add(G1JacH::from_affine(zcr).mul(xie));
        beta = beta * (Fr::one() + xi);
    }
    const G1AffineH fa = g1_at(p), fc = g1_at(p + 192), fw1 = g1_at(p + 512), fw2 = g1_at(p + 576);
    const G2AffineH fb = g2_at(p + 64), fv1 = g2_at(p + 256), fv2 = g2_at(p + 384);
    const Fr z = next_challenge(x, p, FINAL_BYTES);
    p += FINAL_BYTES;
    const G2AffineH pv1 = g2_at(p), pv2 = g2_at(p + G2_BYTES);
    const G1AffineH pw1 = g1_at(p + 2 * G2_BYTES), pw2 = g1_at(p + 2 * G2_BYTES + G1_BYTES);

    // GIPA: the folded commitments open to the folded vectors and keys
    if (!(z_ab == gt_pairing_product({{fa, fb}}))) return false;
    if (!(t_ab == gt_pairing_product({{fa, fv1}, {fw1, fb}})) || !(u_ab == gt_pairing_product({{fa, fv2}, {fw2, fb}}))) return false;
    const G1AffineH zc_aff = z_c.to_affine(), bc = G1JacH::from_affine(fc).mul(beta.to_u256()).to_affine();
    if (!(zc_aff.x == bc.x && zc_aff.y == bc.y)) return false;
    if (!(t_c == gt_pairing_product({{fc, fv1}})) || !(u_c == gt_pairing_product({{fc, fv2}}))) return false;
    // KZG: v = h^f_v(tau), w = g^F_w(tau) for tau = a, b, opened at z
    std::vector<Fr> cv, cw;
    fold_polys(xs, r.inv(), n, cv, cw);
    const U256 ze = z.to_u256(), fvz = poly_eval(cv, z).to_u256(), fwz = poly_eval(cw, z).to_u256();
    const Gt one = gt_one();
    auto neg1 = [](G1AffineH a) { a.y = a.y.neg(); return a; };
    const G1AffineH gz = G1JacH::from_affine(avk.g).mul(ze).to_affine();
    const G2AffineH hz = G2JacH::from_affine(avk.h).mul(ze).to_affine();
    const G2AffineH hfv = G2JacH::from_affine(avk.h).mul(fvz).to_affine();
    const G1AffineH gfw = G1JacH::from_affine(avk.g).mul(fwz).to_affine();
    const G1AffineH ga[2] = {avk.g_a, avk.g_b}, fw[2] = {fw1, fw2}, pw[2] = {pw1, pw2};
    const G2AffineH ha[2] = {avk.h_a, avk.h_b}, fv[2] = {fv1, fv2}, pv[2] = {pv1, pv2};
    for (int t = 0; t < 2; ++t) {
        const G1AffineH lhs = G1JacH::from_affine(ga[t]).add(G1JacH::from_affine(neg1(gz))).to_affine();
        const G2AffineH rhs = G2JacH::from_affine(fv[t]).add(G2JacH::from_affine(hfv).neg()).to_affine();
        if (!(gt_pairing_product({{lhs, pv[t]}, {neg1(avk.g), rhs}}) == one)) return false;
        const G2AffineH hl = G2JacH::from_affine(ha[t]).add(G2JacH::from_affine(hz).neg()).to_affine();
        const G1AffineH wr = G1JacH::from_affine(fw[t]).add(G1JacH::from_affine(neg1(gfw))).to_affine();
        if (!(gt_pairing_product({{pw[t], hl}, {neg1(wr), avk.h}}) == one)) return false;
    }
    // Groth16 in aggregated form: Z_AB = e(alpha, beta)^(sum r^i) e(sum_i r^i vk_x_i, gamma) e(Z_C, delta)
    std::vector<Fr> coeff(np + 1, Fr::zero());
    Fr ri = Fr::one();
    for (size_t i = 0; i < n; ++i, ri = ri * r) {
        coeff[0] = coeff[0] + ri;
        for (size_t j = 0; j < np; ++j) coeff[j + 1] = coeff[j + 1] + ri * pub[i * np + j];
    }
    G1JacH vkx = G1JacH::inf();
    for (size_t j = 0; j <= np; ++j) vkx = vkx.add(G1JacH::from_affine(vk.ic[j]).mul(coeff[j].to_u256()));
    const G1AffineH sa = G1JacH::from_affine(vk.alpha1).mul(coeff[0].to_u256()).to_affine();
    return z_ab0 == gt_pairing_product({{sa, vk.beta2}, {vkx.to_affine(), vk.gamma2}, {z_c0, vk.delta2}});
}

}  // namespace agg
}  // namespace zke

using namespace zke;

extern "C" int zke_agg_verify(const char* agg_vk_json, const char* vkey_json, size_t n, const uint8_t* publics, const uint8_t* agg,
                              size_t agg_len, char* err, size_t errcap) {
    try {
        if (!agg_vk_json || !vkey_json || !agg) throw std::runtime_error("null argument");
        const agg::AggVk avk = agg::agg_vk_from_json(agg_vk_json);
        const VerifyingKey vk = vkey_from_json(vkey_json);
        if (vk.ic.size() > 1 && !publics) throw std::runtime_error("null argument");
        return agg::verify(avk, vk, n, publics, agg, agg_len) ? 1 : 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}
