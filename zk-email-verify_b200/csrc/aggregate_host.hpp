// Host side of Groth16 proof aggregation (SnarkPack; DESIGN.md "Proof aggregation"): the byte layout of an aggregate,
// the SHA-256 transcript, the folded-key polynomials, the GT arithmetic the verifier needs, and the verifier itself.
// The prover (aggregate.cu) and the verifier (aggregate_host.cpp) share everything here, so they replay one transcript.
#pragma once
#include "ec_host.hpp"
#include <array>
#include <string>
#include <vector>

namespace zke {
namespace agg {

constexpr size_t GT_BYTES = 384, G1_BYTES = 64, G2_BYTES = 128;
constexpr int ROUND_GT = 10;                                          // ZL ZR TL TR UL UR TCL TCR UCL UCR
constexpr size_t HEAD_BYTES = 5 * GT_BYTES + G1_BYTES;                // T_AB U_AB T_C U_C Z_AB Z_C
constexpr size_t ROUND_BYTES = ROUND_GT * GT_BYTES + 2 * G1_BYTES;    // ... ZCL ZCR
constexpr size_t FINAL_BYTES = 4 * G1_BYTES + 3 * G2_BYTES;           // A B C v1 v2 w1 w2
constexpr size_t TAIL_BYTES = FINAL_BYTES + 2 * G2_BYTES + 2 * G1_BYTES;   // + pi_v1 pi_v2 pi_w1 pi_w2
constexpr uint32_t MAX_PROOFS = 8192;
inline unsigned log2_exact(size_t n) { unsigned k = 0; while (((size_t)1 << k) < n) ++k; return k; }
inline size_t agg_bytes(size_t n) { return HEAD_BYTES + log2_exact(n) * ROUND_BYTES + TAIL_BYTES; }
// refuses an n that is not a power of two in [2, MAX_PROOFS]
void check_count(size_t n);

// The verifier key: g, h and their images under the two secrets
struct AggVk { G1AffineH g, g_a, g_b; G2AffineH h, h_a, h_b; };
AggVk agg_vk_from_json(const char* json);   // capi_json.cpp
std::string agg_vk_to_json(const AggVk& vk);

// SHA-256 (FIPS 180-4)
void sha256(const uint8_t* data, size_t len, uint8_t out[32]);
// SHA-256 of the concatenation, read little-endian and reduced mod r; throws on a zero challenge
Fr challenge(const std::vector<uint8_t>& bytes);
// r = H(tag, Groth16 key, n as u32, T_AB U_AB T_C U_C, public signals); every later challenge H(previous, messages)
Fr first_challenge(const VerifyingKey& vk, size_t n, const uint8_t* com, const uint8_t* publics);
Fr next_challenge(const Fr& prev, const uint8_t* msg, size_t len);
// the Groth16 key and the public signals as the first challenge hashes them
void put_vkey(std::vector<uint8_t>& out, const VerifyingKey& vk);
G1AffineH g1_at(const uint8_t* p);   // load_g1 + on the curve
G2AffineH g2_at(const uint8_t* p);   // load_g2 + on the twist and in the order-r subgroup

// Coefficients (low to high) of the folded-key polynomials after the rounds with challenges xs:
//   v: f_v(X) = prod_j (1 + x_j^-1 (X / r)^(n / 2^(j+1))), n coefficients
//   w: F_w(X) = X^n prod_j (1 + x_j X^(n / 2^(j+1))), 2n coefficients
void fold_polys(const std::vector<Fr>& xs, const Fr& r_inv, size_t n, std::vector<Fr>& cv, std::vector<Fr>& cw);
std::vector<Fr> kzg_quotient(const std::vector<Fr>& coeffs, const Fr& z);   // (f(X) - f(z)) / (X - z)
Fr poly_eval(const std::vector<Fr>& coeffs, const Fr& z);

// GT in pairing_host.cpp's dense representation, values normalised like snarkjs' vk_alphabeta_12
struct Gt { std::array<Fq, 12> c; bool operator==(const Gt& o) const { return c == o.c; } };
Gt gt_one();
Gt gt_mul(const Gt& a, const Gt& b);
Gt gt_pow(const Gt& a, const U256& e);
Gt gt_pairing_product(const std::vector<std::pair<G1AffineH, G2AffineH>>& terms);
void gt_store(const Gt& a, uint8_t out[384]);   // tower layout of vk_alphabeta_12, standard form LE
Gt gt_load(const uint8_t* in);                  // the inverse; throws on an unreduced coordinate

// 1 if `agg` (agg_bytes(n) bytes) proves n valid proofs of these public signals (n x nPublic x 32 bytes, standard form LE)
// under `vk`, 0 if not; throws on malformed input (bad n, wrong lengths, unreduced or invalid points)
bool verify(const AggVk& avk, const VerifyingKey& vk, size_t n, const uint8_t* publics, const uint8_t* agg, size_t agg_len);

}  // namespace agg
}  // namespace zke
