#pragma once
#include "circuit.hpp"
#include <vector>

namespace zke {

// Field-side result of the toy trusted setup: per-variable QAP evaluations at tau and the H-basis scalars.
struct SetupScalars {
    unsigned log_n = 0;
    Fr tau, alpha, beta, gamma, delta;
    std::vector<Fr> a;    // a_j(tau)                          -> A points (G1)
    std::vector<Fr> b;    // b_j(tau)                          -> B1 (G1) and B2 (G2) points
    std::vector<Fr> kc;   // (beta a_j + alpha b_j + c_j)/gamma for j <= nPublic (IC), /delta otherwise (C / "L")
    std::vector<Fr> h;    // N scalars of the H points
};
SetupScalars compute_setup_scalars(const Circuit& c, uint64_t seed);
// tau, alpha, beta, gamma, delta derived from the seed (the KNOWN toxic waste of the toy setup)
void derive_toxic(uint64_t seed, Fr out[5]);
// out[i] = numer * omega^i / (x - omega^i), i < 2^log_n, omega a primitive 2^log_n-th root; with numer = (x^N - 1) / N
// these are the Lagrange basis polynomials of that domain evaluated at x.  x must not lie in the domain.
void lagrange_like(const Fr& x, const Fr& numer, unsigned log_n, std::vector<Fr>& out);

}  // namespace zke
