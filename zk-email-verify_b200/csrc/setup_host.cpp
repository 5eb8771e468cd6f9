// Host part of the (toy, seeded) Groth16 trusted setup: evaluates the QAP polynomials at tau.
//
// Stands in for `snarkjs groth16 setup` + contributions of the reference's offline flow
// (/root/reference/docs/zk-email-docs/UsageGuide/README.md:139-153).  The toxic waste (tau, alpha, beta, gamma,
// delta) is derived from a seed and therefore KNOWN - keys produced here are for benchmarking and testing only.
// The polynomial conventions are the snarkjs / ark-circom ones (SURVEY A.7): rows n_constraints .. n_constraints+l
// are the extra A-only rows 1 * w_j, the quotient is evaluated on the coset g*H with g a primitive 2N-th root,
// where Z(x) = x^N - 1 is the constant -2, so H_i = [ -L_i(tau / g) Z(tau) / (2 delta) ]_1.
#include "setup_host.hpp"
#include <thread>

namespace zke {

static Fr fr_from_seed(uint64_t seed, uint64_t stream) {
    // splitmix64 expanded to 4 limbs, reduced mod r (top 2 bits cleared first so one subtraction suffices)
    uint64_t x = seed * 0x9E3779B97F4A7C15ull + stream * 0xD1B54A32D192ED03ull + 0x2545F4914F6CDD1Dull;
    U256 v;
    for (int i = 0; i < 4; ++i) {
        x += 0x9E3779B97F4A7C15ull;
        uint64_t z = x;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        v.v[i] = z ^ (z >> 31);
    }
    v.v[3] &= 0x3FFFFFFFFFFFFFFFull;
    if (u256_cmp(v, fr_params().p) >= 0) u256_sub(v, v, fr_params().p);
    if (v.is_zero()) v.v[0] = 7;
    return Fr::from_u256(v);
}

void derive_toxic(uint64_t seed, Fr out[5]) { for (int i = 0; i < 5; ++i) out[i] = fr_from_seed(seed, (uint64_t)i + 1); }

// out[i] = numer * omega^i / (x - omega^i) for i in [0, N)
void lagrange_like(const Fr& x, const Fr& numer, unsigned log_n, std::vector<Fr>& out) {
    const size_t N = (size_t)1 << log_n;
    out.resize(N);
    const Fr omega = fr_root_of_unity(log_n);
    const unsigned T = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; ++t) {
        th.emplace_back([&, t]() {
            size_t beg = N * t / T, end = N * (t + 1) / T;
            if (beg >= end) return;
            U256 e = {{(uint64_t)beg, 0, 0, 0}};
            Fr w = omega.pow(e);
            std::vector<Fr> pw(end - beg);
            for (size_t i = beg; i < end; ++i) { pw[i - beg] = w; out[i] = x - w; w = w * omega; }
            batch_inverse(out.data() + beg, end - beg);   // (a zero denominator means tau is in the domain: excluded by the caller)
            for (size_t i = beg; i < end; ++i) out[i] = out[i] * pw[i - beg] * numer;
        });
    }
    for (auto& x2 : th) x2.join();
}

SetupScalars compute_setup_scalars(const Circuit& c, uint64_t seed) {
    SetupScalars S;
    S.log_n = c.domain_log2();
    const size_t N = (size_t)1 << S.log_n;
    const uint32_t m = c.n_vars, l = c.n_public();
    Fr tox[5];
    derive_toxic(seed, tox);
    S.tau = tox[0]; S.alpha = tox[1]; S.beta = tox[2]; S.gamma = tox[3]; S.delta = tox[4];

    U256 eN = {{(uint64_t)N, 0, 0, 0}};
    const Fr tauN = S.tau.pow(eN);
    const Fr z_tau = tauN - Fr::one();                    // Z(tau)
    if (z_tau.is_zero()) throw std::runtime_error("setup: tau lies in the evaluation domain");
    const Fr n_inv = Fr::from_u64(N).inv();

    // L_c(tau) = Z(tau)/N * omega^c / (tau - omega^c)
    std::vector<Fr> lag;
    lagrange_like(S.tau, z_tau * n_inv, S.log_n, lag);

    std::vector<Fr> coef(c.coefs.size());
    for (size_t i = 0; i < coef.size(); ++i) coef[i] = Fr::from_u256(c.coefs[i]);

    S.a.assign(m, Fr::zero()); S.b.assign(m, Fr::zero());
    std::vector<Fr> cc(m, Fr::zero());
    auto accumulate = [&](const std::vector<uint32_t>& ptr, const std::vector<uint32_t>& var, const std::vector<uint32_t>& cf, std::vector<Fr>& dst) {
        for (uint32_t row = 0; row < c.n_constraints; ++row) {
            const Fr& L = lag[row];
            for (uint32_t k = ptr[row]; k < ptr[row + 1]; ++k) {
                const uint32_t ci = cf[k];
                if (ci == 0) dst[var[k]] += L;
                else if (ci == 1) dst[var[k]] -= L;
                else dst[var[k]] += coef[ci] * L;
            }
        }
    };
    std::thread ta([&]() { accumulate(c.a_ptr, c.a_var, c.a_coef, S.a); });
    std::thread tb([&]() { accumulate(c.b_ptr, c.b_var, c.b_coef, S.b); });
    accumulate(c.c_ptr, c.c_var, c.c_coef, cc);
    ta.join(); tb.join();
    for (uint32_t j = 0; j <= l; ++j) S.a[j] += lag[c.n_constraints + j];   // extra public rows: A = w_j

    const Fr gamma_inv = S.gamma.inv(), delta_inv = S.delta.inv();
    S.kc.resize(m);
    for (uint32_t j = 0; j < m; ++j) {
        Fr v = S.beta * S.a[j] + S.alpha * S.b[j] + cc[j];
        S.kc[j] = v * (j <= l ? gamma_inv : delta_inv);
    }

    // H_i = -L_i(tau/g) Z(tau) / (2 delta),  L_i(tau/g) = ((tau/g)^N - 1)/N * omega^i / (tau/g - omega^i),  (tau/g)^N = -tau^N
    const Fr g = fr_root_of_unity(S.log_n + 1);
    const Fr tau_g = S.tau * g.inv();
    const Fr zc = (Fr::zero() - tauN) - Fr::one();
    const Fr two_inv = Fr::from_u64(2).inv();
    const Fr numer = (Fr::zero() - (zc * n_inv * z_tau * two_inv * delta_inv));
    lagrange_like(tau_g, numer, S.log_n, S.h);
    return S;
}

}  // namespace zke
