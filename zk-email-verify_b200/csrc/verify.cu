// Batch Groth16 verification on the GPU (SURVEY 8(f) rank 4): zke_verifier_open / zke_verifier_batch /
// zke_selftest_pairing_gpu (include/zkemail_b200.h).  For n proofs under one key:
//   1. every proof is validated, one thread each: coordinates below q, A and C on G1, B on the twist and in the
//      order-r subgroup, public signals below r;
//   2. if all are valid, the weighted terms are formed: -r_i A_i, r_i C_i (128-bit weights), the IC coefficients
//      coeff_j = sum_i r_i s_ij mod r (coeff_0 = sum_i r_i), X = sum_j coeff_j IC_j and coeff_0 alpha;
//   3. the n Miller loops (B_i, -r_i A_i) run on the fly, the three of (coeff_0 alpha, X, sum r_i C_i) against beta2,
//      gamma2, delta2 replay line tables made when the verifier opened; the n + 3 values are multiplied in a tree and
//      one final exponentiation decides;
//   4. if some proof is malformed or the combined check fails, every proof is verified on its own, one thread each:
//      e(-A, B) e(X_i, gamma2) e(C, delta2) in one shared Miller loop, times e(alpha, beta) kept in GT.
// The verdicts are those of the host path (zke_verify_batch_json: groth16_verify_batch, then groth16_verify per proof).
#include "pairing.cuh"
#include "device_engine.cuh"
#include "cuda_host.hpp"
#include "../../include/zkemail_b200.h"
#include "engine.hpp"
#include "ec_host.hpp"
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace zke {
namespace dev {

ZKE_DEFINE_CONSTANT_UPLOAD(upload_constants_verify)

static const int VERIFY_THREADS = 64;
static const uint32_t FOLD = 32;     // elements combined per thread and level of a tree reduction

struct FixedLines { const uint8_t* p[3]; };   // line tables of beta2, gamma2, delta2 (null: the point is at infinity)

__device__ __forceinline__ G1Affine g1_zero() { G1Affine r; r.x = Fq::zero(); r.y = Fq::zero(); return r; }
__device__ __forceinline__ G2Affine g2_zero() { G2Affine r; r.x = Fq2::zero(); r.y = Fq2::zero(); return r; }

// proofs: [n][8][32] standard form (A.x, A.y, B.x.c0, B.x.c1, B.y.c0, B.y.c1, C.x, C.y), all-zero points = infinity.
// mont: the same points in Montgomery form; valid[i]: the checks of groth16_verify on proof i
__global__ void __launch_bounds__(VERIFY_THREADS)
verify_validate_kernel(const uint8_t* __restrict__ proofs, const uint8_t* __restrict__ publics, uint32_t n, uint32_t np,
                       uint8_t* __restrict__ mont, uint8_t* __restrict__ valid) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool ok = true;
    Fq c[8];
    for (int k = 0; k < 8; ++k) {
        const Fq x = Fq::load(proofs + 256ull * i + 32 * k);
        ok = ok && below_modulus(x);
        c[k] = x.to_mont();
    }
    for (uint32_t j = 0; j < np; ++j) ok = ok && below_modulus(Fr::load(publics + 32ull * ((size_t)i * np + j)));
    G1Affine a, cc; G2Affine b;
    a.x = c[0]; a.y = c[1]; b.x.c0 = c[2]; b.x.c1 = c[3]; b.y.c0 = c[4]; b.y.c1 = c[5]; cc.x = c[6]; cc.y = c[7];
    ok = ok && g1_on_curve(a) && g1_on_curve(cc) && g2_on_curve(b);
    ok = ok && g2_in_subgroup(b);
    a.store(mont + 256ull * i);
    b.store(mont + 256ull * i + 64);
    cc.store(mont + 256ull * i + 192);
    valid[i] = ok ? 1 : 0;
}

// neg_ra[i] = -r_i A_i (affine), rc[i] = r_i C_i (XYZZ); rand32: [n][32] weights below 2^128, standard form
__global__ void __launch_bounds__(VERIFY_THREADS)
verify_weight_kernel(const uint8_t* __restrict__ mont, const uint8_t* __restrict__ rand32, uint32_t n,
                     uint8_t* __restrict__ neg_ra, uint8_t* __restrict__ rc) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr r = Fr::load(rand32 + 32ull * i);
    G1Affine ra = g1_to_affine(scalar_mul(G1Affine::load(mont + 256ull * i), r.v, 128));
    ra.y = ra.y.neg();
    ra.store(neg_ra + 64ull * i);
    scalar_mul(G1Affine::load(mont + 256ull * i + 192), r.v, 128).store(rc + 128ull * i);
}

// terms[i][0] = r_i, terms[i][1 + j] = r_i s_ij mod r (standard form: the Montgomery product of r_i R and s_ij)
__global__ void __launch_bounds__(VERIFY_THREADS)
verify_coeff_terms_kernel(const uint8_t* __restrict__ rand32, const uint8_t* __restrict__ publics, uint32_t n, uint32_t np,
                          uint8_t* __restrict__ terms) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr r = Fr::load(rand32 + 32ull * i), rm = r.to_mont();
    uint8_t* t = terms + 32ull * (np + 1) * i;
    r.store(t);
    for (uint32_t j = 0; j < np; ++j) (rm * Fr::load(publics + 32ull * ((size_t)i * np + j))).store(t + 32 * (j + 1));
}

struct FrSumOp {
    typedef Fr T;
    static const int BYTES = 32;
    static __device__ __forceinline__ T load(const uint8_t* p) { return Fr::load(p); }
    static __device__ __forceinline__ void store(const T& v, uint8_t* p) { v.store(p); }
    static __device__ __forceinline__ T combine(const T& a, const T& b) { return a + b; }
};
struct G1SumOp {
    typedef G1XYZZ T;
    static const int BYTES = 128;
    static __device__ __forceinline__ T load(const uint8_t* p) { return G1XYZZ::load(p); }
    static __device__ __forceinline__ void store(const T& v, uint8_t* p) { v.store(p); }
    static __device__ __forceinline__ T combine(T a, const T& b) { a.add(b); return a; }
};
struct F12ProdOp {
    typedef Fq12 T;
    static const int BYTES = 384;
    static __device__ __forceinline__ T load(const uint8_t* p) { return Fq12::load(p); }
    static __device__ __forceinline__ void store(const T& v, uint8_t* p) { v.store(p); }
    static __device__ __forceinline__ T combine(const T& a, const T& b) { return a * b; }
};

// One level of a tree reduction over `count` rows of `width` elements: out[g][w] = fold of in[g FOLD .. ][w]
template <class Op>
__global__ void __launch_bounds__(VERIFY_THREADS)
verify_fold_kernel(const uint8_t* __restrict__ in, uint32_t count, uint32_t width, uint8_t* __restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t groups = (count + FOLD - 1) / FOLD;
    if (t >= groups * width) return;
    const uint32_t g = t / width, w = t % width;
    const uint32_t end = min(count, (g + 1) * FOLD);
    typename Op::T acc = Op::load(in + (size_t)Op::BYTES * ((size_t)g * FOLD * width + w));
    for (uint32_t k = g * FOLD + 1; k < end; ++k) acc = Op::combine(acc, Op::load(in + (size_t)Op::BYTES * ((size_t)k * width + w)));
    Op::store(acc, out + (size_t)Op::BYTES * t);
}

// products[j] = coeff_j IC_j (j <= np), products[np + 1] = coeff_0 alpha (XYZZ)
__global__ void __launch_bounds__(VERIFY_THREADS)
verify_ic_mul_kernel(const uint8_t* __restrict__ coeff, const uint8_t* __restrict__ ic, const uint8_t* __restrict__ alpha,
                     uint32_t np, uint8_t* __restrict__ products) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > np + 1) return;
    const Fr k = Fr::load(coeff + 32ull * (j <= np ? j : 0));
    const G1Affine p = G1Affine::load(j <= np ? ic + 64ull * j : alpha);
    scalar_mul(p, k.v, 254).store(products + 128ull * j);
}

// fixed_p = {coeff_0 alpha, X = sum_j coeff_j IC_j, sum_i r_i C_i} (affine): the G1 sides of the three fixed pairs
__global__ void verify_fixed_points_kernel(const uint8_t* __restrict__ products, uint32_t np, const uint8_t* __restrict__ csum,
                                           uint8_t* __restrict__ fixed_p) {
    if (blockIdx.x * blockDim.x + threadIdx.x != 0) return;
    G1XYZZ x = G1XYZZ::load(products);
    for (uint32_t j = 1; j <= np; ++j) x.add(G1XYZZ::load(products + 128ull * j));
    g1_to_affine(G1XYZZ::load(products + 128ull * (np + 1))).store(fixed_p);
    g1_to_affine(x).store(fixed_p + 64);
    g1_to_affine(G1XYZZ::load(csum)).store(fixed_p + 128);
}

// f[i] = ML(B_i, -r_i A_i) for i < n (lines on the fly); f[n + k] = ML(fixed G2 point k, fixed_p[k]) from its line table
__global__ void __launch_bounds__(VERIFY_THREADS)
verify_miller_kernel(const uint8_t* __restrict__ mont, const uint8_t* __restrict__ neg_ra, uint32_t n, FixedLines fl,
                     const uint8_t* __restrict__ fixed_p, uint8_t* __restrict__ f) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        miller_loop<0>(true, G2Affine::load(mont + 256ull * i + 64), G1Affine::load(neg_ra + 64ull * i), nullptr, nullptr, nullptr)
            .store(f + 384ull * i);
    } else if (i < n + 3) {
        const uint32_t k = i - n;
        const uint8_t* tab[1] = {fl.p[k]};
        const G1Affine p = G1Affine::load(fixed_p + 64ull * k);
        miller_loop<1>(false, g2_zero(), g1_zero(), tab, &p, nullptr).store(f + 384ull * i);
    }
}

__global__ void verify_final_kernel(const uint8_t* __restrict__ f, uint8_t* __restrict__ result) {
    if (blockIdx.x * blockDim.x + threadIdx.x != 0) return;
    *result = final_exponentiation(Fq12::load(f)).is_one() ? 1 : 0;
}

// One proof per thread: e(-A, B) e(X_i, gamma2) e(C, delta2) e(alpha, beta) == 1 with X_i = IC_0 + sum_j s_ij IC_j
__global__ void __launch_bounds__(VERIFY_THREADS)
verify_single_kernel(const uint8_t* __restrict__ mont, const uint8_t* __restrict__ publics, const uint8_t* __restrict__ valid,
                     uint32_t n, uint32_t np, const uint8_t* __restrict__ ic, FixedLines fl, const uint8_t* __restrict__ e_ab,
                     uint8_t* __restrict__ ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!valid[i]) { ok[i] = 0; return; }
    // all np scalar multiplications share one doubling chain (s_ij < r < 2^254)
    const uint32_t* s = reinterpret_cast<const uint32_t*>(publics + 32ull * np * i);
    G1XYZZ x = G1XYZZ::inf();
    for (int bit = 253; bit >= 0; --bit) {
        x.dbl();
        for (uint32_t j = 0; j < np; ++j)
            if ((s[8 * j + (bit >> 5)] >> (bit & 31)) & 1) x.madd(G1Affine::load(ic + 64ull * (j + 1)), false);
    }
    x.madd(G1Affine::load(ic), false);
    G1Affine a = G1Affine::load(mont + 256ull * i);
    a.y = a.y.neg();
    const uint8_t* tab[2] = {fl.p[1], fl.p[2]};
    const G1Affine fp[2] = {g1_to_affine(x), G1Affine::load(mont + 256ull * i + 192)};
    const Fq12 f = miller_loop<2>(true, G2Affine::load(mont + 256ull * i + 64), a, tab, fp, nullptr);
    ok[i] = (final_exponentiation(f) * Fq12::load(e_ab)).is_one() ? 1 : 0;
}

// Open time: thread k < 3 records the lines of fixed G2 point k (evaluated at the generator of G1; only the table is kept)
__global__ void verify_lines_kernel(const uint8_t* __restrict__ g2, uint8_t* __restrict__ lines) {
    const uint32_t k = threadIdx.x;
    if (k >= 3) return;
    G1Affine gen; gen.x = Fq::one(); gen.y = Fq::one().dbl();
    miller_loop<0>(true, G2Affine::load(g2 + 128 * k), gen, nullptr, nullptr, lines + (size_t)k * ATE_LINES * LINE_BYTES);
}
// e(alpha, beta) after the final exponentiation, from beta2's line table
__global__ void verify_alphabeta_kernel(const uint8_t* __restrict__ alpha, FixedLines fl, uint8_t* __restrict__ out) {
    if (threadIdx.x != 0) return;
    const uint8_t* tab[1] = {fl.p[0]};
    const G1Affine a = G1Affine::load(alpha);
    final_exponentiation(miller_loop<1>(false, g2_zero(), g1_zero(), tab, &a, nullptr)).store(out);
}

// Diagnostic pairing: standard-form points in, e(P_i, Q_i) out as 12 standard-form Fq (vk_alphabeta_12 layout)
__global__ void __launch_bounds__(VERIFY_THREADS)
pairing_selftest_kernel(const uint8_t* __restrict__ g1, const uint8_t* __restrict__ g2, uint32_t n, uint8_t* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1Affine p; G2Affine q;
    p.x = Fq::load(g1 + 64ull * i).to_mont(); p.y = Fq::load(g1 + 64ull * i + 32).to_mont();
    q.x.c0 = Fq::load(g2 + 128ull * i).to_mont(); q.x.c1 = Fq::load(g2 + 128ull * i + 32).to_mont();
    q.y.c0 = Fq::load(g2 + 128ull * i + 64).to_mont(); q.y.c1 = Fq::load(g2 + 128ull * i + 96).to_mont();
    const Fq12 e = final_exponentiation(miller_loop<0>(true, q, p, nullptr, nullptr, nullptr));
    for (int k = 0; k < 6; ++k) {
        const Fq2& c = e.at(k / 3, k % 3);
        c.c0.from_mont().store(out + 384ull * i + 64 * k);
        c.c1.from_mont().store(out + 384ull * i + 64 * k + 32);
    }
}

}  // namespace dev
}  // namespace zke

using namespace zke;

namespace {

unsigned blocks(size_t threads) { return (unsigned)((threads + dev::VERIFY_THREADS - 1) / dev::VERIFY_THREADS); }

// Montgomery images of points, the format the verification kernels read (not the standard form of ec_host.hpp)
void put_fq_mont(std::vector<uint8_t>& out, const Fq& x) { const uint8_t* b = reinterpret_cast<const uint8_t*>(x.m.v); out.insert(out.end(), b, b + 32); }
void put_g1_mont(std::vector<uint8_t>& out, const G1AffineH& p) { put_fq_mont(out, p.x); put_fq_mont(out, p.y); }
void put_g2_mont(std::vector<uint8_t>& out, const G2AffineH& p) { put_fq_mont(out, p.x.c0); put_fq_mont(out, p.x.c1); put_fq_mont(out, p.y.c0); put_fq_mont(out, p.y.c1); }

// Folds `count` rows of `width` elements to one row, level by level between two scratch buffers; returns the row
template <class Op>
const uint8_t* fold_all(const uint8_t* in, uint32_t count, uint32_t width, uint8_t* s0, uint8_t* s1, cudaStream_t st) {
    uint8_t* bufs[2] = {s0, s1};
    int b = 0;
    while (count > 1) {
        const uint32_t groups = (count + dev::FOLD - 1) / dev::FOLD;
        dev::verify_fold_kernel<Op><<<blocks((size_t)groups * width), dev::VERIFY_THREADS, 0, st>>>(in, count, width, bufs[b]);
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        in = bufs[b];
        b ^= 1;
        count = groups;
    }
    return in;
}

size_t fold_scratch(size_t count) { return (count + dev::FOLD - 1) / dev::FOLD; }

}  // namespace

struct zke_verifier {
    int device = 0;
    uint32_t n_public = 0;
    cudaStream_t stream = nullptr;
    DevBuf ic, alpha, g2, lines, e_ab;
    dev::FixedLines fl{{nullptr, nullptr, nullptr}};
    // per-call buffers
    DevBuf proofs, publics, rand32, mont, valid, ok, neg_ra, rc, rc_s0, rc_s1, terms, terms_s0, terms_s1, products, fixed_p, f,
        f_s0, f_s1, flag;
    ~zke_verifier() {
        if (stream) cudaStreamDestroy(stream);
    }
};

extern "C" {

zke_verifier* zke_verifier_open(const char* vkey_json, int device, char* err, size_t errcap) {
    try {
        if (!vkey_json) throw std::runtime_error("null argument");
        const VerifyingKey vk = vkey_from_json(vkey_json);
        if (!g1_on_curve(vk.alpha1)) throw std::runtime_error("vkey: vk_alpha_1 is not on the curve");
        for (size_t j = 0; j < vk.ic.size(); ++j)
            if (!g1_on_curve(vk.ic[j])) throw std::runtime_error("vkey: IC[" + std::to_string(j) + "] is not on the curve");
        const G2AffineH* g2s[3] = {&vk.beta2, &vk.gamma2, &vk.delta2};
        const char* names[3] = {"vk_beta_2", "vk_gamma_2", "vk_delta_2"};
        for (int k = 0; k < 3; ++k) {
            if (!g2_on_curve(*g2s[k])) throw std::runtime_error(std::string("vkey: ") + names[k] + " is not on the twist curve");
            if (!g2_in_subgroup(*g2s[k])) throw std::runtime_error(std::string("vkey: ") + names[k] + " is not in the order-r subgroup");
        }
        std::unique_ptr<zke_verifier> v(new zke_verifier());
        v->device = device;
        v->n_public = (uint32_t)(vk.ic.size() - 1);
        select_device(device);
        CUDA_OK(cudaStreamCreateWithFlags(&v->stream, cudaStreamNonBlocking));
        std::vector<uint8_t> ic, alpha, g2;
        for (auto& p : vk.ic) put_g1_mont(ic, p);
        put_g1_mont(alpha, vk.alpha1);
        for (int k = 0; k < 3; ++k) put_g2_mont(g2, *g2s[k]);
        CUDA_OK(cudaMemcpy(v->ic.reserve(ic.size()), ic.data(), ic.size(), cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(v->alpha.reserve(64), alpha.data(), 64, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(v->g2.reserve(384), g2.data(), 384, cudaMemcpyHostToDevice));
        const size_t table = (size_t)dev::ATE_LINES * dev::LINE_BYTES;
        uint8_t* lines = v->lines.reserve(3 * table);
        for (int k = 0; k < 3; ++k) v->fl.p[k] = g2s[k]->is_inf() ? nullptr : lines + k * table;
        dev::verify_lines_kernel<<<1, 32, 0, v->stream>>>(v->g2.p, lines);
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        dev::verify_alphabeta_kernel<<<1, 32, 0, v->stream>>>(v->alpha.p, v->fl, v->e_ab.reserve(384));
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        CUDA_OK(cudaStreamSynchronize(v->stream));
        return v.release();
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}

void zke_verifier_close(zke_verifier* v) {
    if (!v) return;
    cudaSetDevice(v->device);
    delete v;
}

int zke_verifier_batch(zke_verifier* v, size_t n, const uint8_t* proofs, const uint8_t* publics, const uint8_t* rand16,
                       uint8_t* ok, char* err, size_t errcap) {
    try {
        if (!v) throw std::runtime_error("null verifier");
        if (n == 0) return 0;
        const uint32_t np = v->n_public;
        if (!proofs || (np && !publics)) throw std::runtime_error("null argument");
        if (n > (size_t)1 << 26) throw std::runtime_error("batch too large");
        CUDA_OK(cudaSetDevice(v->device));
        cudaStream_t st = v->stream;
        // weights: 128 bits, a zero weight replaced by 1 (as zke_verify_batch_json)
        std::vector<uint8_t> rnd(32 * n, 0), r16(16 * n);
        if (rand16) memcpy(r16.data(), rand16, 16 * n);
        else random_bytes(r16.data(), r16.size());
        for (size_t i = 0; i < n; ++i) {
            memcpy(&rnd[32 * i], &r16[16 * i], 16);
            bool zero = true;
            for (int k = 0; k < 16; ++k) zero = zero && r16[16 * i + k] == 0;
            if (zero) rnd[32 * i] = 1;
        }
        const uint32_t nn = (uint32_t)n;
        uint8_t* d_proofs = v->proofs.reserve(256 * n);
        uint8_t* d_pub = v->publics.reserve(32 * n * (np ? np : 1));
        uint8_t* d_rand = v->rand32.reserve(32 * n);
        uint8_t* d_mont = v->mont.reserve(256 * n);
        uint8_t* d_valid = v->valid.reserve(n);
        CUDA_OK(cudaMemcpyAsync(d_proofs, proofs, 256 * n, cudaMemcpyHostToDevice, st));
        if (np) CUDA_OK(cudaMemcpyAsync(d_pub, publics, 32 * n * np, cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaMemcpyAsync(d_rand, rnd.data(), 32 * n, cudaMemcpyHostToDevice, st));
        dev::verify_validate_kernel<<<blocks(n), dev::VERIFY_THREADS, 0, st>>>(d_proofs, d_pub, nn, np, d_mont, d_valid);
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        std::vector<uint8_t> valid(n);
        CUDA_OK(cudaMemcpyAsync(valid.data(), d_valid, n, cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
        bool all_valid = true;
        for (size_t i = 0; i < n; ++i) all_valid = all_valid && valid[i];

        if (all_valid) {
            uint8_t* d_nra = v->neg_ra.reserve(64 * n);
            uint8_t* d_rc = v->rc.reserve(128 * n);
            dev::verify_weight_kernel<<<blocks(n), dev::VERIFY_THREADS, 0, st>>>(d_mont, d_rand, nn, d_nra, d_rc);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            const size_t w = np + 1;
            uint8_t* d_terms = v->terms.reserve(32 * w * n);
            dev::verify_coeff_terms_kernel<<<blocks(n), dev::VERIFY_THREADS, 0, st>>>(d_rand, d_pub, nn, np, d_terms);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            const uint8_t* coeff = fold_all<dev::FrSumOp>(d_terms, nn, (uint32_t)w, v->terms_s0.reserve(32 * w * fold_scratch(n)),
                                                          v->terms_s1.reserve(32 * w * fold_scratch(n)), st);
            const uint8_t* csum = fold_all<dev::G1SumOp>(d_rc, nn, 1, v->rc_s0.reserve(128 * fold_scratch(n)),
                                                         v->rc_s1.reserve(128 * fold_scratch(n)), st);
            uint8_t* d_prod = v->products.reserve(128 * (np + 2));
            dev::verify_ic_mul_kernel<<<blocks(np + 2), dev::VERIFY_THREADS, 0, st>>>(coeff, v->ic.p, v->alpha.p, np, d_prod);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            uint8_t* d_fixed = v->fixed_p.reserve(192);
            dev::verify_fixed_points_kernel<<<1, 32, 0, st>>>(d_prod, np, csum, d_fixed);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            uint8_t* d_f = v->f.reserve(384 * (n + 3));
            dev::verify_miller_kernel<<<blocks(n + 3), dev::VERIFY_THREADS, 0, st>>>(d_mont, d_nra, nn, v->fl, d_fixed, d_f);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            const uint8_t* prod = fold_all<dev::F12ProdOp>(d_f, nn + 3, 1, v->f_s0.reserve(384 * fold_scratch(n + 3)),
                                                           v->f_s1.reserve(384 * fold_scratch(n + 3)), st);
            uint8_t* d_flag = v->flag.reserve(1);
            dev::verify_final_kernel<<<1, 32, 0, st>>>(prod, d_flag);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            uint8_t flag = 0;
            CUDA_OK(cudaMemcpyAsync(&flag, d_flag, 1, cudaMemcpyDeviceToHost, st));
            CUDA_OK(cudaStreamSynchronize(st));
            if (flag) {
                if (ok) memset(ok, 1, n);
                return (int)n;
            }
        }
        // per-proof verdicts
        uint8_t* d_ok = v->ok.reserve(n);
        dev::verify_single_kernel<<<blocks(n), dev::VERIFY_THREADS, 0, st>>>(d_mont, d_pub, d_valid, nn, np, v->ic.p, v->fl,
                                                                            v->e_ab.p, d_ok);
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        std::vector<uint8_t> res(n);
        CUDA_OK(cudaMemcpyAsync(res.data(), d_ok, n, cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
        int count = 0;
        for (size_t i = 0; i < n; ++i) {
            if (ok) ok[i] = res[i];
            count += res[i];
        }
        return count;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_selftest_pairing_gpu(int device, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* out, char* err, size_t errcap) {
    try {
        if (n == 0) return 0;
        if (!g1 || !g2 || !out) throw std::runtime_error("null argument");
        for (size_t i = 0; i < n; ++i) {
            const G1AffineH p = load_g1(g1 + 64 * i);
            const G2AffineH q = load_g2(g2 + 128 * i);
            if (!g1_on_curve(p) || !g2_on_curve(q)) throw std::runtime_error("point " + std::to_string(i) + " is not on its curve");
        }
        select_device(device);
        DevBuf d1, d2, d3;
        CUDA_OK(cudaMemcpy(d1.reserve(64 * n), g1, 64 * n, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(d2.reserve(128 * n), g2, 128 * n, cudaMemcpyHostToDevice));
        dev::pairing_selftest_kernel<<<blocks(n), dev::VERIFY_THREADS>>>(d1.p, d2.p, (uint32_t)n, d3.reserve(384 * n));
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        CUDA_OK(cudaDeviceSynchronize());
        CUDA_OK(cudaMemcpy(out, d3.p, 384 * n, cudaMemcpyDeviceToHost));
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

}  // extern "C"
