// Engine: device-resident proving key + circuit, trusted setup on the GPU, batched witness + Groth16 prove.
// This is the translation unit nvcc compiles (it includes the kernel files so that the __constant__ field
// parameters exist once); everything CUDA-facing of the C ABI lives here.
#include "ff.cuh"
namespace zke { namespace dev { unsigned long long g_kernel_launches = 0; } }
#include "witness.cu"
#include "matvec.cu"
#include "ntt.cu"
#include "msm.cuh"
#include "fixed_base.cuh"
namespace zke { namespace dev {
ZKE_DEFINE_CONSTANT_UPLOAD(upload_constants_engine)
cudaError_t upload_constants_msm_g1(const FieldConsts*, const FieldConsts*);
cudaError_t upload_constants_msm_g2(const FieldConsts*, const FieldConsts*);
cudaError_t upload_constants_fixed_base(const FieldConsts*, const FieldConsts*);
cudaError_t upload_constants_verify(const FieldConsts*, const FieldConsts*);
cudaError_t upload_constants_registry(const FieldConsts*, const FieldConsts*);
} }

#include "../../include/zkemail_b200.h"
#include "cuda_host.hpp"
#include "engine.hpp"
#include "witness_program.hpp"
#include "binfile.hpp"
#include "ec_host.hpp"
#include "setup_host.hpp"
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>

using namespace zke;

void zke::select_device(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) throw std::runtime_error("no CUDA device available (this library has no CPU fallback)");
    if (device < 0 || device >= n) throw std::runtime_error("bad device index");
    CUDA_OK(cudaSetDevice(device));
    dev::FieldConsts fr, fq;
    fill_consts(fr, fr_params());
    fill_consts(fq, fq_params());
    CUDA_OK(dev::upload_constants_engine(&fr, &fq));
    CUDA_OK(dev::upload_constants_msm_g1(&fr, &fq));
    CUDA_OK(dev::upload_constants_msm_g2(&fr, &fq));
    CUDA_OK(dev::upload_constants_fixed_base(&fr, &fq));
    CUDA_OK(dev::upload_constants_verify(&fr, &fq));
    CUDA_OK(dev::upload_constants_registry(&fr, &fq));
    CUDA_OK(dev::configure_witness_kernel());   // per-device function attribute (> 48 KB dynamic shared memory)
}

namespace {

// 32 x 256 window table of multiples of a generator, affine Montgomery, entry d = 0 is infinity
template <class F>
std::vector<AffineH<F>> window_table(const AffineH<F>& gen) {
    std::vector<AffineH<F>> t(32 * 256, AffineH<F>::inf());
    JacobianH<F> base = JacobianH<F>::from_affine(gen);
    for (int w = 0; w < 32; ++w) {
        JacobianH<F> acc = JacobianH<F>::inf();
        for (int d = 1; d < 256; ++d) {
            acc = acc.add(base);
            t[w * 256 + d] = acc.to_affine();
        }
        for (int k = 0; k < 8; ++k) base = base.dbl();
    }
    return t;
}

std::vector<U256> to_standard(const std::vector<Fr>& v) {
    std::vector<U256> out(v.size());
    const unsigned T = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; ++t)
        th.emplace_back([&, t]() { for (size_t i = v.size() * t / T; i < v.size() * (t + 1) / T; ++i) out[i] = v[i].to_u256(); });
    for (auto& x : th) x.join();
    return out;
}

}  // namespace

struct zke_zkey {
    uint32_t n_vars = 0, n_public = 0, log_n = 0;
    int device = 0;
    bool toy = false;         // made by zke_setup (the toxic waste is known) or by zke_zkey_from_ptau (delta = 1)
    bool delta_one = false;   // made by zke_zkey_from_ptau and not yet contributed to: toy until a contribution
    G1AffineH alpha1, beta1, delta1;
    G2AffineH beta2, gamma2, delta2;
    std::vector<G1AffineH> ic;
    DevBuf A, B1, B2, C, H;   // affine Montgomery points on the device; H holds h_levels window levels [level][N]
    int h_levels = 1;         // > 1: level j = 2^(c j) * H (fixed-base table for the H multi-exponentiation)
    dev::MsmConfig cfg_h;
    // Coefficient matrices of `.zkey` section 4 (loaded keys only): A and B of the QAP as CSR over the 2^log_n domain
    // rows, including the n_public + 1 extra rows of A; `coefs` is the interned coefficient table in standard form.
    bool has_coefs = false;
    std::vector<uint32_t> a_ptr, a_var, a_coef, b_ptr, b_var, b_coef;
    std::vector<U256> coefs;
};

struct zke_ctx {
    const zke_circuit* circuit = nullptr;   // may be null for a context opened from a loaded `.zkey` alone
    const zke_zkey* zkey = nullptr;
    int device = 0;
    uint32_t max_batch = 0;
    uint32_t n_vars = 0, n_public = 0, n_inputs = 0;
    cudaStream_t stream = nullptr;          // witness stream (highest priority)
    // circuit on device
    DevBuf ops, iter_hdr, lc_terms, aux, coop, coef_r, small_inv;
    std::vector<uint32_t> coef_word;   // per interned coefficient: index | k << 16 | kind << 24 (lc_term.cuh)
    std::vector<uint32_t> iter_info;   // per iteration {first op's record word 1, live ops, terms} (diagnostics)
    DevBuf a_ptr, a_terms, b_ptr, b_terms, c_ptr, c_terms;
    dev::DevProgram prog;
    dev::DevR1cs r1cs;
    // ntt
    DevBuf tw_fwd, tw_inv, coset_scale;
    dev::NttTables ntt;
    size_t stride = 0;           // witness elements per email (n_vars + n_temps)
    DevBuf inputs, check_flag;   // inputs made resident by zke_upload_inputs; flag words of the witness validation
    uint32_t inputs_resident = 0;
    // Batch slots.  The synchronous entry points use slot 0; zke_fullprove_submit alternates between the two, so that
    // the witness kernel of one batch (latency-bound, a few CTAs) runs while the proving kernels of the previous batch
    // saturate the multiplier pipe.  Slot 1 is allocated on first use.
    struct Slot {
        bool allocated = false, busy = false;
        DevBuf w_all, inputs, results, first_bad;
        uint8_t* results_host = nullptr;      // pinned, [max_batch][ZKE_RESULT_STRIDE]
        uint8_t* publics_host = nullptr;      // pinned, [max_batch][n_public][32]
        std::vector<cudaEvent_t> done;        // per email
        cudaEvent_t witness_done = nullptr;
        uint32_t loaded = 0;                  // witnesses resident in w_all
        uint32_t batch = 0;                   // batch of the pending submission
        std::vector<uint8_t> rs;              // its blinding scalars ([batch][2][32]) or empty
    };
    Slot slots[2];
    uint64_t n_submitted = 0, n_collected = 0;
    // intra-proof sharding (zke_shard_*): this GPU's place among `shard_world` GPUs proving ONE witness together
    int shard_rank = -1, shard_world = 0, shard_log_g = 0, shard_stage = 0;
    // proving lanes: emails are dealt round-robin to `n_lanes` streams, each with its own NTT vectors and MSM
    // workspace, so that the latency-bound tails of one email's kernels overlap the saturating kernels of another
    // Each lane owns two streams: `st` (high priority) carries the latency- / memory-bound kernels, `heavy` (low
    // priority) the kernels that saturate the integer pipe (NTT passes, bucket accumulation of the H MSM).  When a
    // block of a saturating kernel retires, the block scheduler serves pending high-priority blocks first, so the
    // light kernels of one proof run inside the heavy kernels of another instead of queueing behind them.
    struct Lane { cudaStream_t st = nullptr, heavy = nullptr; cudaEvent_t ev[6] = {}; DevBuf va, vb, vc, vd, msm_ws; };
    Lane lanes[ZKE_MAX_LANES];
    int n_lanes = 1, lanes_alloc = 0;
    int finish_threads = 4;      // host threads that finish the MSMs / assemble the proofs (ZKE_FINISH_THREADS)
    dev::MsmConfig cfg_w, cfg_h;
    bool split_streams = true;   // ZKE_SPLIT_STREAMS=0: everything of a lane on one stream (experiments)
    std::vector<uint32_t> bad_host;
    // optional stage profiling (CUDA events on `stream`)
    bool profile = false;
    std::vector<cudaEvent_t> ev_pool;
    size_t ev_used = 0;
    struct Span { int stage; size_t e0, e1; };
    std::vector<Span> spans;
    double stage_ms[ZKE_N_STAGES] = {0};
    uint64_t stage_count[ZKE_N_STAGES] = {0};
    cudaEvent_t ev(size_t* idx) {
        if (ev_used == ev_pool.size()) { cudaEvent_t e; cudaEventCreate(&e); ev_pool.push_back(e); }
        *idx = ev_used;
        return ev_pool[ev_used++];
    }
    size_t mark(cudaStream_t st) { size_t i; cudaEventRecord(ev(&i), st); return i; }
    size_t mark() { return mark(stream); }
    void collect() {   // call after the stream has been synchronised
        for (auto& s : spans) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, ev_pool[s.e0], ev_pool[s.e1]) == cudaSuccess) { stage_ms[s.stage] += ms; stage_count[s.stage]++; }
        }
        spans.clear();
        ev_used = 0;
    }
};

// ------------------------------------------------------------------------------------------------ H table
// zk->H holds level 0 (the N points of `.zkey` section 9) in its first N entries and is sized for h_levels levels:
// level j = 2^(c j) * level 0, the fixed-base table that lets all windows of the H multi-exponentiation share one
// bucket set (msm.cuh).
static const uint32_t SETUP_SLAB = 1u << 20;
static void h_table_config(zke_zkey* zk, size_t N) {
    const char* e = getenv("ZKE_H_PRECOMP");
    const bool precomp = !(e && atoi(e) == 0);
    zk->cfg_h = dev::msm_config_full((uint32_t)N, precomp);
    zk->h_levels = precomp ? dev::msm_windows(zk->cfg_h) : 1;
}
static void build_h_levels(zke_zkey* zk, size_t N, uint8_t* scratch, cudaStream_t st) {
    for (int lvl = 1; lvl < zk->h_levels; ++lvl) {
        const uint8_t* prev = zk->H.p + (size_t)(lvl - 1) * N * sizeof(dev::G1Affine);
        uint8_t* cur = zk->H.p + (size_t)lvl * N * sizeof(dev::G1Affine);
        for (size_t off = 0; off < N; off += SETUP_SLAB) {
            uint32_t cnt = (uint32_t)std::min<size_t>(SETUP_SLAB, N - off);
            dev::scale_pow2_batch<dev::Fq>(prev + sizeof(dev::G1Affine) * off, cnt, zk->cfg_h.c, scratch, cur + sizeof(dev::G1Affine) * off, st);
        }
    }
    CHECK_LAUNCH();
    CUDA_OK(cudaStreamSynchronize(st));
}

// ------------------------------------------------------------------------------------------------ setup
static zke_zkey* do_setup(const zke_circuit* zc, uint64_t seed, int device) {
    select_device(device);
    const Circuit& c = zc->c;
    SetupScalars S = compute_setup_scalars(c, seed);
    std::unique_ptr<zke_zkey> zk(new zke_zkey());
    zk->n_vars = c.n_vars; zk->n_public = c.n_public(); zk->log_n = S.log_n; zk->device = device;
    zk->toy = true;
    const size_t N = (size_t)1 << S.log_n;
    const uint32_t m = c.n_vars, l = c.n_public();

    G1JacH g1 = G1JacH::from_affine(g1_generator());
    G2JacH g2 = G2JacH::from_affine(g2_generator());
    zk->alpha1 = g1.mul(S.alpha.to_u256()).to_affine();
    zk->beta1 = g1.mul(S.beta.to_u256()).to_affine();
    zk->delta1 = g1.mul(S.delta.to_u256()).to_affine();
    zk->beta2 = g2.mul(S.beta.to_u256()).to_affine();
    zk->gamma2 = g2.mul(S.gamma.to_u256()).to_affine();
    zk->delta2 = g2.mul(S.delta.to_u256()).to_affine();

    DevBuf t1, t2, scal, scratch;
    t1.upload(window_table<Fq>(g1_generator()));
    t2.upload(window_table<Fq2>(g2_generator()));
    const uint32_t SLAB = SETUP_SLAB;
    scratch.alloc((size_t)SLAB * sizeof(dev::G2XYZZ));
    cudaStream_t st = nullptr;

    auto run_g1 = [&](const std::vector<Fr>& s, DevBuf& out) {
        std::vector<U256> std_s = to_standard(s);
        scal.upload(std_s);
        out.alloc(s.size() * sizeof(dev::G1Affine));
        for (size_t off = 0; off < s.size(); off += SLAB) {
            uint32_t cnt = (uint32_t)std::min<size_t>(SLAB, s.size() - off);
            dev::fixed_base_batch<dev::Fq>(t1.p, scal.p + 32 * off, cnt, scratch.p, out.p + sizeof(dev::G1Affine) * off, st);
        }
        CHECK_LAUNCH();
        CUDA_OK(cudaStreamSynchronize(st));
    };
    run_g1(S.a, zk->A);
    run_g1(S.b, zk->B1);
    run_g1(S.kc, zk->C);
    {
        // H points, then (unless ZKE_H_PRECOMP=0) the fixed-base table levels 2^(c j) * H_i
        h_table_config(zk.get(), N);
        std::vector<U256> std_s = to_standard(S.h);
        scal.upload(std_s);
        zk->H.alloc((size_t)zk->h_levels * N * sizeof(dev::G1Affine));
        for (size_t off = 0; off < N; off += SLAB) {
            uint32_t cnt = (uint32_t)std::min<size_t>(SLAB, N - off);
            dev::fixed_base_batch<dev::Fq>(t1.p, scal.p + 32 * off, cnt, scratch.p, zk->H.p + sizeof(dev::G1Affine) * off, st);
        }
        build_h_levels(zk.get(), N, scratch.p, st);
    }
    {
        std::vector<U256> std_s = to_standard(S.b);
        scal.upload(std_s);
        zk->B2.alloc((size_t)m * sizeof(dev::G2Affine));
        for (size_t off = 0; off < m; off += SLAB) {
            uint32_t cnt = (uint32_t)std::min<size_t>(SLAB, m - off);
            dev::fixed_base_batch<dev::Fq2>(t2.p, scal.p + 32 * off, cnt, scratch.p, zk->B2.p + sizeof(dev::G2Affine) * off, st);
        }
        CHECK_LAUNCH();
        CUDA_OK(cudaStreamSynchronize(st));
    }
    // IC = first l+1 entries of the kc points; they are not part of the C ("L") section
    zk->ic.resize(l + 1);
    CUDA_OK(cudaMemcpy(zk->ic.data(), zk->C.p, sizeof(G1AffineH) * (l + 1), cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemset(zk->C.p, 0, sizeof(G1AffineH) * (l + 1)));
    return zk.release();
}

// ------------------------------------------------------------------------------------------------ .zkey reader
// iden3 binfile container: magic[4], u32 version, u32 nSections, then {u32 type, u64 size, payload} per section.
// zkey v1 (Groth16): 1 {u32 protocol = 1}; 2 {n8q, q, n8r, r, nVars, nPublic, domainSize, alpha1, beta1, beta2, gamma2,
// delta1, delta2}; 3 IC; 4 {u32 n, (u32 matrix, u32 constraint, u32 signal, value[n8r]) x n}; 5 A; 6 B1; 7 B2;
// 8 C (private signals only); 9 H; 10 contributions.  Points are affine with Montgomery-form little-endian
// coordinates (G2: x.c0, x.c1, y.c0, y.c1), infinity = all-zero bytes - the device image of this engine, so the point
// sections are uploaded as they are; coefficient values are stored multiplied by R^2 (snarkjs multiplies them with
// the raw witness in Montgomery arithmetic twice).  The formats live in the un-vendored @iden3/binfileutils /
// snarkjs 0.5.0 (SURVEY 8(b)); the call sites are chunked-zkey.ts:80-84 and UsageGuide/README.md:139-195.
namespace {
void split_container(const uint8_t* b, size_t len, SecView sec[11]) {
    if (!b || len < 12 || memcmp(b, "zkey", 4) != 0) throw std::runtime_error("not a .zkey file (bad magic)");
    if (rd32(b + 4) != 1) throw std::runtime_error("unsupported .zkey version");
    for (const BinSection& s : binfile_sections(b, len, ".zkey"))
        if (s.type >= 1 && s.type <= 10) sec[s.type] = s.view;
}

// Runs launch(flag) for a kernel that atomicMin's the index of each failing item into *flag (device); returns the
// smallest such index, or -1 if none failed.
template <class Launch>
int64_t first_flagged(uint32_t* flag, Launch launch) {
    CUDA_OK(cudaMemset(flag, 0xff, 4));
    launch(flag);
    ZKE_COUNT_LAUNCH(1);
    CHECK_LAUNCH();
    uint32_t first = 0;
    CUDA_OK(cudaMemcpy(&first, flag, 4, cudaMemcpyDeviceToHost));
    return first == 0xffffffffu ? -1 : (int64_t)first;
}

// every point either all-zero (infinity) or on y^2 = x^3 + b with canonical (< q) coordinates
template <class F>
__global__ void validate_points_kernel(const uint8_t* __restrict__ pts, uint32_t n, F b, uint32_t* bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const dev::Affine<F> p = dev::Affine<F>::load(pts + sizeof(dev::Affine<F>) * (size_t)i);
    if (p.is_inf()) return;
    if (!dev::below_modulus(p.x) || !dev::below_modulus(p.y) || !(p.y.sqr() == p.x.sqr() * p.x + b)) atomicMin(bad, i);
}

// -1 if every point of pts[0, n) (device) passes validate_points_kernel, else the first index that does not
template <class F, class HostF>
int64_t first_invalid_point(const uint8_t* pts, size_t n, const HostF& b_host, uint32_t* flag) {
    if (!n) return -1;
    F b;
    static_assert(sizeof(F) == sizeof(HostF), "host / device field images differ");
    memcpy(&b, &b_host, sizeof(F));
    return first_flagged(flag, [&](uint32_t* f) { validate_points_kernel<F><<<(unsigned)((n + 127) / 128), 128>>>(pts, (uint32_t)n, b, f); });
}

Fq2 g2_twist_b() { return Fq2{Fq::from_u64(3), Fq::zero()} * Fq2{Fq::from_u64(9), Fq::one()}.inv(); }

struct U256HashE {
    size_t operator()(const U256& x) const { return (size_t)(x.v[0] * 0x9E3779B97F4A7C15ull ^ x.v[1] * 31 ^ x.v[2] * 131 ^ x.v[3]); }
};
}  // namespace

static zke_zkey* do_zkey_load(const SecView sec[11], int device) {
    select_device(device);
    for (int s = 1; s <= 9; ++s) if (!sec[s].p) throw std::runtime_error(".zkey section " + std::to_string(s) + " is missing");
    if (sec[1].n < 4 || rd32(sec[1].p) != 1) throw std::runtime_error("not a Groth16 .zkey (protocol id)");
    const uint8_t* h = sec[2].p;
    const size_t HDR = 4 + 32 + 4 + 32 + 12 + 64 + 64 + 128 + 128 + 64 + 128;
    if (sec[2].n < HDR) throw std::runtime_error(".zkey header section too short");
    if (rd32(h) != 32 || memcmp(h + 4, fq_params().p.v, 32) != 0) throw std::runtime_error(".zkey is not over the BN254 base field");
    if (rd32(h + 36) != 32 || memcmp(h + 40, fr_params().p.v, 32) != 0) throw std::runtime_error(".zkey is not over the BN254 scalar field");
    std::unique_ptr<zke_zkey> zk(new zke_zkey());
    zk->device = device;
    zk->n_vars = rd32(h + 72); zk->n_public = rd32(h + 76);
    const uint32_t domain = rd32(h + 80);
    if (domain == 0 || (domain & (domain - 1)) || domain > (1u << 28)) throw std::runtime_error(".zkey domain size is not a power of two <= 2^28");
    zk->log_n = 0;
    while ((1u << zk->log_n) < domain) zk->log_n++;
    const uint32_t m = zk->n_vars, l = zk->n_public;
    if (m == 0 || l + 1 > m) throw std::runtime_error(".zkey header: nPublic + 1 > nVars");
    const size_t N = domain;
    auto need = [&](int s, size_t bytes) {
        if (sec[s].n != bytes) throw std::runtime_error(".zkey section " + std::to_string(s) + " has " + std::to_string(sec[s].n) + " bytes, expected " + std::to_string(bytes));
    };
    need(3, (size_t)(l + 1) * 64); need(5, (size_t)m * 64); need(6, (size_t)m * 64); need(7, (size_t)m * 128);
    need(8, (size_t)(m - l - 1) * 64); need(9, N * 64);

    // header points and IC: host copies, checked on the host
    const uint8_t* q = h + 84;
    memcpy(&zk->alpha1, q, 64); memcpy(&zk->beta1, q + 64, 64); memcpy(&zk->beta2, q + 128, 128);
    memcpy(&zk->gamma2, q + 256, 128); memcpy(&zk->delta1, q + 384, 64); memcpy(&zk->delta2, q + 448, 128);
    auto fq_ok = [](const Fq& x) { return u256_cmp(x.m, fq_params().p) < 0; };
    auto g1_ok = [&](const G1AffineH& p) { return fq_ok(p.x) && fq_ok(p.y) && g1_on_curve(p); };
    auto g2_ok = [&](const G2AffineH& p) { return fq_ok(p.x.c0) && fq_ok(p.x.c1) && fq_ok(p.y.c0) && fq_ok(p.y.c1) && g2_on_curve(p); };
    if (!g1_ok(zk->alpha1) || !g1_ok(zk->beta1) || !g1_ok(zk->delta1) || !g2_ok(zk->beta2) || !g2_ok(zk->gamma2) || !g2_ok(zk->delta2))
        throw std::runtime_error(".zkey header: a key point is not on its curve");
    zk->ic.resize(l + 1);
    memcpy(zk->ic.data(), sec[3].p, (size_t)(l + 1) * 64);
    for (auto& p : zk->ic) if (!g1_ok(p)) throw std::runtime_error(".zkey section 3: an IC point is not on the curve");

    // section 4 -> CSR of A and B over the N domain rows
    {
        if (sec[4].n < 4) throw std::runtime_error(".zkey section 4 too short");
        const uint32_t n_rec = rd32(sec[4].p);
        if (sec[4].n != 4 + (size_t)n_rec * 44) throw std::runtime_error(".zkey section 4: size does not match its record count");
        const uint8_t* rec = sec[4].p + 4;
        zk->a_ptr.assign(N + 1, 0); zk->b_ptr.assign(N + 1, 0);
        for (uint32_t k = 0; k < n_rec; ++k) {
            const uint8_t* r = rec + 44 * (size_t)k;
            const uint32_t mat = rd32(r), row = rd32(r + 4), sig = rd32(r + 8);
            if (mat > 1 || row >= N || sig >= m) throw std::runtime_error(".zkey section 4: record " + std::to_string(k) + " out of range");
            (mat == 0 ? zk->a_ptr : zk->b_ptr)[row + 1]++;
        }
        for (size_t i = 0; i < N; ++i) { zk->a_ptr[i + 1] += zk->a_ptr[i]; zk->b_ptr[i + 1] += zk->b_ptr[i]; }
        zk->a_var.resize(zk->a_ptr[N]); zk->a_coef.resize(zk->a_ptr[N]);
        zk->b_var.resize(zk->b_ptr[N]); zk->b_coef.resize(zk->b_ptr[N]);
        std::vector<uint32_t> ca(zk->a_ptr.begin(), zk->a_ptr.end() - 1), cb(zk->b_ptr.begin(), zk->b_ptr.end() - 1);
        // stored value = c R^2 mod r; interned on the stored image, converted once per distinct value
        const Fr r_elem = Fr::from_u256(fr_params().r);          // the field element R mod r
        const Fr rinv2 = (r_elem * r_elem).inv();
        std::unordered_map<U256, uint32_t, U256HashE> index;
        for (uint32_t k = 0; k < n_rec; ++k) {
            const uint8_t* r = rec + 44 * (size_t)k;
            const uint32_t mat = rd32(r), row = rd32(r + 4), sig = rd32(r + 8);
            U256 raw;
            memcpy(raw.v, r + 12, 32);
            auto it = index.find(raw);
            if (it == index.end()) {
                if (u256_cmp(raw, fr_params().p) >= 0) throw std::runtime_error(".zkey section 4: coefficient not reduced mod r");
                it = index.emplace(raw, (uint32_t)zk->coefs.size()).first;
                zk->coefs.push_back((Fr::from_u256(raw) * rinv2).to_u256());
            }
            if (mat == 0) { const uint32_t pos = ca[row]++; zk->a_var[pos] = sig; zk->a_coef[pos] = it->second; }
            else { const uint32_t pos = cb[row]++; zk->b_var[pos] = sig; zk->b_coef[pos] = it->second; }
        }
        if (zk->coefs.size() >= (1u << 24)) throw std::runtime_error(".zkey has more than 2^24 distinct coefficients");
        zk->has_coefs = true;
    }

    // point sections: the file image is the device image
    DevBuf flag, scratch;
    flag.alloc(4);
    const Fq b1 = Fq::from_u64(3);
    const Fq2 b2 = g2_twist_b();
    auto up = [&](DevBuf& dst, const uint8_t* src, size_t bytes, size_t skip) {
        dst.alloc(skip + bytes);
        if (skip) CUDA_OK(cudaMemset(dst.p, 0, skip));
        if (bytes) CUDA_OK(cudaMemcpy(dst.p + skip, src, bytes, cudaMemcpyHostToDevice));
    };
    auto refuse = [](int64_t bad, const char* what) {
        if (bad >= 0) throw std::runtime_error(std::string(".zkey section ") + what + ": point " + std::to_string(bad) + " is not on the curve");
    };
    uint32_t* fl = (uint32_t*)flag.p;
    up(zk->A, sec[5].p, sec[5].n, 0);   refuse(first_invalid_point<dev::Fq>(zk->A.p, m, b1, fl), "5 (A)");
    up(zk->B1, sec[6].p, sec[6].n, 0);  refuse(first_invalid_point<dev::Fq>(zk->B1.p, m, b1, fl), "6 (B1)");
    up(zk->B2, sec[7].p, sec[7].n, 0);  refuse(first_invalid_point<dev::Fq2>(zk->B2.p, m, b2, fl), "7 (B2)");
    up(zk->C, sec[8].p, sec[8].n, (size_t)(l + 1) * 64);   // C / "L": infinity for the public signals
    refuse(first_invalid_point<dev::Fq>(zk->C.p, m, b1, fl), "8 (C)");
    h_table_config(zk.get(), N);
    zk->H.alloc((size_t)zk->h_levels * N * sizeof(dev::G1Affine));
    CUDA_OK(cudaMemcpy(zk->H.p, sec[9].p, N * 64, cudaMemcpyHostToDevice));
    refuse(first_invalid_point<dev::Fq>(zk->H.p, N, b1, fl), "9 (H)");
    scratch.alloc((size_t)SETUP_SLAB * sizeof(dev::G1XYZZ));
    build_h_levels(zk.get(), N, scratch.p, nullptr);
    return zk.release();
}

// `.zkey` writer (sections in file order 1..10; the record order of section 4 is A rows, B rows, then the extra rows)
static int64_t do_zkey_write(const zke_zkey* zk, const zke_circuit* zc, uint8_t* out, size_t cap) {
    const uint32_t m = zk->n_vars, l = zk->n_public;
    const size_t N = (size_t)1 << zk->log_n;
    const Circuit* c = zc ? &zc->c : nullptr;
    if (!zk->has_coefs) {
        if (!c) throw std::runtime_error("a key made by zke_setup needs its circuit to write the coefficient section");
        if (c->n_vars != m || c->n_public() != l || c->domain_log2() != zk->log_n) throw std::runtime_error("zkey does not belong to this circuit");
    }
    size_t n_rec;
    if (zk->has_coefs) n_rec = zk->a_var.size() + zk->b_var.size();
    else n_rec = c->a_var.size() + c->b_var.size() + l + 1;
    const size_t HDR = 4 + 32 + 4 + 32 + 12 + 64 + 64 + 128 + 128 + 64 + 128;
    const size_t sizes[11] = {0, 4, HDR, (size_t)(l + 1) * 64, 4 + n_rec * 44, (size_t)m * 64, (size_t)m * 64, (size_t)m * 128,
                              (size_t)(m - l - 1) * 64, N * 64, 68};
    size_t total = 12;
    for (int s = 1; s <= 10; ++s) total += 12 + sizes[s];
    if (!out) return (int64_t)total;
    if (cap < total) return -2;
    CUDA_OK(cudaSetDevice(zk->device));
    BinWriter w{out};
    w.header("zkey", 1, 10);
    w.section(1, sizes[1]); w.u32(1);
    w.section(2, sizes[2]);
    w.u32(32); w.bytes(fq_params().p.v, 32); w.u32(32); w.bytes(fr_params().p.v, 32); w.u32(m); w.u32(l); w.u32((uint32_t)N);
    w.bytes(&zk->alpha1, 64); w.bytes(&zk->beta1, 64); w.bytes(&zk->beta2, 128); w.bytes(&zk->gamma2, 128); w.bytes(&zk->delta1, 64); w.bytes(&zk->delta2, 128);
    w.section(3, sizes[3]); w.bytes(zk->ic.data(), (size_t)(l + 1) * 64);
    w.section(4, sizes[4]); w.u32((uint32_t)n_rec);
    {
        const std::vector<U256>& coefs = zk->has_coefs ? zk->coefs : c->coefs;
        const Fr r_elem = Fr::from_u256(fr_params().r);
        const Fr r2 = r_elem * r_elem;
        std::vector<U256> stored(coefs.size());
        for (size_t i = 0; i < coefs.size(); ++i) stored[i] = (Fr::from_u256(coefs[i]) * r2).to_u256();
        auto rows = [&](uint32_t mat, const std::vector<uint32_t>& ptr, const std::vector<uint32_t>& var, const std::vector<uint32_t>& coef, size_t n_rows) {
            for (size_t row = 0; row < n_rows; ++row)
                for (uint32_t k = ptr[row]; k < ptr[row + 1]; ++k) { w.u32(mat); w.u32((uint32_t)row); w.u32(var[k]); w.bytes(stored[coef[k]].v, 32); }
        };
        if (zk->has_coefs) {
            rows(0, zk->a_ptr, zk->a_var, zk->a_coef, N);
            rows(1, zk->b_ptr, zk->b_var, zk->b_coef, N);
        } else {
            rows(0, c->a_ptr, c->a_var, c->a_coef, c->n_constraints);
            rows(1, c->b_ptr, c->b_var, c->b_coef, c->n_constraints);
            const U256 one_r2 = r2.to_u256();
            for (uint32_t j = 0; j <= l; ++j) { w.u32(0); w.u32(c->n_constraints + j); w.u32(j); w.bytes(one_r2.v, 32); }
        }
    }
    auto dev_sec = [&](int s, const DevBuf& b, size_t skip) {
        w.section(s, sizes[s]);
        if (sizes[s]) CUDA_OK(cudaMemcpy(w.p, b.p + skip, sizes[s], cudaMemcpyDeviceToHost));
        w.p += sizes[s];
    };
    dev_sec(5, zk->A, 0); dev_sec(6, zk->B1, 0); dev_sec(7, zk->B2, 0); dev_sec(8, zk->C, (size_t)(l + 1) * 64); dev_sec(9, zk->H, 0);
    w.section(10, sizes[10]); memset(w.p, 0, 68); w.p += 68;    // circuit hash placeholder, zero contributions
    return (int64_t)(w.p - out);
}

// ------------------------------------------------------------------------------------------------ ctx
static void alloc_slot(zke_ctx* x, zke_ctx::Slot& S) {
    if (S.allocated) return;
    S.w_all.alloc(x->stride * 32 * x->max_batch);
    S.inputs.alloc((size_t)std::max(1u, x->n_inputs) * 32 * x->max_batch);
    S.first_bad.alloc(4 * (size_t)x->max_batch);
    if (x->zkey) {
        S.results.alloc((size_t)x->max_batch * ZKE_RESULT_STRIDE);
        CUDA_OK(cudaHostAlloc((void**)&S.results_host, (size_t)x->max_batch * ZKE_RESULT_STRIDE, cudaHostAllocDefault));
        CUDA_OK(cudaHostAlloc((void**)&S.publics_host, (size_t)x->max_batch * std::max(1u, x->n_public) * 32, cudaHostAllocDefault));
        S.done.resize(x->max_batch);
        for (auto& e : S.done) CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        CUDA_OK(cudaEventCreateWithFlags(&S.witness_done, cudaEventDisableTiming));
    }
    S.allocated = true;
}

// The key's A and B (`.zkey` section 4 form: CSR over the 2^log_n domain rows) against the circuit's, compared as linear
// forms: a row's terms sorted by signal, duplicates added, zero terms dropped.  Rows of the circuit, then the n_public + 1
// extra rows of A (1 * w_j), then nothing.  Rows whose terms are listed identically are compared without the sort.
static void check_key_matrices(const Circuit& c, const zke_zkey& zk) {
    const size_t N = (size_t)1 << zk.log_n;
    const uint32_t nc = c.n_constraints, l = c.n_public();
    typedef std::vector<std::pair<uint32_t, Fr>> Form;
    auto canonical = [](Form& f) {
        std::sort(f.begin(), f.end(), [](const std::pair<uint32_t, Fr>& a, const std::pair<uint32_t, Fr>& b) { return a.first < b.first; });
        size_t o = 0;
        for (size_t i = 0; i < f.size();) {
            std::pair<uint32_t, Fr> t = f[i++];
            while (i < f.size() && f[i].first == t.first) t.second = t.second + f[i++].second;
            if (!t.second.is_zero()) f[o++] = t;
        }
        f.resize(o);
    };
    Form x, y;
    auto compare = [&](const char* name, const std::vector<uint32_t>& kp, const std::vector<uint32_t>& kv, const std::vector<uint32_t>& kc,
                       const std::vector<uint32_t>& cp, const std::vector<uint32_t>& cv, const std::vector<uint32_t>& cc, bool extra) {
        for (size_t row = 0; row < N; ++row) {
            const uint32_t kb = kp[row], ke = kp[row + 1];
            if (row < nc) {
                const uint32_t b = cp[row], e = cp[row + 1];
                bool same = e - b == ke - kb;
                for (uint32_t k = 0; same && k < e - b; ++k) same = cv[b + k] == kv[kb + k] && c.coefs[cc[b + k]] == zk.coefs[kc[kb + k]];
                if (same) continue;
            }
            x.clear(); y.clear();
            for (uint32_t k = kb; k < ke; ++k) x.emplace_back(kv[k], Fr::from_u256(zk.coefs[kc[k]]));
            if (row < nc) {
                for (uint32_t k = cp[row]; k < cp[row + 1]; ++k) y.emplace_back(cv[k], Fr::from_u256(c.coefs[cc[k]]));
            } else if (extra && row <= (size_t)nc + l) {
                y.emplace_back((uint32_t)(row - nc), Fr::one());
            }
            canonical(x); canonical(y);
            bool same = x.size() == y.size();
            for (size_t i = 0; same && i < x.size(); ++i) same = x[i].first == y[i].first && x[i].second == y[i].second;
            if (!same) throw std::runtime_error(std::string("zkey does not belong to this circuit: ") + name + " row " + std::to_string(row) + " differs");
        }
    };
    compare("A", zk.a_ptr, zk.a_var, zk.a_coef, c.a_ptr, c.a_var, c.a_coef, true);
    compare("B", zk.b_ptr, zk.b_var, zk.b_coef, c.b_ptr, c.b_var, c.b_coef, false);
}

// Lowers the circuit's witness program into the kernel's stream (witness_program.cpp) with the options of this process and
// context, and makes it resident.
static void upload_program(zke_ctx* x, const Circuit& c) {
    const uint32_t max_batch = x->max_batch;
    LowerOptions opt;
    // ZKE_NATIVE_SHA=0 keeps the Sha256compression gadget's own ops, ZKE_NATIVE_REGEX=0 turns the regex state seeding off,
    // ZKE_COOP_FPMUL=0: the sequential single-thread hint
    if (const char* e = getenv("ZKE_NATIVE_SHA")) opt.native_sha = atoi(e) != 0;
    if (const char* e = getenv("ZKE_NATIVE_REGEX")) opt.native_regex = atoi(e) != 0;
    if (const char* e = getenv("ZKE_NATIVE_POSEIDON")) opt.native_poseidon = atoi(e) != 0;   // 0: the recorded Poseidon gadgets' own ops
    if (const char* e = getenv("ZKE_COOP_FPMUL")) opt.coop_fpmul = atoi(e) != 0;
    // ZKE_WITNESS_CLUSTER = 2 / 4 / 8: thread-block cluster of that many CTAs per email (witness.cu); every level is padded to
    // whole rounds of `cluster` iterations, iteration k belongs to CTA k % cluster
    // (default: as many CTAs per email as still fit one wave of the GPU's SMs at this context's batch size - a witness
    // CTA owns an SM; ZKE_WITNESS_CLUSTER=1 keeps one CTA per email).
    const uint32_t sms = (uint32_t)dev::sm_count();
    opt.cluster = max_batch <= 8 ? 8 : (max_batch <= 32 ? 4 : (2 * max_batch <= sms ? 2 : 1));
    if (const char* e = getenv("ZKE_WITNESS_CLUSTER")) { const int v = atoi(e); if (v == 1 || v == 2 || v == 4 || v == 8) opt.cluster = (uint32_t)v; }
    WitnessStream S = lower_witness_program(c, x->coef_word, opt);
    x->ops.upload(S.ops);
    x->iter_hdr.upload(S.iter_hdr);
    x->lc_terms.upload(S.terms);
    x->aux.upload(S.aux);
    x->coop.upload(S.coop);
    x->iter_info = std::move(S.iter_info);
    const uint32_t NSMALL = 4096;
    std::vector<Fr> inv(NSMALL);
    for (uint32_t i = 0; i < NSMALL; ++i) inv[i] = Fr::from_u64(i);
    batch_inverse(inv.data(), NSMALL);
    std::vector<U256> inv_std(NSMALL);
    for (uint32_t i = 0; i < NSMALL; ++i) inv_std[i] = inv[i].to_u256();
    x->small_inv.upload(inv_std);
    dev::DevProgram& P = x->prog;
    P.ops = (const uint4*)x->ops.p; P.iter_hdr = (const uint4*)x->iter_hdr.p; P.coop = (const uint32_t*)x->coop.p;
    P.terms = (const uint2*)x->lc_terms.p; P.aux = (const uint32_t*)x->aux.p; P.coef_r = x->coef_r.p;
    P.small_inv = x->small_inv.p; P.n_small_inv = NSMALL;
    P.trace = nullptr;
    P.cluster = S.cluster;
    P.n_iters = S.n_iters; P.n_ops = (uint32_t)c.ops.size(); P.n_vars = c.n_vars; P.n_temps = c.n_temps;
    P.n_outputs = c.n_outputs; P.n_inputs = c.n_inputs();
}

// R1CS (the circuit's A, B, C) or the QAP matrices of the key (A, B incl. the extra public rows; no C)
static void upload_r1cs(zke_ctx* x, const Circuit* cp, const zke_zkey* zk) {
    auto up_terms = [&](const std::vector<uint32_t>& var, const std::vector<uint32_t>& coef, DevBuf& dst) {
        std::vector<uint32_t> t(2 * var.size() + 2);
        for (size_t i = 0; i < var.size(); ++i) { t[2 * i] = var[i]; t[2 * i + 1] = x->coef_word[coef[i]]; }
        dst.upload(t);
    };
    dev::DevR1cs& R = x->r1cs;
    if (cp) {
        const Circuit& c = *cp;
        x->a_ptr.upload(c.a_ptr); x->b_ptr.upload(c.b_ptr); x->c_ptr.upload(c.c_ptr);
        up_terms(c.a_var, c.a_coef, x->a_terms); up_terms(c.b_var, c.b_coef, x->b_terms); up_terms(c.c_var, c.c_coef, x->c_terms);
        R.c_ptr = (const uint32_t*)x->c_ptr.p; R.c_terms = (const uint2*)x->c_terms.p;
        R.n_constraints = c.n_constraints; R.n_public = c.n_public();
    } else {
        x->a_ptr.upload(zk->a_ptr); x->b_ptr.upload(zk->b_ptr);
        up_terms(zk->a_var, zk->a_coef, x->a_terms); up_terms(zk->b_var, zk->b_coef, x->b_terms);
        R.c_ptr = nullptr; R.c_terms = nullptr;
        R.n_constraints = 1u << zk->log_n; R.n_public = 0;    // every domain row comes from the key's matrices
    }
    R.a_ptr = (const uint32_t*)x->a_ptr.p; R.b_ptr = (const uint32_t*)x->b_ptr.p;
    R.a_terms = (const uint2*)x->a_terms.p; R.b_terms = (const uint2*)x->b_terms.p;
    R.coef_r = x->coef_r.p; R.n_vars = x->n_vars;
}

namespace {
// Fixed-operand form of a constant w (ff.cuh: Fp::mul_shoup): {w in standard form, floor(w 2^256 / r)}.  With
// w 2^256 = q r + rem the remainder is the Montgomery image of w, so q = (w 2^256 - rem) / r exactly, and an exact
// quotient is a product with r^-1 modulo 2^256: q = rem * (-r^-1 mod 2^256) mod 2^256 - no division.
struct ShoupPair { U256 w, wq; };
U256 mul_lo256(const U256& a, const U256& b) {
    uint64_t t[4] = {0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) {
        u128 c = 0;
        for (int j = 0; i + j < 4; ++j) {
            c += (u128)a.v[j] * b.v[i] + t[i + j];
            t[i + j] = (uint64_t)c;
            c >>= 64;
        }
    }
    return U256{{t[0], t[1], t[2], t[3]}};
}
const U256& fr_neg_inv256() {     // -r^-1 mod 2^256 (Newton iteration from the 64-bit constant of the Montgomery product)
    static const U256 v = [] {
        const U256& p = fr_params().p;
        U256 y = {{(uint64_t)0 - fr_params().inv, 0, 0, 0}};          // r^-1 mod 2^64
        for (int it = 0; it < 2; ++it) {                               // y <- y (2 - r y): 64 -> 128 -> 256 bits
            U256 t = mul_lo256(p, y), two = {{2, 0, 0, 0}}, d;
            u256_sub(d, two, t);
            y = mul_lo256(y, d);
        }
        U256 zero = {{0, 0, 0, 0}}, n;
        u256_sub(n, zero, y);
        return n;
    }();
    return v;
}
ShoupPair shoup_pair(const Fr& w) { return ShoupPair{w.to_u256(), mul_lo256(w.m, fr_neg_inv256())}; }
}  // namespace

static void build_ntt_tables(zke_ctx* x, unsigned log_n) {
    const size_t N = (size_t)1 << log_n;
    // twiddles omega^k, omega^-k (k < N/2) and the bit-reversed coset scale g^j / N
    const Fr omega = fr_root_of_unity(log_n), omega_inv = omega.inv();
    const Fr g = fr_root_of_unity(log_n + 1);
    const Fr n_inv = Fr::from_u64(N).inv();
    // constants of the transforms: Montgomery form (32 bytes) or fixed-operand pairs (64 bytes) - ZKE_NTT_SHOUP
    bool shoup = false;
    if (const char* e = getenv("ZKE_NTT_SHOUP")) shoup = atoi(e) != 0;
    const size_t esz = shoup ? 64 : 32;
    std::vector<uint8_t> fw(esz * std::max<size_t>(1, N / 2)), iv(esz * std::max<size_t>(1, N / 2)), cs(esz * N);
    auto put = [&](std::vector<uint8_t>& tab, size_t i, const Fr& w) {
        if (shoup) { const ShoupPair sp = shoup_pair(w); memcpy(&tab[64 * i], sp.w.v, 32); memcpy(&tab[64 * i + 32], sp.wq.v, 32); }
        else memcpy(&tab[32 * i], w.m.v, 32);
    };
    const unsigned T = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; ++t) {
        th.emplace_back([&, t]() {
            size_t beg = (N / 2) * t / T, end = (N / 2) * (t + 1) / T;
            if (beg < end) {
                U256 e = {{(uint64_t)beg, 0, 0, 0}};
                Fr a = omega.pow(e), b = omega_inv.pow(e);
                for (size_t i = beg; i < end; ++i) { put(fw, i, a); put(iv, i, b); a = a * omega; b = b * omega_inv; }
            }
            beg = N * t / T; end = N * (t + 1) / T;
            if (beg < end) {
                U256 e = {{(uint64_t)beg, 0, 0, 0}};
                Fr a = g.pow(e) * n_inv;
                for (size_t j = beg; j < end; ++j) {
                    size_t p = 0;
                    for (unsigned bit = 0; bit < log_n; ++bit) if (j & ((size_t)1 << bit)) p |= (size_t)1 << (log_n - 1 - bit);
                    put(cs, p, a);
                    a = a * g;
                }
            }
        });
    }
    for (auto& t : th) t.join();
    if (N == 1) { put(fw, 0, Fr::one()); put(iv, 0, Fr::one()); }
    x->tw_fwd.upload(fw); x->tw_inv.upload(iv); x->coset_scale.upload(cs);
    x->ntt.tw_fwd = x->tw_fwd.p; x->ntt.tw_inv = x->tw_inv.p; x->ntt.log_n = (int)log_n; x->ntt.shoup = shoup;
}

// The proving lanes of a context with a key: streams, NTT vectors and MSM workspace each.
static void open_lanes(zke_ctx* x, size_t N, int prio_least, int prio_greatest) {
    const uint32_t max_batch = x->max_batch;
    x->cfg_w = dev::msm_config_witness();
    x->cfg_h = x->zkey->cfg_h;
    size_t ws = std::max(dev::MsmPlan<dev::Fq>::workspace_bytes(x->n_vars, x->cfg_w),
                         dev::MsmPlan<dev::Fq>::workspace_bytes((uint32_t)N, x->cfg_h));
    ws = std::max(ws, dev::MsmPlan<dev::Fq2>::workspace_bytes(x->n_vars, x->cfg_w));
    int want = 8;
    if (const char* e = getenv("ZKE_LANES")) want = atoi(e);
    if (const char* e = getenv("ZKE_SPLIT_STREAMS")) x->split_streams = atoi(e) != 0;
    if (const char* e = getenv("ZKE_FINISH_THREADS")) x->finish_threads = std::max(1, std::min(32, atoi(e)));
    want = std::max(1, std::min(ZKE_MAX_LANES, std::min<int>(want, (int)max_batch)));
    {   // lanes only buy overlap: open no more than fit in device memory beside the second witness slot (allocated by
        // the first zke_fullprove_submit) and 1 GiB for per-call buffers - at 2^24 eight lanes alone exceed 80 GB
        size_t free_b = 0, total_b = 0;
        CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
        const size_t lane_bytes = 4 * N * 32 + ws;
        const size_t keep = x->stride * 32 * max_batch + ((size_t)1 << 30);
        const size_t fit = free_b > keep ? (free_b - keep) / lane_bytes : 0;
        want = std::max(1, std::min<int>(want, (int)std::min<size_t>(fit, ZKE_MAX_LANES)));
    }
    // the lanes' light streams sit one priority step below the witness stream (when the device offers three levels)
    const int prio_light = prio_greatest < prio_least - 1 ? prio_greatest + 1 : prio_greatest;
    for (int i = 0; i < want; ++i) {
        zke_ctx::Lane& L = x->lanes[i];
        CUDA_OK(cudaStreamCreateWithPriority(&L.st, cudaStreamNonBlocking, prio_light));
        CUDA_OK(cudaStreamCreateWithPriority(&L.heavy, cudaStreamNonBlocking, prio_least));
        for (auto& e : L.ev) CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        L.va.alloc(N * 32); L.vb.alloc(N * 32); L.vc.alloc(N * 32); L.vd.alloc(N * 32);
        L.msm_ws.alloc(ws);
    }
    x->lanes_alloc = x->n_lanes = want;
}

static zke_ctx* do_open(const zke_circuit* zc, const zke_zkey* zk, int device, uint32_t max_batch) {
    select_device(device);
    const Circuit* cp = zc ? &zc->c : nullptr;
    if (!cp && !(zk && zk->has_coefs)) throw std::runtime_error("a context needs a circuit, or a proving key loaded from a .zkey");
    if (zk && cp && (zk->n_vars != cp->n_vars || zk->n_public != cp->n_public() || zk->log_n != cp->domain_log2()))
        throw std::runtime_error("zkey does not belong to this circuit");
    if (zk && zk->device != device) throw std::runtime_error("zkey lives on another device");
    if (max_batch == 0) throw std::runtime_error("max_batch must be positive");
    std::unique_ptr<zke_ctx> x(new zke_ctx());
    x->circuit = zc; x->zkey = zk; x->device = device; x->max_batch = max_batch;
    x->n_vars = cp ? cp->n_vars : zk->n_vars;
    x->n_public = cp ? cp->n_public() : zk->n_public;
    x->n_inputs = cp ? cp->n_inputs() : 0;
    int prio_least = 0, prio_greatest = 0;
    CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    CUDA_OK(cudaStreamCreateWithPriority(&x->stream, cudaStreamNonBlocking, prio_greatest));

    // coefficient words (lc_term.cuh) of the circuit's - or the key's - interned coefficient table
    const std::vector<U256>& coefs = cp ? cp->coefs : zk->coefs;
    x->coef_word = coef_words(coefs);
    {   // coefficient table scaled by R: as Montgomery numbers these are just the Montgomery forms
        std::vector<Fr> cr(std::max<size_t>(1, coefs.size()));
        for (size_t i = 0; i < coefs.size(); ++i) cr[i] = Fr::from_u256(coefs[i]);
        x->coef_r.upload(cr);
    }

    // a circuit read from an `.r1cs` and a key that carries its own coefficient matrices: they must be the same system
    if (zk && cp && cp->r1cs_only && zk->has_coefs) check_key_matrices(*cp, *zk);

    // witness program (none for a circuit read from an `.r1cs`: its witnesses are loaded)
    if (cp && !cp->r1cs_only) upload_program(x.get(), *cp);
    upload_r1cs(x.get(), cp, zk);
    x->stride = (size_t)x->n_vars + (cp ? cp->n_temps : 0);
    x->inputs.alloc((size_t)std::max(1u, x->n_inputs) * 32 * max_batch);
    x->check_flag.alloc(8);
    x->bad_host.resize(max_batch);
    alloc_slot(x.get(), x->slots[0]);

    if (zk) {
        build_ntt_tables(x.get(), zk->log_n);
        open_lanes(x.get(), (size_t)1 << zk->log_n, prio_least, prio_greatest);
    }
    CUDA_OK(cudaDeviceSynchronize());
    return x.release();
}

static std::string assert_message(const zke_ctx* x, uint32_t email, uint32_t row) {
    std::string scope = "?";
    if (x->circuit) {
        const Circuit& c = x->circuit->c;
        if (row < c.scope_of_constraint.size()) scope = c.scopes[c.scope_of_constraint[row]];
    }
    return "Assert Failed: constraint " + std::to_string(row) + " in template " + scope + " @ email " + std::to_string(email);
}

static void require_idle(const zke_ctx* x) {
    if (x->n_submitted != x->n_collected) throw std::runtime_error("a submitted batch is still in flight: call zke_fullprove_collect first");
}

// Runs the witness kernel of `batch` emails into slot S.  inputs: host memory, or NULL for the resident inputs.
static void do_witness(zke_ctx* x, zke_ctx::Slot& S, const uint8_t* inputs, size_t batch) {
    if (!x->circuit) throw std::runtime_error("this context was opened from a .zkey alone: it has no witness program (use zke_load_witness / zke_wtns_prove)");
    const Circuit& c = x->circuit->c;
    if (c.r1cs_only) throw std::runtime_error(R1CS_NO_PROGRAM);
    if (batch == 0 || batch > x->max_batch) throw std::runtime_error("batch exceeds the context's max_batch");
    CUDA_OK(cudaSetDevice(x->device));
    const uint8_t* in_dev = x->inputs.p;
    if (inputs) {
        if (c.n_inputs()) CUDA_OK(cudaMemcpyAsync(S.inputs.p, inputs, (size_t)c.n_inputs() * 32 * batch, cudaMemcpyHostToDevice, x->stream));
        in_dev = S.inputs.p;
    } else if (x->inputs_resident < batch) {
        throw std::runtime_error("inputs == NULL but no (or too few) inputs are resident: call zke_upload_inputs first");
    }
    size_t p0 = 0;
    if (x->profile) p0 = x->mark();
    if (const char* tp = getenv("ZKE_WITNESS_TRACE")) {   // diagnostics: per-iteration clock of CTA 0 -> file
        DevBuf tr;
        tr.alloc(8 * ((size_t)x->prog.n_iters + 1));
        dev::DevProgram P = x->prog;
        P.trace = (unsigned long long*)tr.p;
        dev::launch_witness(P, S.w_all.p, x->stride, in_dev, (uint32_t)batch, x->stream);
        CUDA_OK(cudaStreamSynchronize(x->stream));
        std::vector<unsigned long long> h(x->prog.n_iters);
        CUDA_OK(cudaMemcpy(h.data(), tr.p, 8 * h.size(), cudaMemcpyDeviceToHost));
        if (FILE* f = fopen(tp, "wb")) {
            fwrite(h.data(), 8, h.size(), f);
            fwrite(x->iter_info.data(), 4, x->iter_info.size(), f);
            fclose(f);
        }
    }
    dev::launch_witness(x->prog, S.w_all.p, x->stride, in_dev, (uint32_t)batch, x->stream);
    CHECK_LAUNCH();
    if (x->profile) x->spans.push_back({ZKE_STAGE_WITNESS, p0, x->mark()});
    S.loaded = (uint32_t)batch;
}

// constraint check only (no zkey needed): uses scratch a/b vectors sized to n_constraints
static int do_check(zke_ctx* x, zke_ctx::Slot& S, size_t batch, int32_t* status, std::string& msg) {
    CUDA_OK(cudaMemsetAsync(S.first_bad.p, 0xff, 4 * batch, x->stream));
    dev::launch_check_rows(x->r1cs, S.w_all.p, x->stride, (uint32_t)batch, (uint32_t*)S.first_bad.p, x->stream);   // one launch, no a / b vectors
    CHECK_LAUNCH();
    CUDA_OK(cudaMemcpyAsync(x->bad_host.data(), S.first_bad.p, 4 * batch, cudaMemcpyDeviceToHost, x->stream));
    CUDA_OK(cudaStreamSynchronize(x->stream));
    if (x->profile) x->collect();
    int bad = 0;
    for (size_t e = 0; e < batch; ++e) {
        int32_t s = x->bad_host[e] == 0xffffffffu ? -1 : (int32_t)x->bad_host[e];
        if (status) status[e] = s;
        if (s >= 0) { if (!bad) msg = assert_message(x, (uint32_t)e, (uint32_t)s); ++bad; }
    }
    return bad;
}

// Serial tail of one MSM on the host: sum of the unit-scalar partials + Horner over the window sums.
template <class F>
static AffineH<F> finish_msm(const uint8_t* block, const dev::MsmConfig& cfg) {
    const XyzzH<F>* slots = reinterpret_cast<const XyzzH<F>*>(block);
    const int n_windows = cfg.precomputed ? 1 : (255 + cfg.c - 1) / cfg.c;   // precomputed tables: one bucket set, no Horner
    XyzzH<F> acc = XyzzH<F>::inf();
    for (int j = n_windows - 1; j >= 0; --j) {
        if (!acc.is_inf()) for (int k = 0; k < cfg.c; ++k) acc.dbl();
        acc.add(slots[dev::MSM_ONES_SLOTS + j]);
    }
    if (cfg.classify) for (int i = 0; i < dev::MSM_ONES_SLOTS; ++i) acc.add(slots[i]);
    return acc.to_affine();
}

// Enqueues the witness multi-exponentiations A, B1, C and B2 over the wires [lo, hi) on `st`, in that order, into their
// blocks of `res`; `queued(stage)` runs after each one is queued.
template <class Queued>
static void enqueue_witness_msms(const zke_ctx* x, const uint8_t* w, uint32_t lo, uint32_t hi, uint8_t* ws, uint8_t* res,
                                 cudaStream_t st, Queued queued) {
    const zke_zkey* zk = x->zkey;
    w += 32ull * lo;
    dev::MsmPlan<dev::Fq>::run(zk->A.p + 64ull * lo, w, hi - lo, x->cfg_w, ws, res + RES_A * ZKE_RES_G1_BLOCK, st);
    queued(ZKE_STAGE_MSM_A);
    dev::MsmPlan<dev::Fq>::run(zk->B1.p + 64ull * lo, w, hi - lo, x->cfg_w, ws, res + RES_B1 * ZKE_RES_G1_BLOCK, st);
    queued(ZKE_STAGE_MSM_B1);
    dev::MsmPlan<dev::Fq>::run(zk->C.p + 64ull * lo, w, hi - lo, x->cfg_w, ws, res + RES_C * ZKE_RES_G1_BLOCK, st);
    queued(ZKE_STAGE_MSM_C);
    dev::MsmPlan<dev::Fq2>::run(zk->B2.p + 128ull * lo, w, hi - lo, x->cfg_w, ws, res + RES_B2 * ZKE_RES_G1_BLOCK, st);
    CHECK_LAUNCH();
    queued(ZKE_STAGE_MSM_B2);
}

struct MsmSums { G1AffineH a, b1, c, h; G2AffineH b2; };

// The host tail of the five multi-exponentiations of a result buffer copied back from the device
static MsmSums finish_msms(const uint8_t* res, const dev::MsmConfig& cfg_w, const dev::MsmConfig& cfg_h) {
    return MsmSums{finish_msm<Fq>(res + RES_A * ZKE_RES_G1_BLOCK, cfg_w), finish_msm<Fq>(res + RES_B1 * ZKE_RES_G1_BLOCK, cfg_w),
                   finish_msm<Fq>(res + RES_C * ZKE_RES_G1_BLOCK, cfg_w), finish_msm<Fq>(res + RES_H * ZKE_RES_G1_BLOCK, cfg_h),
                   finish_msm<Fq2>(res + RES_B2 * ZKE_RES_G1_BLOCK, cfg_w)};
}

// The proving key's fixed points that the assembly of a proof adds
struct KeyPoints { G1AffineH alpha1, beta1, delta1; G2AffineH beta2, delta2; };

// Writes the 256-byte proof pi_A, pi_B, pi_C:  pi_A = alpha1 + A + r delta1 ; pi_B = beta2 + B2 + s delta2 ;
// pi_C = C + H + s pi_A + r pi_B1 - r s delta1 with pi_B1 = beta1 + B1 + s delta1
static void assemble_proof(const KeyPoints& kp, const G1JacH& a, const G1JacH& b1, const G1JacH& c, const G1JacH& h, const G2JacH& b2,
                           const U256& r, const U256& s, uint8_t out[256]) {
    const G1JacH delta1 = G1JacH::from_affine(kp.delta1);
    const G1JacH pa = G1JacH::from_affine(kp.alpha1).add(a).add(delta1.mul(r));
    const G2JacH pb2 = G2JacH::from_affine(kp.beta2).add(b2).add(G2JacH::from_affine(kp.delta2).mul(s));
    const G1JacH pb1 = G1JacH::from_affine(kp.beta1).add(b1).add(delta1.mul(s));
    const U256 rs_prod = (Fr::from_u256(r) * Fr::from_u256(s)).to_u256();
    const G1JacH pc = c.add(h).add(pa.mul(s)).add(pb1.mul(r)).add(delta1.mul(rs_prod).neg());
    store_g1(out, pa.to_affine());
    store_g2(out + 64, pb2.to_affine());
    store_g1(out + 192, pc.to_affine());
}

static void sync_lanes(zke_ctx* x) {
    cudaStreamSynchronize(x->stream);
    for (int i = 0; i < x->lanes_alloc; ++i) { cudaStreamSynchronize(x->lanes[i].st); cudaStreamSynchronize(x->lanes[i].heavy); }
}

// Enqueues every proving kernel of the `batch` witnesses resident in slot S (no host synchronisation).
static void enqueue_prove(zke_ctx* x, zke_ctx::Slot& S, size_t batch, const uint8_t* rs) {
    const zke_zkey* zk = x->zkey;
    if (!zk) throw std::runtime_error("context was opened without a proving key");
    if (batch == 0 || batch > S.loaded) throw std::runtime_error("no witness loaded for this batch (call zke_witness first)");
    if (rs) {   // validated before any GPU work is queued
        for (size_t e = 0; e < 2 * batch; ++e) {
            U256 v;
            memcpy(v.v, rs + 32 * e, 32);
            if (u256_cmp(v, fr_params().p) >= 0) throw std::runtime_error("r / s not reduced mod the group order");
        }
        S.rs.assign(rs, rs + 64 * batch);
    } else {
        S.rs.clear();
    }
    CUDA_OK(cudaSetDevice(x->device));
    const uint32_t N = 1u << zk->log_n, m = x->n_vars, l = x->n_public;
    const bool prof = x->profile;
    const int n_lanes = prof ? 1 : x->n_lanes;     // stage timing is only meaningful without overlap
    if (const char* e = getenv("ZKE_SPLIT_STREAMS")) x->split_streams = atoi(e) != 0;
    // the witnesses were produced on the main stream; the lanes start after it (and after the public signals copy)
    if (l) CUDA_OK(cudaMemcpy2DAsync(S.publics_host, (size_t)l * 32, S.w_all.p + 32, x->stride * 32, (size_t)l * 32, batch, cudaMemcpyDeviceToHost, x->stream));
    CUDA_OK(cudaEventRecord(S.witness_done, x->stream));
    for (int i = 0; i < n_lanes; ++i) CUDA_OK(cudaStreamWaitEvent(x->lanes[i].st, S.witness_done, 0));
    for (size_t e = 0; e < batch; ++e) {
        zke_ctx::Lane& L = x->lanes[e % n_lanes];
        cudaStream_t st = L.st;
        const uint8_t* w = S.w_all.p + 32 * x->stride * e;
        uint8_t* res = S.results.p + (size_t)ZKE_RESULT_STRIDE * e;
        uint32_t* flag = (uint32_t*)(res + ZKE_RES_FLAG_OFF);
        size_t t0 = 0, t1 = 0;
        CUDA_OK(cudaMemsetAsync(flag, 0xff, 4, st));
        if (prof) t0 = x->mark(st);
        auto span = [&](int stage) { if (prof) { t1 = x->mark(st); x->spans.push_back({stage, t0, t1}); t0 = t1; } };
        // `hv` = the lane's low-priority stream for the saturating kernels (profiling: everything on `st`)
        cudaStream_t hv = (prof || !x->split_streams) ? st : L.heavy;
        dev::launch_build_ab(x->r1cs, w, L.va.p, L.vb.p, L.vc.p, N, flag, st);
        span(ZKE_STAGE_MATVEC);
        if (hv != st) { CUDA_OK(cudaEventRecord(L.ev[0], st)); CUDA_OK(cudaStreamWaitEvent(hv, L.ev[0], 0)); }
        dev::launch_intt_dif(L.va.p, x->ntt, x->coset_scale.p, hv);
        dev::launch_intt_dif(L.vb.p, x->ntt, x->coset_scale.p, hv);
        dev::launch_intt_dif(L.vc.p, x->ntt, x->coset_scale.p, hv);
        dev::launch_ntt_dit(L.va.p, x->ntt, hv);
        dev::launch_ntt_dit(L.vb.p, x->ntt, hv);
        dev::launch_ntt_dit(L.vc.p, x->ntt, hv);
        dev::launch_quotient(L.va.p, L.vb.p, L.vc.p, L.vd.p, N, hv);
        CHECK_LAUNCH();
        if (hv != st) CUDA_OK(cudaEventRecord(L.ev[1], hv));
        span(ZKE_STAGE_NTT);
        // the witness MSMs do not depend on the transforms: with split streams they run on `st` while the lane's NTT
        // passes are still in flight on `hv` (the MSM workspace is only touched from `st`-ordered work)
        enqueue_witness_msms(x, w, 0, m, L.msm_ws.p, res, st, span);
        if (hv != st) CUDA_OK(cudaStreamWaitEvent(st, L.ev[1], 0));
        const dev::MsmPlan<dev::Fq>::Heavy heavy{hv, L.ev[2], L.ev[3]};
        size_t i0 = 0, i1 = 0;
        cudaEvent_t evs[2] = {prof ? x->ev(&i0) : nullptr, prof ? x->ev(&i1) : nullptr};   // profiling: the bucket kernel alone
        dev::MsmPlan<dev::Fq>::run(zk->H.p, L.vd.p, N, x->cfg_h, L.msm_ws.p, res + RES_H * ZKE_RES_G1_BLOCK, st, prof ? evs : nullptr, &heavy);
        if (prof) x->spans.push_back({ZKE_STAGE_MSM_H_BUCKETS, i0, i1});
        span(ZKE_STAGE_MSM_H);
        CHECK_LAUNCH();
        CUDA_OK(cudaMemcpyAsync(S.results_host + (size_t)ZKE_RESULT_STRIDE * e, res, ZKE_RESULT_STRIDE, cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaEventRecord(S.done[e], st));
        // the lane's next email reuses va..vd on `hv`; its first kernels run on `st` (after this point) and `hv`
        // only starts after an event recorded on `st`, so the order is already enforced
    }
    S.batch = (uint32_t)batch;
}

// Host tail of a batch enqueued by enqueue_prove: waits per email, finishes the MSMs, assembles pi_A, pi_B, pi_C.
// `finish_threads` host threads share the emails (3 ms of big-integer work each), overlapped with the GPU work of the
// later emails and of the next submitted batch.
static int finish_prove(zke_ctx* x, zke_ctx::Slot& S, uint8_t* proofs_out, uint8_t* publics_out, int32_t* status, std::string& msg) {
    const zke_zkey* zk = x->zkey;
    const size_t batch = S.batch;
    const uint32_t l = x->n_public;
    const KeyPoints kp{zk->alpha1, zk->beta1, zk->delta1, zk->beta2, zk->delta2};
    std::vector<int32_t> st_local(batch, -1);
    std::string first_error;
    std::mutex err_mutex;
    auto one = [&](size_t e) {
        CUDA_OK(cudaEventSynchronize(S.done[e]));
        const uint8_t* res = S.results_host + (size_t)ZKE_RESULT_STRIDE * e;
        uint32_t flag;
        memcpy(&flag, res + ZKE_RES_FLAG_OFF, 4);
        const int32_t s = flag == 0xffffffffu ? -1 : (int32_t)flag;
        st_local[e] = s;
        uint8_t* out = proofs_out + 256 * e;
        if (s >= 0) { memset(out, 0, 256); return; }
        U256 r, sc;
        if (!S.rs.empty()) { memcpy(r.v, S.rs.data() + 64 * e, 32); memcpy(sc.v, S.rs.data() + 64 * e + 32, 32); }
        else { random_scalar(r); random_scalar(sc); }
        const MsmSums m = finish_msms(res, x->cfg_w, x->cfg_h);
        assemble_proof(kp, G1JacH::from_affine(m.a), G1JacH::from_affine(m.b1), G1JacH::from_affine(m.c), G1JacH::from_affine(m.h),
                       G2JacH::from_affine(m.b2), r, sc, out);
    };
    const int T = (int)std::max<size_t>(1, std::min<size_t>((size_t)x->finish_threads, batch));
    std::atomic<size_t> next{0};
    auto worker = [&]() {
        try {
            cudaSetDevice(x->device);
            for (;;) {
                const size_t e = next.fetch_add(1);
                if (e >= batch) break;
                one(e);
            }
        } catch (const std::exception& ex) {
            std::lock_guard<std::mutex> lock(err_mutex);
            if (first_error.empty()) first_error = ex.what();
        }
    };
    if (T == 1) worker();
    else {
        std::vector<std::thread> th;
        for (int t = 0; t < T; ++t) th.emplace_back(worker);
        for (auto& t : th) t.join();
    }
    // everything of this batch has completed (each email's `done` event closes its lane work; the publics copy
    // precedes the lanes on the witness stream)
    if (x->profile) { sync_lanes(x); x->collect(); }
    if (!first_error.empty()) { sync_lanes(x); throw std::runtime_error(first_error); }
    int bad = 0;
    for (size_t e = 0; e < batch; ++e) {
        if (status) status[e] = st_local[e];
        if (st_local[e] >= 0) { if (!bad) msg = assert_message(x, (uint32_t)e, (uint32_t)st_local[e]); ++bad; }
    }
    if (publics_out && l) memcpy(publics_out, S.publics_host, (size_t)l * 32 * batch);
    return bad;
}

static int do_prove(zke_ctx* x, zke_ctx::Slot& S, size_t batch, const uint8_t* rs, uint8_t* proofs_out, uint8_t* publics_out, int32_t* status, std::string& msg) {
    try {
        enqueue_prove(x, S, batch, rs);
    } catch (...) {
        sync_lanes(x);      // nothing of a half-queued batch may keep writing into the result buffers
        throw;
    }
    return finish_prove(x, S, proofs_out, publics_out, status, msg);
}

// iden3 `.wtns` v2: section 1 {u32 n8, q[n8], u32 nWitness}, section 2 nWitness x n8 bytes (standard form)
static const uint8_t* parse_wtns(const uint8_t* b, size_t len, uint32_t expect_vars) {
    if (!b || len < 12 || memcmp(b, "wtns", 4) != 0) throw std::runtime_error("not a .wtns file (bad magic)");
    std::vector<BinSection> secs;
    try { secs = binfile_sections(b, len, ".wtns"); }
    catch (const std::runtime_error&) { throw std::runtime_error("truncated .wtns"); }   // without the section detail
    const uint8_t *s1 = nullptr, *s2 = nullptr;
    size_t n1 = 0, n2 = 0;
    for (const BinSection& s : secs) {
        if (s.type == 1) { s1 = s.view.p; n1 = s.view.n; }
        if (s.type == 2) { s2 = s.view.p; n2 = s.view.n; }
    }
    if (!s1 || !s2 || n1 < 40) throw std::runtime_error(".wtns sections missing");
    if (rd32(s1) != 32 || memcmp(s1 + 4, fr_params().p.v, 32) != 0) throw std::runtime_error(".wtns is not over the BN254 scalar field");
    const uint32_t n = rd32(s1 + 36);
    if (n != expect_vars) throw std::runtime_error(".wtns has " + std::to_string(n) + " values, the key expects " + std::to_string(expect_vars));
    if (n2 != (size_t)n * 32) throw std::runtime_error(".wtns data section has the wrong size");
    return s2;
}

static void load_witness(zke_ctx* x, zke_ctx::Slot& S, const uint8_t* wtns, size_t batch) {
    if (batch == 0 || batch > x->max_batch) throw std::runtime_error("batch exceeds the context's max_batch");
    CUDA_OK(cudaSetDevice(x->device));
    const size_t m = x->n_vars;
    CUDA_OK(cudaMemcpy2DAsync(S.w_all.p, x->stride * 32, wtns, m * 32, m * 32, batch, cudaMemcpyHostToDevice, x->stream));
    // externally computed witnesses are validated: every value canonical (< r) and w[0] == 1
    CUDA_OK(cudaMemsetAsync(x->check_flag.p, 0, 8, x->stream));
    dev::launch_check_witness(S.w_all.p, x->stride, (uint32_t)m, (uint32_t)batch, (uint32_t*)x->check_flag.p, x->stream);
    CHECK_LAUNCH();
    uint32_t flags[2] = {0, 0};
    CUDA_OK(cudaMemcpyAsync(flags, x->check_flag.p, 8, cudaMemcpyDeviceToHost, x->stream));
    CUDA_OK(cudaStreamSynchronize(x->stream));
    S.loaded = 0;
    if (flags[0]) throw std::runtime_error("witness value not reduced mod r");
    if (flags[1]) throw std::runtime_error("witness[0] must be 1");
    S.loaded = (uint32_t)batch;
}

// ------------------------------------------------------------------------------------------------ sharded proving
// One proof across G = 2, 4 or 8 GPUs (SURVEY 8(e)(ii), BASELINE configs[3]/[4]).  Every GPU holds the key and the
// witness; the work of the proof is partitioned:
//   * the quotient: the N-point transforms are split 4-step style.  The vectors live at their global positions; a GPU
//     works either on its ROW block (positions [rank * M, (rank + 1) * M), M = N / G) or on its COLUMN range (columns
//     [rank * M / G, (rank + 1) * M / G) of every block).  begin: mat-vec for the rows of the column range + the top
//     log2 G inverse stages (cross-block, in registers).  [exchange columns -> rows, done by the caller with NCCL
//     all-to-all on the device pointers of zke_shard_vector]  mid: the block-local inverse stages, coset scale and
//     block-local forward stages.  [exchange rows -> columns]  end: the top forward stages and a o b - c on the column
//     range: this GPU's share of the H scalars (zero elsewhere);
//   * the multi-exponentiations: A, B1, C, B2 over the contiguous point range [rank m / G, (rank + 1) m / G), H over the
//     column range; each GPU finishes its partial sums to five affine points (ZKE_SHARD_PARTIAL_BYTES);
//   * combine (host): the partial points of all GPUs (an all-gather of 388 bytes per GPU) are added and the proof is
//     assembled - the group law makes the result bit-identical to the single-GPU proof.
static void shard_geometry(const zke_ctx* x, int& log_m, int& log_cols, uint32_t& col0) {
    log_m = (int)x->zkey->log_n - x->shard_log_g;
    log_cols = log_m - x->shard_log_g;
    col0 = (uint32_t)x->shard_rank << log_cols;
}

static void shard_begin(zke_ctx* x, int rank, int world) {
    const zke_zkey* zk = x->zkey;
    if (!zk) throw std::runtime_error("context was opened without a proving key");
    require_idle(x);
    int log_g = 0;
    while ((1 << log_g) < world) ++log_g;
    if (world < 2 || world > 8 || (1 << log_g) != world) throw std::runtime_error("sharded proving supports 2, 4 or 8 GPUs");
    if (rank < 0 || rank >= world) throw std::runtime_error("bad shard rank");
    if ((int)zk->log_n < 2 * log_g + 10) throw std::runtime_error("domain too small to shard (use batch parallelism)");
    zke_ctx::Slot& S = x->slots[0];
    if (S.loaded < 1) throw std::runtime_error("no witness loaded (call zke_witness / zke_load_witness on every rank first)");
    CUDA_OK(cudaSetDevice(x->device));
    x->shard_rank = rank; x->shard_world = world; x->shard_log_g = log_g;
    int log_m, log_cols; uint32_t col0;
    shard_geometry(x, log_m, log_cols, col0);
    zke_ctx::Lane& L = x->lanes[0];
    cudaStream_t st = L.st;
    CUDA_OK(cudaStreamSynchronize(x->stream));
    uint32_t* flag = (uint32_t*)(S.results.p + ZKE_RES_FLAG_OFF);
    CUDA_OK(cudaMemsetAsync(flag, 0xff, 4, st));
    dev::RowMap map;
    map.log_cols = log_cols; map.log_m = log_m; map.col0 = col0;
    const uint32_t n_rows = (uint32_t)world << log_cols;
    dev::launch_build_ab(x->r1cs, S.w_all.p, L.va.p, L.vb.p, L.vc.p, n_rows, flag, st, &map);
    const uint32_t n_cols = 1u << log_cols;
    dev::launch_intt_cross(L.va.p, x->ntt, log_g, col0, n_cols, st);
    dev::launch_intt_cross(L.vb.p, x->ntt, log_g, col0, n_cols, st);
    dev::launch_intt_cross(L.vc.p, x->ntt, log_g, col0, n_cols, st);
    CHECK_LAUNCH();
    CUDA_OK(cudaStreamSynchronize(st));
    x->shard_stage = 1;
}

static void shard_mid(zke_ctx* x) {
    if (x->shard_stage != 1) throw std::runtime_error("zke_shard_mid out of order");
    CUDA_OK(cudaSetDevice(x->device));
    int log_m, log_cols; uint32_t col0;
    shard_geometry(x, log_m, log_cols, col0);
    zke_ctx::Lane& L = x->lanes[0];
    cudaStream_t st = L.st;
    const size_t block_off = ((size_t)x->shard_rank << log_m);
    for (uint8_t* v : {L.va.p, L.vb.p, L.vc.p}) {
        dev::launch_intt_dif_block(v + 32 * block_off, x->ntt, log_m, x->coset_scale.p + (x->ntt.shoup ? 64 : 32) * block_off, st);
        dev::launch_ntt_dit_block(v + 32 * block_off, x->ntt, log_m, st);
    }
    CHECK_LAUNCH();
    CUDA_OK(cudaStreamSynchronize(st));
    x->shard_stage = 2;
}

// A GPU's share of a proof (ZKE_SHARD_PARTIAL_BYTES): A, B1, C, H, B2 in the host point format, then the first violated
// row of its rows (u32).  The reader refuses unreduced coordinates and points off their curves (no subgroup check).
static const char PARTIAL_COORD[] = "partial point coordinate";
static void write_partial(const MsmSums& m, uint32_t first_bad, uint8_t* out) {
    store_g1(out, m.a); store_g1(out + 64, m.b1); store_g1(out + 128, m.c); store_g1(out + 192, m.h); store_g2(out + 256, m.b2);
    memcpy(out + 384, &first_bad, 4);
}
static MsmSums read_partial(const uint8_t* p, uint32_t& first_bad) {
    const MsmSums m{load_g1(p, PARTIAL_COORD), load_g1(p + 64, PARTIAL_COORD), load_g1(p + 128, PARTIAL_COORD),
                    load_g1(p + 192, PARTIAL_COORD), load_g2(p + 256, PARTIAL_COORD)};
    if (!g1_on_curve(m.a) || !g1_on_curve(m.b1) || !g1_on_curve(m.c) || !g1_on_curve(m.h) || !g2_on_curve(m.b2)) throw std::runtime_error("partial point not on the curve");
    memcpy(&first_bad, p + 384, 4);
    return m;
}

static void shard_end(zke_ctx* x, uint8_t* partial_out, uint8_t* publics_out) {
    if (x->shard_stage != 2) throw std::runtime_error("zke_shard_end out of order");
    const zke_zkey* zk = x->zkey;
    CUDA_OK(cudaSetDevice(x->device));
    int log_m, log_cols; uint32_t col0;
    shard_geometry(x, log_m, log_cols, col0);
    zke_ctx::Slot& S = x->slots[0];
    zke_ctx::Lane& L = x->lanes[0];
    cudaStream_t st = L.st;
    const uint32_t N = 1u << zk->log_n, m = x->n_vars, l = x->n_public;
    const int G = x->shard_world, log_g = x->shard_log_g;
    const uint32_t n_cols = 1u << log_cols;
    dev::launch_ntt_cross(L.va.p, x->ntt, log_g, col0, n_cols, st);
    dev::launch_ntt_cross(L.vb.p, x->ntt, log_g, col0, n_cols, st);
    dev::launch_ntt_cross(L.vc.p, x->ntt, log_g, col0, n_cols, st);
    CUDA_OK(cudaMemsetAsync(L.vd.p, 0, (size_t)N * 32, st));
    dev::launch_quotient_cols(L.va.p, L.vb.p, L.vc.p, L.vd.p, (int)zk->log_n, log_g, col0, (uint32_t)log_cols, st);
    CHECK_LAUNCH();
    // witness multi-exponentiations over this GPU's point range, H over its columns (all other scalars are zero)
    const uint32_t lo = (uint32_t)((uint64_t)m * x->shard_rank / G), hi = (uint32_t)((uint64_t)m * (x->shard_rank + 1) / G);
    uint8_t* res = S.results.p;
    enqueue_witness_msms(x, S.w_all.p, lo, hi, L.msm_ws.p, res, st, [](int) {});
    dev::MsmPlan<dev::Fq>::run(zk->H.p, L.vd.p, N, x->cfg_h, L.msm_ws.p, res + RES_H * ZKE_RES_G1_BLOCK, st);
    CHECK_LAUNCH();
    CUDA_OK(cudaMemcpyAsync(S.results_host, res, ZKE_RESULT_STRIDE, cudaMemcpyDeviceToHost, st));
    if (l) CUDA_OK(cudaMemcpyAsync(S.publics_host, S.w_all.p + 32, (size_t)l * 32, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    uint32_t first_bad;     // first violated row among this GPU's rows (0xffffffff: none)
    memcpy(&first_bad, S.results_host + ZKE_RES_FLAG_OFF, 4);
    write_partial(finish_msms(S.results_host, x->cfg_w, x->cfg_h), first_bad, partial_out);
    if (publics_out && l) memcpy(publics_out, S.publics_host, (size_t)l * 32);
    x->shard_stage = 0;
}

// host only: sums the partial points of all GPUs and assembles the proof
static int shard_combine(const KeyPoints& kp, const uint8_t* partials, int world, const uint8_t* rs, uint8_t* out, int32_t* status) {
    G1JacH sa = G1JacH::inf(), sb1 = G1JacH::inf(), sc = G1JacH::inf(), sh = G1JacH::inf();
    G2JacH sb2 = G2JacH::inf();
    uint32_t first_bad = 0xffffffffu;
    for (int r = 0; r < world; ++r) {
        uint32_t f;
        const MsmSums m = read_partial(partials + (size_t)ZKE_SHARD_PARTIAL_BYTES * r, f);
        sa = sa.add_affine(m.a); sb1 = sb1.add_affine(m.b1); sc = sc.add_affine(m.c); sh = sh.add_affine(m.h); sb2 = sb2.add_affine(m.b2);
        first_bad = std::min(first_bad, f);
    }
    if (status) *status = first_bad == 0xffffffffu ? -1 : (int32_t)first_bad;
    if (first_bad != 0xffffffffu) { memset(out, 0, 256); return 1; }
    U256 r, s;
    if (rs) { memcpy(r.v, rs, 32); memcpy(s.v, rs + 32, 32); }
    else { random_scalar(r); random_scalar(s); }
    if (u256_cmp(r, fr_params().p) >= 0 || u256_cmp(s, fr_params().p) >= 0) throw std::runtime_error("r / s not reduced mod the group order");
    assemble_proof(kp, sa, sb1, sc, sh, sb2, r, s, out);
    return 0;
}

// ------------------------------------------------------------------------------------------------ C ABI
extern "C" {

int zke_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

zke_zkey* zke_setup(const zke_circuit* c, uint64_t seed, int device, char* err, size_t errcap) {
    try { if (!c) throw std::runtime_error("null circuit"); return do_setup(c, seed, device); }
    catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}
zke_zkey* zke_zkey_load(const void* zkey_bytes, size_t len, int device, char* err, size_t errcap) {
    try {
        SecView sec[11];
        split_container((const uint8_t*)zkey_bytes, len, sec);
        return do_zkey_load(sec, device);
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}
zke_zkey* zke_zkey_load_chunks(const void* const* chunks, const size_t* lens, size_t n_chunks, int device, char* err, size_t errcap) {
    try {
        if (!chunks || !lens || n_chunks < 9) throw std::runtime_error("expected the chunk files b..j (sections 1-9; k is optional)");
        SecView sec[11];
        for (size_t i = 0; i < n_chunks && i < 10; ++i) sec[i + 1] = SecView{(const uint8_t*)chunks[i], lens[i]};
        return do_zkey_load(sec, device);
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}
int64_t zke_zkey_write(const zke_zkey* z, const zke_circuit* c, uint8_t* out, size_t cap) {
    try { if (!z) return -1; return do_zkey_write(z, c, out, cap); }
    catch (const std::exception&) { return -3; }
}
int zke_zkey_is_toy(const zke_zkey* z) { return z ? (z->toy ? 1 : 0) : -1; }
void zke_zkey_free(zke_zkey* z) { if (z) { cudaSetDevice(z->device); delete z; } }

int zke_zkey_info(const zke_zkey* z, uint32_t* n_vars, uint32_t* n_public, uint32_t* domain_log2) {
    if (!z) return -1;
    if (n_vars) *n_vars = z->n_vars;
    if (n_public) *n_public = z->n_public;
    if (domain_log2) *domain_log2 = z->log_n;
    return 0;
}

// Copies one section of the proving key to the host as affine points with standard-form little-endian
// coordinates (G1: x, y = 64 bytes; G2: x.c0, x.c1, y.c0, y.c1 = 128 bytes); infinity = all zero.
int64_t zke_zkey_section(const zke_zkey* z, int section, uint8_t* out, size_t cap) {
    if (!z) return -1;
    try {
        CUDA_OK(cudaSetDevice(z->device));
        const size_t N = (size_t)1 << z->log_n;
        auto g1_host = [&](const G1AffineH* pts, size_t n) -> int64_t {
            if (!out) return (int64_t)n;
            if (cap < n * 64) return -2;
            for (size_t i = 0; i < n; ++i) store_g1(out + 64 * i, pts[i]);
            return (int64_t)n;
        };
        auto g1_dev = [&](const DevBuf& b, size_t n) -> int64_t {
            if (!out) return (int64_t)n;
            std::vector<G1AffineH> h(n);
            CUDA_OK(cudaMemcpy(h.data(), b.p, n * sizeof(G1AffineH), cudaMemcpyDeviceToHost));
            return g1_host(h.data(), n);
        };
        auto g2_host = [&](const G2AffineH* pts, size_t n) -> int64_t {
            if (!out) return (int64_t)n;
            if (cap < n * 128) return -2;
            for (size_t i = 0; i < n; ++i) store_g2(out + 128 * i, pts[i]);
            return (int64_t)n;
        };
        switch (section) {
            case ZKE_SEC_ALPHA1: return g1_host(&z->alpha1, 1);
            case ZKE_SEC_BETA1: return g1_host(&z->beta1, 1);
            case ZKE_SEC_DELTA1: return g1_host(&z->delta1, 1);
            case ZKE_SEC_BETA2: return g2_host(&z->beta2, 1);
            case ZKE_SEC_GAMMA2: return g2_host(&z->gamma2, 1);
            case ZKE_SEC_DELTA2: return g2_host(&z->delta2, 1);
            case ZKE_SEC_IC: return g1_host(z->ic.data(), z->ic.size());
            case ZKE_SEC_A: return g1_dev(z->A, z->n_vars);
            case ZKE_SEC_B1: return g1_dev(z->B1, z->n_vars);
            case ZKE_SEC_C: return g1_dev(z->C, z->n_vars);
            case ZKE_SEC_H: return g1_dev(z->H, N);
            case ZKE_SEC_B2: {
                if (!out) return z->n_vars;
                std::vector<G2AffineH> h(z->n_vars);
                CUDA_OK(cudaMemcpy(h.data(), z->B2.p, h.size() * sizeof(G2AffineH), cudaMemcpyDeviceToHost));
                return g2_host(h.data(), h.size());
            }
            default: return -1;
        }
    } catch (const std::exception&) { return -3; }
}

zke_ctx* zke_ctx_open(const zke_circuit* c, const zke_zkey* zkey, int device, uint32_t max_batch, char* err, size_t errcap) {
    try { return do_open(c, zkey, device, max_batch); }
    catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}
void zke_ctx_close(zke_ctx* x) {
    if (!x) return;
    cudaSetDevice(x->device);
    sync_lanes(x);
    for (auto e : x->ev_pool) cudaEventDestroy(e);
    for (auto& S : x->slots) {
        for (auto e : S.done) cudaEventDestroy(e);
        if (S.witness_done) cudaEventDestroy(S.witness_done);
        if (S.results_host) cudaFreeHost(S.results_host);
        if (S.publics_host) cudaFreeHost(S.publics_host);
    }
    for (int i = 0; i < x->lanes_alloc; ++i) {
        if (x->lanes[i].st) cudaStreamDestroy(x->lanes[i].st);
        if (x->lanes[i].heavy) cudaStreamDestroy(x->lanes[i].heavy);
        for (auto e : x->lanes[i].ev) if (e) cudaEventDestroy(e);
    }
    if (x->stream) cudaStreamDestroy(x->stream);
    delete x;
}

int zke_upload_inputs(zke_ctx* x, const uint8_t* inputs, size_t batch, char* err, size_t errcap) {
    try {
        if (!x || !inputs) throw std::runtime_error("null argument");
        if (x->circuit && x->circuit->c.r1cs_only) throw std::runtime_error(R1CS_NO_PROGRAM);
        if (batch == 0 || batch > x->max_batch) throw std::runtime_error("batch exceeds the context's max_batch");
        require_idle(x);
        CUDA_OK(cudaSetDevice(x->device));
        const size_t n = x->n_inputs;
        if (n) CUDA_OK(cudaMemcpy(x->inputs.p, inputs, n * 32 * batch, cudaMemcpyHostToDevice));
        x->inputs_resident = (uint32_t)batch;
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_ctx_set_lanes(zke_ctx* x, int n) {
    if (!x || n < 1) return -1;
    x->n_lanes = n > x->lanes_alloc ? x->lanes_alloc : n;
    return x->n_lanes;
}
int zke_ctx_profile(zke_ctx* x, int enable) {
    if (!x) return -1;
    x->profile = enable != 0;
    for (int i = 0; i < ZKE_N_STAGES; ++i) { x->stage_ms[i] = 0; x->stage_count[i] = 0; }
    return 0;
}
int zke_ctx_profile_get(const zke_ctx* x, double* ms_out, uint64_t* count_out) {
    if (!x) return -1;
    for (int i = 0; i < ZKE_N_STAGES; ++i) { if (ms_out) ms_out[i] = x->stage_ms[i]; if (count_out) count_out[i] = x->stage_count[i]; }
    return ZKE_N_STAGES;
}
void* zke_ctx_stream(const zke_ctx* x) { return x ? (void*)x->stream : nullptr; }
uint64_t zke_kernel_launches(void) { return dev::g_kernel_launches; }

int zke_witness(zke_ctx* x, const uint8_t* inputs, size_t batch, uint8_t* wtns_out, int32_t* status, char* err, size_t errcap) {
    try {
        if (!x) throw std::runtime_error("null context");
        require_idle(x);
        zke_ctx::Slot& S = x->slots[0];
        do_witness(x, S, inputs, batch);
        std::string msg;
        int bad = do_check(x, S, batch, status, msg);
        if (wtns_out) {
            const size_t m = x->n_vars;
            CUDA_OK(cudaMemcpy2D(wtns_out, m * 32, S.w_all.p, x->stride * 32, m * 32, batch, cudaMemcpyDeviceToHost));
        }
        if (bad) { set_err(err, errcap, msg); return bad; }
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_load_witness(zke_ctx* x, const uint8_t* wtns, size_t batch, char* err, size_t errcap) {
    try {
        if (!x || !wtns) throw std::runtime_error("null argument");
        require_idle(x);
        load_witness(x, x->slots[0], wtns, batch);
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_check_witness(zke_ctx* x, size_t batch, int32_t* status, char* err, size_t errcap) {
    try {
        if (!x) throw std::runtime_error("null context");
        if (!x->circuit) throw std::runtime_error("this context was opened from a .zkey alone: it has no C matrix to check witnesses against (open it with the circuit)");
        require_idle(x);
        zke_ctx::Slot& S = x->slots[0];
        if (batch == 0 || batch > S.loaded) throw std::runtime_error("no witness loaded for this batch (call zke_load_witness first)");
        CUDA_OK(cudaSetDevice(x->device));
        std::string msg;
        int bad = do_check(x, S, batch, status, msg);
        if (bad) { set_err(err, errcap, msg); return bad; }
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_prove(zke_ctx* x, size_t batch, const uint8_t* rs, uint8_t* proofs_out, uint8_t* publics_out, int32_t* status, char* err, size_t errcap) {
    try {
        if (!x || !proofs_out) throw std::runtime_error("null argument");
        require_idle(x);
        std::string msg;
        int bad = do_prove(x, x->slots[0], batch, rs, proofs_out, publics_out, status, msg);
        if (bad) { set_err(err, errcap, msg); return bad; }
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_wtns_prove(zke_ctx* x, const void* wtns_bytes, size_t len, const uint8_t* rs, uint8_t* proof_out, uint8_t* publics_out,
                   char* err, size_t errcap) {
    try {
        if (!x || !proof_out) throw std::runtime_error("null argument");
        require_idle(x);
        const uint8_t* data = parse_wtns((const uint8_t*)wtns_bytes, len, x->n_vars);
        load_witness(x, x->slots[0], data, 1);
        std::string msg;
        int32_t status = -1;
        int bad = do_prove(x, x->slots[0], 1, rs, proof_out, publics_out, &status, msg);
        if (bad) { set_err(err, errcap, msg); return bad; }
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_fullprove_submit(zke_ctx* x, const uint8_t* inputs, size_t batch, const uint8_t* rs, char* err, size_t errcap) {
    try {
        if (!x) throw std::runtime_error("null context");
        if (x->profile) throw std::runtime_error("stage profiling needs the synchronous entry points");
        if (x->n_submitted - x->n_collected >= 2) throw std::runtime_error("two batches are already in flight: collect one first");
        CUDA_OK(cudaSetDevice(x->device));
        zke_ctx::Slot& S = x->slots[x->n_submitted & 1];
        alloc_slot(x, S);
        try {
            do_witness(x, S, inputs, batch);
            enqueue_prove(x, S, batch, rs);
        } catch (...) { sync_lanes(x); throw; }
        S.busy = true;
        x->n_submitted++;
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_fullprove_collect(zke_ctx* x, uint8_t* proofs_out, uint8_t* publics_out, int32_t* status, char* err, size_t errcap) {
    try {
        if (!x || !proofs_out) throw std::runtime_error("null argument");
        if (x->n_submitted == x->n_collected) throw std::runtime_error("nothing was submitted");
        zke_ctx::Slot& S = x->slots[x->n_collected & 1];
        x->n_collected++;      // the slot is released whatever happens below
        S.busy = false;
        std::string msg;
        int bad = finish_prove(x, S, proofs_out, publics_out, status, msg);
        if (bad) { set_err(err, errcap, msg); return bad; }
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_fullprove(zke_ctx* x, const uint8_t* inputs, size_t batch, const uint8_t* rs, uint8_t* proofs_out, uint8_t* publics_out,
                  int32_t* status, char* err, size_t errcap) {
    try {
        if (!x || !proofs_out) throw std::runtime_error("null argument");
        require_idle(x);
        zke_ctx::Slot& S = x->slots[0];
        do_witness(x, S, inputs, batch);
        std::string msg;
        int bad = do_prove(x, S, batch, rs, proofs_out, publics_out, status, msg);
        if (bad) { set_err(err, errcap, msg); return bad; }
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_shard_begin(zke_ctx* x, int rank, int world, char* err, size_t errcap) {
    try { if (!x) throw std::runtime_error("null context"); shard_begin(x, rank, world); return 0; }
    catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}
void* zke_shard_vector(zke_ctx* x, int which, size_t* n_elems) {
    if (!x || !x->zkey || which < 0 || which > 2 || x->lanes_alloc < 1) return nullptr;
    if (n_elems) *n_elems = (size_t)1 << x->zkey->log_n;
    zke_ctx::Lane& L = x->lanes[0];
    return which == 0 ? L.va.p : (which == 1 ? L.vb.p : L.vc.p);
}
int zke_shard_mid(zke_ctx* x, char* err, size_t errcap) {
    try { if (!x) throw std::runtime_error("null context"); shard_mid(x); return 0; }
    catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}
int zke_shard_end(zke_ctx* x, uint8_t* partial_out, uint8_t* publics_out, char* err, size_t errcap) {
    try { if (!x || !partial_out) throw std::runtime_error("null argument"); shard_end(x, partial_out, publics_out); return 0; }
    catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}
int zke_shard_combine(const zke_zkey* z, const uint8_t* partials, int world, const uint8_t* rs, uint8_t* proof_out, int32_t* status,
                      char* err, size_t errcap) {
    try {
        if (!z || !partials || !proof_out || world < 1) throw std::runtime_error("bad argument");
        const KeyPoints kp{z->alpha1, z->beta1, z->delta1, z->beta2, z->delta2};
        int bad = shard_combine(kp, partials, world, rs, proof_out, status);
        if (bad) set_err(err, errcap, "Assert Failed: constraint " + std::to_string(status ? *status : 0));
        return bad;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}
int zke_shard_combine_raw(const uint8_t* key_points, const uint8_t* partials, int world, const uint8_t* rs, uint8_t* proof_out,
                          int32_t* status, char* err, size_t errcap) {
    try {
        if (!key_points || !partials || !proof_out || world < 1) throw std::runtime_error("bad argument");
        const KeyPoints kp{load_g1(key_points, PARTIAL_COORD), load_g1(key_points + 64, PARTIAL_COORD), load_g1(key_points + 128, PARTIAL_COORD),
                          load_g2(key_points + 192, PARTIAL_COORD), load_g2(key_points + 320, PARTIAL_COORD)};
        int bad = shard_combine(kp, partials, world, rs, proof_out, status);
        if (bad) set_err(err, errcap, "Assert Failed: constraint " + std::to_string(status ? *status : 0));
        return bad;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

}  // extern "C"

// Key construction from a Powers-of-Tau file, phase-2 contributions and their check: part of this translation unit,
// because it builds zke_zkey objects the same way do_setup / do_zkey_load do.
#include "setup.cu"
#include "ptau.cu"
#include "aggregate.cu"
