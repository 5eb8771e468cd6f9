// Aggregation of n Groth16 proofs under one key into one O(log n) proof on the GPU (SnarkPack: TIPP for
// prod e(A_i, B_i)^(r^i), MIPP for sum r^i C_i, keys committed with KZG).  Protocol, byte layout and transcript: DESIGN.md
// "Proof aggregation"; the verifier and the transcript helpers are in aggregate_host.cpp.  Included at the end of
// engine.cu after setup.cu and ptau.cu, whose `.ptau` reader and point validation it uses.
//
// Device work, all in place in HBM across the rounds:
//   pairings     every GT value is a product of columns, a column a list of (G1, G2) pairs of equal length; one thread
//                per pair runs its Miller loop (pairing.cuh), the rows of each column are multiplied in a tree of
//                FOLD-wide levels, and one thread per value multiplies its columns and runs the final exponentiation;
//   scaling      A_i, C_i times r^i and the v keys times r^-i (one thread per point);
//   folding      L + x R over the G1 vectors (A, C, w1, w2) and L + x^-1 R over the G2 vectors (B, v1, v2) of a round;
//   sums         the C halves for the MIPP cross terms (tree of XYZZ additions);
//   openings     the KZG quotients (host: O(n) field operations) as MSMs over the SRS (MsmPlan).
#include "pairing.cuh"
#include "aggregate_host.hpp"

namespace zke {
namespace dev {

static const int AGG_THREADS = 64;
static const uint32_t AGG_FOLD = 32;
static const int AGG_MAX_COLS = 14;
struct AggCols { const uint8_t* p[AGG_MAX_COLS]; const uint8_t* q[AGG_MAX_COLS]; };   // G1 / G2 vectors (Montgomery affine)
struct AggGroups { uint32_t first[AGG_MAX_COLS + 1]; };                               // value k = columns [first[k], first[k+1])

template <class F>
__device__ __forceinline__ Affine<F> agg_to_affine(const XYZZ<F>& a) {
    Affine<F> r;
    if (a.is_inf()) { r.x = F::zero(); r.y = F::zero(); return r; }
    const F zzz_inv = a.zzz.inv();
    const F zz_inv = (a.zz * zzz_inv).sqr();   // zz^3 = zzz^2
    r.x = a.x * zz_inv; r.y = a.y * zzz_inv;
    return r;
}

// proofs: [n][8][32] standard form as zke_prove writes them -> A, C (G1) and B (G2) in Montgomery form; bad[0] = the
// first proof with an unreduced coordinate, a point off its curve or B outside the order-r subgroup
__global__ void __launch_bounds__(AGG_THREADS)
agg_load_kernel(const uint8_t* __restrict__ proofs, uint32_t n, uint8_t* __restrict__ a, uint8_t* __restrict__ b,
                uint8_t* __restrict__ c, uint32_t* bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool ok = true;
    Fq w[8];
    for (int k = 0; k < 8; ++k) {
        const Fq x = Fq::load(proofs + 256ull * i + 32 * k);
        ok = ok && below_modulus(x);
        w[k] = x.to_mont();
    }
    G1Affine pa, pc; G2Affine pb;
    pa.x = w[0]; pa.y = w[1]; pb.x.c0 = w[2]; pb.x.c1 = w[3]; pb.y.c0 = w[4]; pb.y.c1 = w[5]; pc.x = w[6]; pc.y = w[7];
    ok = ok && g1_on_curve(pa) && g1_on_curve(pc) && g2_on_curve(pb) && g2_in_subgroup(pb);
    if (!ok) atomicMin(bad, i);
    pa.store(a + 64ull * i); pb.store(b + 128ull * i); pc.store(c + 64ull * i);
}

// f[row][col] = MillerLoop(q_col[row], p_col[row])
__global__ void __launch_bounds__(AGG_THREADS)
agg_miller_kernel(AggCols cols, uint32_t ncols, uint32_t rows, uint8_t* __restrict__ f) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= rows * ncols) return;
    const uint32_t row = t / ncols, col = t % ncols;
    miller_loop<0>(true, G2Affine::load(cols.q[col] + 128ull * row), G1Affine::load(cols.p[col] + 64ull * row), nullptr, nullptr,
                   nullptr).store(f + 384ull * t);
}

// one level of a tree product over `rows` rows of `width` Fq12 values: out[g][w] = prod in[g FOLD ..][w]
__global__ void __launch_bounds__(AGG_THREADS)
agg_prod_kernel(const uint8_t* __restrict__ in, uint32_t rows, uint32_t width, uint8_t* __restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t groups = (rows + AGG_FOLD - 1) / AGG_FOLD;
    if (t >= groups * width) return;
    const uint32_t g = t / width, w = t % width, end = min(rows, (g + 1) * AGG_FOLD);
    Fq12 acc = Fq12::load(in + 384ull * ((size_t)g * AGG_FOLD * width + w));
    for (uint32_t k = g * AGG_FOLD + 1; k < end; ++k) acc = acc * Fq12::load(in + 384ull * ((size_t)k * width + w));
    acc.store(out + 384ull * t);
}

// value k = final exponentiation of the product of its columns, in the tower layout of vk_alphabeta_12, standard form
__global__ void agg_final_kernel(const uint8_t* __restrict__ colprod, AggGroups g, uint32_t nvals, uint8_t* __restrict__ out) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nvals) return;
    Fq12 f = Fq12::load(colprod + 384ull * g.first[k]);
    for (uint32_t c = g.first[k] + 1; c < g.first[k + 1]; ++c) f = f * Fq12::load(colprod + 384ull * c);
    const Fq12 e = final_exponentiation(f);
    for (int m = 0; m < 6; ++m) {
        const Fq2& c = e.at(m / 3, m % 3);
        c.c0.from_mont().store(out + 384ull * k + 64 * m);
        c.c1.from_mont().store(out + 384ull * k + 64 * m + 32);
    }
}

// pts[i] <- s_i pts[i] (s: [n][32] standard form), in place
template <class F>
__global__ void __launch_bounds__(AGG_THREADS)
agg_scale_kernel(uint8_t* __restrict__ pts, const uint8_t* __restrict__ s, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr k = Fr::load(s + 32ull * i);
    agg_to_affine(scalar_mul(Affine<F>::load(pts + sizeof(Affine<F>) * (size_t)i), k.v, 254)).store(pts + sizeof(Affine<F>) * (size_t)i);
}

// One GIPA round over up to 4 vectors of 2h points: v[i] <- v[i] + x_k v[h + i] for i < h, in place
struct AggFold { uint8_t* v[4]; uint32_t x[4][8]; };
template <class F>
__global__ void __launch_bounds__(AGG_THREADS)
agg_fold_kernel(AggFold a, uint32_t nvec, uint32_t h) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nvec * h) return;
    const uint32_t k = t / h, i = t % h;
    uint8_t* v = a.v[k];
    XYZZ<F> acc = scalar_mul(Affine<F>::load(v + sizeof(Affine<F>) * ((size_t)h + i)), a.x[k], 254);
    acc.madd(Affine<F>::load(v + sizeof(Affine<F>) * (size_t)i), false);
    agg_to_affine(acc).store(v + sizeof(Affine<F>) * (size_t)i);
}

// one level of a tree sum of G1 points: out[g] = sum in[g FOLD ..]; `affine` input (Montgomery) or XYZZ
__global__ void __launch_bounds__(AGG_THREADS)
agg_sum_kernel(const uint8_t* __restrict__ in, bool affine, uint32_t count, uint8_t* __restrict__ out) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (count + AGG_FOLD - 1) / AGG_FOLD) return;
    G1XYZZ acc = G1XYZZ::inf();
    for (uint32_t k = g * AGG_FOLD; k < min(count, (g + 1) * AGG_FOLD); ++k) {
        if (affine) acc.madd(G1Affine::load(in + 64ull * k), false);
        else acc.add(G1XYZZ::load(in + 128ull * k));
    }
    acc.store(out + 128ull * g);
}

}  // namespace dev
}  // namespace zke

struct zke_agg_srs {
    int device = 0;
    uint32_t n_max = 0;
    zke::DevBuf ga, gb, ha, hb;   // g^(a^i), g^(b^i), i < 2 n_max; h^(a^i), h^(b^i), i < n_max (Montgomery affine)
    zke::agg::AggVk vk;
};

namespace {

using namespace zke;

unsigned agg_blocks(size_t threads) { return (unsigned)((threads + dev::AGG_THREADS - 1) / dev::AGG_THREADS); }

Fq fq_mont_at(const uint8_t* p) { Fq x; memcpy(x.m.v, p, 32); return x; }
G1AffineH g1_mont_at(const uint8_t* p) { return G1AffineH{fq_mont_at(p), fq_mont_at(p + 32)}; }
G2AffineH g2_mont_at(const uint8_t* p) {
    return G2AffineH{Fq2{fq_mont_at(p), fq_mont_at(p + 32)}, Fq2{fq_mont_at(p + 64), fq_mont_at(p + 96)}};
}

// Per-call device state of one aggregation
struct AggRun {
    cudaStream_t st = nullptr;
    DevBuf f, f0, f1, vals, sums0, sums1, scal;
    // GT values of `ngroups` column groups over `rows` rows -> host bytes (384 each)
    void gt_values(const dev::AggCols& cols, uint32_t ncols, const dev::AggGroups& g, uint32_t ngroups, uint32_t rows, uint8_t* out) {
        uint8_t* d_f = f.reserve(384ull * rows * ncols);
        dev::agg_miller_kernel<<<agg_blocks((size_t)rows * ncols), dev::AGG_THREADS, 0, st>>>(cols, ncols, rows, d_f);
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        const size_t scratch = 384ull * ncols * ((rows + dev::AGG_FOLD - 1) / dev::AGG_FOLD);
        uint8_t* bufs[2] = {f0.reserve(scratch), f1.reserve(scratch)};
        const uint8_t* in = d_f;
        for (int b = 0; rows > 1; b ^= 1) {
            const uint32_t groups = (rows + dev::AGG_FOLD - 1) / dev::AGG_FOLD;
            dev::agg_prod_kernel<<<agg_blocks((size_t)groups * ncols), dev::AGG_THREADS, 0, st>>>(in, rows, ncols, bufs[b]);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            in = bufs[b];
            rows = groups;
        }
        uint8_t* d_v = vals.reserve(384ull * ngroups);
        dev::agg_final_kernel<<<1, 32, 0, st>>>(in, g, ngroups, d_v);
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        CUDA_OK(cudaMemcpyAsync(out, d_v, 384ull * ngroups, cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
    }
    // sum of `count` G1 points (Montgomery affine, device) on the host
    G1JacH g1_sum(const uint8_t* pts, uint32_t count) {
        const size_t scratch = 128ull * ((count + dev::AGG_FOLD - 1) / dev::AGG_FOLD);
        uint8_t* bufs[2] = {sums0.reserve(scratch), sums1.reserve(scratch)};
        const uint8_t* in = pts;
        bool affine = true;
        int b = 0;
        do {
            const uint32_t groups = (count + dev::AGG_FOLD - 1) / dev::AGG_FOLD;
            dev::agg_sum_kernel<<<agg_blocks(groups), dev::AGG_THREADS, 0, st>>>(in, affine, count, bufs[b]);
            ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
            in = bufs[b]; b ^= 1; affine = false; count = groups;
        } while (count > 1);
        XyzzH<Fq> s;
        CUDA_OK(cudaMemcpyAsync(&s, in, 128, cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
        const G1AffineH a = s.to_affine();
        return G1JacH::from_affine(a);
    }
    // pts[i] *= s_i (F: the device field of the points)
    template <class F>
    void scale(uint8_t* pts, const std::vector<Fr>& s) {
        std::vector<uint8_t> b(32 * s.size());
        for (size_t i = 0; i < s.size(); ++i) store_fr(&b[32 * i], s[i]);
        uint8_t* d = scal.reserve(b.size());
        CUDA_OK(cudaMemcpyAsync(d, b.data(), b.size(), cudaMemcpyHostToDevice, st));
        dev::agg_scale_kernel<F><<<agg_blocks(s.size()), dev::AGG_THREADS, 0, st>>>(pts, d, (uint32_t)s.size());
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
        CUDA_OK(cudaStreamSynchronize(st));   // `b` is pageable host memory
    }
    template <class F>
    void fold(std::initializer_list<uint8_t*> vecs, const Fr& x, uint32_t h) {
        dev::AggFold a{};
        uint32_t k = 0;
        const U256 xs = x.to_u256();
        for (uint8_t* v : vecs) { a.v[k] = v; memcpy(a.x[k], xs.v, 32); ++k; }
        dev::agg_fold_kernel<F><<<agg_blocks((size_t)k * h), dev::AGG_THREADS, 0, st>>>(a, k, h);
        ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
    }
    template <class F>
    AffineH<F> msm(const uint8_t* points, const std::vector<Fr>& s) {
        const uint32_t n = (uint32_t)s.size();
        std::vector<uint8_t> b(32 * s.size());
        for (size_t i = 0; i < s.size(); ++i) store_fr(&b[32 * i], s[i]);
        DevBuf d_s, ws, res;
        CUDA_OK(cudaMemcpyAsync(d_s.reserve(b.size()), b.data(), b.size(), cudaMemcpyHostToDevice, st));
        typedef typename std::conditional<sizeof(F) == sizeof(Fq), dev::Fq, dev::Fq2>::type DF;
        const dev::MsmConfig cfg = dev::msm_config_full(n, false);
        const size_t slot = sizeof(dev::XYZZ<DF>);
        res.reserve(slot * dev::MSM_RESULT_SLOTS);
        CUDA_OK(cudaMemsetAsync(res.p, 0, slot * dev::MSM_RESULT_SLOTS, st));
        dev::MsmPlan<DF>::run(points, d_s.p, n, cfg, ws.reserve(dev::MsmPlan<DF>::workspace_bytes(n, cfg)), res.p, st);
        CHECK_LAUNCH();
        std::vector<uint8_t> block(slot * dev::MSM_RESULT_SLOTS);
        CUDA_OK(cudaMemcpyAsync(block.data(), res.p, block.size(), cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
        return finish_msm<F>(block.data(), cfg);
    }
    ~AggRun() { if (st) cudaStreamDestroy(st); }
};

void put_point(uint8_t*& o, const G1AffineH& p) { store_g1(o, p); o += agg::G1_BYTES; }
void put_point(uint8_t*& o, const G2AffineH& p) { store_g2(o, p); o += agg::G2_BYTES; }

std::vector<Fr> powers(const Fr& x, size_t n) {
    std::vector<Fr> p(n);
    Fr acc = Fr::one();
    for (size_t i = 0; i < n; ++i) { p[i] = acc; acc = acc * x; }
    return p;
}

int64_t do_aggregate(zke_agg_srs* s, const char* vkey_json, size_t n, const uint8_t* proofs, const uint8_t* publics, uint8_t* out,
                     size_t cap) {
    agg::check_count(n);
    if (n > s->n_max) throw std::runtime_error(std::to_string(n) + " proofs exceed the SRS size " + std::to_string(s->n_max));
    const VerifyingKey vk = vkey_from_json(vkey_json);
    const size_t np = vk.ic.size() - 1;
    if (np && !publics) throw std::runtime_error("null argument");
    for (size_t i = 0; i < n * np; ++i) {
        U256 v; memcpy(v.v, publics + 32 * i, 32);
        if (u256_cmp(v, fr_params().p) >= 0) throw std::runtime_error("public signal " + std::to_string(i % np) + " of proof " + std::to_string(i / np) + " is not below r");
    }
    const size_t total = agg::agg_bytes(n);
    if (!out || cap < total) throw std::runtime_error("output buffer needs " + std::to_string(total) + " bytes");
    select_device(s->device);
    AggRun run;
    CUDA_OK(cudaStreamCreateWithFlags(&run.st, cudaStreamNonBlocking));
    cudaStream_t st = run.st;
    const uint32_t nn = (uint32_t)n;
    DevBuf d_proofs, A, B, C, v1, v2, w1, w2, flag;
    CUDA_OK(cudaMemcpyAsync(d_proofs.reserve(256 * n), proofs, 256 * n, cudaMemcpyHostToDevice, st));
    A.reserve(64 * n); B.reserve(128 * n); C.reserve(64 * n);
    CUDA_OK(cudaMemsetAsync(flag.reserve(4), 0xff, 4, st));
    dev::agg_load_kernel<<<agg_blocks(n), dev::AGG_THREADS, 0, st>>>(d_proofs.p, nn, A.p, B.p, C.p, (uint32_t*)flag.p);
    ZKE_COUNT_LAUNCH(1); CHECK_LAUNCH();
    uint32_t bad = 0;
    CUDA_OK(cudaMemcpyAsync(&bad, flag.p, 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    if (bad != 0xffffffffu)
        throw std::runtime_error("proof " + std::to_string(bad) + ": a coordinate is not reduced, a point is off its curve or B is outside the order-r subgroup");
    CUDA_OK(cudaMemcpyAsync(v1.reserve(128 * n), s->ha.p, 128 * n, cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(v2.reserve(128 * n), s->hb.p, 128 * n, cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(w1.reserve(64 * n), s->ga.p + 64 * n, 64 * n, cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(w2.reserve(64 * n), s->gb.p + 64 * n, 64 * n, cudaMemcpyDeviceToDevice, st));

    uint8_t* o = out;
    // commitments: T_AB = e(A, v1) e(w1, B), U_AB = e(A, v2) e(w2, B), T_C = e(C, v1), U_C = e(C, v2)
    {
        const dev::AggCols cols{{A.p, w1.p, A.p, w2.p, C.p, C.p}, {v1.p, B.p, v2.p, B.p, v1.p, v2.p}};
        const dev::AggGroups g{{0, 2, 4, 5, 6}};
        run.gt_values(cols, 6, g, 4, nn, o);
    }
    const Fr r = agg::first_challenge(vk, n, o, publics);
    o += 4 * agg::GT_BYTES;
    const std::vector<Fr> rp = powers(r, n), rinv = powers(r.inv(), n);
    run.scale<dev::Fq>(A.p, rp);
    run.scale<dev::Fq>(C.p, rp);
    run.scale<dev::Fq2>(v1.p, rinv);
    run.scale<dev::Fq2>(v2.p, rinv);
    {
        const dev::AggCols cols{{A.p}, {B.p}};
        const dev::AggGroups g{{0, 1}};
        run.gt_values(cols, 1, g, 1, nn, o);   // Z_AB
        o += agg::GT_BYTES;
    }
    put_point(o, run.g1_sum(C.p, nn).to_affine());   // Z_C
    Fr x = r, beta = Fr::one();
    std::vector<Fr> xs;
    for (uint32_t h = nn / 2; h >= 1; h /= 2) {
        uint8_t* msg = o;
        // columns: ZL, ZR | TL = e(A_R, v1_L) e(w1_R, B_L) | TR = e(A_L, v1_R) e(w1_L, B_R) | UL | UR (v2, w2) | TCL TCR UCL UCR
        uint8_t *AL = A.p, *AR = A.p + 64ull * h, *CL = C.p, *CR = C.p + 64ull * h, *BL = B.p, *BR = B.p + 128ull * h;
        uint8_t *w1L = w1.p, *w1R = w1.p + 64ull * h, *w2L = w2.p, *w2R = w2.p + 64ull * h;
        uint8_t *v1L = v1.p, *v1R = v1.p + 128ull * h, *v2L = v2.p, *v2R = v2.p + 128ull * h;
        const dev::AggCols c{{AR, AL, AR, w1R, AL, w1L, AR, w2R, AL, w2L, CR, CL, CR, CL},
                             {BL, BR, v1L, BL, v1R, BR, v2L, BL, v2R, BR, v1L, v1R, v2L, v2R}};
        const dev::AggGroups g{{0, 1, 2, 4, 6, 8, 10, 11, 12, 13, 14}};
        run.gt_values(c, 14, g, 10, h, o);
        o += agg::ROUND_GT * agg::GT_BYTES;
        const U256 be = beta.to_u256();
        put_point(o, run.g1_sum(CR, h).mul(be).to_affine());   // ZCL = <b_L, C_R>: b is the constant vector beta
        put_point(o, run.g1_sum(CL, h).mul(be).to_affine());   // ZCR = <b_R, C_L>
        x = agg::next_challenge(x, msg, agg::ROUND_BYTES);
        xs.push_back(x);
        const Fr xi = x.inv();
        run.fold<dev::Fq>({A.p, C.p, w1.p, w2.p}, x, h);
        run.fold<dev::Fq2>({B.p, v1.p, v2.p}, xi, h);
        beta = beta * (Fr::one() + xi);
    }
    // final vectors and keys, then the KZG openings at z
    uint8_t fin[agg::FINAL_BYTES];
    {
        uint8_t* f = fin;
        uint8_t raw[128];
        auto g1 = [&](const DevBuf& v) { CUDA_OK(cudaMemcpyAsync(raw, v.p, 64, cudaMemcpyDeviceToHost, st)); CUDA_OK(cudaStreamSynchronize(st)); put_point(f, g1_mont_at(raw)); };
        auto g2 = [&](const DevBuf& v) { CUDA_OK(cudaMemcpyAsync(raw, v.p, 128, cudaMemcpyDeviceToHost, st)); CUDA_OK(cudaStreamSynchronize(st)); put_point(f, g2_mont_at(raw)); };
        g1(A); g2(B); g1(C); g2(v1); g2(v2); g1(w1); g1(w2);
    }
    memcpy(o, fin, sizeof fin);
    o += sizeof fin;
    const Fr z = agg::next_challenge(x, fin, sizeof fin);
    std::vector<Fr> cv, cw;
    agg::fold_polys(xs, r.inv(), n, cv, cw);
    const std::vector<Fr> qv = agg::kzg_quotient(cv, z), qw = agg::kzg_quotient(cw, z);
    put_point(o, run.msm<Fq2>(s->ha.p, qv));
    put_point(o, run.msm<Fq2>(s->hb.p, qv));
    put_point(o, run.msm<Fq>(s->ga.p, qw));
    put_point(o, run.msm<Fq>(s->gb.p, qw));
    if ((size_t)(o - out) != total) throw std::runtime_error("internal error: aggregate size");
    return (int64_t)total;
}

zke_agg_srs* do_agg_srs_from_ptau(const uint8_t* fa, size_t la, const uint8_t* fb, size_t lb, uint32_t n_max, int device) {
    agg::check_count(n_max);
    const PtauView va = parse_ptau(fa, la, true), vb = parse_ptau(fb, lb, true);
    unsigned need = 1;
    while (((size_t)1 << (need - 1)) < n_max) ++need;
    for (const PtauView* v : {&va, &vb})
        if (v->power < need)
            throw std::runtime_error(".ptau of power " + std::to_string(v->power) + " is too small for " + std::to_string(n_max) + " proofs: it needs power " +
                                     std::to_string(need) + " or more");
    select_device(device);
    std::unique_ptr<zke_agg_srs> s(new zke_agg_srs());
    s->device = device;
    s->n_max = n_max;
    DevBuf flag;
    flag.reserve(4);
    const char* which[2] = {"first", "second"};
    const PtauView* vs[2] = {&va, &vb};
    DevBuf* g1s[2] = {&s->ga, &s->gb};
    DevBuf* g2s[2] = {&s->ha, &s->hb};
    for (int t = 0; t < 2; ++t) {
        CUDA_OK(cudaMemcpy(g1s[t]->reserve(128ull * n_max), vs[t]->sec[2].p, 128ull * n_max, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(g2s[t]->reserve(128ull * n_max), vs[t]->sec[3].p, 128ull * n_max, cudaMemcpyHostToDevice));
        std::string why = section_points_problem(2, g1s[t]->p, 2ull * n_max, 0, (uint32_t*)flag.p);
        if (why.empty()) why = section_points_problem(3, g2s[t]->p, n_max, 0, (uint32_t*)flag.p);
        if (!why.empty()) throw std::runtime_error(std::string("the ") + which[t] + " " + why);
    }
    const G1AffineH g = g1_mont_at(va.sec[2].p), gb0 = g1_mont_at(vb.sec[2].p);
    const G2AffineH h = g2_mont_at(va.sec[3].p), hb0 = g2_mont_at(vb.sec[3].p);
    if (g.is_inf() || h.is_inf() || !(g.x == gb0.x && g.y == gb0.y) || !(h.x == hb0.x && h.y == hb0.y))
        throw std::runtime_error("the two .ptau files do not start from the same generators");
    s->vk = agg::AggVk{g, g1_mont_at(va.sec[2].p + 64), g1_mont_at(vb.sec[2].p + 64), h, g2_mont_at(va.sec[3].p + 128), g2_mont_at(vb.sec[3].p + 128)};
    if (s->vk.g_a.x == s->vk.g_b.x && s->vk.g_a.y == s->vk.g_b.y) throw std::runtime_error("the two .ptau files share their tau: aggregation needs independent secrets");
    return s.release();
}

}  // namespace

extern "C" {

zke_agg_srs* zke_agg_srs_from_ptau(const void* ptau_a, size_t len_a, const void* ptau_b, size_t len_b, uint32_t n_max, int device,
                                   char* err, size_t errcap) {
    try {
        return do_agg_srs_from_ptau((const uint8_t*)ptau_a, len_a, (const uint8_t*)ptau_b, len_b, n_max, device);
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}

void zke_agg_srs_free(zke_agg_srs* s) {
    if (!s) return;
    cudaSetDevice(s->device);
    delete s;
}

uint32_t zke_agg_srs_n_max(const zke_agg_srs* s) { return s ? s->n_max : 0; }

int zke_agg_vk_json(const zke_agg_srs* s, char* out, size_t* len) {
    if (!s || !len) return -1;
    const std::string j = agg::agg_vk_to_json(s->vk);
    const size_t cap = *len;
    *len = j.size() + 1;
    if (!out || cap < j.size() + 1) return -2;
    memcpy(out, j.c_str(), j.size() + 1);
    return 0;
}

int64_t zke_aggregate(zke_agg_srs* s, const char* vkey_json, size_t n, const uint8_t* proofs, const uint8_t* publics, uint8_t* out,
                      size_t cap, char* err, size_t errcap) {
    try {
        if (!s || !vkey_json || !proofs) throw std::runtime_error("null argument");
        return do_aggregate(s, vkey_json, n, proofs, publics, out, cap);
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

size_t zke_agg_bytes(size_t n) { return (n >= 2 && n <= zke::agg::MAX_PROOFS && !(n & (n - 1))) ? zke::agg::agg_bytes(n) : 0; }

}  // extern "C"
