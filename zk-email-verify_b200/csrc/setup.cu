// Groth16 keys from a prepared Powers-of-Tau file (`snarkjs groth16 setup` / `zkey new`), phase-2 contributions
// (`snarkjs zkey contribute`, without its transcript) and the ratio check of `snarkjs zkey verify`.
// Included at the end of engine.cu: it builds zke_zkey objects exactly as do_setup / do_zkey_load do.
//
// A key is a set of sparse sums of Lagrange-basis points: for every signal j
//     A_j  = sum_k a_kj [L_k(tau)]_1          B1_j = sum_k b_kj [L_k(tau)]_1        B2_j = sum_k b_kj [L_k(tau)]_2
//     IC_j (j <= l), C_j (j > l) = sum_k a_kj [beta L_k(tau)]_1 + b_kj [alpha L_k(tau)]_1 + c_kj [L_k(tau)]_1
// with the rows n_constraints + j (j <= l) of A holding 1 * w_j, as in setup_host.cpp.  The sums run on the GPU:
// the circuit's row-major CSR is transposed on the host to signal-major term lists, every signal's list is cut into
// chunks of SETUP_CHUNK terms, one thread sums one chunk, and the partial sums of a signal are added in further passes
// of at most SETUP_FANIN partials each - so the constant wire, with hundreds of thousands of terms, does not serialise
// a warp.  The key has gamma = delta = 1: anyone who knows it can forge proofs, so it reports itself as a toy until a
// contribution replaces delta.
#include "ec_ntt.cuh"
#include <chrono>

namespace {

// ------------------------------------------------------------------------------------------------ .ptau reader
// Prepared phase-2 Powers-of-Tau file of snarkjs (`powersoftau prepare phase2`), restated from the snarkjs 0.5 sources
// (un-vendored here; no file of this layout can be checked against them in this repository):
//   iden3 binfile: magic "ptau", u32 version 1, u32 nSections, then {u32 type, u64 size, payload} per section;
//   1  header: u32 n8q = 32, q (n8q bytes, LE), u32 power, u32 ceremonyPower
//   2  tauG1       [tau^i]_1,          i < 2^(power+1) - 1
//   3  tauG2       [tau^i]_2,          i < 2^power
//   4  alphaTauG1  [alpha tau^i]_1,    i < 2^power
//   5  betaTauG1   [beta tau^i]_1,     i < 2^power
//   6  betaG2      [beta]_2
//   7  contributions (not read)
//   12 lTauG1, 13 lTauG2, 14 lAlphaTauG1, 15 lBetaTauG1: the same four families in the Lagrange bases of the domains
//      of size 1, 2, 4, ..., 2^power, back to back - the size-2^k basis starts at point 2^k - 1, and its point i is
//      [L_i(tau)]  with  L_i(x) = (x^N - 1) / N * omega^i / (x - omega^i)  (times alpha / beta in 14 / 15).
// Points are affine with Montgomery-form little-endian coordinates (G2: x.c0, x.c1, y.c0, y.c1), as in `.zkey`.
struct PtauView {
    uint32_t power = 0, ceremony_power = 0;
    SecView sec[16];
    const uint8_t* base = nullptr;
    bool prepared = false;   // sections 12-15 present
};

const char* ptau_section_name(int s) {
    switch (s) {
        case 2: return "tauG1"; case 3: return "tauG2"; case 4: return "alphaTauG1"; case 5: return "betaTauG1";
        case 6: return "betaG2"; case 12: return "lTauG1"; case 13: return "lTauG2"; case 14: return "lAlphaTauG1";
        case 15: return "lBetaTauG1"; default: return "?";
    }
}
// bytes of section s at `power`
size_t ptau_section_bytes(int s, uint32_t power) {
    const size_t n = (size_t)1 << power;
    switch (s) {
        case 2: return (2 * n - 1) * 64;
        case 3: return n * 128;
        case 4: case 5: return n * 64;
        case 6: return 128;
        case 12: case 14: case 15: return (2 * n - 1) * 64;
        case 13: return (2 * n - 1) * 128;
        default: return 0;
    }
}
const int PTAU_POINT_SECTIONS[] = {2, 3, 4, 5, 6, 12, 13, 14, 15};
const size_t PTAU_HEADER_BYTES = 4 + 32 + 4 + 4;
const uint32_t PTAU_MAX_POWER = 28;

// Structure only (sizes, modulus, power); the points are validated on the device where they are used.  With
// lagrange_optional, sections 12-15 may be absent (an unprepared file), but only all four together.
PtauView parse_ptau(const uint8_t* b, size_t len, bool lagrange_optional = false) {
    PtauView v;
    v.base = b;
    if (!b || len < 12 || memcmp(b, "ptau", 4) != 0) throw std::runtime_error("not a .ptau file (bad magic)");
    if (rd32(b + 4) != 1) throw std::runtime_error("unsupported .ptau version " + std::to_string(rd32(b + 4)));
    for (const BinSection& s : binfile_sections(b, len, ".ptau")) {
        if (s.type >= 16) continue;
        if (v.sec[s.type].p) throw std::runtime_error(".ptau section " + std::to_string(s.type) + " appears twice");
        v.sec[s.type] = s.view;
    }
    const SecView& h = v.sec[1];
    if (!h.p) throw std::runtime_error(".ptau header section 1 is missing");
    if (h.n != PTAU_HEADER_BYTES || rd32(h.p) != 32 || memcmp(h.p + 4, fq_params().p.v, 32) != 0)
        throw std::runtime_error(".ptau is not over the BN254 base field");
    v.power = rd32(h.p + 36);
    v.ceremony_power = rd32(h.p + 40);
    if (v.power < 1 || v.power > PTAU_MAX_POWER) throw std::runtime_error(".ptau power " + std::to_string(v.power) + " is outside [1, 28]");
    v.prepared = v.sec[12].p || v.sec[13].p || v.sec[14].p || v.sec[15].p;
    for (int s : PTAU_POINT_SECTIONS) {
        if (lagrange_optional && s >= 12 && !v.prepared) continue;
        if (!v.sec[s].p) throw std::runtime_error(".ptau section " + std::to_string(s) + " (" + ptau_section_name(s) + ") is missing");
        const size_t want = ptau_section_bytes(s, v.power);
        if (v.sec[s].n != want)
            throw std::runtime_error(".ptau section " + std::to_string(s) + " (" + ptau_section_name(s) + ") has " + std::to_string(v.sec[s].n) +
                                     " bytes, expected " + std::to_string(want) + " for power " + std::to_string(v.power));
    }
    return v;
}

// the H points need the Lagrange basis of size 2N
void ptau_fits_circuit(const PtauView& v, const Circuit& c) {
    const uint32_t need = c.domain_log2() + 1;
    if (v.power < need)
        throw std::runtime_error(".ptau of power " + std::to_string(v.power) + " is too small for this circuit: its domain 2^" +
                                 std::to_string(c.domain_log2()) + " needs power " + std::to_string(need) + " or more");
}

// first point of the size-2^k basis of Lagrange section s
const uint8_t* ptau_basis(const PtauView& v, int s, unsigned k) {
    return v.sec[s].p + (((size_t)1 << k) - 1) * (s == 13 ? 128 : 64);
}

// ------------------------------------------------------------------------------------------------ signal-major terms
// one matrix of the circuit whose terms are added to every signal's list: point index = base + row
struct TermSource {
    const std::vector<uint32_t>* ptr; const std::vector<uint32_t>* var; const std::vector<uint32_t>* coef;
    uint32_t rows, base;
    bool extra_rows;   // also the rows n_rows + j (j <= n_public) of A: 1 * w_j
};

// Counting sort of the terms by signal; within a signal, the sources in order and each in row order.
void signal_major(const std::vector<TermSource>& src, uint32_t m, uint32_t n_public, std::vector<uint32_t>& sig_ptr, std::vector<uint2>& terms) {
    sig_ptr.assign((size_t)m + 1, 0);
    for (const TermSource& s : src) {
        for (uint32_t k = 0; k < (*s.ptr)[s.rows]; ++k) sig_ptr[(*s.var)[k] + 1]++;
        if (s.extra_rows) for (uint32_t j = 0; j <= n_public; ++j) sig_ptr[j + 1]++;
    }
    for (uint32_t j = 0; j < m; ++j) sig_ptr[j + 1] += sig_ptr[j];
    terms.resize(sig_ptr[m]);
    std::vector<uint32_t> pos(sig_ptr.begin(), sig_ptr.end() - 1);
    for (const TermSource& s : src) {
        for (uint32_t row = 0; row < s.rows; ++row)
            for (uint32_t k = (*s.ptr)[row]; k < (*s.ptr)[row + 1]; ++k) terms[pos[(*s.var)[k]]++] = make_uint2(s.base + row, (*s.coef)[k]);
        if (s.extra_rows) for (uint32_t j = 0; j <= n_public; ++j) terms[pos[j]++] = make_uint2(s.base + s.rows + j, 0u);
    }
}

// Cuts segments (ptr[i], ptr[i+1]) into chunks of at most `width` items.  chunk_ptr: item boundaries of the chunks;
// seg_chunks: the new segmentation (chunk boundaries per segment).  Empty segments get no chunk.
void cut_chunks(const std::vector<uint32_t>& ptr, uint32_t width, std::vector<uint32_t>& chunk_ptr, std::vector<uint32_t>& seg_chunks) {
    const size_t n_seg = ptr.size() - 1;
    chunk_ptr.assign(1, ptr[0]);
    seg_chunks.assign(n_seg + 1, 0);
    for (size_t i = 0; i < n_seg; ++i) {
        for (uint32_t b = ptr[i]; b < ptr[i + 1]; b += width) chunk_ptr.push_back(std::min(b + width, ptr[i + 1]));
        seg_chunks[i + 1] = (uint32_t)(chunk_ptr.size() - 1);
    }
}

// Coefficient table of the device sums: the magnitude of the smaller of v and r - v, with bit 255 set when it is r - v
// (so -1 is "1, negative", and a term with it is one mixed subtraction).
std::vector<U256> signed_coefs(const std::vector<U256>& coefs) {
    U256 half = fr_params().p;
    for (int i = 0; i < 4; ++i) half.v[i] = (half.v[i] >> 1) | (i < 3 ? half.v[i + 1] << 63 : 0);
    std::vector<U256> out(coefs.size());
    for (size_t i = 0; i < coefs.size(); ++i) {
        if (u256_cmp(coefs[i], half) > 0) { u256_sub(out[i], fr_params().p, coefs[i]); out[i].v[3] |= 1ull << 63; }
        else out[i] = coefs[i];
    }
    return out;
}

}  // namespace

namespace zke { namespace dev {

static const uint32_t SETUP_CHUNK = 32;   // terms summed by one thread in the first pass
static const uint32_t SETUP_FANIN = 32;   // partial sums added by one thread in each further pass

// acc += coef * P for a term {point index, coefficient index}; a coefficient of magnitude 1 is one mixed addition,
// any other a double-and-add over its bits.  The loop starts from P at the top bit rather than calling ec.cuh's
// scalar_mul: the scalar_mul form made the device part of `from_ptau` 3.6% slower (H100 80GB HBM3, 700 W).
template <class F>
__device__ __forceinline__ void add_term(XYZZ<F>& acc, const uint8_t* __restrict__ points, uint2 t, const uint32_t* __restrict__ coefs) {
    const Affine<F> p = Affine<F>::load(points + sizeof(Affine<F>) * (size_t)t.x);
    const uint32_t* k = coefs + 8 * (size_t)t.y;
    const bool neg = k[7] >> 31;
    int top = -1;
    for (int w = 7; w >= 0 && top < 0; --w) {
        const uint32_t v = w == 7 ? (k[7] & 0x7fffffffu) : k[w];
        if (v) top = 32 * w + 31 - __clz(v);
    }
    if (top < 0) return;
    if (top == 0) { acc.madd(p, neg); return; }
    XYZZ<F> q = XYZZ<F>::from_affine(p);
    for (int i = top - 1; i >= 0; --i) {
        q.dbl();
        uint32_t limb = k[i >> 5];
        if ((i >> 5) == 7) limb &= 0x7fffffffu;
        if ((limb >> (i & 31)) & 1) q.madd(p, false);
    }
    if (neg) q.negate();
    acc.add(q);
}

// out[c] = sum of the terms [chunk_ptr[c], chunk_ptr[c + 1])
template <class F>
__global__ void __launch_bounds__(128)
setup_term_sum_kernel(const uint8_t* __restrict__ points, const uint2* __restrict__ terms, const uint32_t* __restrict__ chunk_ptr,
                      uint32_t n_chunks, const uint32_t* __restrict__ coefs, uint8_t* __restrict__ out_xyzz) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks) return;
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t k = chunk_ptr[c]; k < chunk_ptr[c + 1]; ++k) add_term(acc, points, terms[k], coefs);
    acc.store(out_xyzz + sizeof(XYZZ<F>) * (size_t)c);
}

// out[s] = sum of the partial sums [ptr[s], ptr[s + 1]) (infinity for an empty segment)
template <class F>
__global__ void __launch_bounds__(128)
setup_partial_sum_kernel(const uint8_t* __restrict__ in_xyzz, const uint32_t* __restrict__ ptr, uint32_t n_seg, uint8_t* __restrict__ out_xyzz) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t k = ptr[s]; k < ptr[s + 1]; ++k) acc.add(XYZZ<F>::load(in_xyzz + sizeof(XYZZ<F>) * (size_t)k));
    acc.store(out_xyzz + sizeof(XYZZ<F>) * (size_t)s);
}

// first index i < n with a[i] != b[i] (16-byte words) -> atomicMin(first)
__global__ void words_differ_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint32_t n, uint32_t* first) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4 x = a[i], y = b[i];
    if (x.x != y.x || x.y != y.y || x.z != y.z || x.w != y.w) atomicMin(first, i);
}

} }  // namespace zke::dev

namespace {

// Sums every signal's term list on the device and writes the n_sig affine results to `out`.
template <class F>
void signal_sums(const uint8_t* points_dev, const std::vector<uint32_t>& sig_ptr, const std::vector<uint2>& terms, const DevBuf& coefs_dev,
                 DevBuf& out, cudaStream_t st) {
    using XY = dev::XYZZ<F>;
    const uint32_t n_sig = (uint32_t)(sig_ptr.size() - 1);
    out.alloc((size_t)n_sig * sizeof(dev::Affine<F>));
    std::vector<uint32_t> chunk_ptr, seg;
    cut_chunks(sig_ptr, dev::SETUP_CHUNK, chunk_ptr, seg);
    DevBuf d_terms, d_ptr, part[2];
    d_terms.upload(terms);
    d_ptr.upload(chunk_ptr);
    uint32_t n_items = (uint32_t)(chunk_ptr.size() - 1);
    part[0].alloc(std::max<size_t>(1, n_items) * sizeof(XY));
    if (n_items) {
        dev::setup_term_sum_kernel<F><<<(n_items + 127) / 128, 128, 0, st>>>(points_dev, (const uint2*)d_terms.p, (const uint32_t*)d_ptr.p,
                                                                           n_items, (const uint32_t*)coefs_dev.p, part[0].p);
        ZKE_COUNT_LAUNCH(1);
        CHECK_LAUNCH();
    }
    // further passes while some signal has more than SETUP_FANIN partials, then one pass per signal
    int cur = 0;
    for (;;) {
        uint32_t widest = 0;
        for (uint32_t j = 0; j < n_sig; ++j) widest = std::max(widest, seg[j + 1] - seg[j]);
        const bool last = widest <= dev::SETUP_FANIN;
        std::vector<uint32_t> next_ptr, next_seg;
        if (last) next_ptr = seg;
        else cut_chunks(seg, dev::SETUP_FANIN, next_ptr, next_seg);
        const uint32_t n_out = (uint32_t)(next_ptr.size() - 1);
        CUDA_OK(cudaStreamSynchronize(st));   // the previous pass still reads d_ptr and writes part[cur]
        DevBuf& dst = part[1 - cur];
        dst.alloc(std::max<size_t>(1, n_out) * sizeof(XY));
        d_ptr.upload(next_ptr);
        if (n_out) {
            dev::setup_partial_sum_kernel<F><<<(n_out + 127) / 128, 128, 0, st>>>(part[cur].p, (const uint32_t*)d_ptr.p, n_out, dst.p);
            ZKE_COUNT_LAUNCH(1);
            CHECK_LAUNCH();
        }
        cur = 1 - cur;
        if (last) break;
        seg.swap(next_seg);
    }
    dev::xyzz_to_affine_batch<F>(part[cur].p, n_sig, out.p, st);
    CHECK_LAUNCH();
    CUDA_OK(cudaStreamSynchronize(st));
}

// out[i] = k_i * in[i] for n affine points on the device (k_i = k[i * stride], standard form, device; stride 0: one
// scalar for all), through `x` (n XYZZ points)
template <class F>
void scale_each(const uint8_t* in, size_t n, const uint8_t* k, uint32_t stride, uint8_t* x, uint8_t* out, cudaStream_t st) {
    if (!n) return;
    dev::scale_each_kernel<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(in, (uint32_t)n, (const uint32_t*)k, stride, 0, x);
    ZKE_COUNT_LAUNCH(1);
    dev::xyzz_to_affine_batch<F>(x, (uint32_t)n, out, st);
    CHECK_LAUNCH();
}

// sum_i w_i P_i over the affine device points P_0 .. P_{n-1} (w: standard form, below r), affine host image: one
// segment of n terms {point i, weight i} through the signal sums
template <class F, class H>
H weighted_sum(const uint8_t* pts, const std::vector<U256>& w) {
    H r = H::inf();
    const uint32_t n = (uint32_t)w.size();
    if (!n) return r;
    const std::vector<uint32_t> ptr = {0u, n};
    std::vector<uint2> terms(n);
    for (uint32_t i = 0; i < n; ++i) terms[i] = make_uint2(i, i);
    DevBuf weights, out;
    weights.upload(w);
    signal_sums<F>(pts, ptr, terms, weights, out, nullptr);
    CUDA_OK(cudaMemcpy(&r, out.p, sizeof r, cudaMemcpyDeviceToHost));
    return r;
}

// a contribution secret in [2, r); `name` (may be null) follows "contribution secret" in the messages
Fr contribution_secret(const uint8_t* b32, const char* name = nullptr) {
    U256 s;
    memcpy(s.v, b32, 32);
    const std::string what = name ? std::string("contribution secret ") + name : std::string("contribution secret");
    if (s.is_zero()) throw std::runtime_error(what + " is zero");
    if (u256_cmp(s, fr_params().p) >= 0) throw std::runtime_error(what + " is not below the group order r");
    if (s.v[0] == 1 && !s.v[1] && !s.v[2] && !s.v[3]) throw std::runtime_error(what + " is one (it would change nothing)");
    return Fr::from_u256(s);
}

bool g1_valid(const G1AffineH& p) { return u256_cmp(p.x.m, fq_params().p) < 0 && u256_cmp(p.y.m, fq_params().p) < 0 && g1_on_curve(p); }
bool g2_valid(const G2AffineH& p) {
    for (const Fq* c : {&p.x.c0, &p.x.c1, &p.y.c0, &p.y.c1}) if (u256_cmp(c->m, fq_params().p) >= 0) return false;
    return g2_on_curve(p);
}
bool g1_eq(const G1AffineH& a, const G1AffineH& b) { return memcmp(&a, &b, sizeof a) == 0; }
bool g2_eq(const G2AffineH& a, const G2AffineH& b) { return memcmp(&a, &b, sizeof a) == 0; }

double ms_since(const std::chrono::steady_clock::time_point& t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

// ------------------------------------------------------------------------------------------------ zke_zkey_from_ptau
struct SetupTiming { double host_ms = 0, gpu_ms = 0; };
static thread_local SetupTiming g_last_setup_timing;

static zke_zkey* do_zkey_from_ptau(const zke_circuit* zc, const uint8_t* file, size_t len, int device) {
    const auto t0 = std::chrono::steady_clock::now();
    const Circuit& c = zc->c;
    const PtauView v = parse_ptau(file, len);
    ptau_fits_circuit(v, c);
    const unsigned log_n = c.domain_log2();
    const size_t N = (size_t)1 << log_n;
    const uint32_t m = c.n_vars, l = c.n_public(), nc = c.n_constraints;

    // header points: host copies, checked on the host
    std::unique_ptr<zke_zkey> zk(new zke_zkey());
    zk->n_vars = m; zk->n_public = l; zk->log_n = log_n; zk->device = device;
    zk->toy = true; zk->delta_one = true;
    memcpy(&zk->alpha1, v.sec[4].p, 64);
    memcpy(&zk->beta1, v.sec[5].p, 64);
    memcpy(&zk->beta2, v.sec[6].p, 128);
    if (!g1_valid(zk->alpha1) || zk->alpha1.is_inf()) throw std::runtime_error(".ptau section 4 (alphaTauG1): point 0 is not on the curve");
    if (!g1_valid(zk->beta1) || zk->beta1.is_inf()) throw std::runtime_error(".ptau section 5 (betaTauG1): point 0 is not on the curve");
    if (!g2_valid(zk->beta2) || zk->beta2.is_inf() || !g2_in_subgroup(zk->beta2)) throw std::runtime_error(".ptau section 6 (betaG2): the point is not in G2");
    zk->delta1 = g1_generator();
    zk->gamma2 = g2_generator();
    zk->delta2 = g2_generator();

    // signal-major term lists; G1 bases are [lTau | lAlphaTau | lBetaTau] of size N each
    std::vector<uint32_t> ab_ptr, cc_ptr, a_ptr;
    std::vector<uint2> a_terms, b_terms, c_terms;
    signal_major({TermSource{&c.a_ptr, &c.a_var, &c.a_coef, nc, 0, true}}, m, l, a_ptr, a_terms);
    signal_major({TermSource{&c.b_ptr, &c.b_var, &c.b_coef, nc, 0, false}}, m, l, ab_ptr, b_terms);
    signal_major({TermSource{&c.a_ptr, &c.a_var, &c.a_coef, nc, (uint32_t)(2 * N), true},
                  TermSource{&c.b_ptr, &c.b_var, &c.b_coef, nc, (uint32_t)N, false},
                  TermSource{&c.c_ptr, &c.c_var, &c.c_coef, nc, 0, false}}, m, l, cc_ptr, c_terms);
    // the key's own coefficient matrices (`.zkey` section 4 form: CSR over the N domain rows, extra rows of A included)
    zk->coefs = c.coefs;
    zk->a_ptr.assign(N + 1, 0); zk->b_ptr.assign(N + 1, 0);
    for (uint32_t row = 0; row < nc; ++row) { zk->a_ptr[row + 1] = c.a_ptr[row + 1]; zk->b_ptr[row + 1] = c.b_ptr[row + 1]; }
    for (size_t row = nc; row < N; ++row) { zk->a_ptr[row + 1] = zk->a_ptr[row] + (row <= (size_t)nc + l ? 1 : 0); zk->b_ptr[row + 1] = zk->b_ptr[row]; }
    zk->a_var.assign(c.a_var.begin(), c.a_var.begin() + c.a_ptr[nc]); zk->a_coef.assign(c.a_coef.begin(), c.a_coef.begin() + c.a_ptr[nc]);
    for (uint32_t j = 0; j <= l; ++j) { zk->a_var.push_back(j); zk->a_coef.push_back(0); }
    zk->b_var.assign(c.b_var.begin(), c.b_var.begin() + c.b_ptr[nc]); zk->b_coef.assign(c.b_coef.begin(), c.b_coef.begin() + c.b_ptr[nc]);
    zk->has_coefs = true;
    const std::vector<U256> scoefs = signed_coefs(c.coefs);
    const double host_ms = ms_since(t0);

    const auto t1 = std::chrono::steady_clock::now();
    select_device(device);
    cudaStream_t st = nullptr;
    DevBuf flag, g1b, g2b, coefs_dev;
    flag.alloc(4);
    coefs_dev.upload(scoefs);
    const Fq b1 = Fq::from_u64(3);
    const Fq2 b2 = g2_twist_b();
    g1b.alloc(3 * N * 64);
    CUDA_OK(cudaMemcpy(g1b.p, ptau_basis(v, 12, log_n), N * 64, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(g1b.p + N * 64, ptau_basis(v, 14, log_n), N * 64, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(g1b.p + 2 * N * 64, ptau_basis(v, 15, log_n), N * 64, cudaMemcpyHostToDevice));
    auto refuse = [](int64_t bad, const char* what) {
        if (bad >= 0) throw std::runtime_error(std::string(".ptau section ") + what + ": point " + std::to_string(bad) + " is not on the curve");
    };
    uint32_t* fl = (uint32_t*)flag.p;
    refuse(first_invalid_point<dev::Fq>(g1b.p, N, b1, fl), "12 (lTauG1)");
    refuse(first_invalid_point<dev::Fq>(g1b.p + N * 64, N, b1, fl), "14 (lAlphaTauG1)");
    refuse(first_invalid_point<dev::Fq>(g1b.p + 2 * N * 64, N, b1, fl), "15 (lBetaTauG1)");
    g2b.alloc(N * 128);
    CUDA_OK(cudaMemcpy(g2b.p, ptau_basis(v, 13, log_n), N * 128, cudaMemcpyHostToDevice));
    refuse(first_invalid_point<dev::Fq2>(g2b.p, N, b2, fl), "13 (lTauG2)");

    signal_sums<dev::Fq>(g1b.p, a_ptr, a_terms, coefs_dev, zk->A, st);
    signal_sums<dev::Fq>(g1b.p, ab_ptr, b_terms, coefs_dev, zk->B1, st);
    signal_sums<dev::Fq2>(g2b.p, ab_ptr, b_terms, coefs_dev, zk->B2, st);
    signal_sums<dev::Fq>(g1b.p, cc_ptr, c_terms, coefs_dev, zk->C, st);
    g2b.release();
    zk->ic.resize(l + 1);
    CUDA_OK(cudaMemcpy(zk->ic.data(), zk->C.p, sizeof(G1AffineH) * (l + 1), cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemset(zk->C.p, 0, sizeof(G1AffineH) * (l + 1)));

    // H_i = point 2i + 1 of the size-2N lTauG1 basis:  L_{2i+1}^{(2N)}(tau) = (tau^2N - 1)/(2N) g omega^i / (tau - g omega^i)
    // = -L_i(tau/g) Z(tau) / 2, the engine's H scalar (setup_host.cpp) at delta = 1 (g a primitive 2N-th root, g^2 = omega)
    g1b.release();
    h_table_config(zk.get(), N);
    zk->H.alloc((size_t)zk->h_levels * N * sizeof(dev::G1Affine));
    CUDA_OK(cudaMemcpy2D(zk->H.p, 64, ptau_basis(v, 12, log_n + 1) + 64, 128, 64, N, cudaMemcpyHostToDevice));
    refuse(first_invalid_point<dev::Fq>(zk->H.p, N, b1, fl), "12 (lTauG1, size-2N basis)");
    DevBuf scratch;
    scratch.alloc((size_t)SETUP_SLAB * sizeof(dev::G1XYZZ));
    build_h_levels(zk.get(), N, scratch.p, st);
    g_last_setup_timing = SetupTiming{host_ms, ms_since(t1)};
    return zk.release();
}

// ------------------------------------------------------------------------------------------------ zke_zkey_contribute
static zke_zkey* do_zkey_contribute(const zke_zkey* prev, const uint8_t* secret32) {
    const Fr sf = contribution_secret(secret32);
    const U256 s = sf.to_u256();
    CUDA_OK(cudaSetDevice(prev->device));
    select_device(prev->device);
    const uint32_t m = prev->n_vars;
    const size_t N = (size_t)1 << prev->log_n;
    std::unique_ptr<zke_zkey> zk(new zke_zkey());
    zk->n_vars = prev->n_vars; zk->n_public = prev->n_public; zk->log_n = prev->log_n; zk->device = prev->device;
    zk->toy = prev->toy && !prev->delta_one;   // a key of the seeded setup stays a toy: its tau is known
    zk->delta_one = false;
    zk->alpha1 = prev->alpha1; zk->beta1 = prev->beta1; zk->beta2 = prev->beta2; zk->gamma2 = prev->gamma2; zk->ic = prev->ic;
    zk->has_coefs = prev->has_coefs;
    zk->a_ptr = prev->a_ptr; zk->a_var = prev->a_var; zk->a_coef = prev->a_coef;
    zk->b_ptr = prev->b_ptr; zk->b_var = prev->b_var; zk->b_coef = prev->b_coef; zk->coefs = prev->coefs;
    zk->delta1 = G1JacH::from_affine(prev->delta1).mul(s).to_affine();
    zk->delta2 = G2JacH::from_affine(prev->delta2).mul(s).to_affine();

    auto copy = [&](DevBuf& dst, const DevBuf& src, size_t bytes) { dst.alloc(bytes); CUDA_OK(cudaMemcpy(dst.p, src.p, bytes, cudaMemcpyDeviceToDevice)); };
    copy(zk->A, prev->A, (size_t)m * 64);
    copy(zk->B1, prev->B1, (size_t)m * 64);
    copy(zk->B2, prev->B2, (size_t)m * 128);
    cudaStream_t st = nullptr;
    DevBuf s_inv, scratch;
    s_inv.upload(std::vector<U256>{sf.inv().to_u256()});
    scratch.alloc((size_t)SETUP_SLAB * sizeof(dev::G1XYZZ));
    auto scale = [&](const uint8_t* in, size_t n, uint8_t* out) {   // out = s^-1 in, slab by slab
        for (size_t off = 0; off < n; off += SETUP_SLAB)
            scale_each<dev::Fq>(in + 64 * off, std::min<size_t>(SETUP_SLAB, n - off), s_inv.p, 0, scratch.p, out + 64 * off, st);
        CUDA_OK(cudaStreamSynchronize(st));
    };
    zk->C.alloc((size_t)m * 64);
    scale(prev->C.p, m, zk->C.p);        // the public rows are infinity and stay so
    zk->cfg_h = prev->cfg_h; zk->h_levels = prev->h_levels;
    zk->H.alloc((size_t)zk->h_levels * N * sizeof(dev::G1Affine));
    scale(prev->H.p, N, zk->H.p);
    build_h_levels(zk.get(), N, scratch.p, st);
    return zk.release();
}

// ------------------------------------------------------------------------------------------------ zke_zkey_check_contribution
// 128-bit weights from a 16-byte seed (SplitMix64 streams keyed by both halves)
static void derive_weights(const uint8_t* rand16, size_t n, std::vector<U256>& out) {
    uint64_t k0, k1;
    memcpy(&k0, rand16, 8); memcpy(&k1, rand16 + 8, 8);
    auto mix = [](uint64_t z) {
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    };
    out.resize(n);
    for (size_t i = 0; i < n; ++i) {
        const uint64_t a = mix(k0 + 0x9E3779B97F4A7C15ull * (2 * i + 1)) ^ mix(k1 ^ (0xD1B54A32D192ED03ull * (i + 1)));
        const uint64_t b = mix(k1 + 0x9E3779B97F4A7C15ull * (2 * i + 2)) ^ mix(k0 ^ (0xD1B54A32D192ED03ull * (i + 7)));
        out[i] = U256{{a, b | 1, 0, 0}};    // never zero
    }
}

// 1: next follows from prev by one or more contributions; 0: it does not (reason in `why`)
static int do_check_contribution(const zke_zkey* a, const zke_zkey* b, const uint8_t* rand16, std::string& why) {
    if (a->device != b->device) throw std::runtime_error("the two keys live on different devices");
    if (a->n_vars != b->n_vars || a->n_public != b->n_public || a->log_n != b->log_n) { why = "the keys have different shapes (signals, public signals or domain)"; return 0; }
    if (!a->has_coefs || !b->has_coefs) throw std::runtime_error("a key of the seeded setup carries no coefficient matrices; write and load it first");
    if (!g1_eq(a->alpha1, b->alpha1) || !g1_eq(a->beta1, b->beta1) || !g2_eq(a->beta2, b->beta2) || !g2_eq(a->gamma2, b->gamma2)) {
        why = "header points alpha, beta or gamma differ"; return 0;
    }
    for (size_t j = 0; j < a->ic.size(); ++j) if (!g1_eq(a->ic[j], b->ic[j])) { why = "IC point " + std::to_string(j) + " differs"; return 0; }
    {
        auto same_rows = [&](const std::vector<uint32_t>& pa, const std::vector<uint32_t>& va, const std::vector<uint32_t>& ca,
                             const std::vector<uint32_t>& pb, const std::vector<uint32_t>& vb, const std::vector<uint32_t>& cb) {
            if (pa != pb || va != vb) return false;
            for (size_t k = 0; k < ca.size(); ++k) if (u256_cmp(a->coefs[ca[k]], b->coefs[cb[k]]) != 0) return false;
            return true;
        };
        if (!same_rows(a->a_ptr, a->a_var, a->a_coef, b->a_ptr, b->a_var, b->a_coef) ||
            !same_rows(a->b_ptr, a->b_var, a->b_coef, b->b_ptr, b->b_var, b->b_coef)) { why = "the coefficient matrices differ"; return 0; }
    }
    CUDA_OK(cudaSetDevice(a->device));
    select_device(a->device);
    const uint32_t m = a->n_vars, l = a->n_public;
    const size_t N = (size_t)1 << a->log_n;
    DevBuf flag;
    flag.alloc(4);
    auto differ = [&](const DevBuf& x, const DevBuf& y, size_t bytes, size_t point_bytes) -> int64_t {
        const uint32_t words = (uint32_t)(bytes / 16);
        if (!words) return -1;
        const int64_t first = first_flagged((uint32_t*)flag.p, [&](uint32_t* f) {
            dev::words_differ_kernel<<<(words + 255) / 256, 256>>>((const uint4*)x.p, (const uint4*)y.p, words, f);
        });
        return first < 0 ? -1 : first * 16 / (int64_t)point_bytes;
    };
    int64_t d;
    if ((d = differ(a->A, b->A, (size_t)m * 64, 64)) >= 0) { why = "A point " + std::to_string(d) + " differs"; return 0; }
    if ((d = differ(a->B1, b->B1, (size_t)m * 64, 64)) >= 0) { why = "B1 point " + std::to_string(d) + " differs"; return 0; }
    if ((d = differ(a->B2, b->B2, (size_t)m * 128, 128)) >= 0) { why = "B2 point " + std::to_string(d) + " differs"; return 0; }

    // delta1' and delta2' have the same discrete log: e(delta1', G2) == e(G1, delta2')
    if (b->delta1.is_inf() || b->delta2.is_inf() || !g2_in_subgroup(b->delta2)) { why = "delta is not a valid group element"; return 0; }
    {
        G1AffineH neg_g1 = g1_generator();
        neg_g1.y = neg_g1.y.neg();
        if (!pairing_product_is_one({{b->delta1, g2_generator()}, {neg_g1, b->delta2}})) { why = "delta1 and delta2 have different discrete logarithms"; return 0; }
    }
    // L and H scaled by one common factor, the inverse of delta's: e(X', delta2') == e(X, delta2) for
    // X = sum_i r_i L_i + sum_j t_j H_j with random 128-bit weights
    std::vector<U256> wc, wh;
    derive_weights(rand16, (size_t)m + N, wc);
    wh.assign(wc.begin() + m, wc.end());
    wc.resize(m);
    for (uint32_t j = 0; j <= l; ++j) wc[j] = U256{{0, 0, 0, 0}};    // the public rows of C are infinity
    auto x_of = [&](const zke_zkey* k) {
        return G1JacH::from_affine(weighted_sum<dev::Fq, G1AffineH>(k->C.p, wc)).add(G1JacH::from_affine(weighted_sum<dev::Fq, G1AffineH>(k->H.p, wh))).to_affine();
    };
    const G1AffineH xa = x_of(a), xb = x_of(b);
    G1AffineH neg_xa = xa;
    neg_xa.y = neg_xa.y.neg();
    if (xa.is_inf() != xb.is_inf() || !pairing_product_is_one({{xb, b->delta2}, {neg_xa, a->delta2}})) {
        why = "the L and H points are not the previous key's scaled by the inverse of the new delta"; return 0;
    }
    return 1;
}

// ------------------------------------------------------------------------------------------------ toy .ptau writer
// x^i for i < n (threads start at x^beg)
static std::vector<Fr> powers_of(const Fr& x, size_t n) {
    std::vector<Fr> out(n);
    const unsigned T = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; ++t)
        th.emplace_back([&, t]() {
            const size_t beg = n * t / T, end = n * (t + 1) / T;
            if (beg >= end) return;
            Fr w = x.pow(U256{{(uint64_t)beg, 0, 0, 0}});
            for (size_t i = beg; i < end; ++i) { out[i] = w; w = w * x; }
        });
    for (auto& x2 : th) x2.join();
    return out;
}

static int64_t do_ptau_toy(uint32_t power, const uint8_t* tab96, int device, uint8_t* out, size_t cap) {
    if (power < 1 || power > PTAU_MAX_POWER) throw std::runtime_error("power must lie in [1, 28]");
    const int order[] = {1, 2, 3, 4, 5, 6, 7, 12, 13, 14, 15};
    auto sec_bytes = [&](int s) -> size_t { return s == 1 ? PTAU_HEADER_BYTES : s == 7 ? 4 : ptau_section_bytes(s, power); };
    size_t total = 12;
    for (int s : order) total += 12 + sec_bytes(s);
    if (!out) return (int64_t)total;
    if (cap < total) return -2;
    Fr tox[3];
    for (int i = 0; i < 3; ++i) {
        U256 x;
        memcpy(x.v, tab96 + 32 * i, 32);
        if (x.is_zero() || u256_cmp(x, fr_params().p) >= 0) throw std::runtime_error("tau, alpha and beta must lie in [1, r)");
        tox[i] = Fr::from_u256(x);
    }
    const Fr tau = tox[0], alpha = tox[1], beta = tox[2];
    const size_t n = (size_t)1 << power;
    if (tau.pow(U256{{(uint64_t)n, 0, 0, 0}}) == Fr::one()) throw std::runtime_error("tau lies in an evaluation domain of this power");
    select_device(device);
    DevBuf t1, t2, scal, scratch, pts;
    t1.upload(window_table<Fq>(g1_generator()));
    t2.upload(window_table<Fq2>(g2_generator()));
    scratch.alloc((size_t)SETUP_SLAB * sizeof(dev::G2XYZZ));
    pts.alloc((size_t)SETUP_SLAB * sizeof(dev::G2Affine));
    cudaStream_t st = nullptr;

    BinWriter w{out};
    auto sec_hdr = [&](int s) { w.section(s, sec_bytes(s)); };
    // [k_i]_1 or [k_i]_2 for the scalars k, appended at w.p
    auto emit = [&](const std::vector<Fr>& k, bool g2) {
        const std::vector<U256> std_k = to_standard(k);
        scal.upload(std_k);
        const size_t ps = g2 ? 128 : 64;
        for (size_t off = 0; off < k.size(); off += SETUP_SLAB) {
            const uint32_t cnt = (uint32_t)std::min<size_t>(SETUP_SLAB, k.size() - off);
            if (g2) dev::fixed_base_batch<dev::Fq2>(t2.p, scal.p + 32 * off, cnt, scratch.p, pts.p, st);
            else dev::fixed_base_batch<dev::Fq>(t1.p, scal.p + 32 * off, cnt, scratch.p, pts.p, st);
            CHECK_LAUNCH();
            CUDA_OK(cudaMemcpy(w.p, pts.p, cnt * ps, cudaMemcpyDeviceToHost));
            w.p += cnt * ps;
        }
    };
    auto scaled = [](std::vector<Fr> v, const Fr& k) { for (auto& x : v) x = x * k; return v; };

    w.header("ptau", 1, (uint32_t)(sizeof order / sizeof order[0]));
    sec_hdr(1); w.u32(32); w.bytes(fq_params().p.v, 32); w.u32(power); w.u32(power);
    {
        std::vector<Fr> pw = powers_of(tau, 2 * n - 1);
        sec_hdr(2); emit(pw, false);
        pw.resize(n);
        sec_hdr(3); emit(pw, true);
        sec_hdr(4); emit(scaled(pw, alpha), false);
        sec_hdr(5); emit(scaled(pw, beta), false);
        sec_hdr(6); emit({beta}, true);
        sec_hdr(7); w.u32(0);
    }
    {
        // Lagrange bases of the domains 2^0 .. 2^power at tau, back to back
        std::vector<Fr> lag, part;
        lag.reserve(2 * n - 1);
        for (uint32_t k = 0; k <= power; ++k) {
            const size_t nk = (size_t)1 << k;
            const Fr numer = (tau.pow(U256{{(uint64_t)nk, 0, 0, 0}}) - Fr::one()) * Fr::from_u64(nk).inv();
            lagrange_like(tau, numer, k, part);
            lag.insert(lag.end(), part.begin(), part.end());
        }
        sec_hdr(12); emit(lag, false);
        sec_hdr(13); emit(lag, true);
        sec_hdr(14); emit(scaled(lag, alpha), false);
        sec_hdr(15); emit(scaled(lag, beta), false);
    }
    CUDA_OK(cudaStreamSynchronize(st));
    return (int64_t)(w.p - out);
}

extern "C" {

int zke_ptau_info(const zke_circuit* c, const void* ptau, size_t len, uint32_t* power, uint64_t* offsets16, uint64_t* sizes16,
                  char* err, size_t errcap) {
    try {
        const PtauView v = parse_ptau((const uint8_t*)ptau, len);
        if (c) ptau_fits_circuit(v, c->c);
        if (power) *power = v.power;
        for (int s = 0; s < 16; ++s) {
            if (offsets16) offsets16[s] = v.sec[s].p ? (uint64_t)(v.sec[s].p - v.base) : 0;
            if (sizes16) sizes16[s] = v.sec[s].p ? (uint64_t)v.sec[s].n : 0;
        }
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

zke_zkey* zke_zkey_from_ptau(const zke_circuit* c, const void* ptau, size_t len, int device, char* err, size_t errcap) {
    try {
        if (!c) throw std::runtime_error("null circuit");
        return do_zkey_from_ptau(c, (const uint8_t*)ptau, len, device);
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}

int zke_zkey_from_ptau_timing(double* host_ms, double* gpu_ms) {
    if (host_ms) *host_ms = g_last_setup_timing.host_ms;
    if (gpu_ms) *gpu_ms = g_last_setup_timing.gpu_ms;
    return 0;
}

zke_zkey* zke_zkey_contribute(const zke_zkey* prev, const uint8_t* secret32, char* err, size_t errcap) {
    try {
        if (!prev || !secret32) throw std::runtime_error("null argument");
        return do_zkey_contribute(prev, secret32);
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}

int zke_zkey_check_contribution(const zke_zkey* prev, const zke_zkey* next, const uint8_t* rand16, char* err, size_t errcap) {
    try {
        if (!prev || !next) throw std::runtime_error("null key");
        uint8_t seed[16];
        if (rand16) memcpy(seed, rand16, 16);
        else random_bytes(seed, 16);
        std::string why;
        const int ok = do_check_contribution(prev, next, seed, why);
        set_err(err, errcap, why);
        return ok;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int64_t zke_ptau_toy(uint32_t power, const uint8_t* tau_alpha_beta96, int device, uint8_t* out, size_t cap, char* err, size_t errcap) {
    try {
        if (!tau_alpha_beta96) throw std::runtime_error("null argument");
        const int64_t r = do_ptau_toy(power, tau_alpha_beta96, device, out, cap);
        if (r == -2) set_err(err, errcap, "output buffer too small");
        return r;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

}  // extern "C"
