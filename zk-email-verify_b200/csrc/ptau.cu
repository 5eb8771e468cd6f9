// Phase 1 of the Powers-of-Tau ceremony on the GPU: `snarkjs powersoftau new`, `contribute`, `prepare phase2` and the
// algebraic part of `verify`.  Included at the end of engine.cu after setup.cu, whose file layout (top of setup.cu) and
// reader (parse_ptau) it uses.  An UNPREPARED file holds sections 1-7, a PREPARED one also 12-15.
//
//   new        header (power, ceremonyPower = power), sections 2-6 filled with the generators, section 7 = count 0.
//   contribute tauG1[i] *= t^i, tauG2[i] *= t^i, alphaTauG1[i] *= a t^i, betaTauG1[i] *= b t^i, betaG2 *= b for secrets
//              (t, a, b).  Every point is multiplied by its own scalar on the device (ec_ntt.cuh: scale_each_kernel).
//              The output is unprepared (sections 12-15 of a prepared input would be stale and are dropped); sections 1
//              and 7 are copied byte for byte.  The contribution is NOT recorded in section 7: no snarkjs transcript
//              (contribution records, BLAKE2b challenge hashes, proofs of knowledge) is written, as for zkey
//              contributions, so snarkjs cannot audit a chain made here.  The public part of the contribution is the
//              receipt ([t]_2, [a]_2, [b]_2), which zke_ptau_verify checks against the previous file.
//   prepare    for every k <= power, the size-2^k Lagrange basis of each family is the inverse DFT of its first 2^k points,
//              L_i = n^-1 sum_j omega^(-ij) T_j (omega = fr_root_of_unity(k)), computed by the point transform of
//              ec_ntt.cuh in HBM, one launch per stage.
//   verify     points on their curves and in range, G2 points in the order-r subgroup, the generators at index 0; every
//              family a sequence of consecutive powers of one tau (one random linear combination and one pairing
//              equation per family); the Lagrange sections (one group equation per family, no pairing); optionally the
//              link to the previous file through the receipt.
#include "ec_ntt.cuh"

namespace zke { namespace dev {

// first index i < n whose G2 point is not in the order-r subgroup -> atomicMin(bad); the points must be on the twist
__global__ void __launch_bounds__(128)
g2_subgroup_kernel(const uint8_t* __restrict__ pts, uint32_t n, uint32_t* bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && !g2_in_subgroup(G2Affine::load(pts + sizeof(G2Affine) * (size_t)i))) atomicMin(bad, i);
}

} }  // namespace zke::dev

namespace {

const int PTAU_PHASE1_SECTIONS[] = {2, 3, 4, 5, 6};

size_t ptau_point_bytes(int s) { return s == 3 || s == 6 || s == 13 ? 128 : 64; }
std::string ptau_sec_label(int s) { return "section " + std::to_string(s) + " (" + ptau_section_name(s) + ")"; }

// -1 if every G2 point of pts[0, n) (on the twist) lies in the order-r subgroup, else the first index that does not
int64_t first_off_subgroup(const uint8_t* pts, size_t n, uint32_t* flag) {
    if (!n) return -1;
    return first_flagged(flag, [&](uint32_t* f) { dev::g2_subgroup_kernel<<<(unsigned)((n + 127) / 128), 128>>>(pts, (uint32_t)n, f); });
}

// "" if the n points of section s at pts (device; index 0 = point `first` of the section) are valid, else the reason
std::string section_points_problem(int s, const uint8_t* pts, size_t n, size_t first, uint32_t* flag) {
    const bool g2 = ptau_point_bytes(s) == 128;
    const int64_t bad = g2 ? first_invalid_point<dev::Fq2>(pts, n, g2_twist_b(), flag) : first_invalid_point<dev::Fq>(pts, n, Fq::from_u64(3), flag);
    if (bad >= 0) return ".ptau " + ptau_sec_label(s) + ": point " + std::to_string(first + bad) + " is not on the curve";
    if (g2) {
        const int64_t off = first_off_subgroup(pts, n, flag);
        if (off >= 0) return ".ptau " + ptau_sec_label(s) + ": point " + std::to_string(first + off) + " is not in the order-r subgroup";
    }
    return "";
}

// Section s of the contribution: point i of `in` (host) times factor * pw[i], slab by slab, into `out` (host).
// Every input point is validated on the device first, G2 points also against the subgroup.
template <class F>
void contribute_family(int s, const uint8_t* in, size_t n, const std::vector<Fr>& pw, const Fr& factor, bool scaled, uint8_t* out, uint32_t* flag) {
    const size_t ps = sizeof(dev::Affine<F>);
    const size_t slab = std::min<size_t>(SETUP_SLAB, n);
    DevBuf pts, x, k;
    pts.alloc(slab * ps);
    x.alloc(slab * sizeof(dev::XYZZ<F>));
    std::vector<Fr> ks(slab);
    cudaStream_t st = nullptr;
    for (size_t off = 0; off < n; off += slab) {
        const size_t cnt = std::min(slab, n - off);
        ks.assign(pw.begin() + off, pw.begin() + off + cnt);
        if (scaled) for (Fr& v : ks) v = v * factor;
        k.upload(to_standard(ks));
        CUDA_OK(cudaMemcpy(pts.p, in + off * ps, cnt * ps, cudaMemcpyHostToDevice));
        const std::string bad = section_points_problem(s, pts.p, cnt, off, flag);
        if (!bad.empty()) throw std::runtime_error(bad);
        scale_each<F>(pts.p, cnt, k.p, 1, x.p, pts.p, st);
        CUDA_OK(cudaMemcpy(out + off * ps, pts.p, cnt * ps, cudaMemcpyDeviceToHost));
    }
}

// The Lagrange bases of sizes 1, 2, ..., 2^power of one family, back to back into `out` (host): `first` holds the
// family's first 2^power points (host), tw the twiddles omega_N^-j, j < N/2 (device, standard form, N = 2^power).
template <class F>
void lagrange_family(int s, const uint8_t* first, uint32_t power, const DevBuf& tw, uint8_t* out, uint32_t* flag) {
    const size_t N = (size_t)1 << power, ps = sizeof(dev::Affine<F>);
    DevBuf in, a, x, n_inv;
    in.alloc(N * ps);
    a.alloc(N * ps);
    x.alloc(N * sizeof(dev::XYZZ<F>));
    CUDA_OK(cudaMemcpy(in.p, first, N * ps, cudaMemcpyHostToDevice));
    const std::string bad = section_points_problem(s, in.p, N, 0, flag);
    if (!bad.empty()) throw std::runtime_error(bad);
    cudaStream_t st = nullptr;
    for (uint32_t k = 0; k <= power; ++k) {
        const uint32_t n = 1u << k;
        n_inv.upload(std::vector<U256>{Fr::from_u64(n).inv().to_u256()});
        // X[i] = n^-1 T[bitrev(i)], then one launch per stage
        dev::scale_each_kernel<F><<<(n + 127) / 128, 128, 0, st>>>(in.p, n, (const uint32_t*)n_inv.p, 0, (int)k, x.p);
        ZKE_COUNT_LAUNCH(1);
        dev::xyzz_to_affine_batch<F>(x.p, n, a.p, st);
        for (uint32_t m = 1; m < n; m <<= 1) {
            dev::point_ntt_stage_kernel<F><<<(n / 2 + 127) / 128, 128, 0, st>>>(a.p, n / 2, m, (const uint32_t*)tw.p, (uint32_t)(N / (2 * m)), x.p);
            ZKE_COUNT_LAUNCH(1);
            dev::xyzz_to_affine_batch<F>(x.p, n, a.p, st);
        }
        CHECK_LAUNCH();
        CUDA_OK(cudaMemcpy(out + (size_t)(n - 1) * ps, a.p, n * ps, cudaMemcpyDeviceToHost));
    }
}

// In-place inverse DFT over Fr, natural order in and out, scaled by 1/n: a_i <- n^-1 sum_j omega^(-ij) a_j
void fr_intt(std::vector<Fr>& a, unsigned log_n) {
    const size_t n = (size_t)1 << log_n;
    if (n == 1) return;
    for (size_t i = 1, j = 0; i < n; ++i) {
        size_t bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) std::swap(a[i], a[j]);
    }
    const std::vector<Fr> tw = powers_of(fr_root_of_unity(log_n).inv(), n / 2);
    const unsigned T = n >= (1u << 14) ? std::max(1u, std::min(16u, std::thread::hardware_concurrency())) : 1u;
    for (size_t len = 2; len <= n; len <<= 1) {
        const size_t half = len / 2, stride = n / len;
        auto run = [&](size_t beg, size_t end) {   // butterflies [beg, end) of n / 2
            for (size_t t = beg; t < end; ++t) {
                const size_t j = t % half, i0 = (t / half) * len + j, i1 = i0 + half;
                const Fr v = a[i1] * tw[j * stride];
                a[i1] = a[i0] - v;
                a[i0] = a[i0] + v;
            }
        };
        if (T == 1) run(0, n / 2);
        else {
            std::vector<std::thread> th;
            for (unsigned t = 0; t < T; ++t) th.emplace_back(run, n / 2 * t / T, n / 2 * (t + 1) / T);
            for (auto& x : th) x.join();
        }
    }
    const Fr n_inv = Fr::from_u64(n).inv();
    for (Fr& v : a) v = v * n_inv;
}

template <class H>
H neg_point(H p) { if (!p.is_inf()) p.y = p.y.neg(); return p; }

G1AffineH g1_at(const PtauView& v, int s, size_t i) { G1AffineH p; memcpy(&p, v.sec[s].p + 64 * i, 64); return p; }
G2AffineH g2_at(const PtauView& v, int s, size_t i) { G2AffineH p; memcpy(&p, v.sec[s].p + 128 * i, 128); return p; }

}  // namespace

// ------------------------------------------------------------------------------------------------ new
static int64_t do_ptau_new(uint32_t power, uint8_t* out, size_t cap) {
    if (power < 1 || power > PTAU_MAX_POWER) throw std::runtime_error("power must lie in [1, 28]");
    size_t total = 12 + 12 + PTAU_HEADER_BYTES + 12 + 4;
    for (int s : PTAU_PHASE1_SECTIONS) total += 12 + ptau_section_bytes(s, power);
    if (!out) return (int64_t)total;
    if (cap < total) return -2;
    const G1AffineH g1 = g1_generator();
    const G2AffineH g2 = g2_generator();
    BinWriter w{out};
    w.header("ptau", 1, 7);
    w.section(1, PTAU_HEADER_BYTES); w.u32(32); w.bytes(fq_params().p.v, 32); w.u32(power); w.u32(power);
    for (int s : PTAU_PHASE1_SECTIONS) {
        const size_t bytes = ptau_section_bytes(s, power), ps = ptau_point_bytes(s);
        w.section(s, bytes);
        for (size_t i = 0; i < bytes / ps; ++i) w.bytes(ps == 64 ? (const void*)&g1 : (const void*)&g2, ps);
    }
    w.section(7, 4); w.u32(0);
    return (int64_t)(w.p - out);
}

// ------------------------------------------------------------------------------------------------ contribute
static size_t unprepared_bytes(const PtauView& v) {
    size_t total = 12 + 12 + v.sec[1].n + 12 + v.sec[7].n;
    for (int s : PTAU_PHASE1_SECTIONS) total += 12 + v.sec[s].n;
    return total;
}

static int64_t do_ptau_contribute(const uint8_t* in, size_t len, const uint8_t* secrets96, int device, uint8_t* out, size_t cap,
                                  uint8_t* receipt384) {
    const PtauView v = parse_ptau(in, len, true);
    if (!v.sec[7].p) throw std::runtime_error(".ptau section 7 (contributions) is missing");
    const size_t total = unprepared_bytes(v);
    if (!out) return (int64_t)total;
    if (cap < total) return -2;
    Fr sec[3];
    const char* names[3] = {"tau", "alpha", "beta"};
    for (int i = 0; i < 3; ++i) {
        if (secrets96) { sec[i] = contribution_secret(secrets96 + 32 * i, names[i]); continue; }
        U256 r;
        do random_scalar(r); while (r.v[0] < 2 && !r.v[1] && !r.v[2] && !r.v[3]);
        sec[i] = Fr::from_u256(r);
    }
    const Fr tau = sec[0], alpha = sec[1], beta = sec[2];
    const G2AffineH beta2 = g2_at(v, 6, 0);
    if (!g2_valid(beta2) || !g2_in_subgroup(beta2)) throw std::runtime_error(".ptau section 6 (betaG2): the point is not in G2");
    select_device(device);
    const size_t n = (size_t)1 << v.power;
    DevBuf flag;
    flag.alloc(4);

    BinWriter w{out};
    w.header("ptau", 1, 7);
    w.section(1, v.sec[1].n); w.bytes(v.sec[1].p, v.sec[1].n);
    {
        const std::vector<Fr> pw = powers_of(tau, 2 * n - 1);
        w.section(2, v.sec[2].n); contribute_family<dev::Fq>(2, v.sec[2].p, 2 * n - 1, pw, Fr::one(), false, w.p, (uint32_t*)flag.p); w.p += v.sec[2].n;
        w.section(3, v.sec[3].n); contribute_family<dev::Fq2>(3, v.sec[3].p, n, pw, Fr::one(), false, w.p, (uint32_t*)flag.p); w.p += v.sec[3].n;
        w.section(4, v.sec[4].n); contribute_family<dev::Fq>(4, v.sec[4].p, n, pw, alpha, true, w.p, (uint32_t*)flag.p); w.p += v.sec[4].n;
        w.section(5, v.sec[5].n); contribute_family<dev::Fq>(5, v.sec[5].p, n, pw, beta, true, w.p, (uint32_t*)flag.p); w.p += v.sec[5].n;
    }
    const G2AffineH nb = G2JacH::from_affine(beta2).mul(beta.to_u256()).to_affine();
    w.section(6, 128); w.bytes(&nb, 128);
    w.section(7, v.sec[7].n); w.bytes(v.sec[7].p, v.sec[7].n);
    if (receipt384)
        for (int i = 0; i < 3; ++i) {
            const G2AffineH r = G2JacH::from_affine(g2_generator()).mul(sec[i].to_u256()).to_affine();
            memcpy(receipt384 + 128 * i, &r, 128);
        }
    return (int64_t)(w.p - out);
}

// ------------------------------------------------------------------------------------------------ prepare
struct PrepareTiming { double g1_ms = 0, g2_ms = 0; };
static thread_local PrepareTiming g_last_prepare_timing;

static int64_t do_ptau_prepare(const uint8_t* in, size_t len, int device, uint8_t* out, size_t cap) {
    const PtauView v = parse_ptau(in, len, true);
    if (v.prepared) throw std::runtime_error(".ptau is already prepared (it holds sections 12-15)");
    if (!v.sec[7].p) throw std::runtime_error(".ptau section 7 (contributions) is missing");
    size_t total = unprepared_bytes(v);
    for (int s : {12, 13, 14, 15}) total += 12 + ptau_section_bytes(s, v.power);
    if (!out) return (int64_t)total;
    if (cap < total) return -2;
    const size_t N = (size_t)1 << v.power;
    select_device(device);
    {   // the largest transform: 2^power G2 points as input, working copy and XYZZ stage output, plus the twiddles
        const size_t need = N * (2 * sizeof(dev::G2Affine) + sizeof(dev::G2XYZZ)) + N / 2 * 32;
        size_t free_b = 0, total_b = 0;
        CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
        if (need > free_b)
            throw std::runtime_error("prepare of a power-" + std::to_string(v.power) + " .ptau needs " + std::to_string(need) +
                                     " bytes of device memory for its largest transform; " + std::to_string(free_b) + " are free");
    }
    DevBuf flag, tw;
    flag.alloc(4);
    tw.upload(to_standard(powers_of(fr_root_of_unity(v.power).inv(), N / 2)));

    BinWriter w{out};
    w.header("ptau", 1, 11);
    for (int s : {1, 2, 3, 4, 5, 6, 7}) { w.section(s, v.sec[s].n); w.bytes(v.sec[s].p, v.sec[s].n); }
    const auto t0 = std::chrono::steady_clock::now();
    double g2_ms = 0;
    for (int s : {12, 13, 14, 15}) {
        w.section(s, ptau_section_bytes(s, v.power));
        const int src = s - 10;
        if (s == 13) {
            const auto t1 = std::chrono::steady_clock::now();
            lagrange_family<dev::Fq2>(src, v.sec[src].p, v.power, tw, w.p, (uint32_t*)flag.p);
            g2_ms = ms_since(t1);
        } else lagrange_family<dev::Fq>(src, v.sec[src].p, v.power, tw, w.p, (uint32_t*)flag.p);
        w.p += ptau_section_bytes(s, v.power);
    }
    g_last_prepare_timing = PrepareTiming{ms_since(t0) - g2_ms, g2_ms};
    return (int64_t)(w.p - out);
}

// ------------------------------------------------------------------------------------------------ verify
// 1: the file passes every check; 0: it does not (the first failure in `why`)
static int do_ptau_verify(const uint8_t* f, size_t len, const uint8_t* pf, size_t plen, const uint8_t* receipt, const uint8_t* seed, int device,
                          std::string& why) {
    const PtauView v = parse_ptau(f, len, true);
    PtauView pv;
    if (pf) pv = parse_ptau(pf, plen, true);
    const size_t n = (size_t)1 << v.power;
    const G1AffineH g1 = g1_generator();
    const G2AffineH g2 = g2_generator();
    select_device(device);
    DevBuf flag;
    flag.alloc(4);

    // points: every section on its curve and in range, G2 in the subgroup; the phase-1 families stay on the device
    DevBuf d[6];
    for (int s : {2, 3, 4, 5}) {
        d[s].alloc(v.sec[s].n);
        CUDA_OK(cudaMemcpy(d[s].p, v.sec[s].p, v.sec[s].n, cudaMemcpyHostToDevice));
        why = section_points_problem(s, d[s].p, v.sec[s].n / ptau_point_bytes(s), 0, (uint32_t*)flag.p);
        if (!why.empty()) return 0;
    }
    const G2AffineH beta2 = g2_at(v, 6, 0);
    if (!g2_valid(beta2)) { why = ".ptau section 6 (betaG2): the point is not on the curve"; return 0; }
    if (!g2_in_subgroup(beta2)) { why = ".ptau section 6 (betaG2): the point is not in the order-r subgroup"; return 0; }
    if (v.prepared)
        for (int s : {12, 13, 14, 15}) {
            DevBuf l;
            l.alloc(v.sec[s].n);
            CUDA_OK(cudaMemcpy(l.p, v.sec[s].p, v.sec[s].n, cudaMemcpyHostToDevice));
            why = section_points_problem(s, l.p, v.sec[s].n / ptau_point_bytes(s), 0, (uint32_t*)flag.p);
            if (!why.empty()) return 0;
        }
    if (!g1_eq(g1_at(v, 2, 0), g1)) { why = ".ptau section 2 (tauG1): point 0 is not the G1 generator"; return 0; }
    if (!g2_eq(g2_at(v, 3, 0), g2)) { why = ".ptau section 3 (tauG2): point 0 is not the G2 generator"; return 0; }
    const G1AffineH tau1 = g1_at(v, 2, 1);
    const G2AffineH tau2 = g2_at(v, 3, 1);
    if (tau1.is_inf()) { why = ".ptau section 2 (tauG1): point 1 is infinity (tau = 0)"; return 0; }
    const G1AffineH neg_g1 = neg_point(g1);

    // consecutive powers: with random 128-bit weights r_i, sum r_i P_{i+1} = tau * sum r_i P_i, checked by one pairing
    {
        std::vector<U256> r;
        derive_weights(seed, 2 * n - 2, r);
        for (int s : {2, 4, 5}) {
            const size_t cnt = v.sec[s].n / 64 - 1;
            const std::vector<U256> rs(r.begin(), r.begin() + cnt);
            const G1AffineH lo = weighted_sum<dev::Fq, G1AffineH>(d[s].p, rs), hi = weighted_sum<dev::Fq, G1AffineH>(d[s].p + 64, rs);
            if (!pairing_product_is_one({{hi, g2}, {neg_point(lo), tau2}})) {
                why = ".ptau " + ptau_sec_label(s) + ": the points are not consecutive powers of the tau of tauG2[1]"; return 0;
            }
        }
        const std::vector<U256> rs(r.begin(), r.begin() + (n - 1));
        const G2AffineH lo = weighted_sum<dev::Fq2, G2AffineH>(d[3].p, rs), hi = weighted_sum<dev::Fq2, G2AffineH>(d[3].p + 128, rs);
        if (!pairing_product_is_one({{tau1, lo}, {neg_g1, hi}})) {
            why = ".ptau section 3 (tauG2): the points are not consecutive powers of the tau of tauG1[1]"; return 0;
        }
        if (!pairing_product_is_one({{g1_at(v, 5, 0), g2}, {neg_g1, beta2}})) {
            why = ".ptau section 6 (betaG2): its beta is not the beta of betaTauG1[0]"; return 0;
        }
    }

    // Lagrange sections: sum_k sum_i r_ki L^(k)_i = sum_j c_j T_j with c_j = sum_{k: j < 2^k} 2^-k sum_i r_ki omega_k^(-ij)
    if (v.prepared) {
        std::vector<U256> r;
        uint8_t seed2[16];
        for (int i = 0; i < 16; ++i) seed2[i] = seed[i] ^ 0x5a;
        derive_weights(seed2, 2 * n - 1, r);
        std::vector<Fr> c(n, Fr::zero()), part;
        for (uint32_t k = 0; k <= v.power; ++k) {
            const size_t nk = (size_t)1 << k;
            part.resize(nk);
            for (size_t i = 0; i < nk; ++i) part[i] = Fr::from_u256(r[nk - 1 + i]);
            fr_intt(part, k);
            for (size_t j = 0; j < nk; ++j) c[j] = c[j] + part[j];
        }
        const std::vector<U256> cs = to_standard(c);
        for (int s : {12, 13, 14, 15}) {
            const int src = s - 10;
            DevBuf l;
            l.alloc(v.sec[s].n);
            CUDA_OK(cudaMemcpy(l.p, v.sec[s].p, v.sec[s].n, cudaMemcpyHostToDevice));
            bool same;
            if (s == 13) same = g2_eq(weighted_sum<dev::Fq2, G2AffineH>(l.p, r), weighted_sum<dev::Fq2, G2AffineH>(d[src].p, cs));
            else same = g1_eq(weighted_sum<dev::Fq, G1AffineH>(l.p, r), weighted_sum<dev::Fq, G1AffineH>(d[src].p, cs));
            if (!same) { why = ".ptau " + ptau_sec_label(s) + ": the points are not the Lagrange bases of " + ptau_sec_label(src); return 0; }
        }
    }

    // link to the previous file: e(next P, G2) = e(prev P, [secret]_2) for tauG1[1], alphaTauG1[0], betaTauG1[0]
    if (pf) {
        if (pv.power != v.power) { why = "the previous file has power " + std::to_string(pv.power) + ", this one " + std::to_string(v.power); return 0; }
        const char* names[3] = {"tau", "alpha", "beta"};
        const int sec[3] = {2, 4, 5};
        const size_t idx[3] = {1, 0, 0};
        for (int i = 0; i < 3; ++i) {
            G2AffineH rp;
            memcpy(&rp, receipt + 128 * i, 128);
            const std::string what = std::string("receipt point [") + names[i] + "]_2";
            if (rp.is_inf()) { why = what + " is infinity"; return 0; }
            if (!g2_valid(rp)) { why = what + " is not on the curve"; return 0; }
            if (!g2_in_subgroup(rp)) { why = what + " is not in the order-r subgroup"; return 0; }
            if (g2_eq(rp, g2)) { why = what + " is the generator (a secret of one)"; return 0; }
            const G1AffineH prev_p = g1_at(pv, sec[i], idx[i]);
            if (!g1_valid(prev_p)) { why = "the previous file's " + ptau_sec_label(sec[i]) + " point " + std::to_string(idx[i]) + " is not on the curve"; return 0; }
            if (!pairing_product_is_one({{g1_at(v, sec[i], idx[i]), g2}, {neg_point(prev_p), rp}})) {
                why = ".ptau " + ptau_sec_label(sec[i]) + ": point " + std::to_string(idx[i]) + " is not the previous file's times the receipt's " + names[i];
                return 0;
            }
        }
    }
    why.clear();
    return 1;
}

extern "C" {

int64_t zke_ptau_new(uint32_t power, uint8_t* out, size_t cap, char* err, size_t errcap) {
    try {
        const int64_t r = do_ptau_new(power, out, cap);
        if (r == -2) set_err(err, errcap, "output buffer too small");
        return r;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int64_t zke_ptau_contribute(const void* ptau, size_t len, const uint8_t* secrets96, int device, uint8_t* out, size_t cap, uint8_t* receipt384,
                            char* err, size_t errcap) {
    try {
        const int64_t r = do_ptau_contribute((const uint8_t*)ptau, len, secrets96, device, out, cap, receipt384);
        if (r == -2) set_err(err, errcap, "output buffer too small");
        return r;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int64_t zke_ptau_prepare(const void* ptau, size_t len, int device, uint8_t* out, size_t cap, char* err, size_t errcap) {
    try {
        const int64_t r = do_ptau_prepare((const uint8_t*)ptau, len, device, out, cap);
        if (r == -2) set_err(err, errcap, "output buffer too small");
        return r;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_ptau_prepare_timing(double* g1_ms, double* g2_ms) {
    if (g1_ms) *g1_ms = g_last_prepare_timing.g1_ms;
    if (g2_ms) *g2_ms = g_last_prepare_timing.g2_ms;
    return 0;
}

int zke_ptau_verify(const void* ptau, size_t len, const void* prev, size_t prev_len, const uint8_t* receipt384, const uint8_t* rand16,
                    int device, char* err, size_t errcap) {
    try {
        if (!ptau) throw std::runtime_error("null argument");
        if (!prev != !receipt384) throw std::runtime_error("the previous file and the receipt go together: give both or neither");
        uint8_t seed[16];
        if (rand16) memcpy(seed, rand16, 16);
        else random_bytes(seed, 16);
        std::string why;
        const int ok = do_ptau_verify((const uint8_t*)ptau, len, (const uint8_t*)prev, prev_len, receipt384, seed, device, why);
        set_err(err, errcap, why);
        return ok;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

}  // extern "C"
