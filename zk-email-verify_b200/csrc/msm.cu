// Multi-scalar multiplication over BN254 G1 / G2 for the Groth16 prover (pi_A, pi_B, pi_B1, pi_C, H - snarkjs
// groth16_prove step 5, SURVEY 3.2; the reference's implementation is wasmcurves' chunked `multiExpAffine`).
//
// Pipeline (all on one stream, no host synchronisation inside):
//   classify   : scalars 0 / points at infinity are dropped, scalars == 1 go to a "ones" list that is summed by a
//                plain tree reduction (>= 90 % of EmailVerifier witness scalars are bits, SURVEY 8(d)), the rest
//                go to the Pippenger list.
//   pippenger  : signed c-bit digits -> point indices sorted by bucket (counting sort, in two levels for large
//                bucket sets: msm_sort.cuh) -> buckets cut into chunks of at most CHUNK entries so that a
//                heavy bucket (small-valued witness scalars pile into few buckets) is spread over many threads ->
//                per-chunk XYZZ accumulation with coalesced 32/64-byte affine point loads -> per-group running sums
//                -> per-window tree reduction -> Horner over windows.
// The accumulation kernels are bound by the integer (IMAD) pipe, not HBM: one mixed addition is 10 Fq products
// (~300 IMAD each) per 64-byte point (SURVEY 8(d) "Which roofline bounds what").
#include "device_engine.cuh"
#include "msm.cuh"
#include "msm_ba.cuh"
#include "msm_sort.cuh"
#if defined(ZKE_MSM_G1)
#include "msm_tc.cuh"
#endif
#include <algorithm>
#include <cstdlib>
#include <stdexcept>

namespace zke {
namespace dev {

static const int LIST_FANIN = 32;   // affine points summed per thread at the first level of the unit-scalar reduction
static const int TREE_FANIN = 8;    // XYZZ partial sums combined per thread at the following levels
// (chunk = max bucket entries accumulated by one thread, group = buckets per running-sum thread: MsmConfig)

__device__ __forceinline__ Fr load_scalar(const uint8_t* scalars, uint32_t i) { return Fr::load(scalars + 32ull * i); }

// ---------------------------------------------------------------- classify
template <class F>
__global__ void classify_kernel(const uint8_t* __restrict__ points, const uint8_t* __restrict__ scalars, uint32_t n,
                                uint32_t* ones_list, uint32_t* gen_list, uint32_t* counters /* [0]=ones, [1]=general */) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s = load_scalar(scalars, i);
    if (s.is_zero()) return;
    Affine<F> p = Affine<F>::load(points + sizeof(Affine<F>) * (size_t)i);
    if (p.is_inf()) return;
    bool one = s.v[0] == 1 && (s.v[1] | s.v[2] | s.v[3] | s.v[4] | s.v[5] | s.v[6] | s.v[7]) == 0;
    if (one) ones_list[atomicAdd(&counters[0], 1u)] = i;
    else gen_list[atomicAdd(&counters[1], 1u)] = i;
}

// ---------------------------------------------------------------- list sums
// out[t] = sum of points[list[t*FANIN .. )]   (list == nullptr: identity)
template <class F>
__global__ void sum_affine_list_kernel(const uint8_t* __restrict__ points, const uint32_t* __restrict__ list,
                                       const uint32_t* __restrict__ count_ptr, uint32_t count_fixed, uint8_t* out) {
    const uint32_t count = count_ptr ? *count_ptr : count_fixed;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_out = max(1u, (count + LIST_FANIN - 1) / LIST_FANIN);   // slot 0 is always written
    if (t >= n_out) return;
    XYZZ<F> acc = XYZZ<F>::inf();
    // strided assignment keeps a warp's point loads close together
    for (uint32_t k = t; k < count; k += n_out) {
        uint32_t idx = list ? list[k] : k;
        acc.madd(Affine<F>::load(points + sizeof(Affine<F>) * (size_t)idx), false);
    }
    acc.store(out + sizeof(XYZZ<F>) * (size_t)t);
}

// tree step: out[t] = sum_{k = t, t + n_out, ...} in[k].  The size of `in` is derived on the device from the list
// length: level 0 has ceil(count / LIST_FANIN) partial sums, each further level divides by TREE_FANIN (min 1).
// If pad_to > 0 this is the last level: slots [n_out, pad_to) are filled with the point at infinity.
__device__ __forceinline__ uint32_t tree_level_size(uint32_t count, uint32_t level) {
    uint32_t n = max(1u, (count + LIST_FANIN - 1) / LIST_FANIN);
    for (uint32_t d = 0; d < level; ++d) n = max(1u, (n + TREE_FANIN - 1) / TREE_FANIN);
    return n;
}
template <class F>
__global__ void sum_xyzz_kernel(const uint8_t* __restrict__ in, const uint32_t* __restrict__ count_ptr, uint32_t count_fixed,
                                uint32_t level, uint32_t pad_to, uint8_t* out) {
    const uint32_t count = count_ptr ? *count_ptr : count_fixed;
    const uint32_t n_in = tree_level_size(count, level), n_out = tree_level_size(count, level + 1);
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_out) {
        if (t < pad_to) XYZZ<F>::inf().store(out + sizeof(XYZZ<F>) * (size_t)t);
        return;
    }
    XYZZ<F> acc = XYZZ<F>::inf();
    for (uint32_t k = t; k < n_in; k += n_out) acc.add(XYZZ<F>::load(in + sizeof(XYZZ<F>) * (size_t)k));
    acc.store(out + sizeof(XYZZ<F>) * (size_t)t);
}

// ---------------------------------------------------------------- digits
struct Digits {
    int c, n_windows;
    uint32_t half;   // 2^(c-1) buckets per window
    uint32_t chunk;  // max bucket entries accumulated by one thread
    uint32_t group;  // buckets per running-sum thread
    uint32_t window_bucket_stride;  // half, or 0 when all windows share one bucket set (precomputed tables)
    uint32_t window_point_stride;   // 0, or n when window j uses table level j
};

__device__ __forceinline__ uint32_t window_bits(const Fr& s, int bit, int c) {
    const int w = bit >> 5, b = bit & 31;
    uint64_t two = s.v[w];
    if (w + 1 < 8) two |= (uint64_t)s.v[w + 1] << 32;
    return (uint32_t)((two >> b) & ((1u << c) - 1));
}

// Scalars above r/2 are replaced by r - s with the point negated: "negative" witness values (index differences,
// signed carries, -1 coefficients folded into signals) then have one or two non-zero digits instead of 32 identical
// high digits that would all land in the same few buckets.
__device__ __forceinline__ bool minimal_magnitude(Fr& s) {
    const FieldConsts& C = FR_C;
    // s > (r-1)/2  <=>  2s >= r + 1  <=> 2s > r
    Fr n;
    n.v[0] = sub_cc(C.mod[0], s.v[0]);
#pragma unroll
    for (int i = 1; i < 8; ++i) n.v[i] = subc_cc(C.mod[i], s.v[i]);
    (void)subc(0, 0);
    // compare n < s (n = r - s): lexicographic from the top limb
    bool less = false, decided = false;
#pragma unroll
    for (int i = 7; i >= 0; --i) {
        if (!decided && n.v[i] != s.v[i]) { less = n.v[i] < s.v[i]; decided = true; }
    }
    if (less) { s = n; return true; }
    return false;
}

// calls f(window, bucket_in_window, negative) for every non-zero signed digit of (+/-) s
template <class Fn>
__device__ __forceinline__ void for_each_digit(Fr s, const Digits& D, Fn f) {
    const bool flip = minimal_magnitude(s);
    uint32_t carry = 0;
    for (int j = 0; j < D.n_windows; ++j) {
        uint32_t raw = window_bits(s, j * D.c, D.c) + carry;
        if (raw > D.half) {                      // digit = raw - 2^c  (negative or zero), carry 1
            carry = 1;
            const uint32_t mag = (1u << D.c) - raw;   // raw == 2^c (all-ones window plus carry) gives digit 0
            if (mag) f(j, mag - 1, !flip);
        } else {
            carry = 0;
            if (raw) f(j, raw - 1, flip);
        }
    }
}

// ---------------------------------------------------------------- bucket sort of the digits (msm_sort.cuh)
// Output: hist[b] entries in bucket b, offsets[b] = exclusive scan of hist (offsets[n_buckets] = total), entries in
// bucket order, each (window * window_point_stride + point index) | sign << 31.  The order inside a bucket is not fixed.
// A one-level counting sort costs one global atomic and one 4-byte write to a random place in a 200+ MB array per
// digit (13 x 2^22 digits for the H MSM): every store of a warp lands in 32 different sectors, and the L2 write
// transactions, not the bytes, set its time.  Both scatter passes below therefore first sort a block's digits in
// shared memory and then store them in runs: consecutive threads write consecutive words of a partition (coarse pass,
// ~26 digits per partition and block for the H MSM) or of a bucket (fine pass, ~8 per bucket and tile).
static const int SORT_PART_BITS = 8;
static const uint32_t SORT_PARTS = 1u << SORT_PART_BITS;
static const int SORT_MAX_FINE_BITS = 11;     // buckets per partition: n_buckets <= 2^19
static const int SORT_THREADS = 256;          // coarse passes, fine count pass
static const int SORT_FINE_THREADS = 512;     // fine scatter pass
static const uint32_t SORT_STAGE = 6656;      // digits a coarse block stages (6 B each): 512 scalars x 13 windows
static const uint32_t SORT_TILE = 16384;      // digits of a fine tile
// the one-level counting sort is faster for small bucket sets (the witness MSMs: 4096 buckets), whose histogram and
// scatter targets stay in L2, and it needs fewer launches
static const uint32_t SORT_TWO_LEVEL_MIN_BUCKETS = 1u << 16;
// dynamic shared memory of the fine scatter pass: bin offsets, cursors and global positions, scan scratch, the tile
static const size_t SORT_FINE_SMEM = 4 * (3 * ((size_t)1 << SORT_MAX_FINE_BITS) + 1 + SORT_FINE_THREADS + SORT_TILE);

// in-place exclusive scan of s[0, n) by the whole block (tmp: THREADS words); s[n] = the total.  Ends synchronised.
template <int THREADS>
__device__ __forceinline__ void block_exclusive_scan(uint32_t* s, uint32_t n, uint32_t* tmp) {
    const uint32_t per = (n + THREADS - 1) / THREADS, beg = min(n, threadIdx.x * per), end = min(n, beg + per);
    uint32_t local = 0;
    for (uint32_t i = beg; i < end; ++i) local += s[i];
    tmp[threadIdx.x] = local;
    __syncthreads();
    for (uint32_t off = 1; off < THREADS; off <<= 1) {
        const uint32_t v = threadIdx.x >= off ? tmp[threadIdx.x - off] : 0;
        __syncthreads();
        tmp[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = tmp[threadIdx.x] - local;
    for (uint32_t i = beg; i < end; ++i) { const uint32_t v = s[i]; s[i] = run; run += v; }
    if (threadIdx.x == THREADS - 1) s[n] = tmp[THREADS - 1];
    __syncthreads();
}

// mat[part][block] = the block's digits per partition; block k takes scalars [k * tile, (k + 1) * tile) of the list
static __global__ void __launch_bounds__(SORT_THREADS)
sort_coarse_count_kernel(const uint8_t* __restrict__ scalars, const uint32_t* __restrict__ list, const uint32_t* __restrict__ count_ptr,
                         uint32_t count_fixed, Digits D, int fine_bits, uint32_t n_parts, uint32_t tile, uint32_t* mat) {
    __shared__ uint32_t s_bin[SORT_PARTS];
    const uint32_t count = count_ptr ? *count_ptr : count_fixed;
    for (uint32_t i = threadIdx.x; i < n_parts; i += SORT_THREADS) s_bin[i] = 0;
    __syncthreads();
    const uint32_t beg = blockIdx.x * tile, end = min(count, beg + tile);
    for (uint32_t t = beg + threadIdx.x; t < end; t += SORT_THREADS) {
        Fr s = load_scalar(scalars, list ? list[t] : t);
        for_each_digit(s, D, [&](int j, uint32_t b, bool) { atomicAdd(&s_bin[((uint32_t)j * D.window_bucket_stride + b) >> fine_bits], 1u); });
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n_parts; i += SORT_THREADS) mat[(size_t)i * gridDim.x + blockIdx.x] = s_bin[i];
}

// off = the scanned coarse matrix.  The block recomputes the digits of the count pass (tile * n_windows <= SORT_STAGE),
// sorts them by partition in shared memory and stores each partition's run at off[part][block] in stage / stage_fine.
static __global__ void __launch_bounds__(SORT_THREADS)
sort_coarse_scatter_kernel(const uint8_t* __restrict__ scalars, const uint32_t* __restrict__ list, const uint32_t* __restrict__ count_ptr,
                           uint32_t count_fixed, Digits D, int fine_bits, uint32_t n_parts, uint32_t tile, const uint32_t* __restrict__ off,
                           uint32_t* __restrict__ stage, uint16_t* __restrict__ stage_fine) {
    __shared__ uint32_t s_base[SORT_PARTS + 1], s_cur[SORT_PARTS], s_goff[SORT_PARTS], s_tmp[SORT_THREADS];
    __shared__ uint32_t s_word[SORT_STAGE];
    __shared__ uint16_t s_fine[SORT_STAGE];
    const uint32_t count = count_ptr ? *count_ptr : count_fixed;
    for (uint32_t p = threadIdx.x; p < SORT_PARTS; p += SORT_THREADS) {
        const size_t c = (size_t)p * gridDim.x + blockIdx.x;      // the next cell in scan order holds the next offset
        s_goff[p] = p < n_parts ? off[c] : 0;
        s_base[p] = p < n_parts ? off[c + 1] - off[c] : 0;
    }
    __syncthreads();
    block_exclusive_scan<SORT_THREADS>(s_base, SORT_PARTS, s_tmp);
    for (uint32_t p = threadIdx.x; p < SORT_PARTS; p += SORT_THREADS) s_cur[p] = s_base[p];
    __syncthreads();
    const uint32_t beg = blockIdx.x * tile, end = min(count, beg + tile);
    for (uint32_t t = beg + threadIdx.x; t < end; t += SORT_THREADS) {
        const uint32_t idx = list ? list[t] : t;
        Fr s = load_scalar(scalars, idx);
        for_each_digit(s, D, [&](int j, uint32_t b, bool neg) {
            const uint32_t bucket = (uint32_t)j * D.window_bucket_stride + b;
            const uint32_t pos = atomicAdd(&s_cur[bucket >> fine_bits], 1u);
            s_word[pos] = ((uint32_t)j * D.window_point_stride + idx) | (neg ? 0x80000000u : 0u);
            s_fine[pos] = (uint16_t)(bucket & ((1u << fine_bits) - 1));
        });
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < s_base[SORT_PARTS]; i += SORT_THREADS) {
        const uint32_t p = sort_tile_part(s_base, SORT_PARTS, i);
        const uint32_t g = s_goff[p] + (i - s_base[p]);
        stage[g] = s_word[i];
        stage_fine[g] = s_fine[i];
    }
}

// part_count[p] = digits of partition p (from the scanned coarse matrix)
static __global__ void sort_part_count_kernel(const uint32_t* __restrict__ coarse_off, uint32_t coarse_blocks, uint32_t n_parts,
                                              uint32_t* part_count) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n_parts) part_count[p] = coarse_off[(size_t)(p + 1) * coarse_blocks] - coarse_off[(size_t)p * coarse_blocks];
}

// the staged digits [beg, end) of fine tile w (block w of the fine passes); false past the last tile
__device__ __forceinline__ bool sort_fine_tile(const uint32_t* coarse_off, uint32_t coarse_blocks, const uint32_t* tile_base, uint32_t n_parts,
                                               uint32_t w, uint32_t& tb, uint32_t& tiles_p, uint32_t& t, uint32_t& beg, uint32_t& end) {
    if (w >= tile_base[n_parts]) return false;
    const uint32_t p = sort_tile_part(tile_base, n_parts, w);
    tb = tile_base[p]; tiles_p = tile_base[p + 1] - tb; t = w - tb;
    beg = coarse_off[(size_t)p * coarse_blocks] + t * SORT_TILE;
    end = min(coarse_off[(size_t)(p + 1) * coarse_blocks], beg + SORT_TILE);
    return true;
}

// counts fine tile w's digits per fine bin into mat; blocks past the last tile zero their cells, so that the host can
// scan gridDim.x << fine_bits cells
static __global__ void __launch_bounds__(SORT_THREADS)
sort_fine_count_kernel(const uint32_t* __restrict__ coarse_off, uint32_t coarse_blocks, const uint32_t* __restrict__ tile_base,
                       uint32_t n_parts, int fine_bits, const uint16_t* __restrict__ stage_fine, uint32_t* mat) {
    __shared__ uint32_t s_bin[1u << SORT_MAX_FINE_BITS];
    const uint32_t n_fine = 1u << fine_bits;
    uint32_t tb, tiles_p, t, beg, end;
    if (!sort_fine_tile(coarse_off, coarse_blocks, tile_base, n_parts, blockIdx.x, tb, tiles_p, t, beg, end)) {
        for (uint32_t f = threadIdx.x; f < n_fine; f += SORT_THREADS) mat[((size_t)blockIdx.x << fine_bits) + f] = 0;
        return;
    }
    for (uint32_t f = threadIdx.x; f < n_fine; f += SORT_THREADS) s_bin[f] = 0;
    __syncthreads();
    for (uint32_t k = beg + threadIdx.x; k < end; k += SORT_THREADS) atomicAdd(&s_bin[stage_fine[k]], 1u);
    __syncthreads();
    for (uint32_t f = threadIdx.x; f < n_fine; f += SORT_THREADS) mat[sort_cell(tb, tiles_p, f, t, fine_bits)] = s_bin[f];
}

// off = the scanned fine matrix.  Sorts fine tile w by bucket in shared memory (SORT_FINE_SMEM bytes) and stores each
// bucket's run at its offset in entries.
static __global__ void __launch_bounds__(SORT_FINE_THREADS)
sort_fine_scatter_kernel(const uint32_t* __restrict__ coarse_off, uint32_t coarse_blocks, const uint32_t* __restrict__ tile_base,
                         uint32_t n_parts, int fine_bits, const uint32_t* __restrict__ stage, const uint16_t* __restrict__ stage_fine,
                         const uint32_t* __restrict__ off, uint32_t* __restrict__ entries) {
    extern __shared__ uint32_t smem[];
    const uint32_t n_fine = 1u << fine_bits;
    uint32_t* s_base = smem;                     // n_fine + 1
    uint32_t* s_cur = s_base + n_fine + 1;       // n_fine
    uint32_t* s_goff = s_cur + n_fine;           // n_fine
    uint32_t* s_tmp = s_goff + n_fine;           // SORT_FINE_THREADS
    uint32_t* s_word = s_tmp + SORT_FINE_THREADS;   // SORT_TILE
    uint32_t tb, tiles_p, t, beg, end;
    if (!sort_fine_tile(coarse_off, coarse_blocks, tile_base, n_parts, blockIdx.x, tb, tiles_p, t, beg, end)) return;
    for (uint32_t f = threadIdx.x; f < n_fine; f += SORT_FINE_THREADS) {
        const size_t c = sort_cell(tb, tiles_p, f, t, fine_bits);   // the next cell in scan order holds the next offset
        s_goff[f] = off[c];
        s_base[f] = off[c + 1] - off[c];
    }
    __syncthreads();
    block_exclusive_scan<SORT_FINE_THREADS>(s_base, n_fine, s_tmp);
    for (uint32_t f = threadIdx.x; f < n_fine; f += SORT_FINE_THREADS) s_cur[f] = s_base[f];
    __syncthreads();
    for (uint32_t k = beg + threadIdx.x; k < end; k += SORT_FINE_THREADS) s_word[atomicAdd(&s_cur[stage_fine[k]], 1u)] = stage[k];
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < end - beg; i += SORT_FINE_THREADS) {
        const uint32_t f = sort_tile_part(s_base, n_fine, i);
        entries[s_goff[f] + (i - s_base[f])] = s_word[i];
    }
}

// offsets[b] for b in [0, n_buckets], hist[b] = offsets[b + 1] - offsets[b] (hist[n_buckets] = 0)
static __global__ void sort_offsets_kernel(uint32_t n_buckets, int fine_bits, const uint32_t* __restrict__ coarse_off, uint32_t coarse_blocks,
                                           const uint32_t* __restrict__ tile_base, const uint32_t* __restrict__ fine_off,
                                           uint32_t* hist, uint32_t* offsets) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b > n_buckets) return;
    const uint32_t o = sort_bucket_offset(b, n_buckets, fine_bits, coarse_off, coarse_blocks, tile_base, fine_off);
    offsets[b] = o;
    hist[b] = b < n_buckets ? sort_bucket_offset(b + 1, n_buckets, fine_bits, coarse_off, coarse_blocks, tile_base, fine_off) - o : 0;
}

// one-level counting sort (small bucket sets): global histogram, its exclusive scan, scatter with a cursor per bucket
static __global__ void digit_hist_kernel(const uint8_t* __restrict__ scalars, const uint32_t* __restrict__ list,
                                         const uint32_t* __restrict__ count_ptr, uint32_t count_fixed, Digits D, uint32_t* hist) {
    const uint32_t count = count_ptr ? *count_ptr : count_fixed;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < count; t += gridDim.x * blockDim.x) {
        const uint32_t idx = list ? list[t] : t;
        Fr s = load_scalar(scalars, idx);
        for_each_digit(s, D, [&](int j, uint32_t b, bool) { atomicAdd(&hist[(uint32_t)j * D.window_bucket_stride + b], 1u); });
    }
}
static __global__ void digit_scatter_kernel(const uint8_t* __restrict__ scalars, const uint32_t* __restrict__ list,
                                            const uint32_t* __restrict__ count_ptr, uint32_t count_fixed, Digits D,
                                            const uint32_t* __restrict__ offsets, uint32_t* cursor, uint32_t* entries) {
    const uint32_t count = count_ptr ? *count_ptr : count_fixed;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < count; t += gridDim.x * blockDim.x) {
        const uint32_t idx = list ? list[t] : t;
        Fr s = load_scalar(scalars, idx);
        for_each_digit(s, D, [&](int j, uint32_t b, bool neg) {
            const uint32_t bucket = (uint32_t)j * D.window_bucket_stride + b;
            const uint32_t pos = offsets[bucket] + atomicAdd(&cursor[bucket], 1u);
            entries[pos] = ((uint32_t)j * D.window_point_stride + idx) | (neg ? 0x80000000u : 0u);
        });
    }
}

// the batched-affine path works on the points themselves: sorted[k] = the (sign-adjusted) point of entry k
template <class F>
__global__ void __launch_bounds__(256)
gather_points_kernel(const uint32_t* __restrict__ entries, const uint32_t* __restrict__ offsets, uint32_t n_buckets,
                     const uint8_t* __restrict__ points, Affine<F>* __restrict__ sorted) {
    const uint32_t total = offsets[n_buckets];
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
        const uint32_t e = entries[k];
        Affine<F> p = Affine<F>::load(points + sizeof(Affine<F>) * (size_t)(e & 0x7fffffffu));
        if (e >> 31) p.y = p.y.neg();
        p.store(sorted + k);
    }
}

// ---------------------------------------------------------------- exclusive scan over the bucket array
// out[i] = sum_{k<i} f(in[k]); out[n] = total.  f = identity (chunk == 0) or ceil(x / chunk).
// Three phases: per-tile totals, single-block scan of the tile totals, per-tile rescan with the tile's base.
static const int SCAN_TILE = 2048;   // elements per block (256 threads x 8)
static const uint32_t PASS_FANIN = 32;   // partial sums combined per thread in the extra reduction passes
// number of items a bucket with v entries has after the first pass (chunks of `chunk` entries) and `levels` further
// passes of fan-in PASS_FANIN; chunk == 0 means "the raw entry count"
__device__ __forceinline__ uint32_t scan_f(uint32_t v, uint32_t chunk, uint32_t levels = 0) {
    if (!chunk) return v;
    v = (v + chunk - 1) / chunk;
    for (uint32_t l = 0; l < levels; ++l) v = (v + PASS_FANIN - 1) / PASS_FANIN;
    return v;
}

static __global__ void __launch_bounds__(256) scan_tile_totals_kernel(const uint32_t* __restrict__ in, uint32_t n, uint32_t chunk, uint32_t levels, uint32_t* tile_sums) {
    __shared__ uint32_t red[256];
    const uint32_t base = blockIdx.x * SCAN_TILE;
    uint32_t local = 0;
    for (uint32_t i = threadIdx.x; i < SCAN_TILE; i += 256) if (base + i < n) local += scan_f(in[base + i], chunk, levels);
    red[threadIdx.x] = local;
    __syncthreads();
    for (uint32_t off = 128; off > 0; off >>= 1) { if (threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off]; __syncthreads(); }
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = red[0];
}
// exclusive scan of up to 1024 * 8 values in one block (in place)
static __global__ void __launch_bounds__(1024) scan_small_kernel(uint32_t* data, uint32_t n, uint32_t* total_out) {
    __shared__ uint32_t sums[1024];
    const uint32_t tid = threadIdx.x;
    const uint32_t per = (n + 1023) / 1024;
    const uint32_t beg = min(n, tid * per), end = min(n, beg + per);
    uint32_t local = 0;
    for (uint32_t i = beg; i < end; ++i) local += data[i];
    sums[tid] = local;
    __syncthreads();
    for (uint32_t off = 1; off < 1024; off <<= 1) {
        uint32_t v = tid >= off ? sums[tid - off] : 0;
        __syncthreads();
        sums[tid] += v;
        __syncthreads();
    }
    uint32_t run = sums[tid] - local;
    for (uint32_t i = beg; i < end; ++i) { uint32_t v = data[i]; data[i] = run; run += v; }
    if (tid == 1023 && total_out) *total_out = sums[1023];
}
static __global__ void __launch_bounds__(256) scan_tile_apply_kernel(const uint32_t* __restrict__ in, uint32_t n, uint32_t chunk, uint32_t levels,
                                                              const uint32_t* __restrict__ tile_base, uint32_t* out) {
    __shared__ uint32_t sums[256];
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * 8;
    uint32_t v[8], local = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { v[k] = (base + k < n) ? scan_f(in[base + k], chunk, levels) : 0; local += v[k]; }
    sums[threadIdx.x] = local;
    __syncthreads();
    for (uint32_t off = 1; off < 256; off <<= 1) {
        uint32_t x = threadIdx.x >= off ? sums[threadIdx.x - off] : 0;
        __syncthreads();
        sums[threadIdx.x] += x;
        __syncthreads();
    }
    uint32_t run = tile_base[blockIdx.x] + sums[threadIdx.x] - local;
#pragma unroll
    for (int k = 0; k < 8; ++k) { if (base + k < n) out[base + k] = run; run += v[k]; }
}
// host helper: `tiles` is scratch for ceil(n / SCAN_TILE) + 1 words
static void exclusive_scan(const uint32_t* in, uint32_t n, uint32_t chunk, uint32_t levels, uint32_t* out, uint32_t* tiles, cudaStream_t st) {
    const uint32_t n_tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    scan_tile_totals_kernel<<<n_tiles, 256, 0, st>>>(in, n, chunk, levels, tiles);
    scan_small_kernel<<<1, 1024, 0, st>>>(tiles, n_tiles, out + n);
    scan_tile_apply_kernel<<<n_tiles, 256, 0, st>>>(in, n, chunk, levels, tiles, out);
    ZKE_COUNT_LAUNCH(3);
}

// ---------------------------------------------------------------- bucket sort: workspace and launches
struct DigitSort {
    uint32_t n_buckets, n_parts, coarse_tile, coarse_blocks, fine_blocks;
    int fine_bits = 0;
    size_t max_entries, coarse_cells, fine_cells;
    uint32_t *coarse, *coarse_off, *part_count, *tile_base, *fine, *fine_off, *tiles, *stage;
    uint16_t* stage_fine;
    DigitSort(uint32_t n, int n_windows, uint32_t n_buckets_, size_t max_entries_) : n_buckets(n_buckets_), max_entries(max_entries_) {
        while ((n_buckets - 1) >> fine_bits >= SORT_PARTS) ++fine_bits;      // at most SORT_PARTS partitions
        n_parts = sort_parts(n_buckets, fine_bits);
        coarse_tile = SORT_STAGE / (uint32_t)n_windows;      // a scalar has at most n_windows digits
        coarse_blocks = std::max(1u, (n + coarse_tile - 1) / coarse_tile);
        fine_blocks = (uint32_t)(max_entries / SORT_TILE + n_parts);    // >= sum over partitions of ceil(size / SORT_TILE)
        coarse_cells = (size_t)n_parts * coarse_blocks;
        fine_cells = (size_t)fine_blocks << fine_bits;
    }
    // carves the sort's arrays out of the workspace through take(bytes)
    template <class Take> void place(Take take) {
        coarse = (uint32_t*)take(4 * (coarse_cells + 1));
        coarse_off = (uint32_t*)take(4 * (coarse_cells + 1));
        part_count = (uint32_t*)take(4 * ((size_t)n_parts + 1));
        tile_base = (uint32_t*)take(4 * ((size_t)n_parts + 1));
        fine = (uint32_t*)take(4 * (fine_cells + 1));
        fine_off = (uint32_t*)take(4 * (fine_cells + 1));
        tiles = (uint32_t*)take(4 * (std::max(coarse_cells, fine_cells) / SCAN_TILE + 2));
        stage = (uint32_t*)take(4 * max_entries);
        stage_fine = (uint16_t*)take(2 * max_entries);
    }
    // hist / offsets / entries (layout above) of the digits of scalars[list[0 .. *count_ptr)] (list == nullptr:
    // scalars[0 .. count_fixed)); count_fixed is also the upper bound of *count_ptr
    void run(const uint8_t* scalars, const uint32_t* list, const uint32_t* count_ptr, uint32_t count_fixed, const Digits& D,
             uint32_t* hist, uint32_t* offsets, uint32_t* entries, cudaStream_t st) const {
        sort_coarse_count_kernel<<<coarse_blocks, SORT_THREADS, 0, st>>>(scalars, list, count_ptr, count_fixed, D, fine_bits, n_parts, coarse_tile, coarse);
        exclusive_scan(coarse, (uint32_t)coarse_cells, 0, 0, coarse_off, tiles, st);
        sort_coarse_scatter_kernel<<<coarse_blocks, SORT_THREADS, 0, st>>>(scalars, list, count_ptr, count_fixed, D, fine_bits, n_parts, coarse_tile, coarse_off, stage, stage_fine);
        sort_part_count_kernel<<<(n_parts + 255) / 256, 256, 0, st>>>(coarse_off, coarse_blocks, n_parts, part_count);
        exclusive_scan(part_count, n_parts, SORT_TILE, 0, tile_base, tiles, st);
        sort_fine_count_kernel<<<fine_blocks, SORT_THREADS, 0, st>>>(coarse_off, coarse_blocks, tile_base, n_parts, fine_bits, stage_fine, fine);
        exclusive_scan(fine, (uint32_t)fine_cells, 0, 0, fine_off, tiles, st);
        cudaFuncSetAttribute(sort_fine_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SORT_FINE_SMEM);
        sort_fine_scatter_kernel<<<fine_blocks, SORT_FINE_THREADS, SORT_FINE_SMEM, st>>>(coarse_off, coarse_blocks, tile_base, n_parts, fine_bits, stage, stage_fine, fine_off, entries);
        sort_offsets_kernel<<<(n_buckets + 256) / 256, 256, 0, st>>>(n_buckets, fine_bits, coarse_off, coarse_blocks, tile_base, fine_off, hist, offsets);
        ZKE_COUNT_LAUNCH(6);
    }
};

static __global__ void fill_work_kernel(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ chunk_off, uint32_t n_buckets,
                                 uint32_t CHUNK, uint32_t levels, uint32_t* work_bucket) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_buckets) return;
    const uint32_t nch = scan_f(hist[b], CHUNK, levels);
    for (uint32_t i = 0; i < nch; ++i) work_bucket[chunk_off[b] + i] = b;
}

// ---------------------------------------------------------------- chunk order (counting sort by size)
// Bucket sizes are Poisson distributed (104 +- 10 entries for the H points) and a warp runs as long as its largest
// chunk: with chunks taken in index order only 26 of 32 lanes are active on average (ncu: 26.1 threads per
// instruction).  The chunks are therefore counting-sorted by size, largest first: `order[t]` is the chunk thread t
// works on, so the 32 lanes of a warp - and the 4 warps of a block - get chunks of (nearly) equal length, and the
// longest chunks start first.  Two small kernels around the existing exclusive scan: per-block histograms stored
// bin-major (mat[bin][block]) so that ONE flat scan yields every block's write offset for every size.
static const int ORDER_BLOCK = 256;
__device__ __forceinline__ uint32_t chunk_size_of(uint32_t w, const uint32_t* hist, const uint32_t* chunk_off, const uint32_t* work_bucket, uint32_t CHUNK) {
    const uint32_t b = work_bucket[w];
    return min(CHUNK, hist[b] - (w - chunk_off[b]) * CHUNK);
}
static __global__ void __launch_bounds__(ORDER_BLOCK)
chunk_key_hist_kernel(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ chunk_off, const uint32_t* __restrict__ work_bucket,
                      uint32_t n_buckets, uint32_t CHUNK, uint32_t* mat) {
    extern __shared__ uint32_t s_hist[];      // CHUNK bins: bin = CHUNK - size (size >= 1)
    const uint32_t total = chunk_off[n_buckets];
    for (uint32_t i = threadIdx.x; i < CHUNK; i += ORDER_BLOCK) s_hist[i] = 0;
    __syncthreads();
    const uint32_t w = blockIdx.x * ORDER_BLOCK + threadIdx.x;
    if (w < total) atomicAdd(&s_hist[CHUNK - chunk_size_of(w, hist, chunk_off, work_bucket, CHUNK)], 1u);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < CHUNK; i += ORDER_BLOCK) mat[(size_t)i * gridDim.x + blockIdx.x] = s_hist[i];
}
static __global__ void __launch_bounds__(ORDER_BLOCK)
chunk_order_kernel(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ chunk_off, const uint32_t* __restrict__ work_bucket,
                   uint32_t n_buckets, uint32_t CHUNK, const uint32_t* __restrict__ mat_off, uint32_t* order) {
    __shared__ uint32_t s_key[ORDER_BLOCK];
    const uint32_t total = chunk_off[n_buckets];
    const uint32_t w = blockIdx.x * ORDER_BLOCK + threadIdx.x;
    const uint32_t key = w < total ? CHUNK - chunk_size_of(w, hist, chunk_off, work_bucket, CHUNK) : 0xffffffffu;
    s_key[threadIdx.x] = key;
    __syncthreads();
    if (w >= total) return;
    uint32_t local = 0;
    for (uint32_t j = 0; j < threadIdx.x; ++j) local += s_key[j] == key;
    order[mat_off[(size_t)key * gridDim.x + blockIdx.x] + local] = w;
}

// one thread per chunk: partial[w] = sum of (+/-) points of chunk w = order[thread]
template <class F, int MINB>
__global__ void __launch_bounds__(128, MINB)
chunk_sum_kernel(const uint8_t* __restrict__ points, const uint32_t* __restrict__ entries, const uint32_t* __restrict__ offsets,
                 const uint32_t* __restrict__ hist, const uint32_t* __restrict__ chunk_off, const uint32_t* __restrict__ work_bucket,
                 const uint32_t* __restrict__ order, uint32_t n_buckets, uint32_t CHUNK, uint8_t* partial) {
    const uint32_t total = chunk_off[n_buckets];
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const uint32_t w = order[t];
        const uint32_t b = work_bucket[w];
        const uint32_t ci = w - chunk_off[b];
        const uint32_t beg = offsets[b] + ci * CHUNK;
        const uint32_t end = min(offsets[b] + hist[b], beg + CHUNK);
        XYZZ<F> acc = XYZZ<F>::inf();
        for (uint32_t k = beg; k < end; ++k) {
            const uint32_t e = entries[k];
            acc.madd(Affine<F>::load(points + sizeof(Affine<F>) * (size_t)(e & 0x7fffffffu)), (e >> 31) != 0);
        }
        acc.store(partial + sizeof(XYZZ<F>) * (size_t)w);
    }
}

// extra reduction pass: level `level` items of a bucket (XYZZ partial sums, contiguous at off_in[b]) are combined
// PASS_FANIN at a time into level + 1 items at off_out[b]; spreads the partial sums of a heavy bucket (many equal
// small scalars) over threads instead of leaving them to the running-sum thread
template <class F>
__global__ void __launch_bounds__(128)
partial_pass_kernel(const uint8_t* __restrict__ in, const uint32_t* __restrict__ hist, const uint32_t* __restrict__ off_in,
                    const uint32_t* __restrict__ off_out, const uint32_t* __restrict__ work_bucket, uint32_t n_buckets,
                    uint32_t CHUNK, uint32_t level, uint8_t* out) {
    const uint32_t total = off_out[n_buckets];
    for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < total; w += gridDim.x * blockDim.x) {
        const uint32_t b = work_bucket[w];
        const uint32_t i = w - off_out[b];
        const uint32_t n_in = scan_f(hist[b], CHUNK, level);
        const uint32_t beg = off_in[b] + i * PASS_FANIN, end = min(off_in[b] + n_in, beg + PASS_FANIN);
        XYZZ<F> acc = XYZZ<F>::inf();
        for (uint32_t k = beg; k < end; ++k) acc.add(XYZZ<F>::load(in + sizeof(XYZZ<F>) * (size_t)k));
        acc.store(out + sizeof(XYZZ<F>) * (size_t)w);
    }
}

// one thread per GROUP consecutive buckets of one window: sum_b (b+1) B_b restricted to the group, as
// T + first_index * S with T the in-group weighted sum and S the plain sum
// ITEMS = 0: XYZZ partial sums located by chunk_off (per-chunk sums of the XYZZ bucket kernel); 1: one XYZZ sum per
// bucket at index `bucket` (batched-affine path after bucket_finish_kernel)
template <class F, int ITEMS>
__global__ void __launch_bounds__(128)
group_sum_kernel(const uint8_t* __restrict__ partial, const uint32_t* __restrict__ hist, const uint32_t* __restrict__ chunk_off,
                 uint32_t half, uint32_t n_groups_total, uint32_t CHUNK, uint32_t levels, uint32_t GROUP, uint8_t* group_out) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups_total) return;
    const uint32_t groups_per_window = (half + GROUP - 1) / GROUP;
    const uint32_t window = g / groups_per_window, gi = g % groups_per_window;
    const uint32_t lo = gi * GROUP, hi = min(half, lo + GROUP);
    XYZZ<F> running = XYZZ<F>::inf(), total = XYZZ<F>::inf();
    for (uint32_t b = hi; b-- > lo;) {
        const uint32_t bucket = window * half + b;
        if (ITEMS == 1) {
            if (hist[bucket]) running.add(XYZZ<F>::load(partial + sizeof(XYZZ<F>) * (size_t)bucket));
        } else {
            const uint32_t nch = scan_f(hist[bucket], CHUNK, levels);
            for (uint32_t i = 0; i < nch; ++i) running.add(XYZZ<F>::load(partial + sizeof(XYZZ<F>) * (size_t)(chunk_off[bucket] + i)));
        }
        total.add(running);
    }
    // total = sum (b - lo + 1) B_b ; add lo * running  (lo < 2^15)
    if (lo && !running.is_inf()) {
        XYZZ<F> acc = XYZZ<F>::inf();
        for (int bit = 31 - __clz(lo); bit >= 0; --bit) {
            acc.dbl();
            if ((lo >> bit) & 1) acc.add(running);
        }
        total.add(acc);
    }
    total.store(group_out + sizeof(XYZZ<F>) * (size_t)g);
}

// one block per window: tree-reduce the window's group sums in place (global memory), result in slot 0
template <class F>
__global__ void __launch_bounds__(512)
window_reduce_kernel(uint8_t* group_out, uint32_t groups_per_window) {
    uint8_t* base = group_out + sizeof(XYZZ<F>) * (size_t)blockIdx.x * groups_per_window;
    uint32_t n = groups_per_window;
    while (n > 1) {
        const uint32_t halfn = (n + 1) / 2;
        for (uint32_t t = threadIdx.x; t + halfn < n; t += blockDim.x) {
            XYZZ<F> a = XYZZ<F>::load(base + sizeof(XYZZ<F>) * (size_t)t);
            a.add(XYZZ<F>::load(base + sizeof(XYZZ<F>) * (size_t)(t + halfn)));
            a.store(base + sizeof(XYZZ<F>) * (size_t)t);
        }
        __syncthreads();
        n = halfn;
    }
}

// copies slot 0 of every window (the reduced window sum) into the MSM's result block
template <class F>
__global__ void gather_windows_kernel(const uint8_t* __restrict__ group_out, uint32_t groups_per_window, uint32_t n_windows, uint8_t* out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_windows) return;
    XYZZ<F>::load(group_out + sizeof(XYZZ<F>) * (size_t)j * groups_per_window).store(out + sizeof(XYZZ<F>) * (size_t)j);
}

// one thread per bucket: XYZZ sum of the bucket's remaining affine points
template <class F>
__global__ void __launch_bounds__(128)
bucket_finish_kernel(const Affine<F>* __restrict__ pts, const uint32_t* __restrict__ hist, const uint32_t* __restrict__ off,
                     uint32_t n_buckets, uint32_t level, XYZZ<F>* __restrict__ out) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_buckets) return;
    const uint32_t n = ba_level_count(hist[b], level);
    if (n == 0) return;                      // empty bucket: never read by group_sum_kernel<.., 1>
    const Affine<F>* p = pts + off[b];
    XYZZ<F> acc = XYZZ<F>::from_affine(Affine<F>::load(p));
    Affine<F> nxt = n > 1 ? Affine<F>::load(p + 1) : Affine<F>::load(p);
    for (uint32_t i = 1; i < n; ++i) {
        const Affine<F> cur = nxt;
        if (i + 1 < n) nxt = Affine<F>::load(p + i + 1);
        acc.madd(cur, false);
    }
    acc.store(out + b);
}

// ---------------------------------------------------------------- streaming batched-affine path (msm_ba.cuh)
// entries / hist / offsets: the counting-sorted digits.  Produces the per-group running sums in group_out.
// The sweeps (forward, backward) saturate memory / the multiplier pipe and go to the lane's low-priority stream; the
// tiny kernels of the grid-wide inversion stay on the high-priority one so that they slip between other lanes' blocks.
template <class F>
static void run_ba(const MsmConfig& cfg, const uint32_t* hist, const uint32_t* offsets,
                   uint32_t n_buckets, size_t max_entries, uint32_t* tiles, uint8_t* ws, const Digits& D, uint32_t groups, uint8_t* group_out,
                   cudaStream_t st, cudaEvent_t* ev, const typename MsmPlan<F>::Heavy* heavy) {
    const int L = cfg.ba_levels;
    const size_t s1 = BaPlan<F>::slots_bound(max_entries, n_buckets, 1), s2 = BaPlan<F>::slots_bound(max_entries, n_buckets, 2);
    const size_t t1 = (s1 + BA_K - 1) / BA_K;
    uint8_t* p = ws;
    auto take = [&](size_t x) { uint8_t* r = p; p += (x + 255) & ~(size_t)255; return r; };
    Affine<F>* sorted0 = (Affine<F>*)take(sizeof(Affine<F>) * (max_entries + 1));   // first in the workspace: the scatter kernel wrote it
    F* prefix = (F*)take(sizeof(F) * s1);
    Affine<F>* ping = (Affine<F>*)take(sizeof(Affine<F>) * s1);
    Affine<F>* pong = (Affine<F>*)take(sizeof(Affine<F>) * s2);
    uint32_t* slot_bucket = (uint32_t*)take(4 * s1);
    F* tot = (F*)take(sizeof(F) * t1);
    F* binv_scratch = (F*)take(sizeof(F) * binv_scratch_elems(t1));
    const uint32_t* off[8];
    off[0] = offsets;
    for (int l = 1; l <= L; ++l) {
        uint32_t* o = (uint32_t*)take(4 * ((size_t)n_buckets + 1));
        exclusive_scan(hist, n_buckets, 1u << l, 0, o, tiles, st);     // scan of ceil(size / 2^l)
        off[l] = o;
    }
    cudaStream_t hv = (heavy && heavy->st != st) ? heavy->st : st;
    auto to_heavy = [&]() { if (hv != st) { cudaEventRecord(heavy->before, st); cudaStreamWaitEvent(hv, heavy->before, 0); } };
    auto to_light = [&]() { if (hv != st) { cudaEventRecord(heavy->after, hv); cudaStreamWaitEvent(st, heavy->after, 0); } };
    const Affine<F>* in = sorted0;
    Affine<F>* out = ping;
    for (int l = 0; l < L; ++l) {
        const size_t slots = BaPlan<F>::slots_bound(max_entries, n_buckets, l + 1);
        const uint32_t n_threads = (uint32_t)((slots + BA_K - 1) / BA_K);
        const uint32_t blocks = (n_threads + BA_THREADS - 1) / BA_THREADS;
        fill_work_kernel<<<(n_buckets + 255) / 256, 256, 0, st>>>(hist, off[l + 1], n_buckets, 1u << (l + 1), 0, slot_bucket);
        BaLevel lv{hist, off[l], off[l + 1], slot_bucket, n_buckets, (uint32_t)l};
        to_heavy();
        if (ev && l == 0) cudaEventRecord(ev[0], hv);
        ba_forward_kernel<F><<<blocks, BA_THREADS, 0, hv>>>(lv, in, prefix, tot, n_threads);
        to_light();
        batch_inverse<F>(tot, n_threads, binv_scratch, st);
        to_heavy();
        ba_backward_kernel<F><<<blocks, BA_THREADS, 0, hv>>>(lv, in, prefix, tot, out, n_threads);
        if (ev && l == L - 1) cudaEventRecord(ev[1], hv);
        to_light();
        ZKE_COUNT_LAUNCH(3);
        in = out;
        out = (out == ping) ? pong : ping;
    }
    // what is left of every bucket (ceil(size / 2^L) affine points, 6.5 on average for L = 4) is summed by one thread per
    // bucket with mixed additions - fully parallel - before the (latency-bound) running sums over the buckets
    XYZZ<F>* bucket_sum = (XYZZ<F>*)sorted0;     // the level-0 array is free again
    bucket_finish_kernel<F><<<(n_buckets + 127) / 128, 128, 0, st>>>(in, hist, off[L], n_buckets, (uint32_t)L, bucket_sum);
    group_sum_kernel<F, 1><<<(groups + 127) / 128, 128, 0, st>>>((const uint8_t*)bucket_sum, hist, off[L], D.half, groups, 1u << L, 0, D.group, group_out);
    ZKE_COUNT_LAUNCH(2);
}
template <>
void run_ba<Fq2>(const MsmConfig&, const uint32_t*, const uint32_t*, uint32_t, size_t, uint32_t*, uint8_t*, const Digits&,
                 uint32_t, uint8_t*, cudaStream_t, cudaEvent_t*, const MsmPlan<Fq2>::Heavy*) {}

// ---------------------------------------------------------------- host orchestration
#if defined(ZKE_MSM_G1)
MsmConfig msm_config_witness() {
    MsmConfig c; c.c = 8; c.chunk = 32; c.group = 8; c.classify = true; c.extra_passes = 2;
    if (const char* e = getenv("ZKE_W_C")) c.c = std::max(4, std::min(16, atoi(e)));          // experiments
    if (const char* e = getenv("ZKE_W_CHUNK")) c.chunk = (uint32_t)std::max(8, atoi(e));
    if (const char* e = getenv("ZKE_W_GROUP")) c.group = (uint32_t)std::max(2, atoi(e));
    return c;
}
MsmConfig msm_config_full(uint32_t n, bool precomputed) {
    MsmConfig c;
    c.c = n >= (1u << 18) ? 16 : (n >= (1u << 12) ? 12 : 8);
    c.chunk = 256; c.group = n >= (1u << 20) ? 64 : 16; c.classify = false; c.extra_passes = 0;
    c.precomputed = precomputed;
    // Streaming batched-affine bucket accumulation (msm_ba.cuh): the first `ba_levels` levels of every bucket's addition
    // tree in affine coordinates (6 products per addition instead of 10) - opt-in with ZKE_H_BA=<levels> at key-setup
    // time.  It needs fewer multiplier instructions, but the sweeps are memory- and latency-bound where the XYZZ kernel
    // is purely multiplier-bound, so it stays off by default.
    c.ba_levels = 0;
    if (const char* e = getenv("ZKE_H_BA")) c.ba_levels = precomputed ? std::max(0, std::min(6, atoi(e))) : 0;
    if (const char* e = getenv("ZKE_H_GROUP")) c.group = (uint32_t)std::max(2, atoi(e));   // experiments
    if (precomputed) {
        // one shared bucket set of 2^(c-1) buckets: pick c so that the buckets (~ n * W / 2^(c-1) entries each) still
        // number in the hundreds of thousands for parallelism; 13 table levels at 2^22 points (3.5 GB)
        c.c = n >= (1u << 20) ? 20 : (n >= (1u << 16) ? 17 : (n >= (1u << 10) ? 12 : 8));
    }
    return c;
}
#endif

template <class F>
size_t MsmPlan<F>::workspace_bytes(uint32_t n, const MsmConfig& cfg) {
    const int W = (255 + cfg.c - 1) / cfg.c;
    const size_t half = (size_t)1 << (cfg.c - 1);
    const size_t bucket_sets = cfg.precomputed ? 1 : W;
    const size_t n_buckets = half * bucket_sets;
    const size_t max_entries = (size_t)n * W;
    const size_t max_chunks = n_buckets + max_entries / cfg.chunk + 1;
    const size_t groups = ((half + cfg.group - 1) / cfg.group) * bucket_sets;
    size_t b = 0;
    auto al = [&](size_t x) { b += (x + 255) & ~(size_t)255; };
    al(4 * 2);                         // counters
    al(4 * (size_t)n);                 // ones list
    al(4 * (size_t)n);                 // general list
    al(4 * (n_buckets + 1));           // hist
    al(4 * (n_buckets + 1));           // offsets
    al(4 * (n_buckets + 1));           // chunk_off
    al(4 * (n_buckets / SCAN_TILE + 2));  // scan tiles
    al(4 * max_entries);               // entries
    al(4 * max_chunks);                // work_bucket
    al(sizeof(XYZZ<F>) * max_chunks);  // partial
    al(sizeof(XYZZ<F>) * (max_chunks / PASS_FANIN + n_buckets + 1));  // partial (ping-pong for the extra passes)
    al(4 * (n_buckets + 1));           // second offsets array
    al(sizeof(XYZZ<F>) * groups);      // group sums
    al(sizeof(XYZZ<F>) * ((size_t)n / LIST_FANIN + 2));      // list reduction ping-pong: two arrays, each padded as run() takes it
    al(sizeof(XYZZ<F>) * ((size_t)n / LIST_FANIN + 2));
    if (cfg.ba_levels > 0 && sizeof(F) == 32) al(BaPlan<F>::bytes(max_entries, n_buckets, cfg.ba_levels));
    const size_t order_cells = ((max_chunks + ORDER_BLOCK - 1) / ORDER_BLOCK) * cfg.chunk;
    al(4 * max_chunks);                       // order
    al(4 * (order_cells + 1));                // per-block size histograms, bin-major
    al(4 * (order_cells + 1));                // their exclusive scan
    al(4 * (order_cells / SCAN_TILE + 2));    // scan tiles
    if (n_buckets >= SORT_TWO_LEVEL_MIN_BUCKETS) DigitSort((uint32_t)n, W, (uint32_t)n_buckets, max_entries).place([&](size_t x) { al(x); return (uint8_t*)nullptr; });
    else al(4 * (n_buckets + 1));             // cursor
    return b;
}

template <class F>
void MsmPlan<F>::run(const uint8_t* points, const uint8_t* scalars, uint32_t n, const MsmConfig& cfg, uint8_t* ws,
                     uint8_t* result, cudaStream_t st, cudaEvent_t* ev, const Heavy* heavy) {
    Digits D;
    D.c = cfg.c;
    D.n_windows = (255 + cfg.c - 1) / cfg.c;
    D.half = 1u << (cfg.c - 1);
    D.chunk = cfg.chunk;
    D.group = cfg.group;
    D.window_bucket_stride = cfg.precomputed ? 0 : D.half;
    D.window_point_stride = cfg.precomputed ? n : 0;
    if (D.n_windows > MSM_MAX_WINDOWS) return;
    const uint32_t bucket_sets = cfg.precomputed ? 1 : (uint32_t)D.n_windows;
    const uint32_t n_buckets = D.half * bucket_sets;
    const size_t max_entries = (size_t)n * D.n_windows;
    const size_t max_chunks = n_buckets + max_entries / cfg.chunk + 1;
    const uint32_t groups_per_window = (D.half + D.group - 1) / D.group;
    const uint32_t groups = groups_per_window * bucket_sets;
    uint8_t* p = ws;
    auto take = [&](size_t x) { uint8_t* r = p; p += (x + 255) & ~(size_t)255; return r; };
    uint32_t* counters = (uint32_t*)take(8);
    uint32_t* ones_list = (uint32_t*)take(4 * (size_t)n);
    uint32_t* gen_list = (uint32_t*)take(4 * (size_t)n);
    uint32_t* hist = (uint32_t*)take(4 * ((size_t)n_buckets + 1));
    uint32_t* offsets = (uint32_t*)take(4 * ((size_t)n_buckets + 1));
    uint32_t* chunk_off = (uint32_t*)take(4 * ((size_t)n_buckets + 1));
    uint32_t* tiles = (uint32_t*)take(4 * ((size_t)n_buckets / SCAN_TILE + 2));
    uint32_t* entries = (uint32_t*)take(4 * max_entries);
    uint32_t* work_bucket = (uint32_t*)take(4 * max_chunks);
    uint8_t* partial = take(sizeof(XYZZ<F>) * max_chunks);
    uint8_t* partial2 = take(sizeof(XYZZ<F>) * (max_chunks / PASS_FANIN + n_buckets + 1));
    uint32_t* off2 = (uint32_t*)take(4 * ((size_t)n_buckets + 1));
    uint8_t* group_out = take(sizeof(XYZZ<F>) * groups);
    const size_t list_slots = (size_t)n / LIST_FANIN + 2;
    uint8_t* red_a = take(sizeof(XYZZ<F>) * list_slots);
    uint8_t* red_b = take(sizeof(XYZZ<F>) * list_slots);
    const bool use_ba = cfg.ba_levels > 0 && sizeof(F) == 32;      // G1 only
    uint8_t* ba_ws = use_ba ? take(BaPlan<F>::bytes(max_entries, n_buckets, cfg.ba_levels)) : nullptr;
    const size_t order_cells = ((max_chunks + ORDER_BLOCK - 1) / ORDER_BLOCK) * cfg.chunk;
    uint32_t* order = (uint32_t*)take(4 * max_chunks);
    uint32_t* order_mat = (uint32_t*)take(4 * (order_cells + 1));
    uint32_t* order_off = (uint32_t*)take(4 * (order_cells + 1));
    uint32_t* order_tiles = (uint32_t*)take(4 * (order_cells / SCAN_TILE + 2));
    const bool two_level = n_buckets >= SORT_TWO_LEVEL_MIN_BUCKETS;
    DigitSort sort(n, D.n_windows, n_buckets, max_entries);
    if (sort.fine_bits > SORT_MAX_FINE_BITS) throw std::runtime_error("MSM bucket sort: more than 2^19 buckets");
    uint32_t* cursor = nullptr;
    if (two_level) sort.place(take);
    else cursor = (uint32_t*)take(4 * ((size_t)n_buckets + 1));

    // result block: [MSM_ONES_SLOTS partial sums of the unit-scalar points][MSM_MAX_WINDOWS window sums]
    uint8_t* res_ones = result;
    uint8_t* res_windows = result + sizeof(XYZZ<F>) * MSM_ONES_SLOTS;
    cudaMemsetAsync(result, 0, sizeof(XYZZ<F>) * MSM_RESULT_SLOTS, st);   // all-zero XYZZ = infinity

    const uint32_t* gen_count = nullptr;
    const uint32_t* gen_idx = nullptr;
    if (cfg.classify) {
        cudaMemsetAsync(counters, 0, 8, st);
        classify_kernel<F><<<(n + 255) / 256, 256, 0, st>>>(points, scalars, n, ones_list, gen_list, counters);
        // unit scalars: tree reduction; level sizes are recomputed on the device from counters[0], the host only
        // needs the upper bound n to know how many levels to launch
        uint32_t upper = (n + LIST_FANIN - 1) / LIST_FANIN;
        sum_affine_list_kernel<F><<<(upper + 127) / 128, 128, 0, st>>>(points, ones_list, counters, 0, red_a);
        ZKE_COUNT_LAUNCH(2);
        uint8_t *src = red_a, *dst = red_b;
        uint32_t level = 0;
        for (;;) {
            const uint32_t next = (upper + TREE_FANIN - 1) / TREE_FANIN;
            const bool last = next <= MSM_ONES_SLOTS;
            uint8_t* out = last ? res_ones : dst;
            const uint32_t threads = last ? (uint32_t)MSM_ONES_SLOTS : next;
            sum_xyzz_kernel<F><<<(threads + 63) / 64, 64, 0, st>>>(src, counters, 0, level, last ? MSM_ONES_SLOTS : 0, out);
            ZKE_COUNT_LAUNCH(1);
            if (last) break;
            uint8_t* t = src; src = dst; dst = t;
            upper = next;
            ++level;
        }
        gen_count = counters + 1;
        gen_idx = gen_list;
    }
    const int sms = sm_count();
    if (two_level) {
        sort.run(scalars, gen_idx, gen_count, n, D, hist, offsets, entries, st);
    } else {
        cudaMemsetAsync(hist, 0, 4 * ((size_t)n_buckets + 1), st);
        cudaMemsetAsync(cursor, 0, 4 * ((size_t)n_buckets + 1), st);
        digit_hist_kernel<<<sms * 8, 256, 0, st>>>(scalars, gen_idx, gen_count, n, D, hist);
        exclusive_scan(hist, n_buckets, 0, 0, offsets, tiles, st);
        digit_scatter_kernel<<<sms * 8, 256, 0, st>>>(scalars, gen_idx, gen_count, n, D, offsets, cursor, entries);
        ZKE_COUNT_LAUNCH(2);
    }
    if (use_ba) {
        gather_points_kernel<F><<<sms * 8, 256, 0, st>>>(entries, offsets, n_buckets, points, (Affine<F>*)ba_ws);
        ZKE_COUNT_LAUNCH(1);
        run_ba<F>(cfg, hist, offsets, n_buckets, max_entries, tiles, ba_ws, D, groups, group_out, st, ev, heavy);
    } else {
        exclusive_scan(hist, n_buckets, D.chunk, 0, chunk_off, tiles, st);
        fill_work_kernel<<<(n_buckets + 255) / 256, 256, 0, st>>>(hist, chunk_off, n_buckets, D.chunk, 0, work_bucket);
        {   // order[] = chunks sorted by size, largest first
            const uint32_t nblk = (uint32_t)((max_chunks + ORDER_BLOCK - 1) / ORDER_BLOCK);
            chunk_key_hist_kernel<<<nblk, ORDER_BLOCK, 4 * D.chunk, st>>>(hist, chunk_off, work_bucket, n_buckets, D.chunk, order_mat);
            exclusive_scan(order_mat, nblk * D.chunk, 0, 0, order_off, order_tiles, st);
            chunk_order_kernel<<<nblk, ORDER_BLOCK, 0, st>>>(hist, chunk_off, work_bucket, n_buckets, D.chunk, order_off, order);
            ZKE_COUNT_LAUNCH(2);
        }
        cudaStream_t st_light = st;
        if (heavy && heavy->st != st) {
            cudaEventRecord(heavy->before, st);
            cudaStreamWaitEvent(heavy->st, heavy->before, 0);
            st = heavy->st;
        }
        if (ev) cudaEventRecord(ev[0], st);
        {
            // blocks per SM the bucket kernel is compiled for (register cap 128 / 96 / 80): more resident warps hide the
            // IMAD.WIDE carry-chain latency; tunable for experiments with ZKE_CHUNK_MINB
            int minb = sizeof(F) == 32 ? 5 : 4, waves = 4;
            if (const char* e = getenv("ZKE_CHUNK_MINB")) minb = atoi(e);
            if (const char* e = getenv("ZKE_CHUNK_WAVES")) waves = std::max(1, atoi(e));
            bool done = false;
#if defined(ZKE_MSM_G1)
            // ZKE_H_TC=1: Montgomery reductions of the bucket accumulation on the tensor cores (msm_tc.cuh), large G1 sets only
            const char* h_tc_env = getenv("ZKE_H_TC");
            const int h_tc = h_tc_env ? atoi(h_tc_env) : 0;
            if (h_tc > 0 && cfg.precomputed) {
                if (const TcTable* tab = tc_table_fq()) {
                    const uint8_t* pts = reinterpret_cast<const uint8_t*>(points);
                    if (h_tc >= 5) chunk_sum_tc_kernel<5><<<sms * 5 * waves, 128, 0, st>>>(pts, entries, offsets, hist, chunk_off, work_bucket, order, n_buckets, D.chunk, partial, tab);
                    else if (h_tc == 4) chunk_sum_tc_kernel<4><<<sms * 4 * waves, 128, 0, st>>>(pts, entries, offsets, hist, chunk_off, work_bucket, order, n_buckets, D.chunk, partial, tab);
                    else chunk_sum_tc_kernel<3><<<sms * 3 * waves, 128, 0, st>>>(pts, entries, offsets, hist, chunk_off, work_bucket, order, n_buckets, D.chunk, partial, tab);
                    done = true;
                }
            }
#endif
            // ZKE_CHUNK_PAD_SMEM=<bytes <= 48 K>: dynamic shared memory the kernel does not use - caps the resident blocks per SM
            // below what the register file allows, so that blocks of the other lanes' (latency-bound) kernels find room
            // beside a running bucket kernel (experiment; 0 = off)
            size_t pad = 0;
            if (const char* e = getenv("ZKE_CHUNK_PAD_SMEM")) pad = (size_t)std::max(0, std::min(48 * 1024, atoi(e)));
            if (done) {}
            else if (minb >= 6) chunk_sum_kernel<F, 6><<<sms * 6 * waves, 128, pad, st>>>(points, entries, offsets, hist, chunk_off, work_bucket, order, n_buckets, D.chunk, partial);
            else if (minb == 5) chunk_sum_kernel<F, 5><<<sms * 5 * waves, 128, pad, st>>>(points, entries, offsets, hist, chunk_off, work_bucket, order, n_buckets, D.chunk, partial);
            else chunk_sum_kernel<F, 4><<<sms * 4 * waves, 128, pad, st>>>(points, entries, offsets, hist, chunk_off, work_bucket, order, n_buckets, D.chunk, partial);
        }
        if (ev) cudaEventRecord(ev[1], st);
        if (st != st_light) {
            cudaEventRecord(heavy->after, st);
            cudaStreamWaitEvent(st_light, heavy->after, 0);
            st = st_light;
        }
        // extra passes over the per-chunk partial sums
        uint8_t *items = partial, *items_next = partial2;
        uint32_t *off_cur = chunk_off, *off_next = off2;
        uint32_t levels = 0;
        for (uint32_t pass = 0; pass < cfg.extra_passes; ++pass) {
            exclusive_scan(hist, n_buckets, D.chunk, levels + 1, off_next, tiles, st);
            fill_work_kernel<<<(n_buckets + 255) / 256, 256, 0, st>>>(hist, off_next, n_buckets, D.chunk, levels + 1, work_bucket);
            partial_pass_kernel<F><<<sms * 4, 128, 0, st>>>(items, hist, off_cur, off_next, work_bucket, n_buckets, D.chunk, levels, items_next);
            ZKE_COUNT_LAUNCH(2);
            uint8_t* t = items; items = items_next; items_next = t;
            uint32_t* o = off_cur; off_cur = off_next; off_next = o;
            ++levels;
        }
        group_sum_kernel<F, 0><<<(groups + 127) / 128, 128, 0, st>>>(items, hist, off_cur, D.half, groups, D.chunk, levels, D.group, group_out);
    }
    window_reduce_kernel<F><<<bucket_sets, 512, 0, st>>>(group_out, groups_per_window);
    gather_windows_kernel<F><<<1, 64, 0, st>>>(group_out, groups_per_window, bucket_sets, res_windows);
    ZKE_COUNT_LAUNCH(5);
}

#if defined(ZKE_MSM_G1)
template struct MsmPlan<Fq>;
#elif defined(ZKE_MSM_G2)
template struct MsmPlan<Fq2>;
#else
#error "compile msm.cu through msm_g1.cu / msm_g2.cu"
#endif

}  // namespace dev
}  // namespace zke
