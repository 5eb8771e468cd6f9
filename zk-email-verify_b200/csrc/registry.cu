// Batched Poseidon and the Merkle registry of DKIM keys (include/zkemail_b200.h: zke_poseidon_batch, zke_pubkey_hashes,
// zke_domain_key_leaves, zke_merkle_build, and the resident registry zke_registry_*).
//
// One thread runs one Poseidon instance: the Merkle node hash (width 3) with its state in registers, the other widths
// from one instantiation that takes the width at run time (its state in the thread's stack frame).  The round constants and the MDS matrix of the width come from
// gadgets::poseidon_params - the tables the circuits constrain and the witness kernel's native op reads - and every
// block stages them in shared memory in Montgomery form.  The permutation is circomlib's plain schedule: full rounds
// S-box every lane, partial rounds lane 0 only, a dense t x t mix after each round.
//
// The Merkle tree (node H(l, r) = Poseidon(2)([l, r])) is built level by level on the device: one kernel hashes the
// lowest FUSE_LEVELS levels of a 2^FUSE_LEVELS-leaf subtree per block, keeping each level in shared memory, and one launch
// per higher level hashes the pairs of the level below.  A missing right child at level l is zeros[l], the root of an
// empty subtree of height l (computed on the host: at most 32 hashes).  A resident registry (zke_registry_open) keeps the
// levels on the device and updates k leaves in place: one launch per level, one thread per changed node.
#include "ff.cuh"
#include "device_engine.cuh"
#include "cuda_host.hpp"
#include "gadgets.hpp"
#include "../../include/zkemail_b200.h"
#include <algorithm>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace zke {
void set_err(char* err, size_t cap, const std::string& msg);   // capi_circuit.cpp
}

namespace zke {
namespace dev {

ZKE_DEFINE_CONSTANT_UPLOAD(upload_constants_registry)

static const int REG_THREADS = 128;
static const int FUSE_LEVELS = 8;                 // levels 1..8 of a 256-leaf subtree per block of 128 threads
static const uint32_t NO_BAD = 0xffffffffu;

// Montgomery form from 8 little-endian standard-form words; *bad is set when the value is not below r
__device__ __forceinline__ Fr fr_in(const uint32_t w[8], bool* bad) {
    Fr x;
    for (int i = 0; i < 8; ++i) x.v[i] = w[i];
    if (!below_modulus(x)) *bad = true;
    return x.to_mont();
}
__device__ __forceinline__ Fr fr_load(const uint8_t* p, bool* bad) {
    uint32_t w[8];
    const uint4* q = reinterpret_cast<const uint4*>(p);
    const uint4 a = q[0], b = q[1];
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    return fr_in(w, bad);
}
__device__ __forceinline__ void fr_store(uint8_t* p, const Fr& x) { x.from_mont().store(p); }

// constants of width T: rc[(R_F + R_P) * T] then mds[T][T], standard form in global memory -> Montgomery in shared memory
__device__ __forceinline__ void stage_constants(Fr* sh, const uint8_t* g, uint32_t n) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) sh[i] = Fr::load(g + 32ull * i).to_mont();
    __syncthreads();
}

__device__ __forceinline__ Fr sbox(const Fr& x) { Fr x2 = x.sqr(); Fr x4 = x2.sqr(); return x4 * x; }

// circomlib Poseidon(t - 1) of st[1..t-1] (st[0] = 0 on entry); returns the output state[0].  T > 0: the width is a
// compile-time constant and the state lives in registers (the Merkle node hash, T = 3); T = 0: any width t <= MAX_T
// from one instantiation (unrolling the dense mix for all sixteen widths takes nvcc tens of minutes)
static const int MAX_T = 17;
template <int T>
__device__ __forceinline__ Fr permute(Fr* st, int t, const Fr* rc, const Fr* mds, int r_p) {
    if (T > 0) t = T;
    const int rounds = 8 + r_p;
    Fr nx[T > 0 ? T : MAX_T];
#pragma unroll 1
    for (int rnd = 0; rnd < rounds; ++rnd) {
        const Fr* c = rc + rnd * t;
#pragma unroll
        for (int i = 0; i < (T > 0 ? T : t); ++i) st[i] = st[i] + c[i];
        if (rnd < 4 || rnd >= 4 + r_p) {
#pragma unroll
            for (int i = 0; i < (T > 0 ? T : t); ++i) st[i] = sbox(st[i]);
        } else {
            st[0] = sbox(st[0]);
        }
#pragma unroll
        for (int i = 0; i < (T > 0 ? T : t); ++i) {
            Fr acc = mds[i * t] * st[0];
#pragma unroll
            for (int j = 1; j < (T > 0 ? T : t); ++j) acc = acc + mds[i * t + j] * st[j];
            nx[i] = acc;
        }
#pragma unroll
        for (int i = 0; i < (T > 0 ? T : t); ++i) st[i] = nx[i];
    }
    return st[0];
}

__device__ __forceinline__ uint32_t n_constants(int t, int r_p) { return (uint32_t)((8 + r_p) * t + t * t); }

// out[i] = Poseidon(t - 1)(in[i][0..t-2]); the first instance holding an input not below r goes to *bad
__global__ void __launch_bounds__(REG_THREADS)
poseidon_batch_kernel(const uint8_t* __restrict__ in, uint64_t count, int t, const uint8_t* __restrict__ consts, int r_p,
                      uint8_t* __restrict__ out, uint32_t* __restrict__ bad) {
    extern __shared__ uint4 smem[];
    Fr* sh = reinterpret_cast<Fr*>(smem);
    stage_constants(sh, consts, n_constants(t, r_p));
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    bool b = false;
    Fr st[MAX_T];
    st[0] = Fr::zero();
#pragma unroll 1
    for (int k = 1; k < t; ++k) st[k] = fr_load(in + 32ull * ((uint64_t)(t - 1) * i + (k - 1)), &b);
    if (b) atomicMin(bad, (uint32_t)min(i, (uint64_t)NO_BAD - 1));
    fr_store(out + 32ull * i, permute<0>(st, t, sh, sh + (8 + r_p) * t, r_p));
}

// bits [off, off + w) of a little-endian byte string of `len` bytes (bits past the end read as 0), w <= 256
__device__ __forceinline__ void bit_field(const uint8_t* m, uint32_t len, uint32_t off, uint32_t w, uint32_t out[8]) {
    for (int q = 0; q < 8; ++q) {
        const uint32_t lo = 32 * q;
        if (lo >= w) { out[q] = 0; continue; }
        const uint32_t pos = off + lo, byte = pos >> 3;
        uint64_t v = 0;
        for (int k = 0; k < 5; ++k) if (byte + k < len) v |= (uint64_t)m[byte + k] << (8 * k);
        uint32_t x = (uint32_t)(v >> (pos & 7));
        const uint32_t keep = w - lo;
        if (keep < 32) x &= (1u << keep) - 1;
        out[q] = x;
    }
}

// the PoseidonLarge input of one modulus (mlen bytes, little-endian) into st[1..t-1], t - 1 = ceil(k / 2): its k limbs
// of n bits, merged in pairs (limb 2j + limb 2j+1 * 2^n, the last limb alone for odd k) = the 2n-bit chunks of the
// modulus.  A modulus with a bit at or above n k sets *bad.
__device__ __forceinline__ void pubkey_chunks(const uint8_t* m, uint32_t mlen, uint32_t n, uint32_t k, Fr* st, bool* bad) {
    const int t = (int)(k + 1) / 2 + 1;
    const uint32_t nk = n * k;
    for (uint32_t byte = nk >> 3; byte < mlen; ++byte) {
        const uint32_t first = byte == (nk >> 3) ? (nk & 7) : 0;
        if (m[byte] >> first) *bad = true;
    }
#pragma unroll 1
    for (int j = 1; j < t; ++j) {
        const uint32_t off = 2 * n * (j - 1);
        uint32_t w[8];
        bit_field(m, mlen, off, min(2 * n, nk - off), w);
        st[j] = fr_in(w, bad);
    }
}

// PoseidonLarge leaves: out[i] = pubkeyHash of modulus i; the first modulus with a bit at or above n k goes to *bad
__global__ void __launch_bounds__(REG_THREADS)
pubkey_hash_kernel(const uint8_t* __restrict__ moduli, uint64_t count, uint32_t mlen, uint32_t n, uint32_t k,
                   const uint8_t* __restrict__ consts, int r_p, uint8_t* __restrict__ out, uint32_t* __restrict__ bad) {
    extern __shared__ uint4 smem[];
    Fr* sh = reinterpret_cast<Fr*>(smem);
    stage_constants(sh, consts, n_constants((int)(k + 1) / 2 + 1, r_p));
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const int t = (int)(k + 1) / 2 + 1;
    bool b = false;
    Fr st[MAX_T];
    st[0] = Fr::zero();
    pubkey_chunks(moduli + (uint64_t)mlen * i, mlen, n, k, st, &b);
    if (b) atomicMin(bad, (uint32_t)min(i, (uint64_t)NO_BAD - 1));
    fr_store(out + 32ull * i, permute<0>(st, t, sh, sh + (8 + r_p) * t, r_p));
}

__device__ __forceinline__ Fr node_hash(const Fr& l, const Fr& r, const Fr* rc, const Fr* mds, int r_p) {
    Fr st[3] = {Fr::zero(), l, r};
    return permute<3>(st, 3, rc, mds, r_p);
}

// A domain row: DOMAIN_BYTES bytes, the name then zero padding (the byte image of PackBytes(D, 255)), packed into
// DOMAIN_WORDS words of 31 bytes, little-endian.  Canonical: 1..255 bytes, ASCII without upper-case letters, no zero
// byte inside the name, no trailing dot.
static const uint32_t DOMAIN_BYTES = 255, DOMAIN_WORDS = 9, DOMAIN_T = DOMAIN_WORDS + 1;

__device__ __forceinline__ bool domain_canonical(const uint8_t* d) {
    bool ok = d[0] != 0, ended = false;
    uint8_t last = 0;
#pragma unroll 1
    for (uint32_t j = 0; j < DOMAIN_BYTES; ++j) {
        const uint8_t c = d[j];
        if (c == 0) { ended = true; continue; }
        if (ended || c >= 0x80 || (c >= 'A' && c <= 'Z')) ok = false;
        last = c;
    }
    return ok && last != '.';
}

// Domain-bound leaves: out[i] = Poseidon(2)([Poseidon(9)(the 9 words of domain row i), pubkeyHash of modulus i]).
// Shared memory holds the constants of width DOMAIN_T, then those of the key's width tk unless tk == DOMAIN_T (k = 17,
// 18), then those of width 3.  The first bad modulus goes to *bad_key, the first non-canonical row to *bad_domain.
__global__ void __launch_bounds__(REG_THREADS)
domain_key_leaf_kernel(const uint8_t* __restrict__ moduli, const uint8_t* __restrict__ domains, uint64_t count, uint32_t mlen,
                       uint32_t n, uint32_t k, const uint8_t* __restrict__ consts_d, int r_p_d,
                       const uint8_t* __restrict__ consts_k, int r_p_k, const uint8_t* __restrict__ consts_2, int r_p_2,
                       uint8_t* __restrict__ out, uint32_t* __restrict__ bad_key, uint32_t* __restrict__ bad_domain) {
    extern __shared__ uint4 smem[];
    const int tk = (int)(k + 1) / 2 + 1;
    Fr* sh_d = reinterpret_cast<Fr*>(smem);
    Fr* sh_k = sh_d + n_constants(DOMAIN_T, r_p_d);
    stage_constants(sh_d, consts_d, n_constants(DOMAIN_T, r_p_d));
    if (tk == (int)DOMAIN_T) sh_k = sh_d;
    else stage_constants(sh_k, consts_k, n_constants(tk, r_p_k));
    Fr* sh_2 = sh_k + n_constants(tk, r_p_k);
    stage_constants(sh_2, consts_2, n_constants(3, r_p_2));
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint8_t* d = domains + (uint64_t)DOMAIN_BYTES * i;
    if (!domain_canonical(d)) atomicMin(bad_domain, (uint32_t)min(i, (uint64_t)NO_BAD - 1));
    bool b = false;
    Fr st[MAX_T], domain_hash, key_hash;
    // one permutation site at a run-time width for the three hashes: a call at a constant width is unrolled with its
    // state in registers, which takes the kernel from about 50 to about 240 registers
#pragma unroll 1
    for (int job = 0; job < 3; ++job) {
        const Fr* c = job == 0 ? sh_d : job == 1 ? sh_k : sh_2;
        const int t = job == 0 ? (int)DOMAIN_T : job == 1 ? tk : 3, r_p = job == 0 ? r_p_d : job == 1 ? r_p_k : r_p_2;
        st[0] = Fr::zero();
        if (job == 0) {
#pragma unroll 1
            for (uint32_t j = 0; j < DOMAIN_WORDS; ++j) {
                uint32_t w[8];
                bit_field(d, DOMAIN_BYTES, 248 * j, 248, w);     // below 2^248 < r: never bad
                st[j + 1] = fr_in(w, &b);
            }
        } else if (job == 1) {
            pubkey_chunks(moduli + (uint64_t)mlen * i, mlen, n, k, st, &b);
        } else {
            st[1] = domain_hash;
            st[2] = key_hash;
        }
        const Fr h = permute<0>(st, t, c, c + (8 + r_p) * t, r_p);
        if (job == 0) domain_hash = h;
        else if (job == 1) key_hash = h;
        else fr_store(out + 32ull * i, h);
    }
    if (b) atomicMin(bad_key, (uint32_t)min(i, (uint64_t)NO_BAD - 1));
}

// Levels 1..L of the tree (L <= FUSE_LEVELS): block b owns the nodes under its 2^L leaves.  levels: the whole level
// image, level l starting at off[l] with size[l] nodes (level 0 = the leaves, uploaded); zeros[l] standard form.
struct LevelTable { uint64_t off[33], size[33]; };

__global__ void __launch_bounds__(REG_THREADS)
merkle_fused_kernel(uint8_t* __restrict__ levels, LevelTable lt, int L, const uint8_t* __restrict__ consts, int r_p,
                    const uint8_t* __restrict__ zeros, uint32_t* __restrict__ bad) {
    extern __shared__ uint4 smem[];
    Fr* sh = reinterpret_cast<Fr*>(smem);
    const uint32_t nc = n_constants(3, r_p);
    Fr* node = sh + nc;                                   // [REG_THREADS] nodes of the level just built
    stage_constants(sh, consts, nc);
    const Fr* rc = sh;
    const Fr* mds = sh + (8 + r_p) * 3;
    const uint32_t t = threadIdx.x;
    bool b = false;
    for (int l = 1; l <= L; ++l) {
        const uint32_t width = 1u << (L - l);             // nodes of level l under this block
        const uint64_t j = (uint64_t)blockIdx.x * width + t;
        Fr h;
        const bool live = t < width && j < lt.size[l];
        if (live) {
            Fr left, right;
            const bool has_right = 2 * j + 1 < lt.size[l - 1];
            if (l == 1) {
                left = fr_load(levels + 32 * (lt.off[0] + 2 * j), &b);
                right = has_right ? fr_load(levels + 32 * (lt.off[0] + 2 * j + 1), &b) : Fr::zero();
            } else {
                left = node[2 * t];
                right = has_right ? node[2 * t + 1] : fr_load(zeros + 32 * (l - 1), &b);
            }
            h = node_hash(left, right, rc, mds, r_p);
            fr_store(levels + 32 * (lt.off[l] + j), h);
        }
        __syncthreads();                                  // every read of the level below is done
        if (live) node[t] = h;
        __syncthreads();
    }
    if (b) atomicMin(bad, (uint32_t)min((uint64_t)blockIdx.x << FUSE_LEVELS, (uint64_t)NO_BAD - 1));
}

// level l > FUSE_LEVELS from level l - 1 in global memory
__global__ void __launch_bounds__(REG_THREADS)
merkle_level_kernel(uint8_t* __restrict__ levels, uint64_t below_off, uint64_t below_size, uint64_t off, uint64_t size,
                    const uint8_t* __restrict__ consts, int r_p, const uint8_t* __restrict__ zero_below) {
    extern __shared__ uint4 smem[];
    Fr* sh = reinterpret_cast<Fr*>(smem);
    stage_constants(sh, consts, n_constants(3, r_p));
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= size) return;
    bool b = false;
    const Fr left = fr_load(levels + 32 * (below_off + 2 * j), &b);
    const Fr right = fr_load(2 * j + 1 < below_size ? levels + 32 * (below_off + 2 * j + 1) : zero_below, &b);
    fr_store(levels + 32 * (off + j), node_hash(left, right, sh, sh + (8 + r_p) * 3, r_p));
}

// In-place updates of a resident tree (zke_registry_update).  idx[0..k) are the updated leaf indices, sorted and
// distinct.  level 0: leaf i goes to position idx[i]
__global__ void __launch_bounds__(REG_THREADS)
registry_scatter_kernel(uint8_t* __restrict__ levels, const uint64_t* __restrict__ idx, const uint8_t* __restrict__ leaves,
                        uint64_t k) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const uint4* src = reinterpret_cast<const uint4*>(leaves + 32 * i);
    uint4* dst = reinterpret_cast<uint4*>(levels + 32 * idx[i]);
    dst[0] = src[0];
    dst[1] = src[1];
}

// level l from level l - 1: thread i rehashes the ancestor p = idx[i] >> l unless thread i - 1 has the same one (the
// indices are sorted, so equal ancestors are adjacent and this keeps exactly one thread per changed node).  A node that
// appends bring into range at level l covers leaf p 2^l >= the old count, an appended index, so it is always rehashed
// here; so is its parent once its right child comes into range.  That is what lets an update skip every other node.
__global__ void __launch_bounds__(REG_THREADS)
registry_update_level_kernel(uint8_t* __restrict__ levels, const uint64_t* __restrict__ idx, uint64_t k, int l,
                             uint64_t below_off, uint64_t below_size, uint64_t off, const uint8_t* __restrict__ consts,
                             int r_p, const uint8_t* __restrict__ zero_below) {
    extern __shared__ uint4 smem[];
    Fr* sh = reinterpret_cast<Fr*>(smem);
    stage_constants(sh, consts, n_constants(3, r_p));
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const uint64_t p = idx[i] >> l;
    if (i > 0 && (idx[i - 1] >> l) == p) return;
    bool b = false;                                       // every value was checked below r on the host
    const Fr left = fr_load(levels + 32 * (below_off + 2 * p), &b);
    const Fr right = fr_load(2 * p + 1 < below_size ? levels + 32 * (below_off + 2 * p + 1) : zero_below, &b);
    fr_store(levels + 32 * (off + p), node_hash(left, right, sh, sh + (8 + r_p) * 3, r_p));
}

// out[i] = node idx[i] of level lv[i], or zeros[lv[i]] past the level's size (authentication paths, the host mirror)
__global__ void __launch_bounds__(REG_THREADS)
registry_gather_kernel(const uint8_t* __restrict__ levels, LevelTable lt, const uint32_t* __restrict__ lv,
                       const uint64_t* __restrict__ idx, uint64_t k, const uint8_t* __restrict__ zeros, uint8_t* __restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const uint32_t l = lv[i];
    const uint64_t j = idx[i];
    const uint4* src = reinterpret_cast<const uint4*>(j < lt.size[l] ? levels + 32 * (lt.off[l] + j) : zeros + 32 * l);
    uint4* dst = reinterpret_cast<uint4*>(out + 32 * i);
    dst[0] = src[0];
    dst[1] = src[1];
}

}  // namespace dev
}  // namespace zke

using namespace zke;

namespace {

thread_local double g_last_device_ms = 0;     // zke_registry_device_ms

// rc then mds of Poseidon width t, standard form, on the device
struct WidthConsts {
    DevBuf buf;
    int r_p = 0;
    uint32_t n = 0;
    explicit WidthConsts(int t) {
        const gadgets::PoseidonParams& P = gadgets::poseidon_params(t);
        std::vector<U256> v;
        for (const Fr& c : P.rc) v.push_back(c.to_u256());
        for (int i = 0; i < t; ++i) for (int j = 0; j < t; ++j) v.push_back(P.mds[i][j].to_u256());
        r_p = P.r_p;
        n = (uint32_t)v.size();
        buf.upload(v);
    }
    size_t smem() const { return 32ull * n; }
};

struct Timer {
    cudaEvent_t a = nullptr, b = nullptr;
    Timer() { CUDA_OK(cudaEventCreate(&a)); CUDA_OK(cudaEventCreate(&b)); CUDA_OK(cudaEventRecord(a)); }
    ~Timer() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
    void stop() {          // after the last kernel: the device time of the call's kernels
        CUDA_OK(cudaEventRecord(b));
        CUDA_OK(cudaEventSynchronize(b));
        float ms = 0;
        CUDA_OK(cudaEventElapsedTime(&ms, a, b));
        g_last_device_ms = ms;
    }
};

uint32_t read_bad(const DevBuf& bad) {
    uint32_t v = 0;
    CUDA_OK(cudaMemcpy(&v, bad.p, 4, cudaMemcpyDeviceToHost));
    return v;
}

void bad_flag(DevBuf& d) {
    d.alloc(4);
    CUDA_OK(cudaMemset(d.p, 0xff, 4));
}

uint32_t blocks_for(uint64_t count) {
    const uint64_t b = (count + dev::REG_THREADS - 1) / dev::REG_THREADS;
    if (b > 0x7fffffffull) throw std::runtime_error("count too large");
    return (uint32_t)b;
}

template <class K>
void set_smem(K kernel, size_t bytes) {
    CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
}

// the key shapes PoseidonLarge takes (zke_pubkey_hashes, zke_domain_key_leaves)
void check_key_shape(uint32_t modulus_bytes, uint32_t n, uint32_t k) {
    if (k < 17 || k > 32) throw std::runtime_error("k must be 17..32 (PoseidonLarge), not " + std::to_string(k));
    if (n == 0 || 2 * n >= 251) throw std::runtime_error("n must satisfy 0 < 2n < 251 (PoseidonLarge), not " + std::to_string(n));
    if (modulus_bytes == 0) throw std::runtime_error("modulus_bytes must be positive");
}

// why a domain row is not canonical (the device only reports which row)
std::string domain_fault(const uint8_t* d) {
    if (d[0] == 0) return "is empty";
    uint32_t len = 0;
    while (len < dev::DOMAIN_BYTES && d[len]) ++len;
    for (uint32_t j = len; j < dev::DOMAIN_BYTES; ++j)
        if (d[j]) return "has a zero byte at " + std::to_string(len) + " inside the name";
    for (uint32_t j = 0; j < len; ++j) {
        if (d[j] >= 0x80) return "has a non-ASCII byte at " + std::to_string(j) + " (give the A-label form)";
        if (d[j] >= 'A' && d[j] <= 'Z') return "has an upper-case byte at " + std::to_string(j);
    }
    if (d[len - 1] == '.') return "ends with a dot";
    return "";
}

// the refusals of zke_merkle_build and zke_registry_open
void check_tree(const uint8_t* leaves, size_t count, uint32_t depth) {
    if (!leaves) throw std::runtime_error("null argument");
    if (depth < 1 || depth > 32) throw std::runtime_error("depth must be 1..32, not " + std::to_string(depth));
    if (count == 0) throw std::runtime_error("count must be at least 1");
    if ((uint64_t)count > (1ull << depth))
        throw std::runtime_error("count " + std::to_string(count) + " does not fit a tree of depth " + std::to_string(depth));
}

// level l starts at the sum of the sizes of levels below it in a tree of `cap` leaves and holds ceil(count / 2^l) nodes
dev::LevelTable level_table(uint64_t count, uint64_t cap, uint32_t depth, uint64_t* total) {
    dev::LevelTable lt;
    uint64_t pos = 0;
    for (uint32_t l = 0; l <= depth; ++l) {
        lt.off[l] = pos;
        lt.size[l] = (count + (1ull << l) - 1) >> l;
        pos += (cap + (1ull << l) - 1) >> l;
    }
    if (total) *total = pos;
    return lt;
}

// zeros[l], the root of an empty subtree of height l, standard form
std::vector<U256> zero_nodes(uint32_t depth) {
    std::vector<U256> zeros(depth + 1);
    zeros[0] = U256{{0, 0, 0, 0}};
    Fr z = Fr::zero();
    for (uint32_t l = 1; l <= depth; ++l) { z = gadgets::poseidon_hash({z, z}); zeros[l] = z.to_u256(); }
    return zeros;
}

// levels 1..depth of the tree whose `count` leaves are on the device at lt.off[0]; refuses a leaf not below r, naming it
// (the host copy `leaves` is searched: the fused kernel reports the first leaf of the block)
void build_tree(uint8_t* d, const dev::LevelTable& lt, uint64_t count, uint32_t depth, const WidthConsts& C,
                const uint8_t* zeros, const uint8_t* leaves) {
    DevBuf bad;
    bad_flag(bad);
    const int L = depth < (uint32_t)dev::FUSE_LEVELS ? (int)depth : dev::FUSE_LEVELS;
    const size_t smem = C.smem(), smem_fused = smem + 32ull * dev::REG_THREADS;
    set_smem(dev::merkle_fused_kernel, smem_fused);
    Timer tm;
    dev::merkle_fused_kernel<<<(uint32_t)((count + (1ull << L) - 1) >> L), dev::REG_THREADS, smem_fused>>>(d, lt, L, C.buf.p, C.r_p, zeros, reinterpret_cast<uint32_t*>(bad.p));
    ZKE_COUNT_LAUNCH(1);
    CHECK_LAUNCH();
    for (uint32_t l = (uint32_t)L + 1; l <= depth; ++l) {
        dev::merkle_level_kernel<<<blocks_for(lt.size[l]), dev::REG_THREADS, smem>>>(d, lt.off[l - 1], lt.size[l - 1], lt.off[l],
                                                                                   lt.size[l], C.buf.p, C.r_p, zeros + 32ull * (l - 1));
        ZKE_COUNT_LAUNCH(1);
        CHECK_LAUNCH();
    }
    tm.stop();
    const uint32_t b = read_bad(bad);
    if (b != dev::NO_BAD) {
        for (uint64_t i = b; i < count; ++i) {
            U256 x;
            memcpy(x.v, leaves + 32 * i, 32);
            if (u256_cmp(x, fr_params().p) >= 0) throw std::runtime_error("leaf " + std::to_string(i) + " is not below r");
        }
        throw std::runtime_error("a leaf is not below r");
    }
}

}  // namespace

// A tree resident on one device (zke_registry_open): the levels in one buffer laid out as level_table(count, cap),
// where cap >= count leaves have room; appends past cap double it (at most 2^depth) and move each level's live prefix.
struct zke_registry {
    int device;
    uint32_t depth;
    uint64_t count = 0, cap = 0;
    dev::LevelTable lt{};
    DevBuf levels, zeros, io, out;          // io, out: upload and download staging of update / nodes
    WidthConsts C{3};

    zke_registry(int dv, uint32_t d) : device(dv), depth(d) { zeros.upload(zero_nodes(d)); }

    // room for `need` leaves (need <= 2^depth), keeping every live node
    void reserve(uint64_t need) {
        if (need <= cap) return;
        uint64_t c = cap ? cap : need;
        while (c < need) c *= 2;
        c = std::min<uint64_t>(c, 1ull << depth);
        uint64_t total = 0;
        const dev::LevelTable nt = level_table(count, c, depth, &total);
        DevBuf nb;
        nb.alloc(32 * total);
        if (count)
            for (uint32_t l = 0; l <= depth; ++l)
                CUDA_OK(cudaMemcpy(nb.p + 32 * nt.off[l], levels.p + 32 * lt.off[l], 32 * lt.size[l], cudaMemcpyDeviceToDevice));
        std::swap(levels.p, nb.p);
        std::swap(levels.bytes, nb.bytes);
        lt = nt;
        cap = c;
    }
};

extern "C" {

int zke_poseidon_batch(const uint8_t* inputs, uint32_t width, size_t count, int device, uint8_t* out, char* err, size_t errcap) {
    try {
        if (!inputs || !out) throw std::runtime_error("null argument");
        if (width < 1 || width > 16) throw std::runtime_error("width must be 1..16, not " + std::to_string(width));
        if (count == 0) return 0;
        select_device(device);
        const int t = (int)width + 1;
        WidthConsts C(t);
        DevBuf din, dout, bad;
        bad_flag(bad);
        din.alloc(32ull * width * count);
        dout.alloc(32ull * count);
        CUDA_OK(cudaMemcpy(din.p, inputs, din.bytes, cudaMemcpyHostToDevice));
        Timer tm;
        set_smem(dev::poseidon_batch_kernel, C.smem());
        dev::poseidon_batch_kernel<<<blocks_for(count), dev::REG_THREADS, C.smem()>>>(din.p, count, t, C.buf.p, C.r_p, dout.p,
                                                                                     reinterpret_cast<uint32_t*>(bad.p));
        ZKE_COUNT_LAUNCH(1);
        CHECK_LAUNCH();
        tm.stop();
        const uint32_t b = read_bad(bad);
        if (b != dev::NO_BAD) throw std::runtime_error("instance " + std::to_string(b) + ": an input is not below r");
        CUDA_OK(cudaMemcpy(out, dout.p, dout.bytes, cudaMemcpyDeviceToHost));
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_pubkey_hashes(const uint8_t* moduli, size_t count, uint32_t modulus_bytes, uint32_t n, uint32_t k, int device,
                      uint8_t* out, char* err, size_t errcap) {
    try {
        if (!moduli || !out) throw std::runtime_error("null argument");
        check_key_shape(modulus_bytes, n, k);
        if (count == 0) return 0;
        select_device(device);
        const int t = (int)(k + 1) / 2 + 1;
        WidthConsts C(t);
        DevBuf dm, dout, bad;
        bad_flag(bad);
        dm.alloc((size_t)modulus_bytes * count);
        dout.alloc(32ull * count);
        CUDA_OK(cudaMemcpy(dm.p, moduli, dm.bytes, cudaMemcpyHostToDevice));
        Timer tm;
        set_smem(dev::pubkey_hash_kernel, C.smem());
        dev::pubkey_hash_kernel<<<blocks_for(count), dev::REG_THREADS, C.smem()>>>(dm.p, count, modulus_bytes, n, k, C.buf.p, C.r_p,
                                                                                  dout.p, reinterpret_cast<uint32_t*>(bad.p));
        ZKE_COUNT_LAUNCH(1);
        CHECK_LAUNCH();
        tm.stop();
        const uint32_t b = read_bad(bad);
        if (b != dev::NO_BAD)
            throw std::runtime_error("modulus " + std::to_string(b) + " is not below 2^(n k) = 2^" + std::to_string(n * k));
        CUDA_OK(cudaMemcpy(out, dout.p, dout.bytes, cudaMemcpyDeviceToHost));
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_domain_key_leaves(const uint8_t* moduli, size_t count, uint32_t modulus_bytes, uint32_t n, uint32_t k,
                          const uint8_t* domains, int device, uint8_t* out, char* err, size_t errcap) {
    try {
        if (!moduli || !domains || !out) throw std::runtime_error("null argument");
        check_key_shape(modulus_bytes, n, k);
        if (count == 0) return 0;
        select_device(device);
        const int tk = (int)(k + 1) / 2 + 1;
        WidthConsts Cd(dev::DOMAIN_T), Ck(tk), C2(3);
        const size_t smem = Cd.smem() + (tk == (int)dev::DOMAIN_T ? 0 : Ck.smem()) + C2.smem();
        DevBuf dm, dd, dout, bad_key, bad_domain;
        bad_flag(bad_key);
        bad_flag(bad_domain);
        dm.alloc((size_t)modulus_bytes * count);
        dd.alloc((size_t)dev::DOMAIN_BYTES * count);
        dout.alloc(32ull * count);
        CUDA_OK(cudaMemcpy(dm.p, moduli, dm.bytes, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(dd.p, domains, dd.bytes, cudaMemcpyHostToDevice));
        Timer tm;
        set_smem(dev::domain_key_leaf_kernel, smem);     // above the 48 KB default once the key has a width of its own (k >= 19)
        dev::domain_key_leaf_kernel<<<blocks_for(count), dev::REG_THREADS, smem>>>(
            dm.p, dd.p, count, modulus_bytes, n, k, Cd.buf.p, Cd.r_p, Ck.buf.p, Ck.r_p, C2.buf.p, C2.r_p, dout.p,
            reinterpret_cast<uint32_t*>(bad_key.p), reinterpret_cast<uint32_t*>(bad_domain.p));
        ZKE_COUNT_LAUNCH(1);
        CHECK_LAUNCH();
        tm.stop();
        const uint32_t bk = read_bad(bad_key), bd = read_bad(bad_domain);
        if (bk != dev::NO_BAD)
            throw std::runtime_error("modulus " + std::to_string(bk) + " is not below 2^(n k) = 2^" + std::to_string(n * k));
        if (bd != dev::NO_BAD)
            throw std::runtime_error("domain " + std::to_string(bd) + " is not canonical: it " +
                                     domain_fault(domains + (size_t)dev::DOMAIN_BYTES * bd));
        CUDA_OK(cudaMemcpy(out, dout.p, dout.bytes, cudaMemcpyDeviceToHost));
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int64_t zke_merkle_build(const uint8_t* leaves, size_t count, uint32_t depth, int device, uint8_t* levels, size_t cap,
                         char* err, size_t errcap) {
    try {
        check_tree(leaves, count, depth);
        uint64_t total = 0;
        const dev::LevelTable lt = level_table(count, count, depth, &total);
        const int64_t bytes = (int64_t)(32 * total);
        if (!levels) return bytes;
        if (cap < (size_t)bytes) return -2;
        select_device(device);
        WidthConsts C(3);
        DevBuf d, dz;
        dz.upload(zero_nodes(depth));
        d.alloc((size_t)bytes);
        CUDA_OK(cudaMemcpy(d.p, leaves, 32ull * count, cudaMemcpyHostToDevice));
        build_tree(d.p, lt, count, depth, C, dz.p, leaves);
        CUDA_OK(cudaMemcpy(levels, d.p, (size_t)bytes, cudaMemcpyDeviceToHost));
        return bytes;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

zke_registry* zke_registry_open(const uint8_t* leaves, size_t count, uint32_t depth, int device, char* err, size_t errcap) {
    try {
        check_tree(leaves, count, depth);
        select_device(device);
        std::unique_ptr<zke_registry> r(new zke_registry(device, depth));
        r->reserve(count);
        r->count = count;
        r->lt = level_table(count, r->cap, depth, nullptr);
        CUDA_OK(cudaMemcpy(r->levels.p, leaves, 32ull * count, cudaMemcpyHostToDevice));
        build_tree(r->levels.p, r->lt, count, depth, r->C, r->zeros.p, leaves);
        return r.release();
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return nullptr; }
}

int zke_registry_update(zke_registry* r, const uint64_t* indices, const uint8_t* leaves, size_t k, char* err, size_t errcap) {
    try {
        if (!r) throw std::runtime_error("null registry");
        if (k == 0) return 0;
        if (!indices || !leaves) throw std::runtime_error("null argument");
        // every check before the first device write: a refused update leaves the tree as it was
        for (size_t i = 0; i < k; ++i) {
            U256 x;
            memcpy(x.v, leaves + 32 * i, 32);
            if (u256_cmp(x, fr_params().p) >= 0)
                throw std::runtime_error("leaf " + std::to_string(i) + " of the update is not below r");
        }
        std::vector<size_t> ord(k);
        for (size_t i = 0; i < k; ++i) ord[i] = i;
        std::sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return indices[a] < indices[b]; });
        uint64_t appended = 0;
        for (size_t j = 0; j < k; ++j) {
            const uint64_t x = indices[ord[j]];
            if (j > 0 && x == indices[ord[j - 1]]) throw std::runtime_error("index " + std::to_string(x) + " appears twice");
            if (x >= r->count) {
                if (x != r->count + appended)
                    throw std::runtime_error("index " + std::to_string(x) + " leaves a gap after the " +
                                             std::to_string(r->count + appended) + " leaves");
                ++appended;
            }
        }
        const uint64_t count = r->count + appended;
        if (count > (1ull << r->depth))
            throw std::runtime_error(std::to_string(count) + " leaves do not fit a tree of depth " + std::to_string(r->depth));
        // one upload: the leaves in index order, then the sorted indices
        std::vector<uint8_t> host(40 * k);
        uint64_t* idx = reinterpret_cast<uint64_t*>(host.data() + 32 * k);
        for (size_t j = 0; j < k; ++j) {
            memcpy(host.data() + 32 * j, leaves + 32 * ord[j], 32);
            idx[j] = indices[ord[j]];
        }
        CUDA_OK(cudaSetDevice(r->device));
        r->reserve(count);
        r->count = count;
        r->lt = level_table(count, r->cap, r->depth, nullptr);
        r->io.reserve(host.size());
        CUDA_OK(cudaMemcpy(r->io.p, host.data(), host.size(), cudaMemcpyHostToDevice));
        const uint64_t* didx = reinterpret_cast<const uint64_t*>(r->io.p + 32 * k);
        const dev::LevelTable& lt = r->lt;
        Timer tm;
        dev::registry_scatter_kernel<<<blocks_for(k), dev::REG_THREADS>>>(r->levels.p + 32 * lt.off[0], didx, r->io.p, k);
        ZKE_COUNT_LAUNCH(1);
        CHECK_LAUNCH();
        for (uint32_t l = 1; l <= r->depth; ++l) {
            dev::registry_update_level_kernel<<<blocks_for(k), dev::REG_THREADS, r->C.smem()>>>(
                r->levels.p, didx, k, (int)l, lt.off[l - 1], lt.size[l - 1], lt.off[l], r->C.buf.p, r->C.r_p,
                r->zeros.p + 32ull * (l - 1));
            ZKE_COUNT_LAUNCH(1);
            CHECK_LAUNCH();
        }
        tm.stop();
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_registry_nodes(zke_registry* r, const uint32_t* levels, const uint64_t* indices, size_t k, uint8_t* out,
                       char* err, size_t errcap) {
    try {
        if (!r) throw std::runtime_error("null registry");
        if (k == 0) return 0;
        if (!levels || !indices || !out) throw std::runtime_error("null argument");
        for (size_t i = 0; i < k; ++i) {
            if (levels[i] > r->depth)
                throw std::runtime_error("node " + std::to_string(i) + ": level " + std::to_string(levels[i]) +
                                         " is above the root (level " + std::to_string(r->depth) + ")");
            if (indices[i] >= (1ull << (r->depth - levels[i])))
                throw std::runtime_error("node " + std::to_string(i) + ": index " + std::to_string(indices[i]) +
                                         " is outside level " + std::to_string(levels[i]) + " of a tree of depth " +
                                         std::to_string(r->depth));
        }
        CUDA_OK(cudaSetDevice(r->device));
        r->io.reserve(12 * k);
        CUDA_OK(cudaMemcpy(r->io.p, indices, 8 * k, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(r->io.p + 8 * k, levels, 4 * k, cudaMemcpyHostToDevice));
        r->out.reserve(32 * k);
        Timer tm;
        dev::registry_gather_kernel<<<blocks_for(k), dev::REG_THREADS>>>(
            r->levels.p, r->lt, reinterpret_cast<const uint32_t*>(r->io.p + 8 * k), reinterpret_cast<const uint64_t*>(r->io.p),
            k, r->zeros.p, r->out.p);
        ZKE_COUNT_LAUNCH(1);
        CHECK_LAUNCH();
        tm.stop();
        CUDA_OK(cudaMemcpy(out, r->out.p, 32 * k, cudaMemcpyDeviceToHost));
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int64_t zke_registry_levels(zke_registry* r, uint8_t* out, size_t cap, char* err, size_t errcap) {
    try {
        if (!r) throw std::runtime_error("null registry");
        uint64_t total = 0;
        for (uint32_t l = 0; l <= r->depth; ++l) total += r->lt.size[l];
        const int64_t bytes = (int64_t)(32 * total);
        if (!out) return bytes;
        if (cap < (size_t)bytes) return -2;
        CUDA_OK(cudaSetDevice(r->device));
        Timer tm;
        uint64_t pos = 0;
        for (uint32_t l = 0; l <= r->depth; pos += r->lt.size[l], ++l)
            CUDA_OK(cudaMemcpy(out + 32ull * pos, r->levels.p + 32 * r->lt.off[l], 32 * r->lt.size[l], cudaMemcpyDeviceToHost));
        tm.stop();
        return bytes;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

uint64_t zke_registry_count(const zke_registry* r) { return r ? r->count : 0; }

void zke_registry_close(zke_registry* r) {
    if (!r) return;
    cudaSetDevice(r->device);
    delete r;
}

double zke_registry_device_ms(void) { return g_last_device_ms; }

}  // extern "C"
