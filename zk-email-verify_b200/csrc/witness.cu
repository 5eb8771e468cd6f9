// Batched witness generation on the GPU.
//
// Replaces the circom-generated WASM witness calculator that snarkjs' fullProve runs single-threaded
// (/root/reference/packages/helpers/src/chunked-zkey.ts:80-84 -> wtns.calculate, SURVEY 3.2).
//
// Mapping: ONE CTA PER EMAIL.  The witness program is levelised by the front-end (circuit.cpp): all ops of a level
// depend only on earlier levels, so the CTA's threads evaluate a level's ops in parallel and meet at a
// __syncthreads(); the long dependency chains of the circuit (40 chained SHA-256 compressions, 17 chained
// 2048-bit modular multiplications, the 1025-step regex automaton) cost one barrier per level instead of one
// kernel launch per level, and emails are independent so the batch fills the SMs (132 on an H100 -> size the batch in
// multiples of 132 x CTAs/SM for full occupancy).  Witness values live in HBM as 32-byte standard-form
// little-endian words, [email][signal]; the bounding resource is dependent-load latency, not bandwidth
// (SURVEY 8(d): 32*m bytes written per email).
#include "device_engine.cuh"
#include "lc_term.cuh"
#include "bigdiv.hpp"
#include <cstdlib>

namespace zke {
namespace dev {

// Evaluates up to three LCs whose terms are laid out back to back [A | B | C] at `t` (shared memory, or global for an
// oversized iteration).  The gathers of four consecutive terms are issued together - across the LC boundaries - so
// an 8-term `a*b + c` costs two dependent memory round trips instead of one per LC.
__device__ __forceinline__ void eval_lcs(const DevProgram& P, const uint8_t* w, const uint2* t, uint32_t nA, uint32_t nB,
                                         uint32_t nC, Fr& xa, Fr& xb, Fr& xc) {
    xa = Fr::zero(); xb = Fr::zero(); xc = Fr::zero();
    const uint32_t eA = nA, eB = nA + nB, total = nA + nB + nC;
    for (uint32_t j = 0; j < total; j += 4) {
        uint2 tt[4];
        Fr x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) if (j + u < total) tt[u] = t[j + u];
#pragma unroll
        for (int u = 0; u < 4; ++u) if (j + u < total) x[u] = Fr::load(w + 32ull * tt[u].x);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (j + u < total) {
                const TermVal tv = term_value(P.coef_r, tt[u], x[u]);
                const uint32_t idx = j + u;
                if (idx < eA) xa = tv.neg ? xa - tv.v : xa + tv.v;
                else if (idx < eB) xb = tv.neg ? xb - tv.v : xb + tv.v;
                else xc = tv.neg ? xc - tv.v : xc + tv.v;
            }
        }
    }
}

__device__ __forceinline__ bool is_small(const Fr& x, uint32_t bound) {
    return (x.v[1] | x.v[2] | x.v[3] | x.v[4] | x.v[5] | x.v[6] | x.v[7]) == 0 && x.v[0] < bound;
}

__device__ Fr invz(const DevProgram& P, const Fr& x) {   // circomlib IsZero: inv <-- in != 0 ? 1/in : 0
    if (x.is_zero()) return x;
    if (is_small(x, P.n_small_inv)) return Fr::load(P.small_inv + 32ull * x.v[0]);
    Fr n = Fr::zero() - x;
    if (is_small(n, P.n_small_inv)) return Fr::zero() - Fr::load(P.small_inv + 32ull * n.v[0]);
    return x.to_mont().inv().from_mont();
}

__device__ __forceinline__ Fr shrand(const Fr& x, uint32_t shift, uint32_t nbits) {
    Fr o = Fr::zero();
    if (shift < 256) {
        const uint32_t ws = shift >> 5, bs = shift & 31;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            uint32_t lo = (j + ws < 8) ? x.v[(j + ws) & 7] : 0;
            uint32_t hi = (j + ws + 1 < 8) ? x.v[(j + ws + 1) & 7] : 0;
            o.v[j] = bs ? ((lo >> bs) | (hi << (32 - bs))) : lo;
        }
    }
    if (nbits && nbits < 256) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (32u * j >= nbits) o.v[j] = 0;
            else if (32u * (j + 1) > nbits) o.v[j] &= (1u << (nbits - 32u * j)) - 1;
        }
    }
    return o;
}

__device__ void fpmul_hint_dev(const DevProgram& P, uint8_t* w, uint32_t aux_off, uint32_t dst) {
    const uint32_t* ax = P.aux + aux_off;
    const uint32_t n = ax[0], k = ax[1];
    uint32_t a[8 * 20], b[8 * 20], p[8 * 20], q[8 * 20], r[8 * 20];
    if (k > 20) return;
    for (uint32_t i = 0; i < k; ++i) {
        Fr x = Fr::load(w + 32ull * ax[2 + i]), y = Fr::load(w + 32ull * ax[2 + k + i]), z = Fr::load(w + 32ull * ax[2 + 2 * k + i]);
        for (int j = 0; j < 8; ++j) { a[8 * i + j] = x.v[j]; b[8 * i + j] = y.v[j]; p[8 * i + j] = z.v[j]; }
    }
    if (fpmul_hint_words(n, k, a, b, p, q, r) != 0) {
        for (uint32_t i = 0; i < 8 * k; ++i) { q[i] = 0; r[i] = 0; }
    }
    for (uint32_t i = 0; i < k; ++i) {
        Fr x, y;
        for (int j = 0; j < 8; ++j) { x.v[j] = q[8 * i + j]; y.v[j] = r[8 * i + j]; }
        x.store(w + 32ull * (dst + i));
        y.store(w + 32ull * (dst + k + i));
    }
}

// ---- native Sha256compression (circuit.hpp: ShaBlock) ----------------------------------------------------------------
// The gadget's ~30 k signals are all bits of 64-bit quantities of one plain compression: the CTA gathers the 768 input
// bits, one thread runs the compression and leaves the quantities in shared memory, and all threads write the signals -
// one dependency level instead of the gadget's ~320 (the 40 chained compressions of the default EmailVerifier were 60 %
// of the witness kernel's level count).  The CPU oracle still walks the gadget's own ops, so "GPU witness == oracle
// witness" checks this path end to end; tests/test_sha_native_table.py pins the quantity table on the CPU.
__constant__ uint32_t SHA_K_DEV[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01, 0x243185be,
    0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa,
    0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967, 0x27b70a85,
    0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85, 0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3,
    0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f,
    0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
static const uint32_t SHA_Q_WORDS = 17 * 64;      // quantity groups x 64 (circuit.hpp: ShaQuantity)
__device__ __forceinline__ uint32_t rotr32(uint32_t x, int r) { return __funnelshift_r(x, x, r); }

__device__ void sha_coop(const DevProgram& P, uint8_t* w, uint32_t aux_off, unsigned long long* Q, uint32_t* inw) {
    const uint32_t tid = threadIdx.x;
    const uint32_t* ax = P.aux + aux_off;
    const uint32_t n_desc = ax[0];
    const uint32_t* src = ax + 1;
    const uint32_t* desc = ax + 1 + 768;
    if (tid < 24) inw[tid] = 0;
    __syncthreads();
    for (uint32_t i = tid; i < 768; i += WITNESS_THREADS) {
        const uint32_t s = src[i];
        uint32_t bit;
        if (s >= 0xfffffffeu) bit = s & 1u;                                   // SHA_CONST0 / SHA_CONST1
        else bit = *reinterpret_cast<const uint32_t*>(w + 32ull * s) & 1u;
        if (bit) {
            if (i < 256) atomicOr(&inw[i >> 5], 1u << (i & 31));              // chaining words, LSB first
            else { const uint32_t j = i - 256; atomicOr(&inw[8 + (j >> 5)], 1u << (31 - (j & 31))); }   // message words, MSB first
        }
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t W[64];
#pragma unroll
        for (int t = 0; t < 16; ++t) W[t] = inw[8 + t];
#pragma unroll 1
        for (int t = 16; t < 64; ++t) {
            const uint32_t x = W[t - 2], y = W[t - 15];
            const uint32_t s1 = rotr32(x, 17) ^ rotr32(x, 19) ^ (x >> 10), s0 = rotr32(y, 7) ^ rotr32(y, 18) ^ (y >> 3);
            Q[0 * 64 + t] = rotr32(x, 19) & (x >> 10);
            Q[1 * 64 + t] = s1;
            Q[2 * 64 + t] = rotr32(y, 18) & (y >> 3);
            Q[3 * 64 + t] = s0;
            const unsigned long long sum = (unsigned long long)s1 + W[t - 7] + s0 + W[t - 16];
            Q[4 * 64 + t] = sum;
            W[t] = (uint32_t)sum;
        }
        uint32_t a = inw[0], b = inw[1], c = inw[2], d = inw[3], e = inw[4], f = inw[5], g = inw[6], h = inw[7];
#pragma unroll 1
        for (int t = 0; t < 64; ++t) {
            const uint32_t bs1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25), ch = (e & f) ^ (~e & g);
            Q[5 * 64 + t] = rotr32(e, 11) & rotr32(e, 25);
            Q[6 * 64 + t] = bs1;
            Q[7 * 64 + t] = ch;
            const unsigned long long t1 = (unsigned long long)h + bs1 + ch + SHA_K_DEV[t] + W[t];
            Q[8 * 64 + t] = t1;
            const uint32_t bs0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22), mj = (a & b) ^ (a & c) ^ (b & c);
            Q[9 * 64 + t] = rotr32(a, 13) & rotr32(a, 22);
            Q[10 * 64 + t] = bs0;
            Q[11 * 64 + t] = b & c;
            Q[12 * 64 + t] = mj;
            const unsigned long long t2 = (unsigned long long)bs0 + mj;
            Q[13 * 64 + t] = t2;
            const unsigned long long sume = (unsigned long long)d + (uint32_t)t1, suma = (unsigned long long)(uint32_t)t1 + (uint32_t)t2;
            Q[14 * 64 + t] = sume;
            Q[15 * 64 + t] = suma;
            h = g; g = f; f = e; e = (uint32_t)sume; d = c; c = b; b = a; a = (uint32_t)suma;
        }
        const uint32_t st[8] = {a, b, c, d, e, f, g, h};
#pragma unroll
        for (int i = 0; i < 8; ++i) Q[16 * 64 + i] = (unsigned long long)inw[i] + st[i];
    }
    __syncthreads();
    for (uint32_t dd = tid; dd < n_desc; dd += WITNESS_THREADS) {
        const uint32_t var = desc[2 * dd], qk = desc[2 * dd + 1];
        Fr o = Fr::zero();
        o.v[0] = (uint32_t)((Q[qk >> 8] >> (qk & 255u)) & 1ull);
        o.store(w + 32ull * var);
    }
    __syncthreads();
}

// ---- zk-regex state seeding (circuit.hpp: RegexSeed) -------------------------------------------------------------------
// The state signals of a zk-regex instance form a chain as long as the message (position i needs position i - 1); the
// set of live DFA states per position is just an automaton run.  The CTA gathers the message bytes, one thread runs the
// automaton (the live set is a 64-bit mask, or four of them in the wide mode for 65..255 states; state 0 is always live,
// byte 255 - the marker - fires nothing), and all threads write the state signals of every position.  The instance's own
// ops follow at a handful of levels and write the same values again; the CPU oracle walks only those, so "GPU witness ==
// oracle witness" checks the seeding.
// Shared buffer Q (SHA_Q_WORDS 64-bit words): the live sets of up to RX_CHUNK positions (RX_CHUNK / 4 in the wide mode,
// four words each), then the staged bytes from word RX_CHUNK on, the carry in the last word (the last four, wide).
static const uint32_t RX_CHUNK = 896;
static_assert(RX_CHUNK + RX_CHUNK / 8 + 4 <= SHA_Q_WORDS, "regex chunk does not fit the shared buffer");
__device__ void regex_coop(const DevProgram& P, uint8_t* w, uint32_t aux_off, unsigned long long* Q) {
    const uint32_t tid = threadIdx.x;
    const uint32_t* ax = P.aux + aux_off;
    const uint32_t n_desc = ax[0], n_bytes = ax[1], n_states = ax[2] & 0x3fffffffu, wide = (ax[2] >> 30) & 1u, mode = ax[2] >> 31;
    const unsigned long long first = (unsigned long long)ax[3] | ((unsigned long long)ax[4] << 32);
    const uint32_t* bytes = ax + (wide ? 11 : 5);
    const uint8_t* table = reinterpret_cast<const uint8_t*>(bytes + n_bytes);
    const uint8_t* group = table + n_states * 256u;                  // mode 1 only
    const uint32_t* desc = bytes + n_bytes + n_states * 64 * (1 + mode);
    const uint32_t chunk = wide ? RX_CHUNK / 4 : RX_CHUNK;
    uint8_t* staged = reinterpret_cast<uint8_t*>(Q + RX_CHUNK);
    for (uint32_t base = 0; base < n_bytes; base += chunk) {
        const uint32_t cnt = min(chunk, n_bytes - base);
        __syncthreads();                                           // the previous chunk's masks have been consumed
        for (uint32_t j = tid; j < cnt; j += WITNESS_THREADS) {
            const Fr v = Fr::load(w + 32ull * bytes[base + j]);
            const bool is_byte = (v.v[1] | v.v[2] | v.v[3] | v.v[4] | v.v[5] | v.v[6] | v.v[7]) == 0 && v.v[0] < 255u;
            staged[j] = is_byte ? (uint8_t)v.v[0] : (uint8_t)255;  // anything else fires no transition (and fails its range checks)
        }
        __syncthreads();
        if (tid == 0 && wide) {
            unsigned long long live[4];
#pragma unroll
            for (int q = 0; q < 4; ++q)
                live[q] = base == 0 ? (unsigned long long)ax[3 + 2 * q] | ((unsigned long long)ax[4 + 2 * q] << 32) : Q[SHA_Q_WORDS - 4 + q];
            for (uint32_t j = 0; j < cnt; ++j) {
                const uint32_t c = staged[j];
                unsigned long long next[4] = {1ull, 0ull, 0ull, 0ull};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    unsigned long long m = live[q];
                    while (m) {
                        const uint32_t st = 64u * q + (uint32_t)(__ffsll((long long)m) - 1);
                        m &= m - 1;
                        const uint32_t d = table[st * 256u + c];
                        if (d != 0xffu) next[d >> 6] |= 1ull << (d & 63u);
                    }
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) { live[q] = next[q]; Q[4 * j + q] = next[q]; }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) Q[SHA_Q_WORDS - 4 + q] = live[q];
        } else if (tid == 0) {
            unsigned long long mask = base == 0 ? first : Q[SHA_Q_WORDS - 1];
            for (uint32_t j = 0; mode == 1 && j < cnt; ++j) {     // compact shape: one state, Q[j] = the product that fires
                const uint32_t at = (uint32_t)mask * 256u + staged[j];
                const uint32_t d = table[at];
                Q[j] = group[at];
                mask = d != 0xffu ? d : 0u;
            }
            for (uint32_t j = 0; mode == 0 && j < cnt; ++j) {
                const uint32_t c = staged[j];
                unsigned long long next = 1ull, m = mask;
                while (m) {
                    const int st = __ffsll((long long)m) - 1;
                    m &= m - 1;
                    const uint32_t d = table[(uint32_t)st * 256u + c];
                    if (d != 0xffu) next |= 1ull << d;
                }
                mask = next;
                Q[j] = mask;
            }
            Q[SHA_Q_WORDS - 1] = mask;
        }
        __syncthreads();
        for (uint32_t dd = tid; dd < n_desc; dd += WITNESS_THREADS) {
            const uint32_t var = desc[2 * dd], ps = desc[2 * dd + 1], s = ps & 255u;
            const uint32_t j = (ps >> 8) - 1u - base;              // position p reads message byte p - 1
            if (j < cnt) {
                Fr o = Fr::zero();
                if (wide) o.v[0] = (uint32_t)((Q[4 * j + (s >> 6)] >> (s & 63u)) & 1ull);
                else o.v[0] = mode == 1 ? (uint32_t)(Q[j] == s) : (uint32_t)((Q[j] >> s) & 1ull);
                o.store(w + 32ull * var);
            }
        }
    }
    __syncthreads();
}

// ---- cooperative FpMul hint ---------------------------------------------------------------------------------------
// (q, r) = divmod(A * B, P) on 2048-bit integers.  The sequential Knuth division above runs in one thread, and the
// 17 chained calls of RSAVerifier65537 are a long serial stretch of the witness kernel.
// All of them share the modulus, so the CTA keeps Barrett's reciprocal mu = floor(b^(2t) / P) (b = 2^32, t = words of P)
// in shared memory - computed once per email by the sequential division - and every call becomes three cooperative
// products (column sums by 146 threads + one carry sweep): X = A B, q2 = floor(X / b^(t-1)) mu, q3 P, followed by at
// most two corrective subtractions (Handbook of Applied Cryptography 14.42).  Falls back to the sequential routine when
// the operands do not satisfy Barrett's preconditions (A, B >= b^t, a modulus of fewer than four words, or P = b^(t-1),
// whose reciprocal does not fit t + 1 words).  tests/test_bigdiv_hint.py mirrors these decisions on the CPU.
struct FpmulShared {
    uint32_t A[BIGDIV_MAXW], B[BIGDIV_MAXW], P[BIGDIV_MAXW + 1];
    uint32_t Pc[BIGDIV_MAXW + 1], mu[BIGDIV_MAXW + 2];     // cached modulus and its reciprocal
    uint32_t X[2 * BIGDIV_MAXW + 2], q2[2 * BIGDIV_MAXW + 4], qp[2 * BIGDIV_MAXW + 4];
    uint32_t Q[2 * BIGDIV_MAXW + 2], R[BIGDIV_MAXW + 2];
    uint32_t lo[2 * BIGDIV_MAXW + 4], mid[2 * BIGDIV_MAXW + 4], hi[2 * BIGDIV_MAXW + 4];
    int t, t_cached, mode;
};

// out[0 .. nx + ny) = x[0 .. nx) * y[0 .. ny), everything in shared memory; called by the whole CTA
__device__ void coop_mul(uint32_t* out, const uint32_t* x, int nx, const uint32_t* y, int ny, FpmulShared& S) {
    const int nc = nx + ny;
    for (int c = threadIdx.x; c < nc; c += WITNESS_THREADS) {
        unsigned long long acc = 0;
        uint32_t top = 0;
        const int i0 = c - (ny - 1) > 0 ? c - (ny - 1) : 0, i1 = c < nx - 1 ? c : nx - 1;
        for (int i = i0; i <= i1; ++i) {
            const unsigned long long pr = (unsigned long long)x[i] * y[c - i];
            acc += pr;
            top += acc < pr;
        }
        S.lo[c] = (uint32_t)acc; S.mid[c] = (uint32_t)(acc >> 32); S.hi[c] = top;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long carry = 0;
        for (int c = 0; c < nc; ++c) {
            const unsigned long long sum = carry + S.lo[c] + (c >= 1 ? S.mid[c - 1] : 0u) + (c >= 2 ? S.hi[c - 2] : 0u);
            out[c] = (uint32_t)sum;
            carry = sum >> 32;
        }
    }
    __syncthreads();
}

__device__ void fpmul_coop(const DevProgram& P, uint8_t* w, uint32_t aux_off, uint32_t dst, FpmulShared& S) {
    const uint32_t tid = threadIdx.x;
    const uint32_t* ax = P.aux + aux_off;
    const uint32_t n = ax[0], k = ax[1];
    const int W = (int)((n * k + 256 + 31) / 32);
    // assemble the three operands from their n-bit limbs (one thread each; 17 limbs x 9 words)
    if (tid < 3) {
        uint32_t* dstw = tid == 0 ? S.A : (tid == 1 ? S.B : S.P);
        for (int i = 0; i < W; ++i) dstw[i] = 0;
        for (uint32_t i = 0; i < k; ++i) {
            const Fr x = Fr::load(w + 32ull * ax[2 + tid * k + i]);
            bd_add_shifted(dstw, W, x.v, n * i);
        }
    }
    __syncthreads();
    if (tid == 0) {
        int t = W;
        while (t > 0 && S.P[t - 1] == 0) --t;
        S.t = t;
        bool fits = t >= 4;
        for (int i = t; i < W && fits; ++i) fits = S.A[i] == 0 && S.B[i] == 0;       // A, B < b^t  =>  A B < b^(2t)
        // P = b^(t-1) exactly: the reciprocal b^(t+1) needs t + 2 words, and bd_knuth_div writes only t + 1 quotient
        // words (it would leave b^(t+1) - 1) - sequential path
        bool power = fits && S.P[t - 1] == 1;
        for (int i = 0; i < t - 1 && power; ++i) power = S.P[i] == 0;
        if (power) fits = false;
        S.mode = fits ? 1 : 0;
        if (fits) {
            bool same = S.t_cached == t;
            for (int i = 0; i < t && same; ++i) same = S.Pc[i] == S.P[i];
            if (!same) {
                // mu = floor(b^(2t) / P) < b^(t+1): sequential division, once per modulus (scratch: q2 = dividend,
                // qp = divisor copy, X = quotient)
                for (int i = 0; i < 2 * t + 2; ++i) S.q2[i] = 0;
                S.q2[2 * t] = 1;
                for (int i = 0; i < t; ++i) S.qp[i] = S.P[i];
                for (int i = 0; i < 2 * t + 1; ++i) S.X[i] = 0;
                bd_knuth_div(S.q2, 2 * t, S.qp, t, S.X);
                for (int i = 0; i <= t; ++i) S.mu[i] = S.X[i];
                for (int i = 0; i < t; ++i) S.Pc[i] = S.P[i];
                S.t_cached = t;
            }
        }
    }
    __syncthreads();
    if (S.mode == 0) {
        if (tid == 0) fpmul_hint_dev(P, w, aux_off, dst);          // sequential fallback (also t == 0: zeros)
        __syncthreads();
        return;
    }
    const int t = S.t;
    coop_mul(S.X, S.A, t, S.B, t, S);                              // X = A B, 2t words
    coop_mul(S.q2, S.X + (t - 1), t + 1, S.mu, t + 1, S);          // q1 mu, q1 = floor(X / b^(t-1))
    coop_mul(S.qp, S.q2 + (t + 1), t + 1, S.P, t, S);              // q3 P,  q3 = floor(q2 / b^(t+1))
    if (tid == 0) {
        uint32_t* q3 = S.q2 + (t + 1);
        // R = X - q3 P  (mod b^(t+1): 0 <= R < 3 P fits t + 1 words)
        unsigned long long borrow = 0;
        for (int i = 0; i <= t; ++i) {
            const unsigned long long d = (unsigned long long)S.X[i] - S.qp[i] - borrow;
            S.R[i] = (uint32_t)d;
            borrow = (d >> 32) & 1;
        }
        for (int i = 0; i <= t; ++i) S.Q[i] = q3[i];
        for (int i = t + 1; i < 2 * W + 1; ++i) S.Q[i] = 0;
        for (int round = 0; round < 3; ++round) {                  // at most two corrections
            bool ge = S.R[t] != 0;
            if (!ge) {
                ge = true;
                for (int i = t - 1; i >= 0; --i) if (S.R[i] != S.P[i]) { ge = S.R[i] > S.P[i]; break; }
            }
            if (!ge) break;
            unsigned long long br = 0;
            for (int i = 0; i <= t; ++i) {
                const unsigned long long d = (unsigned long long)S.R[i] - (i < t ? S.P[i] : 0u) - br;
                S.R[i] = (uint32_t)d;
                br = (d >> 32) & 1;
            }
            for (int i = 0; i <= t; ++i) { if (++S.Q[i] != 0) break; }
        }
        for (int i = t; i < W + 2; ++i) S.R[i] = 0;
    }
    __syncthreads();
    if (tid < 2 * k) {
        const uint32_t i = tid < k ? tid : tid - k;
        Fr o;
        if (tid < k) bd_extract(S.Q, 2 * W + 1, n * i, n, o.v);
        else bd_extract(S.R, W + 2, n * i, n, o.v);
        o.store(w + 32ull * (dst + tid));
    }
    __syncthreads();
}

// ---- native Poseidon (circuit.hpp: PoseidonBlock) ---------------------------------------------------------------------
// The gadget's signals are the lanes of one permutation's state round by round; walked as ops they are ~4 dependency
// levels per round (x^2, x^4, x^5, mix), each holding a handful of ops.  Here ONE WARP runs the whole permutation: lane i
// holds state element i (t <= 17) in standard form, full rounds run the S-box on every lane and partial rounds on lane 0,
// the mix gathers the state with shuffles, and every lane writes the signals the gadget created for it (the slot table of
// witness_program.hpp: POSEIDON_AUX; slot 0 = no signal).  The CPU oracle walks the gadget's own ops, so "GPU witness ==
// oracle witness" checks this path; tests/test_app_commit.py checks the record on the CPU.
__device__ __forceinline__ void put_signal(uint8_t* w, uint32_t var, const Fr& x) { if (var) x.store(w + 32ull * var); }

__device__ void poseidon_coop(const DevProgram& P, uint8_t* w, uint32_t aux_off) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t* ax = P.aux + aux_off;
    const uint32_t t = ax[0], r_p = ax[1], rounds = 8 + r_p;
    const uint32_t* rc = P.aux + ax[2];              // [rounds][t] standard form, 8 words each
    const uint32_t* mds = rc + 8 * rounds * t;       // [t][t] times R
    const uint32_t* in = ax + 3;
    const uint32_t* slot = in + (t - 1);
    const bool on = lane < t;
    Fr st = Fr::zero();
    if (on && lane > 0) { st = Fr::load(w + 32ull * in[lane - 1]); put_signal(w, slot[lane], st); }
#pragma unroll 1
    for (uint32_t r = 0; r < rounds; ++r) {
        const uint32_t* sl = slot + t + 4 * (r * t + lane);
        if (on) {
            st = st + Fr::load(rc + 8 * (r * t + lane));
            if (lane == 0 || r < 4 || r >= 4 + r_p) {   // S-box: x^5 from xR = x (x) R^2 as x^2 = xR (x) x, x^4 = x^2 R (x) x^2
                const Fr xr = st * Fr::r2();
                const Fr x2 = xr * st, x2r = xr * xr;
                const Fr x4 = x2r * x2;
                st = x4 * xr;
                put_signal(w, sl[0], x2); put_signal(w, sl[1], x4); put_signal(w, sl[2], st);
            }
        }
        Fr acc = Fr::zero();
#pragma unroll 1
        for (uint32_t j = 0; j < t; ++j) {
            Fr sj;
#pragma unroll
            for (int q = 0; q < 8; ++q) sj.v[q] = __shfl_sync(0xffffffffu, st.v[q], (int)j);
            if (on) acc = acc + Fr::load(mds + 8 * (lane * t + j)) * sj;
        }
        st = acc;
        if (on) put_signal(w, sl[3], st);
    }
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// stages the term block of one iteration into shared memory (16-byte chunks, coalesced); blocks larger than the
// buffer are not staged - the ops of such an iteration read their terms from global memory instead
__device__ __forceinline__ void stage_terms(const DevProgram& P, uint2* buf, const uint4& hdr) {
    if (hdr.y > WITNESS_TERM_BUF) return;
    const uint4* src = reinterpret_cast<const uint4*>(P.terms + hdr.x);
    uint4* dst = reinterpret_cast<uint4*>(buf);
    for (uint32_t i = threadIdx.x; i < hdr.y / 2; i += WITNESS_THREADS) cp_async16(dst + i, src + i);
}

// MINB = 2 caps the kernel at 64 registers per thread (half of an SM's register file per CTA instead of all of it), so
// that the proving kernels of the previous batch can share the SM with a witness CTA when batches are pipelined
// (zke_fullprove_submit): a witness CTA is latency-bound and leaves the multiplier pipe idle.
template <int MINB>
__global__ void __launch_bounds__(WITNESS_THREADS, MINB)
witness_kernel(DevProgram P, uint8_t* __restrict__ w_all, size_t stride_elems, const uint8_t* __restrict__ inputs, uint32_t batch) {
    extern __shared__ uint4 witness_smem[];
    uint2* const term_buf = reinterpret_cast<uint2*>(witness_smem);   // 2 x WITNESS_TERM_BUF
    __shared__ unsigned long long sha_q[SHA_Q_WORDS];
    __shared__ uint32_t sha_in[24];
    __shared__ FpmulShared fpmul_s;
    if (threadIdx.x == 0) fpmul_s.t_cached = -1;        // no reciprocal cached yet (ordered by the first barrier below)
    // thread-block cluster of P.cluster CTAs per email: the iterations of a level are dealt round-robin to the CTAs
    // (iteration k -> CTA k % cluster; the host pads every level to whole rounds), a cluster barrier with release /
    // acquire semantics ends each level.  cluster == 1 is the plain one-CTA-per-email kernel.
    const uint32_t CL = P.cluster ? P.cluster : 1;
    uint32_t rank = 0;
    if (CL > 1) asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    const uint32_t email = blockIdx.x / CL;
    if (email >= batch) return;                          // (whole clusters: every CTA of a cluster shares `email`)
    uint8_t* w = w_all + 32ull * stride_elems * email;
    const uint32_t tid = threadIdx.x;

    // constant one and inputs
    if (tid == 0) { Fr one = Fr::zero(); one.v[0] = 1; one.store(w); }
    const uint8_t* in = inputs + 32ull * P.n_inputs * email;
    for (uint32_t i = tid; i < P.n_inputs; i += blockDim.x) {
        // inputs cross the ABI as raw 32-byte integers: reduce them mod r the way snarkjs' witness calculator does
        // (2^256 < 6 r, so at most five subtractions); everything downstream assumes canonical values
        Fr x = Fr::load(in + 32ull * i);
#pragma unroll 1
        for (int k = 0; k < 5; ++k) x.reduce_once();
        x.store(w + 32ull * (1 + P.n_outputs + i));
    }
    if (P.n_iters == 0) return;

    // software pipeline: op records one iteration ahead (registers), term blocks one iteration ahead (cp.async into
    // the other shared-memory buffer), iteration headers two ahead
    uint4 hdr = P.iter_hdr[rank], hdr_next = P.iter_hdr[rank + CL];
    uint4 op = P.ops[(size_t)rank * WITNESS_THREADS + tid];
    stage_terms(P, term_buf, hdr);
    cp_async_wait_all();
    __syncthreads();

    for (uint32_t k = rank, it = 0; k < P.n_iters; k += CL, ++it) {
        const uint4 hdr_next2 = P.iter_hdr[k + 2 * CL];      // the table has 2 * cluster sentinel entries
        uint4 op_next = make_uint4(0, WOP_NOP, 0, 0);
        if (k + CL < P.n_iters) {
            op_next = P.ops[(size_t)(k + CL) * WITNESS_THREADS + tid];
            stage_terms(P, term_buf + ((it + 1) & 1) * WITNESS_TERM_BUF, hdr_next);
        }
        const uint32_t code = op.y & 0xffu;
        if (code <= 1 || code == 5) {   // OP_LIN: dst = A ; OP_QUAD: dst = A*B + C ; OP_SHRLC: dst = (A >> shift) & mask
            const uint32_t nA = (op.y >> 8) & 31u, nB = (op.y >> 13) & 31u, nC = (op.y >> 18) & 31u;
            const uint2* t = hdr.y > WITNESS_TERM_BUF ? P.terms + op.z : term_buf + (it & 1) * WITNESS_TERM_BUF + (op.z - hdr.x);
            Fr xa, xb, xc;
            eval_lcs(P, w, t, nA, nB, nC, xa, xb, xc);
            if (code == 1) {
                // bits and bytes (most of SHA-256 / the regex automaton): the product fits 64 bits, no reduction
                const bool tiny = ((xa.v[1] | xa.v[2] | xa.v[3] | xa.v[4] | xa.v[5] | xa.v[6] | xa.v[7] |
                                    xb.v[1] | xb.v[2] | xb.v[3] | xb.v[4] | xb.v[5] | xb.v[6] | xb.v[7]) == 0);
                if (tiny) {
                    const unsigned long long pr = (unsigned long long)xa.v[0] * xb.v[0];
                    Fr q = Fr::zero();
                    q.v[0] = (uint32_t)pr; q.v[1] = (uint32_t)(pr >> 32);
                    xa = q + xc;
                } else {
                    xa = (xa * xb) * Fr::r2() + xc;
                }
            }
            if (code == 5) xa = shrand(xa, op.w & 0xffffu, op.w >> 16);
            xa.store(w + 32ull * op.x);
        } else if (code == 2) {   // OP_SHRAND
            shrand(Fr::load(w + 32ull * op.z), op.w & 0xffffu, op.w >> 16).store(w + 32ull * op.x);
        } else if (code == 3) {   // OP_INVZ
            invz(P, Fr::load(w + 32ull * op.z)).store(w + 32ull * op.x);
        } else if (code == 4) {   // OP_FPMUL
            fpmul_hint_dev(P, w, op.z, op.x);
        }
        // cooperative ops of this iteration (native Sha256compression, regex seeds, FpMul hints): the whole CTA works on each in
        // turn, native Poseidon instances on a warp each; they only
        // read signals of earlier levels and define signals nothing else in this iteration touches
        const uint32_t n_coop = hdr.w & 0xffffu;
        for (uint32_t q = 0; q < n_coop; ++q) {
            const uint32_t c0 = P.coop[2 * (hdr.z + q)], c1 = P.coop[2 * (hdr.z + q) + 1];
            if ((c0 >> 30) == 3u) {          // a run of native Poseidon instances (the level's last coop ops): one warp each
                uint32_t e = q + 1;
                while (e < n_coop && (P.coop[2 * (hdr.z + e)] >> 30) == 3u) ++e;
                for (uint32_t p = q + tid / 32u; p < e; p += WITNESS_THREADS / 32) poseidon_coop(P, w, P.coop[2 * (hdr.z + p)] & 0x3fffffffu);
                __syncthreads();
                q = e - 1;
            }
            else if (c0 >> 31) fpmul_coop(P, w, c0 & 0x7fffffffu, c1, fpmul_s);
            else if (c0 & 0x40000000u) regex_coop(P, w, c0 & 0x3fffffffu, sha_q);
            else sha_coop(P, w, c0, sha_q, sha_in);
        }
        cp_async_wait_all();
        __syncthreads();     // level barrier and hand-over of the staged term block
        if (CL > 1 && (hdr.w >> 31))      // last round of a level: the other CTAs' signals become visible here
            asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
        if (P.trace && blockIdx.x == 0 && tid == 0) P.trace[k] = clock64();
        op = op_next; hdr = hdr_next; hdr_next = hdr_next2;
    }
}

static const size_t WITNESS_SMEM = 2 * (size_t)WITNESS_TERM_BUF * sizeof(uint2);   // 128 KB: above the 48 KB default

// The opt-in to > 48 KB of dynamic shared memory is a per-device (per-context) function attribute: the engine calls
// this from select_device() for every device it touches, and checks the result.
cudaError_t configure_witness_kernel() {
    cudaError_t e = cudaFuncSetAttribute(witness_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WITNESS_SMEM);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(witness_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WITNESS_SMEM);
}

void launch_witness(const DevProgram& P, uint8_t* w_all, size_t stride_elems, const uint8_t* inputs, uint32_t batch, cudaStream_t st) {
    static const bool slim = getenv("ZKE_WITNESS_SLIM") && atoi(getenv("ZKE_WITNESS_SLIM")) != 0;
    if (P.cluster > 1) {
        // one thread-block cluster per email (P.cluster CTAs on neighbouring SMs; the program stream was cut for it)
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(batch * P.cluster, 1, 1);
        cfg.blockDim = dim3(WITNESS_THREADS, 1, 1);
        cfg.dynamicSmemBytes = WITNESS_SMEM;
        cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = P.cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        cudaLaunchKernelEx(&cfg, witness_kernel<1>, P, w_all, stride_elems, inputs, batch);
    }
    else if (slim) witness_kernel<2><<<batch, WITNESS_THREADS, WITNESS_SMEM, st>>>(P, w_all, stride_elems, inputs, batch);
    else witness_kernel<1><<<batch, WITNESS_THREADS, WITNESS_SMEM, st>>>(P, w_all, stride_elems, inputs, batch);
    ZKE_COUNT_LAUNCH(1);
}

}  // namespace dev
}  // namespace zke
