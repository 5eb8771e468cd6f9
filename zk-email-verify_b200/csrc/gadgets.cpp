#include "gadgets.hpp"
#include <algorithm>
#include <map>
#include <mutex>
#include <stdexcept>

namespace zke {
namespace gadgets {

static const Fr& fr_one() { static const Fr o = Fr::one(); return o; }
static Fr fr_pow2(uint32_t e) {
    // built completely inside the initialiser: C++11 makes that thread-safe (zke_circuit_build may be called concurrently)
    static const std::vector<Fr> tab = [] {
        std::vector<Fr> t(256);
        t[0] = Fr::one();
        for (int i = 1; i < 256; ++i) t[i] = t[i - 1] + t[i - 1];
        return t;
    }();
    if (e >= 256) throw std::runtime_error("fr_pow2: exponent too large");
    return tab[e];
}
static LC one_lc() { return LC::constant(fr_one()); }
static LC const_u64(uint64_t v) { return LC::constant(Fr::from_u64(v)); }

uint32_t log2_ceil(uint64_t a) {  // utils/functions.circom:7-17
    uint64_t n = a - 1;
    uint32_t r = 0;
    while (n > 0) { r++; n /= 2; }
    return r;
}

// ---------------------------------------------------------------- circomlib bitify
LCVec num2bits(Builder& b, const LC& in_expr, uint32_t n) {
    ScopeGuard g(b, "Num2Bits");
    LC in = b.signal(in_expr);
    Var src = b.source_of(in);
    LCVec out(n);
    LC lc1;
    for (uint32_t i = 0; i < n; ++i) {
        Var bit = b.hint_shrand(src, i, 1);       // out[i] <-- (in >> i) & 1
        out[i] = LC(bit);
        b.enforce_mul(out[i], out[i] - one_lc(), LC());  // out[i] * (out[i] - 1) === 0
        lc1.add_term(bit, fr_pow2(i));
    }
    b.enforce_eq(lc1, in);                         // lc1 === in
    return out;
}

LC bits2num(Builder& b, const LCVec& bits) {
    ScopeGuard g(b, "Bits2Num");
    LC lc1;
    for (size_t i = 0; i < bits.size(); ++i) lc1 += bits[i] * fr_pow2((uint32_t)i);
    return b.signal(lc1);                          // lc1 ==> out
}

LC is_zero(Builder& b, const LC& in_expr) {
    ScopeGuard g(b, "IsZero");
    if (in_expr.is_const()) return in_expr.is_zero() ? one_lc() : LC();   // no hint variable for a compile-time constant
    LC in = b.signal(in_expr);
    Var inv = b.hint_invz(b.source_of(in));        // inv <-- in != 0 ? 1/in : 0
    LC out = b.mul_add(in.neg(), LC(inv), one_lc());   // out <== -in*inv + 1
    b.enforce_mul(in, out, LC());                  // in*out === 0
    return out;
}

LC is_equal(Builder& b, const LC& x, const LC& y) {
    ScopeGuard g(b, "IsEqual");
    return is_zero(b, b.signal(y) - b.signal(x));  // in[1] - in[0] ==> isz.in
}

LC less_than(Builder& b, uint32_t n, const LC& x, const LC& y) {
    ScopeGuard g(b, "LessThan");
    if (n > 252) throw std::runtime_error("LessThan: n > 252");
    LC in0 = b.signal(x), in1 = b.signal(y);
    LCVec bits = num2bits(b, in0 + LC::constant(fr_pow2(n)) - in1, n + 1);
    return b.signal(one_lc() - bits[n]);
}
LC greater_than(Builder& b, uint32_t n, const LC& x, const LC& y) { return less_than(b, n, y, x); }
LC less_eq_than(Builder& b, uint32_t n, const LC& x, const LC& y) { return less_than(b, n, x, b.signal(y) + one_lc()); }

LC gate_and(Builder& b, const LC& x, const LC& y) {
    ScopeGuard g(b, "AND");
    return b.mul(b.signal(x), b.signal(y));
}
LC gate_or(Builder& b, const LC& x, const LC& y) {
    ScopeGuard g(b, "OR");
    LC a = b.signal(x), c = b.signal(y);
    return b.mul_add(a.neg(), c, a + c);           // out <== a + b - a*b
}
LC multi_or(Builder& b, const LCVec& in) {
    ScopeGuard g(b, "MultiOR");
    if (in.size() == 1) return in[0];
    LC sum;
    for (auto& e : in) sum += e;
    return b.signal(one_lc() - is_zero(b, sum));
}

// ---------------------------------------------------------------- circomlib sha256
static const uint32_t SHA_K[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
static const uint32_t SHA_IV[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a,
                                   0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};

static LCVec const_word(uint32_t v) {  // LSB-first bits, as circomlib K(x) / H(x)
    LCVec w(32);
    for (int i = 0; i < 32; ++i) w[i] = ((v >> i) & 1) ? one_lc() : LC();
    return w;
}
LCVec sha256_iv_bits() {
    LCVec out;
    for (int i = 0; i < 8; ++i) { LCVec w = const_word(SHA_IV[i]); out.insert(out.end(), w.begin(), w.end()); }
    return out;
}
static LCVec rotr(const LCVec& in, uint32_t r) { LCVec o(32); for (uint32_t i = 0; i < 32; ++i) o[i] = in[(i + r) % 32]; return o; }
static LCVec shr(const LCVec& in, uint32_t r) { LCVec o(32); for (uint32_t i = 0; i < 32; ++i) o[i] = (i + r >= 32) ? LC() : in[i + r]; return o; }

// Recorder of one Sha256compression instance (circuit.hpp: ShaBlock): whenever a gadget call returns a signal it has just
// created, the signal is noted together with the native quantity and bit whose value it carries.
struct ShaRecorder {
    ShaBlock blk;
    bool ok = true;
    void note(const Builder& b, uint32_t var_mark, const LC& e, uint32_t group, uint32_t index, uint32_t bit) {
        Var v;
        if (b.num_vars() == var_mark) return;                       // the call folded into existing signals / constants
        if (b.num_vars() != var_mark + 1 || !e.is_single_var(&v) || v != var_mark) { ok = false; return; }
        blk.desc.push_back(v);
        blk.desc.push_back(((group * 64 + index) << 8) | bit);
    }
};
static thread_local ShaRecorder* g_sha_rec = nullptr;
#define SHA_NOTE(expr_lc, group, index, bit) do { if (g_sha_rec) g_sha_rec->note(b, mark_, (expr_lc), (group), (index), (bit)); } while (0)

static LCVec xor3(Builder& b, const LCVec& x, const LCVec& y, const LCVec& z, uint32_t q_mid, uint32_t q_out, uint32_t t) {
    // mid[k] <== b[k]*c[k]; out[k] <== a[k] * (1 -2*b[k] -2*c[k] +4*mid[k]) + b[k] + c[k] -2*mid[k];
    const Fr two = Fr::from_u64(2), four = Fr::from_u64(4);
    LCVec o(32);
    for (int k = 0; k < 32; ++k) {
        uint32_t mark_ = b.num_vars();
        LC mid = b.mul(y[k], z[k]);
        SHA_NOTE(mid, q_mid, t, (uint32_t)k);
        mark_ = b.num_vars();
        o[k] = b.mul_add(x[k], one_lc() - y[k] * two - z[k] * two + mid * four, y[k] + z[k] - mid * two);
        SHA_NOTE(o[k], q_out, t, (uint32_t)k);
    }
    return o;
}
static LCVec small_sigma(Builder& b, const LCVec& in, uint32_t ra, uint32_t rb, uint32_t rc, uint32_t q_mid, uint32_t q_out, uint32_t t) {
    return xor3(b, rotr(in, ra), rotr(in, rb), shr(in, rc), q_mid, q_out, t);
}
static LCVec big_sigma(Builder& b, const LCVec& in, uint32_t ra, uint32_t rb, uint32_t rc, uint32_t q_mid, uint32_t q_out, uint32_t t) {
    return xor3(b, rotr(in, ra), rotr(in, rb), rotr(in, rc), q_mid, q_out, t);
}
static LCVec ch_t(Builder& b, const LCVec& x, const LCVec& y, const LCVec& z, uint32_t t) {
    LCVec o(32);
    for (int k = 0; k < 32; ++k) {
        const uint32_t mark_ = b.num_vars();
        o[k] = b.mul_add(x[k], y[k] - z[k], z[k]);   // out <== a*(b-c) + c
        SHA_NOTE(o[k], SHA_Q_CH, t, (uint32_t)k);
    }
    return o;
}
static LCVec maj_t(Builder& b, const LCVec& x, const LCVec& y, const LCVec& z, uint32_t t) {
    const Fr two = Fr::from_u64(2);
    LCVec o(32);
    for (int k = 0; k < 32; ++k) {
        uint32_t mark_ = b.num_vars();
        LC mid = b.mul(y[k], z[k]);
        SHA_NOTE(mid, SHA_Q_MAJMID, t, (uint32_t)k);
        mark_ = b.num_vars();
        o[k] = b.mul_add(x[k], y[k] + z[k] - mid * two, mid);                 // out <== a*(b+c-2*mid) + mid
        SHA_NOTE(o[k], SHA_Q_MAJ, t, (uint32_t)k);
    }
    return o;
}
static uint32_t nbits_of(uint64_t a) { uint64_t n = 1; uint32_t r = 0; while (n - 1 < a) { r++; n *= 2; } return r; }

static LCVec binsum(Builder& b, const std::vector<LCVec>& ins, uint32_t q_sum, uint32_t t) {
    ScopeGuard g(b, "BinSum");
    const uint32_t n = 32, ops = (uint32_t)ins.size();
    const uint32_t nout = nbits_of(((1ull << n) - 1) * ops);
    LC lin;
    for (uint32_t k = 0; k < n; ++k)
        for (uint32_t j = 0; j < ops; ++j) lin += ins[j][k] * fr_pow2(k);
    Var src = b.source_of(lin);
    LCVec out(nout);
    LC lout;
    for (uint32_t k = 0; k < nout; ++k) {
        const uint32_t mark_ = b.num_vars();
        Var bit = b.hint_shrand(src, k, 1);            // out[k] <-- (lin >> k) & 1
        out[k] = LC(bit);
        SHA_NOTE(out[k], q_sum, t, k);
        b.enforce_mul(out[k], out[k] - one_lc(), LC());
        lout.add_term(bit, fr_pow2(k));
    }
    b.enforce_eq(lin, lout);
    return out;
}
static LCVec low32(const LCVec& v) { return LCVec(v.begin(), v.begin() + 32); }

LCVec sha256_compression(Builder& b, const LCVec& hin, const LCVec& inp) {
    ScopeGuard g(b, "Sha256compression");
    if (hin.size() != 256 || inp.size() != 512) throw std::runtime_error("Sha256compression: bad sizes");
    // record the instance for native evaluation (circuit.hpp: ShaBlock) when every input is a signal or a constant bit
    ShaRecorder rec;
    rec.blk.var_begin = b.num_vars();
    rec.blk.temp_begin = b.num_temps();
    rec.blk.inputs.resize(768);
    for (int i = 0; i < 768 && rec.ok; ++i) {
        const LC& e = i < 256 ? hin[i] : inp[i - 256];
        Var v;
        if (e.is_zero()) rec.blk.inputs[i] = SHA_CONST0;
        else if (e.is_const() && e.const_value() == Fr::one()) rec.blk.inputs[i] = SHA_CONST1;
        else if (e.is_single_var(&v)) rec.blk.inputs[i] = v;
        else rec.ok = false;
    }
    ShaRecorder* const outer = g_sha_rec;
    g_sha_rec = rec.ok ? &rec : nullptr;
    struct Restore { ShaRecorder* p; ~Restore() { g_sha_rec = p; } } restore{outer};
    std::vector<LCVec> w(64);
    for (int t = 0; t < 64; ++t) {
        if (t < 16) {
            w[t].resize(32);
            for (int k = 0; k < 32; ++k) w[t][k] = inp[t * 32 + 31 - k];
        } else {
            // SigmaPlus: BinSum(32,4) of sigma1(in2), in7, sigma0(in15), in16
            LCVec s1 = small_sigma(b, w[t - 2], 17, 19, 10, SHA_Q_S1MID, SHA_Q_S1, (uint32_t)t);
            LCVec s0 = small_sigma(b, w[t - 15], 7, 18, 3, SHA_Q_S0MID, SHA_Q_S0, (uint32_t)t);
            w[t] = low32(binsum(b, {s1, w[t - 7], s0, w[t - 16]}, SHA_Q_WSUM, (uint32_t)t));
        }
    }
    LCVec st[8];
    for (int i = 0; i < 8; ++i) st[i] = LCVec(hin.begin() + 32 * i, hin.begin() + 32 * (i + 1));
    LCVec &a = st[0], &bb = st[1], &c = st[2], &d = st[3], &e = st[4], &f = st[5], &gg = st[6], &h = st[7];
    for (int t = 0; t < 64; ++t) {
        // T1 = BinSum(32,5)(h, BigSigma(6,11,25)(e), Ch(e,f,g), k, w)
        LCVec bs1 = big_sigma(b, e, 6, 11, 25, SHA_Q_BS1MID, SHA_Q_BS1, (uint32_t)t);
        LCVec chv = ch_t(b, e, f, gg, (uint32_t)t);
        LCVec t1 = low32(binsum(b, {h, bs1, chv, const_word(SHA_K[t]), w[t]}, SHA_Q_T1SUM, (uint32_t)t));
        // T2 = BinSum(32,2)(BigSigma(2,13,22)(a), Maj(a,b,c))
        LCVec bs0 = big_sigma(b, a, 2, 13, 22, SHA_Q_BS0MID, SHA_Q_BS0, (uint32_t)t);
        LCVec mj = maj_t(b, a, bb, c, (uint32_t)t);
        LCVec t2 = low32(binsum(b, {bs0, mj}, SHA_Q_T2SUM, (uint32_t)t));
        LCVec sume = low32(binsum(b, {d, t1}, SHA_Q_SUME, (uint32_t)t));
        LCVec suma = low32(binsum(b, {t1, t2}, SHA_Q_SUMA, (uint32_t)t));
        h = gg; gg = f; f = e; e = sume; d = c; c = bb; bb = a; a = suma;
    }
    LCVec out(256);
    for (int i = 0; i < 8; ++i) {
        LCVec hi(hin.begin() + 32 * i, hin.begin() + 32 * (i + 1));
        LCVec fs = binsum(b, {hi, st[i]}, SHA_Q_FS, (uint32_t)i);
        for (int k = 0; k < 32; ++k) out[32 * i + 31 - k] = fs[k];
    }
    g_sha_rec = outer;
    rec.blk.var_end = b.num_vars();
    rec.blk.temp_end = b.num_temps();
    // every signal of the instance must have exactly one descriptor - otherwise the instance stays on the generic path
    if (rec.ok && rec.blk.desc.size() == 2 * (size_t)(rec.blk.var_end - rec.blk.var_begin) && rec.blk.var_end > rec.blk.var_begin)
        b.add_sha_block(std::move(rec.blk));
    return out;
}

// ---------------------------------------------------------------- utils/array.circom
LC calculate_total(Builder& b, const LCVec& nums) {
    ScopeGuard g(b, "CalculateTotal");
    LC sum = nums[0];
    for (size_t i = 1; i < nums.size(); ++i) sum = b.signal(sum + nums[i]);   // sums[i] <== sums[i-1] + nums[i]
    return sum;
}

LC item_at_index(Builder& b, const LCVec& in, const LC& index_expr) {
    ScopeGuard g(b, "ItemAtIndex");
    LC index = b.signal(index_expr);
    LCVec vals(in.size()), idxs(in.size());
    for (size_t i = 0; i < in.size(); ++i) {
        LC eq = is_equal(b, const_u64(i), index);
        vals[i] = b.mul(eq, in[i]);               // calcTotalValue.nums[i] <== eqs[i].out * in[i]
        idxs[i] = eq;
    }
    LC total_val = calculate_total(b, vals);
    LC total_idx = calculate_total(b, idxs);
    b.enforce_eq(total_idx, one_lc());            // calcTotalIndex.sum === 1
    return total_val;
}

LCVec var_shift_left(Builder& b, const LCVec& in, const LC& shift, uint32_t max_out_len) {
    ScopeGuard g(b, "VarShiftLeft");
    const uint32_t len = (uint32_t)in.size();
    if (max_out_len > len) throw std::runtime_error("VarShiftLeft: maxOutArrayLen > maxArrayLen");
    const uint32_t bit_length = log2_ceil(len);
    LCVec bits = num2bits(b, shift, bit_length);
    LCVec prev = in;
    for (uint32_t j = 0; j < bit_length; ++j) {
        LCVec cur(len);
        for (uint32_t i = 0; i < len; ++i) {
            uint32_t offset = (uint32_t)(((uint64_t)i + (1ull << j)) % len);
            cur[i] = b.mul_add(bits[j], prev[offset] - prev[i], prev[i]);
        }
        prev.swap(cur);
    }
    return LCVec(prev.begin(), prev.begin() + max_out_len);
}

void assert_zero_padding(Builder& b, const LCVec& in, const LC& start_index) {
    ScopeGuard g(b, "AssertZeroPadding");
    const uint32_t bit_length = log2_ceil(in.size());
    for (size_t i = 0; i < in.size(); ++i) {
        LC lt = less_than(b, bit_length, start_index - one_lc(), const_u64(i));
        b.enforce_mul(lt, in[i], LC());           // lessThans[i].out * in[i] === 0
    }
}

// ---------------------------------------------------------------- utils/bytes.circom
LCVec pack_bits(Builder& b, const LCVec& in, uint32_t bpe) {
    ScopeGuard g(b, "PackBits");
    const uint32_t num_bits = (uint32_t)in.size();
    const uint32_t n_el = (num_bits + bpe - 1) / bpe;
    LCVec out(n_el);
    for (uint32_t i = 0; i < n_el; ++i) {
        LC sum;
        for (uint32_t j = 0; j < bpe; ++j) {
            uint32_t idx = i * bpe + j;
            if (idx < num_bits) sum += in[idx] * fr_pow2(bpe - 1 - j);
        }
        out[i] = b.signal(sum);
    }
    return out;
}

LCVec pack_bytes(Builder& b, const LCVec& in) {
    ScopeGuard g(b, "PackBytes");
    const uint32_t pack_size = 31;                                      // MAX_BYTES_IN_FIELD (utils/constants.circom:13-15)
    const uint32_t max_bytes = (uint32_t)in.size();
    const uint32_t max_ints = (max_bytes + pack_size - 1) / pack_size;  // computeIntChunkLength (utils/bytes.circom:10-20)
    LCVec out(max_ints);
    for (uint32_t i = 0; i < max_ints; ++i) {
        LC sum;                                                         // intSums[i][j] chain (:37-54)
        for (uint32_t j = 0; j < pack_size; ++j) {
            const uint32_t idx = pack_size * i + j;
            if (idx >= max_bytes) break;                                // out of bounds: the previous value is carried
            sum = j == 0 ? b.signal(in[idx]) : b.signal(sum + in[idx] * fr_pow2(8 * j));
        }
        out[i] = sum;
    }
    return out;
}

LCVec pack_regex_reveal(Builder& b, const LCVec& in, const LC& start_index, uint32_t max_reveal_len) {
    ScopeGuard g(b, "PackRegexReveal");
    return pack_bytes(b, select_regex_reveal(b, in, start_index, max_reveal_len));
}

LCVec split_bytes_to_words(Builder& b, const LCVec& in, uint32_t n, uint32_t k) {
    ScopeGuard g(b, "SplitBytesToWords");
    const uint32_t l = (uint32_t)in.size();
    std::vector<LCVec> bits(l);
    for (uint32_t i = 0; i < l; ++i) bits[i] = num2bits(b, in[i], 8);            // :129-133
    LCVec out(k);
    for (uint32_t i = 0; i < k; ++i) {                                           // :134-148: word i = bits [i n, (i+1) n) of the
        LCVec word(n);                                                           // big-endian byte string read as an integer
        for (uint32_t j = 0; j < n; ++j) {
            const uint64_t pos = (uint64_t)i * n + j;
            word[j] = pos >= 8ull * l ? LC() : bits[l - (uint32_t)(pos / 8) - 1][pos % 8];
        }
        out[i] = b.signal(bits2num(b, word));
    }
    return out;
}

// ---------------------------------------------------------------- utils/array.circom (add-on templates)
LCVec select_sub_array(Builder& b, const LCVec& in, const LC& start_index, const LC& length, uint32_t max_sub_len) {
    ScopeGuard g(b, "SelectSubArray");
    if (max_sub_len >= in.size()) throw std::runtime_error("SelectSubArray: maxSubArrayLen >= maxArrayLen");   // :79
    LCVec shifted = var_shift_left(b, in, start_index, max_sub_len);
    const uint32_t bits = log2_ceil(max_sub_len);
    LCVec out(max_sub_len);
    for (uint32_t i = 0; i < max_sub_len; ++i)                                    // :90-97: zero from `length` on
        out[i] = b.mul(greater_than(b, bits, length, const_u64(i)), shifted[i]);
    return out;
}

LC check_substring_match(Builder& b, const LCVec& in, const LCVec& substring) {
    ScopeGuard g(b, "CheckSubstringMatch");
    const size_t n = substring.size();
    b.enforce_eq(is_zero(b, substring[0]), LC());                                 // :199-201 firstElementNonZero === 0
    LC acc = b.signal(one_lc());                                                  // matchAccumulator[0] <== 1
    for (size_t i = 0; i < n; ++i) {
        LC diff = b.mul(in[i] - substring[i], substring[i]);                      // :210 (zero where the pattern is zero-padded)
        acc = b.mul(acc, is_zero(b, diff));                                       // :211-212
    }
    return acc;
}

LC count_substring_occurrences(Builder& b, const LCVec& in, const LCVec& substring) {
    ScopeGuard g(b, "CountSubstringOccurrences");
    const size_t max_len = in.size(), sub_len = substring.size();
    if (max_len < sub_len) throw std::runtime_error("CountSubstringOccurrences: maxLen < maxSubstringLen");   // :227
    LCVec matches(max_len);
    for (size_t i = 0; i < max_len; ++i) {                                        // :234-246
        LCVec window(sub_len);
        for (size_t j = 0; j < sub_len; ++j) window[j] = i + j < max_len ? in[i + j] : LC();
        matches[i] = check_substring_match(b, window, substring);
    }
    return calculate_total(b, matches);                                           // :248-253
}

// ---------------------------------------------------------------- helpers/reveal-substring.circom
LCVec reveal_substring(Builder& b, const LCVec& in, const LC& start_index, const LC& length, uint32_t max_substring_len,
                       bool check_uniqueness) {
    ScopeGuard g(b, "RevealSubstring");
    const uint32_t max_length = (uint32_t)in.size();
    if (max_substring_len >= max_length) throw std::runtime_error("RevealSubstring: maxSubstringLength >= maxLength");   // :14
    b.enforce_eq(less_than(b, log2_ceil(max_length), start_index, const_u64(max_length)), one_lc());                    // :23-24
    b.enforce_eq(less_than(b, log2_ceil(max_substring_len + 1), length, const_u64(max_substring_len + 1)), one_lc());   // :27-28
    LC sum = b.signal(start_index + length);                                                                            // :31
    b.enforce_eq(less_than(b, log2_ceil(max_length + 1), sum, const_u64(max_length + 1)), one_lc());                     // :32-33
    LCVec sub = select_sub_array(b, in, start_index, length, max_substring_len);                                        // :36-39
    if (check_uniqueness) b.enforce_eq(count_substring_occurrences(b, in, sub), one_lc());                              // :41-47
    return sub;
}

// ---------------------------------------------------------------- utils/email.circom
LC clean_email_address(Builder& b, const LCVec& encoded, const LCVec& decoded) {
    ScopeGuard g(b, "CleanEmailAddress");
    const size_t n = encoded.size();
    LCVec all(2 * n);
    for (size_t i = 0; i < n; ++i) { all[i] = encoded[i]; all[n + i] = decoded[i]; }
    LC r = b.signal(poseidon_modular(b, all));                                    // :45-52
    LCVec is_plus(n), is_at(n), neither(n), local(n), should_remove(n);
    for (size_t i = 0; i < n; ++i) {                                              // :54-66
        is_plus[i] = is_equal(b, encoded[i], const_u64(43));
        is_at[i] = is_equal(b, encoded[i], const_u64(64));
        neither[i] = b.mul(one_lc() - is_plus[i], one_lc() - is_at[i]);
        local[i] = i == 0 ? b.signal(neither[0]) : b.mul(local[i - 1], neither[i]);
    }
    LCVec local_period(n);
    for (size_t i = 0; i < n; ++i) local_period[i] = b.mul(local[i], is_equal(b, encoded[i], const_u64(46)));   // :69-72
    LC found_plus = b.signal(is_plus[0]);                                         // :75-78 (running count, not used further)
    for (size_t i = 1; i < n; ++i) found_plus = b.signal(found_plus + is_plus[i]);
    LCVec after_plus(n), after_at(n);
    after_plus[0] = b.signal(one_lc() - is_plus[0]);                              // :81-84
    for (size_t i = 1; i < n; ++i) after_plus[i] = b.mul(after_plus[i - 1], one_lc() - is_plus[i]);
    LC has_alias = b.signal(one_lc() - after_plus[n - 1]);                        // :85
    after_at[0] = b.signal(one_lc() - is_at[0]);                                  // :87-90
    for (size_t i = 1; i < n; ++i) after_at[i] = b.mul(after_at[i - 1], one_lc() - is_at[i]);
    for (size_t i = 0; i < n; ++i) {                                              // :92-100
        LC in_alias = b.mul(has_alias, b.signal(after_at[i] - after_plus[i]));
        should_remove[i] = b.signal(local_period[i] + in_alias);
    }
    LCVec processed(n), r_enc(n), r_dec(n);
    for (size_t i = 0; i < n; ++i) processed[i] = b.mul(one_lc() - should_remove[i], encoded[i]);   // :103-105
    for (size_t i = 0; i < n; ++i) {                                              // :108-120 Mux1: out = (c1 - c0) s + c0
        LC c0 = i == 0 ? r : b.mul(r_enc[i - 1], r);
        LC c1 = i == 0 ? one_lc() : r_enc[i - 1];
        r_enc[i] = b.mul_add(c1 - c0, should_remove[i], c0);
    }
    r_dec[0] = r;                                                                 // :123-126
    for (size_t i = 1; i < n; ++i) r_dec[i] = b.mul(r_dec[i - 1], r);
    LC sum_enc, sum_dec;
    for (size_t i = 0; i < n; ++i) sum_enc = i == 0 ? b.mul(r_enc[0], processed[0]) : b.mul_add(r_enc[i], processed[i], sum_enc);   // :129-132
    for (size_t i = 0; i < n; ++i) sum_dec = i == 0 ? b.mul(r_dec[0], decoded[0]) : b.mul_add(r_dec[i], decoded[i], sum_dec);      // :135-138
    return is_equal(b, sum_enc, sum_dec);                                         // :141
}

// ---------------------------------------------------------------- helpers/email-nullifier.circom
LC email_nullifier(Builder& b, uint32_t bits_per_chunk, const LCVec& signature) {
    ScopeGuard g(b, "EmailNullifier");
    LC sig_hash = b.signal(poseidon_large(b, bits_per_chunk, signature));         // :20
    return poseidon(b, LCVec{sig_hash});                                          // :22
}

LCVec byte_mask(Builder& b, const LCVec& in, const LCVec& mask) {
    ScopeGuard g(b, "ByteMask");
    LCVec out(in.size());
    for (size_t i = 0; i < in.size(); ++i) {
        b.enforce_mul(mask[i], mask[i] - one_lc(), LC());   // AssertBit
        out[i] = b.mul(in[i], mask[i]);
    }
    return out;
}

// ---------------------------------------------------------------- utils/regex.circom
LCVec select_regex_reveal(Builder& b, const LCVec& in, const LC& start_index, uint32_t max_reveal_len) {
    ScopeGuard g(b, "SelectRegexReveal");
    const uint32_t len = (uint32_t)in.size();
    const uint32_t bit_length = log2_ceil(len + max_reveal_len - 1);
    for (uint32_t i = 0; i < len; ++i) {
        LC is_start = is_equal(b, const_u64(i), start_index);
        LC is_z = is_zero(b, in[i]);
        LC is_prev_z = (i == 0) ? one_lc() : is_zero(b, in[i - 1]);
        LC above = greater_than(b, bit_length, const_u64(i), start_index + const_u64(max_reveal_len - 1));
        b.enforce_mul(is_start, is_z, LC());                      // start byte is non-zero
        b.enforce_mul(is_start, one_lc() - is_prev_z, LC());      // byte before start is zero
        b.enforce_mul(above, one_lc() - is_z, LC());              // everything past the window is zero
    }
    return var_shift_left(b, in, start_index, max_reveal_len);
}

// ---------------------------------------------------------------- lib/sha.circom
LCVec sha256_general(Builder& b, const LCVec& padded_in, const LC& padded_in_length, const LCVec* pre_hash) {
    ScopeGuard g(b, pre_hash ? "Sha256Partial" : "Sha256General");
    const uint32_t max_bit_length = (uint32_t)padded_in.size();
    if (max_bit_length % 512 != 0) throw std::runtime_error("Sha256General: maxBitLength % 512 != 0");
    const uint32_t max_blocks = max_bit_length / 512;
    const uint32_t max_bits_padded_bits = log2_ceil(max_bit_length);

    LC len = b.signal(padded_in_length);
    Var in_block_index = b.hint_shrand(b.source_of(len), 9, 0);           // inBlockIndex <-- (paddedInLength >> 9)
    b.enforce_eq(len, LC(in_block_index) * Fr::from_u64(512));             // paddedInLength === inBlockIndex * 512

    LC ok = less_eq_than(b, max_bits_padded_bits, len, const_u64(max_bit_length));
    b.enforce_eq(ok, one_lc());                                            // bitLengthVerifier.out === 1

    LCVec hin(256);
    if (pre_hash) {
        if (pre_hash->size() != 256) throw std::runtime_error("Sha256Partial: preHash must have 256 bits");
        for (int w = 0; w < 8; ++w) for (int k = 0; k < 32; ++k) hin[32 * w + k] = (*pre_hash)[32 * w + 31 - k];
    } else {
        hin = sha256_iv_bits();
    }
    std::vector<LCVec> outs(max_blocks);
    for (uint32_t i = 0; i < max_blocks; ++i) {
        LCVec inp(padded_in.begin() + 512 * i, padded_in.begin() + 512 * (i + 1));
        outs[i] = sha256_compression(b, hin, inp);
        for (int w = 0; w < 8; ++w) for (int k = 0; k < 32; ++k) hin[32 * w + k] = outs[i][32 * w + 31 - k];
    }
    LCVec out(256);
    for (int k = 0; k < 256; ++k) {
        LCVec col(max_blocks);
        for (uint32_t j = 0; j < max_blocks; ++j) col[j] = outs[j][k];
        out[k] = item_at_index(b, col, LC(in_block_index) - one_lc());
    }
    return out;
}

static LCVec bytes_to_bits_msb(Builder& b, const LCVec& bytes) {
    LCVec bits(bytes.size() * 8);
    for (size_t i = 0; i < bytes.size(); ++i) {
        LCVec nb = num2bits(b, bytes[i], 8);
        for (int j = 0; j < 8; ++j) bits[i * 8 + j] = nb[7 - j];
    }
    return bits;
}

LCVec sha256_bytes(Builder& b, const LCVec& padded_in, const LC& padded_in_length) {
    ScopeGuard g(b, "Sha256Bytes");
    LCVec bits = bytes_to_bits_msb(b, padded_in);
    return sha256_general(b, bits, padded_in_length * Fr::from_u64(8), nullptr);
}

LCVec sha256_bytes_partial(Builder& b, const LCVec& padded_in, const LC& padded_in_length, const LCVec& pre_hash) {
    ScopeGuard g(b, "Sha256BytesPartial");
    if (padded_in.size() % 32 != 0 || pre_hash.size() != 32) throw std::runtime_error("Sha256BytesPartial: bad sizes");
    LCVec bits = bytes_to_bits_msb(b, padded_in);
    LCVec state_bits = bytes_to_bits_msb(b, pre_hash);
    return sha256_general(b, bits, padded_in_length * Fr::from_u64(8), &state_bits);
}

// ---------------------------------------------------------------- lib/bigint.circom
LC big_less_than(Builder& b, uint32_t n, const LCVec& x, const LCVec& y) {
    ScopeGuard g(b, "BigLessThan");
    const int k = (int)x.size();
    LCVec lt(k), eq(k);
    for (int i = 0; i < k; ++i) {
        lt[i] = less_than(b, n, x[i], y[i]);
        eq[i] = is_equal(b, x[i], y[i]);
    }
    if (k == 1) return lt[0];
    LC ors, eq_ands;
    for (int i = k - 2; i >= 0; --i) {
        LC ands_i;
        if (i == k - 2) {
            ands_i = gate_and(b, eq[k - 1], lt[k - 2]);
            eq_ands = gate_and(b, eq[k - 1], eq[k - 2]);
            ors = gate_or(b, lt[k - 1], ands_i);
        } else {
            ands_i = gate_and(b, eq_ands, lt[i]);
            LC new_eq_ands = gate_and(b, eq_ands, eq[i]);
            ors = gate_or(b, ors, ands_i);
            eq_ands = new_eq_ands;
        }
    }
    return ors;
}

void check_carry_to_zero(Builder& b, uint32_t n, uint32_t m, const LCVec& in_expr) {
    ScopeGuard g(b, "CheckCarryToZero");
    const uint32_t k = (uint32_t)in_expr.size();
    const uint32_t EPSILON = 3;
    if (k < 2 || m + EPSILON > 253) throw std::runtime_error("CheckCarryToZero: bad parameters");
    LCVec in(k);
    for (uint32_t i = 0; i < k; ++i) in[i] = b.signal(in_expr[i]);   // tCheck.in[i] <== t[i]
    const Fr two_n = fr_pow2(n);
    const Fr inv_two_n = two_n.inv();
    LCVec carry(k);
    for (uint32_t i = 0; i + 1 < k; ++i) {
        LC num = (i == 0) ? in[i] : in[i] + carry[i - 1];
        carry[i] = LC(b.hint_lin(num * inv_two_n));                  // carry[i] <-- (in[i] + carry[i-1]) / (1<<n)
        b.enforce_eq(num, carry[i] * two_n);                         // in[i] + carry[i-1] === carry[i] * (1<<n)
        num2bits(b, carry[i] + LC::constant(fr_pow2(m + EPSILON - n - 1)), m + EPSILON - n);
    }
    b.enforce_eq(in[k - 1] + carry[k - 2], LC());                    // in[k-1] + carry[k-2] === 0
}

// ---------------------------------------------------------------- lib/fp.circom + bigint-func.circom
static uint32_t log_ceil(uint32_t n) {  // lib/bigint-func.circom:14-23
    uint32_t t = n;
    for (uint32_t i = 0; i < 254; ++i) { if (t == 0) return i; t /= 2; }
    return 254;
}
static LC poly_eval(const LCVec& a, uint32_t x) {  // lib/bigint-func.circom:56-62
    LC v;
    Fr xp = Fr::one();
    const Fr fx = Fr::from_u64(x);
    for (size_t i = 0; i < a.size(); ++i) { v += a[i] * xp; xp = xp * fx; }
    return v;
}
// poly_interp (lib/bigint-func.circom:65-103) as a matrix: coefficient j of the polynomial through
// (i, v[i]), i = 0..len-1, is sum_i M[j][i] * v[i].
static std::vector<std::vector<Fr>> poly_interp_matrix(uint32_t len) {
    std::vector<Fr> full(len + 1, Fr::zero());
    full[0] = Fr::one();
    for (uint32_t i = 0; i < len; ++i) {
        full[i + 1] = Fr::zero();
        for (int j = (int)i; j >= 0; --j) {
            full[j + 1] += full[j];
            full[j] *= Fr::from_i64(-(int64_t)i);
        }
    }
    std::vector<std::vector<Fr>> M(len, std::vector<Fr>(len, Fr::zero()));
    for (uint32_t i = 0; i < len; ++i) {
        Fr cur = Fr::one();
        for (uint32_t j = 0; j < len; ++j) if (i != j) cur *= Fr::from_i64((int64_t)i - (int64_t)j);
        Fr cur_v = cur.inv();
        Fr cur_rem = full[len];
        for (int j = (int)len - 1; j >= 0; --j) {
            M[j][i] = cur_v * cur_rem;
            cur_rem = full[j] + Fr::from_u64(i) * cur_rem;
        }
        if (!cur_rem.is_zero()) throw std::runtime_error("poly_interp: non-zero remainder");
    }
    return M;
}
static Var as_var(Builder& b, const LC& e) {
    Var v;
    LC s = b.signal(e);
    if (s.is_single_var(&v)) return v;
    v = b.hint_lin(s);
    b.enforce_eq(LC(v), s);
    return v;
}

LCVec fp_mul(Builder& b, uint32_t n, uint32_t k, const LCVec& x, const LCVec& y, const LCVec& p) {
    ScopeGuard g(b, "FpMul");
    if (n + n + log_ceil(k) + 2 > 252) throw std::runtime_error("FpMul: n too large");
    if (x.size() != k || y.size() != k || p.size() != k) throw std::runtime_error("FpMul: bad operand sizes");
    const uint32_t npts = 2 * k - 1;
    std::vector<Var> av(k), bv(k), pv(k);
    LCVec a(k), bb(k), pp(k);
    for (uint32_t i = 0; i < k; ++i) {
        av[i] = as_var(b, x[i]); bv[i] = as_var(b, y[i]); pv[i] = as_var(b, p[i]);
        a[i] = LC(av[i]); bb[i] = LC(bv[i]); pp[i] = LC(pv[i]);
    }
    LCVec v_ab(npts);
    for (uint32_t xx = 0; xx < npts; ++xx) v_ab[xx] = b.mul(poly_eval(a, xx), poly_eval(bb, xx));   // v_ab[x] <== v_a * v_b

    // q, r <-- long_div(a*b, p)   (lib/fp.circom:32-50; integer divmod of the 2k-limb product, SURVEY A.4)
    Var base = b.hint_fpmul(n, k, av, bv, pv);
    LCVec q(k), r(k);
    for (uint32_t i = 0; i < k; ++i) { q[i] = LC(base + i); r[i] = LC(base + k + i); }
    for (uint32_t i = 0; i < k; ++i) {
        num2bits(b, q[i], n);
        num2bits(b, r[i], n);
    }
    LC lt = big_less_than(b, n, r, pp);
    b.enforce_eq(lt, one_lc());                                      // r_p_lt_check.out === 1

    LCVec v_t(npts);
    for (uint32_t xx = 0; xx < npts; ++xx) {
        LC v_pq_r = b.mul_add(poly_eval(pp, xx), poly_eval(q, xx), poly_eval(r, xx));   // v_pq_r[x] <== v_p*v_q + v_r
        v_t[xx] = b.signal(v_ab[xx] - v_pq_r);                                          // v_t[x] <== v_ab[x] - v_pq_r[x]
    }
    static std::map<uint32_t, std::vector<std::vector<Fr>>> interp_cache;
    static std::mutex interp_mutex;          // zke_circuit_build is callable from several threads (ctypes drops the GIL)
    const std::vector<std::vector<Fr>>* Mp;
    {
        std::lock_guard<std::mutex> lock(interp_mutex);
        auto it = interp_cache.find(npts);
        if (it == interp_cache.end()) it = interp_cache.emplace(npts, poly_interp_matrix(npts)).first;
        Mp = &it->second;                    // std::map nodes are stable: later insertions do not move this entry
    }
    const auto& M = *Mp;
    LCVec t(npts);
    for (uint32_t j = 0; j < npts; ++j) {
        LC e;
        for (uint32_t i = 0; i < npts; ++i) e += v_t[i] * M[j][i];
        t[j] = e;
    }
    check_carry_to_zero(b, n, n + n + log_ceil(k) + 2, t);
    return r;
}

LCVec fp_pow65537_mod(Builder& b, uint32_t n, uint32_t k, const LCVec& base, const LCVec& modulus) {
    ScopeGuard g(b, "FpPow65537Mod");
    LCVec cur = fp_mul(b, n, k, base, base, modulus);                // doublers[0]
    for (int i = 1; i < 16; ++i) cur = fp_mul(b, n, k, cur, cur, modulus);
    return fp_mul(b, n, k, base, cur, modulus);                      // adder
}

// ---------------------------------------------------------------- lib/rsa.circom
LCVec rsa_pad(Builder& b, uint32_t n, uint32_t k, const LCVec& modulus, const LCVec& message) {
    ScopeGuard g(b, "RSAPad");
    const uint32_t base_len = 408, msg_len = 256, nk = n * k;
    if (base_len + 8 + 65 > nk) throw std::runtime_error("RSAPad: modulus too small");
    LCVec modulus_bits(nk), message_bits(nk), padded(nk);
    for (uint32_t i = 0; i < k; ++i) {
        LCVec mb = num2bits(b, message[i], n);
        LCVec nb = num2bits(b, modulus[i], n);
        for (uint32_t j = 0; j < n; ++j) { message_bits[i * n + j] = mb[j]; modulus_bits[i * n + j] = nb[j]; }
    }
    for (uint32_t i = msg_len; i < nk; ++i) b.enforce_eq(message_bits[i], LC());
    for (uint32_t i = 0; i < msg_len; ++i) padded[i] = message_bits[i];
    for (uint32_t i = base_len; i < base_len + 8; ++i) padded[i] = LC();
    {
        // 0x3031300d060960864801650304020105000420 (152 bits), LSB first from bit msgLen
        static const uint8_t DI[19] = {0x30, 0x31, 0x30, 0x0d, 0x06, 0x09, 0x60, 0x86, 0x48, 0x01,
                                       0x65, 0x03, 0x04, 0x02, 0x01, 0x05, 0x00, 0x04, 0x20};
        for (uint32_t i = msg_len; i < base_len; ++i) {
            uint32_t bit = i - msg_len;                  // bit index from the LSB of the big-endian constant
            uint8_t byte = DI[18 - bit / 8];
            padded[i] = ((byte >> (bit % 8)) & 1) ? one_lc() : LC();
        }
    }
    LC modulus_prefix;
    for (int i = (int)nk - 1; i >= (int)(base_len + 8); --i) {
        if ((uint32_t)i + 8 < nk) {
            modulus_prefix += modulus_bits[i + 8];
            if (i % 8 == 0) {
                LC z = is_zero(b, modulus_prefix);
                padded[i] = b.signal(one_lc() - z);
            } else {
                padded[i] = padded[i + 1];
            }
        } else {
            padded[i] = LC();
        }
    }
    for (uint32_t i = base_len + 8; i < base_len + 8 + 65; ++i) b.enforce_eq(padded[i], one_lc());
    LCVec out(k);
    for (uint32_t i = 0; i < k; ++i) out[i] = bits2num(b, LCVec(padded.begin() + i * n, padded.begin() + (i + 1) * n));
    return out;
}

void rsa_verifier65537(Builder& b, uint32_t n, uint32_t k, const LCVec& message, const LCVec& signature,
                       const LCVec& modulus) {
    ScopeGuard g(b, "RSAVerifier65537");
    LCVec padded = rsa_pad(b, n, k, modulus, message);
    for (uint32_t i = 0; i < k; ++i) num2bits(b, signature[i], n);   // signatureRangeCheck
    LC lt = big_less_than(b, n, signature, modulus);
    b.enforce_eq(lt, one_lc());
    LCVec pw = fp_pow65537_mod(b, n, k, signature, modulus);
    for (uint32_t i = 0; i < k; ++i) b.enforce_eq(pw[i], padded[i]);
}

// ---------------------------------------------------------------- lib/base64.circom
LC base64_lookup(Builder& b, const LC& in_expr) {
    ScopeGuard g(b, "Base64Lookup");
    LC in = b.signal(in_expr);
    auto range = [&](uint32_t lo, uint32_t hi) {
        LC le = less_than(b, 8, in, const_u64(hi + 1));
        LC ge = greater_than(b, 8, in, const_u64(lo - 1));
        return b.mul(ge, le);
    };
    LC range_AZ = range(65, 90);
    LC sum_AZ = b.mul(range_AZ, in - const_u64(65));
    LC range_az = range(97, 122);
    LC sum_az = b.mul_add(range_az, in - const_u64(71), sum_AZ);
    LC range_09 = range(48, 57);
    LC sum_09 = b.mul_add(range_09, in + const_u64(4), sum_az);
    LC eq_plus = is_zero(b, in - const_u64(43));
    LC sum_plus = b.mul_add(eq_plus, in + const_u64(19), sum_09);
    LC eq_slash = is_zero(b, in - const_u64(47));
    LC sum_slash = b.mul_add(eq_slash, in + const_u64(16), sum_plus);
    LC eq_eqsign = is_zero(b, in - const_u64(61));
    b.enforce_eq(one_lc(), range_AZ + range_az + range_09 + eq_plus + eq_slash + eq_eqsign);
    return sum_slash;
}

LCVec base64_decode(Builder& b, uint32_t byte_length, const LCVec& in) {
    ScopeGuard g(b, "Base64Decode");
    const uint32_t char_length = 4 * ((byte_length + 2) / 3);
    if (in.size() != char_length) throw std::runtime_error("Base64Decode: bad input length");
    LCVec out(byte_length);
    uint32_t idx = 0;
    for (uint32_t i = 0; i < char_length; i += 4) {
        LCVec bits_in[4];
        for (int j = 0; j < 4; ++j) bits_in[j] = num2bits(b, base64_lookup(b, in[i + j]), 6);
        LCVec o0(8), o1(8), o2(8);
        for (int j = 0; j < 6; ++j) o0[j + 2] = bits_in[0][j];
        o0[0] = bits_in[1][4]; o0[1] = bits_in[1][5];
        for (int j = 0; j < 4; ++j) o1[j + 4] = bits_in[1][j];
        for (int j = 0; j < 4; ++j) o1[j] = bits_in[2][j + 2];
        o2[6] = bits_in[2][0]; o2[7] = bits_in[2][1];
        for (int j = 0; j < 6; ++j) o2[j] = bits_in[3][j];
        LC bytes[3] = {bits2num(b, o0), bits2num(b, o1), bits2num(b, o2)};
        for (int j = 0; j < 3; ++j) if (idx + j < byte_length) out[idx + j] = bytes[j];
        idx += 3;
    }
    return out;
}

// ---------------------------------------------------------------- utils/hash.circom
LC poseidon_large(Builder& b, uint32_t bits_per_chunk, const LCVec& in) {
    ScopeGuard g(b, "PoseidonLarge");
    const uint32_t chunk_size = (uint32_t)in.size();
    if (!(chunk_size > 16 && chunk_size <= 32 && bits_per_chunk * 2 < 251)) throw std::runtime_error("PoseidonLarge: bad parameters");
    uint32_t half = chunk_size >> 1;
    if (chunk_size % 2 == 1) half += 1;
    LCVec pin(half);
    for (uint32_t i = 0; i < half; ++i) {
        if (i == half - 1 && chunk_size % 2 == 1) pin[i] = in[2 * i];
        else pin[i] = b.signal(in[2 * i] + in[2 * i + 1] * fr_pow2(bits_per_chunk));
    }
    return poseidon(b, pin);
}

LC poseidon_modular(Builder& b, const LCVec& in, bool record) {
    ScopeGuard g(b, "PoseidonModular");
    const size_t n = in.size();
    if (n == 0) throw std::runtime_error("PoseidonModular: no inputs");
    LC out;
    for (size_t start = 0, i = 0; start < n; start += 16, ++i) {
        const size_t end = std::min(n, start + 16);
        LC chunk_hash = poseidon(b, LCVec(in.begin() + start, in.begin() + end), record);   // Slice + Poseidon(16 | last_chunk_size)
        out = (i == 0) ? chunk_hash : poseidon(b, {out, chunk_hash}, record);                // _out = Poseidon(2)([_out, chunk_hash])
    }
    return out;
}

// ---------------------------------------------------------------- Merkle registry of keys
LC binary_merkle_root(Builder& b, const LC& leaf, const LC& index, const LCVec& siblings) {
    ScopeGuard g(b, "BinaryMerkleRoot");
    const uint32_t depth = (uint32_t)siblings.size();
    if (depth < 1 || depth > 32) throw std::runtime_error("BinaryMerkleRoot: depth must be 1..32");
    LCVec bits = num2bits(b, index, depth);
    const bool record = b.materialize_linear;           // a record needs its inputs as signals
    LC cur = leaf;
    for (uint32_t l = 0; l < depth; ++l) {
        LC d = b.mul(bits[l], siblings[l] - cur);       // bit = 1: swap, the node is a right child
        LC left = b.signal(cur + d), right = b.signal(siblings[l] - d);
        cur = poseidon(b, {left, right}, record);
    }
    return cur;
}

LC domain_key_leaf(Builder& b, const LCVec& words, const LC& key_hash) {
    ScopeGuard g(b, "DomainKeyLeaf");
    if (words.empty() || words.size() > 9) throw std::runtime_error("DomainKeyLeaf: 1..9 packed words");
    const bool record = b.materialize_linear;           // a record needs its inputs as signals
    // a record takes variables only: one signal constrained to zero fills every padding word (a record may repeat an
    // input), so the hash is PoseidonModular(PackBytes(D, 255)) whatever the part's maxLength
    LCVec in(9);
    const Var zero = words.size() < 9 ? as_var(b, LC()) : 0;
    for (size_t i = 0; i < 9; ++i) in[i] = i < words.size() ? LC(as_var(b, words[i])) : LC(zero);
    LC domain_hash = poseidon(b, in, record);
    return poseidon(b, {LC(as_var(b, domain_hash)), LC(as_var(b, key_hash))}, record);
}

// ---------------------------------------------------------------- helpers/remove-soft-line-breaks.circom
LC remove_soft_line_breaks(Builder& b, const LCVec& encoded, const LCVec& decoded) {
    ScopeGuard g(b, "RemoveSoftLineBreaks");
    const size_t L = encoded.size();
    if (decoded.size() != L || L < 3) throw std::runtime_error("RemoveSoftLineBreaks: bad lengths");
    LCVec hin(encoded);
    hin.insert(hin.end(), decoded.begin(), decoded.end());
    LC r = poseidon_modular(b, hin);                                     // r <== rHasher.out
    LCVec is_eq(L), is_cr(L), is_lf(L), soft(L), should_zero(L), processed(L);
    for (size_t i = 0; i < L; ++i) is_eq[i] = is_equal(b, encoded[i], const_u64(61));
    for (size_t i = 0; i + 1 < L; ++i) is_cr[i] = is_equal(b, encoded[i + 1], const_u64(13));
    for (size_t i = 0; i + 2 < L; ++i) is_lf[i] = is_equal(b, encoded[i + 2], const_u64(10));
    for (size_t i = 0; i + 2 < L; ++i) {
        LC t = b.mul(is_eq[i], is_cr[i]);                                // tempSoftBreak
        soft[i] = b.mul(t, is_lf[i]);                                    // isSoftBreak
    }
    for (size_t i = 0; i < L; ++i) {
        LC e;
        if (i == 0) e = soft[0];
        else if (i == 1) e = soft[1] + soft[0];
        else if (i == L - 1) e = soft[i - 1] + soft[i - 2];
        else e = soft[i] + soft[i - 1] + soft[i - 2];
        should_zero[i] = b.signal(e);
        processed[i] = b.mul(one_lc() - should_zero[i], encoded[i]);     // (1 - shouldZero) * encoded
    }
    // powers of r: Mux1 out = (c1 - c0) * s + c0
    LCVec r_enc(L), r_dec(L);
    r_enc[0] = b.mul_add(one_lc() - r, should_zero[0], r);
    for (size_t i = 1; i < L; ++i) {
        LC c0 = b.mul(r_enc[i - 1], r);                                  // muxEnc[i].c[0] <== rEnc[i-1] * r
        r_enc[i] = b.mul_add(r_enc[i - 1] - c0, should_zero[i], c0);
    }
    r_dec[0] = r;
    for (size_t i = 1; i < L; ++i) r_dec[i] = b.mul(r_dec[i - 1], r);
    LC sum_enc = b.mul(r_enc[0], processed[0]);
    for (size_t i = 1; i < L; ++i) sum_enc = b.mul_add(r_enc[i], processed[i], sum_enc);
    LC sum_dec = b.mul(r_dec[0], decoded[0]);
    for (size_t i = 1; i < L; ++i) sum_dec = b.mul_add(r_dec[i], decoded[i], sum_dec);
    return is_equal(b, sum_enc, sum_dec);                                // isValid
}

// ---------------------------------------------------------------- email-verifier.circom
Circuit build_email_verifier(const EmailVerifierParams& P, bool materialize_linear) {
    AppSpec app;
    app.ev = P;
    if (P.twitter) {
        // Proof-of-Twitter: `email was meant for @(\w+)` in the body, PackRegexReveal(maxBodyLength, 21), public address
        if (P.ignore_body_hash_check) throw std::runtime_error("TwitterVerifier needs the body (ignoreBodyHashCheck = 0)");
        app.expose_header_hash = false;     // EV.shaHi / EV.shaLo: signals of the sub-component
        app.scope = "TwitterVerifier";
        AppRegex rx;
        rx.name = "twitterUsername";
        rx.body = true;
        rx.scope = "TwitterResetRegex";
        rx.parts = {{"email was meant for @", false, 0}, {"[a-zA-Z0-9_]+", true, 21}};
        app.regexes.push_back(rx);
        app.external_inputs.push_back({"address", 0});   // component main { public [ address ] }
    }
    return build_email_app(app, materialize_linear);
}

// every signal name EmailVerifier (or the app wrapper) declares under any flag; an app's names must avoid them
static const char* const EMAIL_VERIFIER_SIGNALS[] = {
    "pubkeyHash", "shaHi", "shaLo", "maskedHeader", "maskedBody", "emailHeader", "emailHeaderLength", "pubkey", "signature",
    "headerMask", "bodyHashIndex", "precomputedSHA", "emailBody", "emailBodyLength", "decodedEmailBodyIn", "bodyMask",
    "emailNullifier"};

static uint32_t packed_len(uint32_t bytes) { return (bytes + 30) / 31; }   // computeIntChunkLength (utils/bytes.circom:10-20)

Circuit build_email_app(const AppSpec& A, bool materialize_linear) {
    const EmailVerifierParams& P = A.ev;
    const uint32_t H = P.max_headers_length, Bd = P.max_body_length, n = P.n, k = P.k;
    if (H % 64 != 0 || Bd % 64 != 0 || !(n * k > 2048) || !(n < 127))
        throw std::runtime_error("EmailVerifier: parameter asserts failed (email-verifier.circom:43-46)");

    // the app's signal names: unique, and none of EmailVerifier's
    std::vector<std::string> taken;
    auto claim = [&](const std::string& field, const std::string& name) {
        if (name.empty()) throw std::runtime_error(field + ": empty name");
        for (const char* r : EMAIL_VERIFIER_SIGNALS)
            if (name == r) throw std::runtime_error(field + ": signal name '" + name + "' collides with an EmailVerifier signal");
        for (const std::string& t : taken)
            if (t == name) throw std::runtime_error(field + ": signal name '" + name + "' is used twice");
        taken.push_back(name);
    };
    struct Reveal { std::string out, index; uint32_t max_length; int reveal; uint32_t salt; };   // salt: index into external_inputs
    std::vector<std::vector<Reveal>> reveals(A.regexes.size());
    for (size_t r = 0; r < A.regexes.size(); ++r) {
        const AppRegex& rx = A.regexes[r];
        const std::string field = "regexes[" + std::to_string(r) + "]";
        if (rx.name.empty()) throw std::runtime_error(field + ".name: empty name");
        if (rx.parts.empty()) throw std::runtime_error(field + ".parts: no parts");
        if (rx.body && P.ignore_body_hash_check)
            throw std::runtime_error(field + ".location: a body regex needs the body (ignoreBodyHashCheck is set)");
        const uint32_t searched = rx.body ? Bd : H;
        uint32_t n_pub = 0;
        for (auto& pt : rx.parts) n_pub += pt.is_public ? 1 : 0;
        uint32_t q = 0;
        for (size_t i = 0; i < rx.parts.size(); ++i) {
            const AppRegexPart& pt = rx.parts[i];
            const std::string pfield = field + ".parts[" + std::to_string(i) + "]";
            if (!pt.is_public) {
                if (pt.reveal_given) throw std::runtime_error(pfield + ".reveal: only a public part is revealed");
                if (!pt.salt.empty()) throw std::runtime_error(pfield + ".salt: only a public part with reveal \"commit\" takes a salt");
                continue;
            }
            uint32_t salt = 0;
            if (pt.reveal == REVEAL_COMMIT) {
                if (pt.salt.empty()) throw std::runtime_error(pfield + ".salt: reveal \"commit\" needs a salt (a private external input)");
                bool found = false;
                for (size_t e = 0; e < A.external_inputs.size() && !found; ++e) {
                    const AppExternalInput& ei = A.external_inputs[e];
                    if (ei.name != pt.salt) continue;
                    found = true;
                    salt = (uint32_t)e;
                    if (ei.is_public) throw std::runtime_error(pfield + ".salt: external input '" + pt.salt + "' is public; a salt must be private");
                    if (ei.max_length) throw std::runtime_error(pfield + ".salt: external input '" + pt.salt + "' is packed; a salt is one field element");
                }
                if (!found) throw std::runtime_error(pfield + ".salt: no external input named '" + pt.salt + "'");
            } else if (!pt.salt.empty()) {
                throw std::runtime_error(pfield + ".salt: a salt needs reveal \"commit\"");
            }
            const std::string pf = pfield + ".maxLength";
            if (pt.max_length == 0) throw std::runtime_error(pf + ": a public part needs maxLength");
            if (pt.max_length > searched)
                throw std::runtime_error(pf + ": " + std::to_string(pt.max_length) + " is larger than the searched " +
                                         (rx.body ? "body" : "header") + " (" + std::to_string(searched) + " bytes)");
            const std::string base = n_pub == 1 ? rx.name : rx.name + std::to_string(q);
            reveals[r].push_back(Reveal{base, base + "Index", pt.max_length, pt.reveal, salt});
            ++q;
        }
    }
    for (size_t r = 0; r < A.regexes.size(); ++r) {
        const std::string field = "regexes[" + std::to_string(r) + "].name";
        if (reveals[r].empty()) claim(field, A.regexes[r].name);      // no signal of its own, but the name stays unique
        for (auto& rv : reveals[r]) { claim(field, rv.out); claim(field, rv.index); }
    }
    for (size_t e = 0; e < A.external_inputs.size(); ++e) claim("externalInputs[" + std::to_string(e) + "].name", A.external_inputs[e].name);

    // the key registry: registryRoot replaces pubkeyHash as the first output, its inputs take the three names
    const uint32_t depth = A.key_registry_depth;
    if (depth > 32) throw std::runtime_error("keyRegistryDepth: at most 32, not " + std::to_string(depth));
    if (depth && P.public_pubkey)
        throw std::runtime_error("keyRegistryDepth: publicPubkey publishes the key the registry hides; drop one of them");
    static const char* const REGISTRY_SIGNALS[] = {"registryRoot", "registryIndex", "registrySiblings"};
    auto check_registry = [&](const std::string& field, const std::string& name) {
        for (const char* r : REGISTRY_SIGNALS)
            if (depth && name == r) throw std::runtime_error(field + ": signal name '" + name + "' is taken by the key registry (keyRegistryDepth)");
    };
    for (size_t r = 0; r < A.regexes.size(); ++r)
        for (auto& rv : reveals[r]) { check_registry("regexes[" + std::to_string(r) + "].name", rv.out); check_registry("regexes[" + std::to_string(r) + "].name", rv.index); }
    for (size_t e = 0; e < A.external_inputs.size(); ++e) check_registry("externalInputs[" + std::to_string(e) + "].name", A.external_inputs[e].name);

    // keyDomain: the public header part whose bytes the registry leaf binds to the key
    size_t kd_regex = 0, kd_part = 0;
    const bool domain_bound = !A.key_domain.empty();
    if (domain_bound) {
        const std::string& kd = A.key_domain;
        if (!depth) throw std::runtime_error("keyDomain: binds the registry leaf to a domain, so it needs keyRegistryDepth");
        bool found = false;
        for (size_t r = 0; r < A.regexes.size() && !found; ++r)
            for (size_t q = 0; q < reveals[r].size() && !found; ++q)
                if (reveals[r][q].out == kd) { found = true; kd_regex = r; kd_part = q; }
        if (!found) throw std::runtime_error("keyDomain: '" + kd + "' is not the output name of a public regex part");
        if (A.regexes[kd_regex].body)
            throw std::runtime_error("keyDomain: '" + kd + "' is a body regex part; the domain must come from the signed header");
        const uint32_t ml = reveals[kd_regex][kd_part].max_length;
        if (ml > 255) throw std::runtime_error("keyDomain: '" + kd + "' has maxLength " + std::to_string(ml) + "; a domain has at most 255 bytes");
    }

    Builder b("EmailVerifier");
    b.materialize_linear = materialize_linear;
    if (P.regex_style >= 0) b.regex_style = P.regex_style;
    ScopeGuard g(b, "EmailVerifier");

    // outputs first (circom witness order)
    Var pubkey_hash = b.declare_outputs(depth ? "registryRoot" : "pubkeyHash", 1)[0];
    Var sha_hi = 0, sha_lo = 0;
    if (A.expose_header_hash) { sha_hi = b.declare_outputs("shaHi", 1)[0]; sha_lo = b.declare_outputs("shaLo", 1)[0]; }
    std::vector<Var> masked_header, masked_body;
    if (P.enable_header_masking) masked_header = b.declare_outputs("maskedHeader", H);
    if (!P.ignore_body_hash_check && P.enable_body_masking) masked_body = b.declare_outputs("maskedBody", Bd);
    std::vector<std::vector<std::vector<Var>>> reveal_out(A.regexes.size());
    for (size_t r = 0; r < A.regexes.size(); ++r)
        for (auto& rv : reveals[r]) reveal_out[r].push_back(b.declare_outputs(rv.out, rv.reveal == REVEAL_BYTES ? packed_len(rv.max_length) : 1));
    Var nullifier = 0;
    if (A.email_nullifier) nullifier = b.declare_outputs("emailNullifier", 1)[0];

    auto to_lcs = [](const std::vector<Var>& v) { LCVec o(v.size()); for (size_t i = 0; i < v.size(); ++i) o[i] = LC(v[i]); return o; };
    // public inputs: the app's external inputs, bound to the proof through their public-input rows of the QAP (SURVEY A.7)
    std::vector<Var> external_first(A.external_inputs.size(), 0);
    for (size_t e = 0; e < A.external_inputs.size(); ++e) {
        const AppExternalInput& ei = A.external_inputs[e];
        if (ei.is_public) external_first[e] = b.declare_inputs(ei.name, ei.max_length ? packed_len(ei.max_length) : 1, true)[0];
    }
    std::vector<Var> pubkey_v;
    if (P.public_pubkey) pubkey_v = b.declare_inputs("pubkey", k, true);
    LCVec email_header = to_lcs(b.declare_inputs("emailHeader", H, false));
    LC email_header_length = LC(b.declare_inputs("emailHeaderLength", 1, false)[0]);
    if (!P.public_pubkey) pubkey_v = b.declare_inputs("pubkey", k, false);
    LCVec pubkey = to_lcs(pubkey_v);
    LCVec signature = to_lcs(b.declare_inputs("signature", k, false));
    LCVec header_mask, body_hash_index_v, precomputed_sha, email_body, email_body_length_v, decoded_in, body_mask;
    if (P.enable_header_masking) header_mask = to_lcs(b.declare_inputs("headerMask", H, false));
    if (!P.ignore_body_hash_check) {
        body_hash_index_v = to_lcs(b.declare_inputs("bodyHashIndex", 1, false));
        precomputed_sha = to_lcs(b.declare_inputs("precomputedSHA", 32, false));
        email_body = to_lcs(b.declare_inputs("emailBody", Bd, false));
        email_body_length_v = to_lcs(b.declare_inputs("emailBodyLength", 1, false));
        if (P.remove_soft_line_breaks) decoded_in = to_lcs(b.declare_inputs("decodedEmailBodyIn", Bd, false));
        if (P.enable_body_masking) body_mask = to_lcs(b.declare_inputs("bodyMask", Bd, false));
    }
    std::vector<std::vector<LC>> reveal_index(A.regexes.size());
    for (size_t r = 0; r < A.regexes.size(); ++r)
        for (auto& rv : reveals[r]) reveal_index[r].push_back(LC(b.declare_inputs(rv.index, 1, false)[0]));
    for (size_t e = 0; e < A.external_inputs.size(); ++e) {     // private external inputs: after everything else
        const AppExternalInput& ei = A.external_inputs[e];
        if (!ei.is_public) external_first[e] = b.declare_inputs(ei.name, ei.max_length ? packed_len(ei.max_length) : 1, false)[0];
    }
    LC registry_index;
    LCVec registry_siblings;
    if (depth) {
        registry_index = LC(b.declare_inputs("registryIndex", 1, false)[0]);
        registry_siblings = to_lcs(b.declare_inputs("registrySiblings", depth, false));
    }

    num2bits(b, email_header_length, log2_ceil(H));                      // :58-59
    assert_zero_padding(b, email_header, email_header_length);           // :63
    LCVec sha = sha256_bytes(b, email_header, email_header_length);      // :67
    LCVec packed = pack_bits(b, sha, 128);                               // :68-71
    if (A.expose_header_hash) { b.assign_output(sha_hi, packed[0]); b.assign_output(sha_lo, packed[1]); }
    else { b.signal(packed[0]); b.signal(packed[1]); }

    const uint32_t rsa_message_size = (256 + n) / n;                     // :74-84
    LCVec rsa_message(k);
    for (uint32_t i = 0; i < rsa_message_size; ++i) {
        LCVec bits(n);
        for (uint32_t j = 0; j < n; ++j) { uint32_t idx = i * n + j; bits[j] = idx < 256 ? sha[255 - idx] : LC(); }
        rsa_message[i] = bits2num(b, bits);
    }
    for (uint32_t i = rsa_message_size; i < k; ++i) rsa_message[i] = LC();
    rsa_verifier65537(b, n, k, rsa_message, signature, pubkey);          // :87-95

    if (P.enable_header_masking) {                                       // :97-105
        LCVec m = byte_mask(b, email_header, header_mask);
        for (uint32_t i = 0; i < H; ++i) b.assign_output(masked_header[i], m[i]);
    }

    if (!P.ignore_body_hash_check) {
        const LC& body_hash_index = body_hash_index_v[0];
        const LC& email_body_length = email_body_length_v[0];
        num2bits(b, email_body_length, log2_ceil(Bd));                   // :116-117
        assert_zero_padding(b, email_body, email_body_length);           // :121
        LCVec rx = body_hash_regex(b, email_header);                     // :126
        b.enforce_eq(rx[0], one_lc());                                   // bhRegexMatch === 1
        LCVec bh_reveal(rx.begin() + 1, rx.end());
        LCVec bh_b64 = select_regex_reveal(b, bh_reveal, body_hash_index, 44);      // :130
        LCVec header_body_hash = base64_decode(b, 32, bh_b64);                       // :131
        LCVec computed = sha256_bytes_partial(b, email_body, email_body_length, precomputed_sha);   // :136
        for (int i = 0; i < 32; ++i) {                                   // :139-146
            LCVec bits(8);
            for (int j = 0; j < 8; ++j) bits[7 - j] = computed[i * 8 + j];
            b.enforce_eq(bits2num(b, bits), header_body_hash[i]);
        }
        if (P.remove_soft_line_breaks) {                                 // :148-156
            LC valid = remove_soft_line_breaks(b, email_body, decoded_in);
            b.enforce_eq(valid, one_lc());                               // qpEncodingChecker.isValid === 1
        }
        if (P.enable_body_masking) {                                     // :158-166
            LCVec m = byte_mask(b, email_body, body_mask);
            for (uint32_t i = 0; i < Bd; ++i) b.assign_output(masked_body[i], m[i]);
        }
    }
    LC key_hash = poseidon_large(b, n, pubkey);                          // :173
    if (!domain_bound) {                 // a domain-bound leaf needs the domain's words: its root follows the regexes
        if (depth) key_hash = binary_merkle_root(b, key_hash, registry_index, registry_siblings);
        b.assign_output(pubkey_hash, key_hash);
    }
    if (A.regexes.empty() && !A.email_nullifier) return b.finalize();

    ScopeGuard ag(b, A.scope);
    LCVec domain_words;                                                  // keyDomain's packed words
    for (size_t r = 0; r < A.regexes.size(); ++r) {                      // the app's regexes (UsageGuide step 2)
        const AppRegex& ar = A.regexes[r];
        const LCVec& msg = ar.body ? (P.remove_soft_line_breaks ? decoded_in : email_body) : email_header;
        std::vector<std::pair<std::string, bool>> parts;
        for (auto& pt : ar.parts) parts.emplace_back(pt.regex, pt.is_public);
        LCVec rx;
        try {
            rx = regex_match_reveals(b, ar.scope.empty() ? ar.name : ar.scope, parts, msg);
        } catch (const std::exception& e) {
            throw std::runtime_error("regexes[" + std::to_string(r) + "] (" + ar.name + "): " + e.what());
        }
        b.enforce_eq(rx[0], one_lc());                                   // the regex must match
        for (size_t q = 0; q < reveals[r].size(); ++q) {
            LCVec reveal(rx.begin() + 1 + q * msg.size(), rx.begin() + 1 + (q + 1) * msg.size());
            const Reveal& rv = reveals[r][q];
            LCVec packs = pack_regex_reveal(b, reveal, reveal_index[r][q], rv.max_length);
            const bool is_domain = domain_bound && r == kd_regex && q == kd_part;
            if (rv.reveal == REVEAL_BYTES) {
                for (size_t i = 0; i < packs.size(); ++i) b.assign_output(reveal_out[r][q][i], packs[i]);
                if (is_domain) domain_words = to_lcs(reveal_out[r][q]);
                continue;
            }
            // hash / commit: the packed words stay intermediate signals; the Poseidon instances are recorded for the
            // engine's native permutation (circuit.hpp: PoseidonBlock)
            for (LC& p : packs) p = b.signal(p);
            if (is_domain) domain_words = packs;
            LC h = poseidon_modular(b, packs, true);
            if (rv.reveal == REVEAL_COMMIT) h = poseidon(b, {h, LC(external_first[rv.salt])}, true);
            b.assign_output(reveal_out[r][q][0], h);
        }
    }
    if (domain_bound) {
        // select_regex_reveal pins the exact matched run (a non-zero first byte after a zero, zeros past it), so the
        // words are the whole part D; the leaf ties D to the key that verified the signature
        LC leaf = domain_key_leaf(b, domain_words, key_hash);
        b.assign_output(pubkey_hash, binary_merkle_root(b, leaf, registry_index, registry_siblings));
    }
    if (A.email_nullifier) b.assign_output(nullifier, email_nullifier(b, n, signature));   // helpers/email-nullifier.circom
    return b.finalize();
}

}  // namespace gadgets
}  // namespace zke
