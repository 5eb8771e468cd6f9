// Poseidon (circomlib parameterisation) - constraint gadget and host permutation.
//
// Follows circomlib 2.0.5 `Poseidon(nInputs)` (un-vendored; pinned at /root/reference/yarn.lock:3619-3621,
// call site /root/reference/packages/circuits/utils/hash.circom:38).  circomlib ships pre-generated constant
// tables and evaluates an algebraically re-arranged schedule; the tables are not part of the reference tree,
// so the constants are regenerated here with the Poseidon Grain-LFSR parameter generator (prime field,
// x^5 S-box, n = 254, t, R_F = 8, R_P from circomlib's N_ROUNDS_P) and the plain permutation is constrained.
// Output values are identical (checked against the published poseidon([1,2]) vector in tests).
#include "gadgets.hpp"
#include <map>
#include <stdexcept>

namespace zke {
namespace gadgets {

namespace {
const int N_BITS = 254;
const int R_F = 8;
const int N_ROUNDS_P[16] = {56, 57, 56, 60, 60, 63, 64, 63, 60, 66, 60, 65, 70, 60, 64, 68};

struct Grain {
    uint8_t s[80];
    int head = 0;
    Grain(int t, int r_f, int r_p) {
        int pos = 0;
        auto put = [&](uint32_t v, int n) { for (int i = n - 1; i >= 0; --i) s[pos++] = (v >> i) & 1; };
        put(1, 2); put(0, 4); put(N_BITS, 12); put((uint32_t)t, 12); put((uint32_t)r_f, 10); put((uint32_t)r_p, 10);
        for (int i = 0; i < 30; ++i) s[pos++] = 1;
        for (int i = 0; i < 160; ++i) step();
    }
    int at(int i) const { return s[(head + i) % 80]; }
    int step() {
        int nb = at(62) ^ at(51) ^ at(38) ^ at(23) ^ at(13) ^ at(0);
        s[head] = (uint8_t)nb;
        head = (head + 1) % 80;
        return nb;
    }
    int bit() {
        for (;;) { int b1 = step(); int b2 = step(); if (b1) return b2; }
    }
    U256 bits254() {
        U256 v = {{0, 0, 0, 0}};
        for (int i = 0; i < N_BITS; ++i) {
            v.v[3] = (v.v[3] << 1) | (v.v[2] >> 63);
            v.v[2] = (v.v[2] << 1) | (v.v[1] >> 63);
            v.v[1] = (v.v[1] << 1) | (v.v[0] >> 63);
            v.v[0] = (v.v[0] << 1) | (uint64_t)bit();
        }
        return v;
    }
};

struct Params {
    int t, r_p;
    std::vector<Fr> rc;                 // (R_F + R_P) * t
    std::vector<std::vector<Fr>> mds;   // t x t
};

const Params& params_for(int t) {
    static std::map<int, Params> cache;
    auto it = cache.find(t);
    if (it != cache.end()) return it->second;
    if (t < 2 || t > 17) throw std::runtime_error("Poseidon: unsupported width");
    Params p;
    p.t = t;
    p.r_p = N_ROUNDS_P[t - 2];
    Grain g(t, R_F, p.r_p);
    const U256& mod = fr_params().p;
    for (int i = 0; i < (R_F + p.r_p) * t; ++i) {
        U256 v;
        do { v = g.bits254(); } while (u256_cmp(v, mod) >= 0);
        p.rc.push_back(Fr::from_u256(v));
    }
    for (;;) {
        std::vector<Fr> vals;
        for (int i = 0; i < 2 * t; ++i) {
            U256 v = g.bits254();
            while (u256_cmp(v, mod) >= 0) u256_sub(v, v, mod);
            vals.push_back(Fr::from_u256(v));
        }
        bool ok = true;
        for (int i = 0; i < 2 * t && ok; ++i) for (int j = i + 1; j < 2 * t; ++j) if (vals[i] == vals[j]) { ok = false; break; }
        for (int i = 0; i < t && ok; ++i) for (int j = 0; j < t; ++j) if ((vals[i] + vals[t + j]).is_zero()) { ok = false; break; }
        if (!ok) continue;
        p.mds.assign(t, std::vector<Fr>(t));
        for (int i = 0; i < t; ++i) for (int j = 0; j < t; ++j) p.mds[i][j] = (vals[i] + vals[t + j]).inv();
        break;
    }
    return cache.emplace(t, std::move(p)).first->second;
}
}  // namespace

Fr poseidon_hash(const std::vector<Fr>& inputs) {
    const int t = (int)inputs.size() + 1;
    const Params& P = params_for(t);
    std::vector<Fr> st(t, Fr::zero());
    for (int i = 1; i < t; ++i) st[i] = inputs[i - 1];
    int k = 0;
    for (int rnd = 0; rnd < R_F + P.r_p; ++rnd) {
        for (int i = 0; i < t; ++i) st[i] += P.rc[k + i];
        k += t;
        bool full = rnd < R_F / 2 || rnd >= R_F / 2 + P.r_p;
        for (int i = 0; i < (full ? t : 1); ++i) { Fr x2 = st[i].sqr(); st[i] = x2.sqr() * st[i]; }
        std::vector<Fr> nx(t, Fr::zero());
        for (int i = 0; i < t; ++i) for (int j = 0; j < t; ++j) nx[i] += P.mds[i][j] * st[j];
        st.swap(nx);
    }
    return st[0];
}

const PoseidonParams& poseidon_params(int t) {
    static std::map<int, PoseidonParams> cache;
    auto it = cache.find(t);
    if (it != cache.end()) return it->second;
    const Params& P = params_for(t);
    PoseidonParams q;
    q.t = t;
    q.r_f = R_F;
    q.r_p = P.r_p;
    q.rc = P.rc;
    q.mds = P.mds;
    return cache.emplace(t, std::move(q)).first->second;
}

LC poseidon(Builder& b, const LCVec& inputs, bool record) {
    ScopeGuard g(b, "Poseidon");
    const int t = (int)inputs.size() + 1;
    const Params& P = params_for(t);
    PoseidonBlock blk;
    if (record) {
        blk.t = (uint32_t)t;
        for (const LC& in : inputs) {
            Var v;
            if (!in.is_single_var(&v)) throw std::runtime_error("Poseidon record: every input must be a signal");
            blk.inputs.push_back(v);
        }
        blk.var_begin = b.num_vars();
        blk.temp_begin = b.num_temps();
    }
    // a signal the gadget created for (round, lane, kind) gets its descriptor (constants and aliases create none)
    auto note = [&](const LC& e, int rnd, int lane, uint32_t kind) {
        Var v;
        if (record && e.is_single_var(&v) && v >= blk.var_begin)
            blk.desc.insert(blk.desc.end(), {v, (uint32_t)rnd << 16 | (uint32_t)lane << 8 | kind});
    };
    LCVec st(t);
    for (int i = 1; i < t; ++i) { st[i] = b.signal(inputs[i - 1]); note(st[i], 0, i, POS_K_INPUT); }
    int k = 0;
    const int rounds = R_F + P.r_p;
    for (int rnd = 0; rnd < rounds; ++rnd) {
        for (int i = 0; i < t; ++i) st[i] += LC::constant(P.rc[k + i]);       // Ark
        k += t;
        bool full = rnd < R_F / 2 || rnd >= R_F / 2 + P.r_p;
        for (int i = 0; i < (full ? t : 1); ++i) {                            // Sigma: in2, in4, out
            LC x = st[i];
            LC x2 = b.mul(x, x);
            LC x4 = b.mul(x2, x2);
            st[i] = b.mul(x4, x);
            note(x2, rnd, i, POS_K_X2); note(x4, rnd, i, POS_K_X4); note(st[i], rnd, i, POS_K_X5);
        }
        LCVec nx(t);                                                          // Mix
        for (int i = 0; i < t; ++i) {
            LC e;
            for (int j = 0; j < t; ++j) e += st[j] * P.mds[i][j];
            // only state[0] is the hash output; it is enough to materialise what later rounds consume
            nx[i] = (rnd == rounds - 1 && i != 0) ? LC() : b.signal(e);
            if (!(rnd == rounds - 1 && i != 0)) note(nx[i], rnd, i, POS_K_MIX);
        }
        st.swap(nx);
    }
    if (record) {
        blk.var_end = b.num_vars();
        blk.temp_end = b.num_temps();
        if (blk.desc.size() / 2 != blk.var_end - blk.var_begin) throw std::runtime_error("Poseidon record: a created signal has no descriptor");
        b.add_poseidon_block(std::move(blk));
    }
    return st[0];
}

}  // namespace gadgets
}  // namespace zke
