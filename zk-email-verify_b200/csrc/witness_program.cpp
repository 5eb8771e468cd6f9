// Lowering of the levelised witness program into the witness kernel's stream (witness_program.hpp).
#include "witness_program.hpp"
#include "gadgets.hpp"
#include <algorithm>
#include <map>
#include <stdexcept>

namespace zke {

std::vector<uint32_t> coef_words(const std::vector<U256>& coefs) {
    std::vector<uint32_t> coef_word(coefs.size(), 0);
    if (coefs.size() >= (1u << 24)) throw std::runtime_error("too many distinct coefficients");
    for (size_t i = 0; i < coefs.size(); ++i) {
        auto log2_exact = [](const U256& v) -> int {   // k if v == 2^k, else -1
            int k = -1, bits = 0;
            for (unsigned b = 0; b < 256; ++b) if (u256_bit(v, b)) { k = (int)b; ++bits; }
            return bits == 1 ? k : -1;
        };
        U256 neg;
        u256_sub(neg, fr_params().p, coefs[i]);
        const int kp = log2_exact(coefs[i]), kn = log2_exact(neg);
        uint32_t kind = 4, k = 0;
        if (kp == 0) kind = 0;
        else if (kn == 0) kind = 1;
        else if (kp > 0 && kp <= 252 && i <= 0xffffu) { kind = 2; k = (uint32_t)kp; }
        else if (kn > 0 && kn <= 252 && i <= 0xffffu) { kind = 3; k = (uint32_t)kn; }
        coef_word[i] = kind == 4 ? ((uint32_t)i | (4u << 24)) : (((uint32_t)i & 0xffffu) | (k << 16) | (kind << 24));
    }
    return coef_word;
}

namespace {

const uint32_t XOP_SHA = 6, XOP_RX = 7, XOP_POS = 8;

struct Levelised {
    std::vector<WOp> xops;                         // code XOP_SHA: a = index of the block; XOP_RX: a = index of the seed;
                                                   // XOP_POS: a = index of the Poseidon block
    std::vector<uint32_t> xlevel_ptr;              // ops of level l: [xlevel_ptr[l], xlevel_ptr[l + 1])
    std::vector<uint32_t> aux;                     // the circuit's aux table, then the regex seed images, the SHA tables and
                                                   // the Poseidon tables and constants
    std::vector<uint32_t> sha_aux_off, rx_aux_off, pos_aux_off; // per block / seed: offset of its table in aux
};

// ---- native Sha256compression (circuit.hpp: ShaBlock): the ops that define the signals / scratch slots of a recorded
// instance are replaced by ONE cooperative op per instance and the program is levelised again - the chained compressions
// then cost one level each instead of ~320.
// ---- zk-regex state seeding (circuit.hpp: RegexSeed): one cooperative op per regex instance runs the automaton over the
// message and writes every state signal; the instance's own ops stay (they write the same values again) but now depend on
// seeded signals instead of on the previous position's gadgets, so the ~4 levels per message byte collapse into a handful
// for the whole message.
// ---- native Poseidon (circuit.hpp: PoseidonBlock): as for SHA, the gadget's ops are replaced by one cooperative op per
// instance - a Poseidon(t - 1) costs one level instead of ~4 per round (~260 for the widths of a PoseidonModular).
Levelised substitute_and_levelise(const Circuit& c, bool native_sha, bool native_rx, bool native_pos) {
    Levelised L;
    std::vector<WOp>& xops = L.xops;
    std::vector<uint32_t>& xlevel_ptr = L.xlevel_ptr;
    std::vector<uint32_t>& aux = L.aux;
    std::vector<uint32_t>& sha_aux_off = L.sha_aux_off, &rx_aux_off = L.rx_aux_off, &pos_aux_off = L.pos_aux_off;
    aux = c.aux;
    sha_aux_off.assign(c.sha_blocks.size(), 0);
    rx_aux_off.assign(c.regex_seeds.size(), 0);
    pos_aux_off.assign(c.poseidon_blocks.size(), 0);
    if (!native_sha && !native_rx && !native_pos) {
        xops = c.ops;
        xlevel_ptr = c.level_ptr;
        return L;
    }
    const uint32_t total = c.n_vars + c.n_temps;
    std::vector<int32_t> owner(total, -1);     // slot -> block that defines it
    std::vector<uint8_t> seeded(total, 0);     // slot written by a regex seed op (its own op stays)
    if (native_rx)
        for (size_t ri = 0; ri < c.regex_seeds.size(); ++ri) {
            const RegexSeed& R = c.regex_seeds[ri];
            rx_aux_off[ri] = (uint32_t)aux.size();
            append_regex_seed(aux, R);
            for (size_t d = 0; d < R.desc.size(); d += 2) seeded[R.desc[d]] = 1;
        }
    if (aux.size() >= (1u << 30)) throw std::runtime_error("witness program: auxiliary table too large");
    for (size_t bi = 0; native_sha && bi < c.sha_blocks.size(); ++bi) {
        const ShaBlock& B = c.sha_blocks[bi];
        for (uint32_t v = B.var_begin; v < B.var_end; ++v) owner[v] = (int32_t)bi;
        for (uint32_t v = B.temp_begin; v < B.temp_end; ++v) owner[v] = (int32_t)bi;
        sha_aux_off[bi] = (uint32_t)aux.size();
        aux.push_back((uint32_t)(B.desc.size() / 2));
        aux.insert(aux.end(), B.inputs.begin(), B.inputs.end());
        aux.insert(aux.end(), B.desc.begin(), B.desc.end());
    }
    if (native_pos) {
        std::map<uint32_t, uint32_t> consts_off;       // width -> offset of its constants
        for (const PoseidonBlock& B : c.poseidon_blocks) {
            if (consts_off.count(B.t)) continue;
            const gadgets::PoseidonParams& Pp = gadgets::poseidon_params((int)B.t);
            while (aux.size() % 8) aux.push_back(0);   // 32-byte rows: the device loads them as two 16-byte words
            consts_off[B.t] = (uint32_t)aux.size();
            for (const Fr& x : Pp.rc) { const U256 u = x.to_u256(); for (int q = 0; q < 4; ++q) aux.insert(aux.end(), {(uint32_t)u.v[q], (uint32_t)(u.v[q] >> 32)}); }
            for (auto& row : Pp.mds) for (const Fr& x : row) for (int q = 0; q < 4; ++q) aux.insert(aux.end(), {(uint32_t)x.m.v[q], (uint32_t)(x.m.v[q] >> 32)});
        }
        for (size_t bi = 0; bi < c.poseidon_blocks.size(); ++bi) {
            const PoseidonBlock& B = c.poseidon_blocks[bi];
            const gadgets::PoseidonParams& Pp = gadgets::poseidon_params((int)B.t);
            if (B.inputs.size() + 1 != B.t) throw std::runtime_error("native Poseidon: a record's inputs do not match its width");
            for (uint32_t v = B.var_begin; v < B.var_end; ++v) owner[v] = (int32_t)bi;
            for (uint32_t v = B.temp_begin; v < B.temp_end; ++v) owner[v] = (int32_t)bi;
            pos_aux_off[bi] = (uint32_t)aux.size();
            aux.insert(aux.end(), {B.t, (uint32_t)Pp.r_p, consts_off[B.t]});
            aux.insert(aux.end(), B.inputs.begin(), B.inputs.end());
            const size_t slots = aux.size(), rounds = (size_t)(Pp.r_f + Pp.r_p);
            aux.resize(slots + B.t + rounds * B.t * 4, 0);
            for (size_t d = 0; d < B.desc.size(); d += 2) {
                const uint32_t rnd = B.desc[d + 1] >> 16, lane = (B.desc[d + 1] >> 8) & 0xff, kind = B.desc[d + 1] & 0xff;
                if (rnd >= rounds || lane >= B.t || kind > POS_K_MIX || (kind == POS_K_INPUT && rnd != 0)) throw std::runtime_error("native Poseidon: bad descriptor");
                aux[slots + (kind == POS_K_INPUT ? lane : B.t + ((size_t)rnd * B.t + lane) * 4 + kind - 1)] = B.desc[d];
            }
        }
        if (aux.size() >= (1u << 30)) throw std::runtime_error("witness program: auxiliary table too large");
    }
    // Order: c.ops is in level order (producers before consumers).  A block's op is inserted right after the
    // producer of its LAST-defined input: everything it reads precedes it, and everything that reads its outputs
    // (the final-sum bits, originally defined after all of the block's inputs) follows it.
    std::vector<int64_t> def_pos(total, -1);
    for (size_t i = 0; i < c.ops.size(); ++i) {
        const WOp& o = c.ops[i];
        const uint32_t nd = o.code == OP_FPMUL ? 2 * c.aux[o.a + 1] : 1;
        for (uint32_t j = 0; j < nd; ++j) def_pos[o.dst + j] = (int64_t)i;
    }
    std::vector<std::vector<uint32_t>> blocks_at(c.ops.size() + 1), seeds_at(c.ops.size() + 1), pos_at(c.ops.size() + 1);
    for (size_t bi = 0; native_pos && bi < c.poseidon_blocks.size(); ++bi) {
        int64_t pos = 0;
        for (uint32_t v : c.poseidon_blocks[bi].inputs) pos = std::max(pos, def_pos[v] + 1);
        pos_at[(size_t)pos].push_back((uint32_t)bi);
    }
    for (size_t bi = 0; native_sha && bi < c.sha_blocks.size(); ++bi) {
        int64_t pos = 0;
        for (uint32_t v : c.sha_blocks[bi].inputs) if (v < SHA_CONST0) pos = std::max(pos, def_pos[v] + 1);
        blocks_at[(size_t)pos].push_back((uint32_t)bi);
    }
    for (size_t ri = 0; native_rx && ri < c.regex_seeds.size(); ++ri) {
        int64_t pos = 0;      // right after the producer of the last message byte: before every op of the instance
        for (uint32_t v : c.regex_seeds[ri].bytes) pos = std::max(pos, def_pos[v] + 1);
        seeds_at[(size_t)pos].push_back((uint32_t)ri);
    }
    std::vector<WOp> kept;
    kept.reserve(c.ops.size());
    for (size_t i = 0; i <= c.ops.size(); ++i) {
        for (uint32_t bi : blocks_at[i]) kept.push_back(WOp{XOP_SHA, c.sha_blocks[bi].var_begin, bi, 0, 0});
        for (uint32_t ri : seeds_at[i]) kept.push_back(WOp{XOP_RX, 0, ri, 0, 0});
        for (uint32_t pi : pos_at[i]) kept.push_back(WOp{XOP_POS, 0, pi, 0, 0});
        if (i < c.ops.size() && owner[c.ops[i].dst] < 0) kept.push_back(c.ops[i]);
    }
    // levelise (the same rules as Builder::finalize, plus the multi-output block op)
    std::vector<uint32_t> level(total, 0), op_level(kept.size(), 0);
    std::vector<uint8_t> defined(total, 0);
    defined[0] = 1;
    for (auto& g : c.groups) if (g.kind != 0) for (uint32_t i = 0; i < g.count; ++i) defined[g.first + i] = 1;
    auto need = [&](uint32_t v) -> uint32_t {
        if (!defined[v]) throw std::runtime_error("native op substitution: an op reads an unassigned signal");
        return level[v];
    };
    auto lc_level = [&](uint32_t id) { uint32_t l = 0; for (uint32_t k = c.lc_ptr[id]; k < c.lc_ptr[id + 1]; ++k) l = std::max(l, need(c.lc_var[k])); return l; };
    uint32_t max_level = 0;
    for (size_t i = 0; i < kept.size(); ++i) {
        const WOp& o = kept[i];
        uint32_t l = 0;
        switch (o.code) {
            case OP_LIN: case OP_SHRLC: l = lc_level(o.a); break;
            case OP_QUAD: l = std::max(lc_level(o.a), std::max(lc_level(o.b), lc_level(o.c))); break;
            case OP_SHRAND: case OP_INVZ: l = need(o.a); break;
            case OP_FPMUL: { const uint32_t kk = c.aux[o.a + 1]; for (uint32_t j = 0; j < 3 * kk; ++j) l = std::max(l, need(c.aux[o.a + 2 + j])); break; }
            case XOP_SHA: for (uint32_t v : c.sha_blocks[o.a].inputs) if (v < SHA_CONST0) l = std::max(l, need(v)); break;
            case XOP_RX: for (uint32_t v : c.regex_seeds[o.a].bytes) l = std::max(l, need(v)); break;
            case XOP_POS: for (uint32_t v : c.poseidon_blocks[o.a].inputs) l = std::max(l, need(v)); break;
            default: throw std::runtime_error("bad opcode");
        }
        l += 1;
        if (o.code == XOP_SHA) {
            const ShaBlock& B = c.sha_blocks[o.a];
            for (uint32_t v = B.var_begin; v < B.var_end; ++v) { defined[v] = 1; level[v] = l; }
        } else if (o.code == XOP_RX) {
            const RegexSeed& R = c.regex_seeds[o.a];
            for (size_t d = 0; d < R.desc.size(); d += 2) { defined[R.desc[d]] = 1; level[R.desc[d]] = l; }
        } else if (o.code == XOP_POS) {
            const PoseidonBlock& B = c.poseidon_blocks[o.a];
            for (size_t d = 0; d < B.desc.size(); d += 2) { defined[B.desc[d]] = 1; level[B.desc[d]] = l; }
        } else if (o.code == OP_FPMUL) {
            const uint32_t kk = c.aux[o.a + 1];
            for (uint32_t j = 0; j < 2 * kk; ++j) { defined[o.dst + j] = 1; level[o.dst + j] = l; }
        } else if (seeded[o.dst]) {
            // the value is already there (same value, written by the seed op at an earlier level): readers keep
            // depending on the seed, this op only has to run after its own operands
            if (!defined[o.dst]) throw std::runtime_error("regex seeding: a seeded signal is produced before its seed op");
        } else {
            defined[o.dst] = 1; level[o.dst] = l;
        }
        op_level[i] = l;
        max_level = std::max(max_level, l);
    }
    xlevel_ptr.assign(max_level + 1, 0);
    for (uint32_t l : op_level) xlevel_ptr[l]++;                 // levels are 1-based here
    { uint32_t run = 0; for (uint32_t l = 1; l <= max_level; ++l) { const uint32_t n = xlevel_ptr[l]; xlevel_ptr[l] = run; run += n; } xlevel_ptr[0] = 0; }
    xops.resize(kept.size());
    { std::vector<uint32_t> cursor(xlevel_ptr.begin(), xlevel_ptr.end()); for (size_t i = 0; i < kept.size(); ++i) xops[cursor[op_level[i]]++] = kept[i]; }
    std::vector<uint32_t> lp(max_level + 1);
    for (uint32_t l = 1; l <= max_level; ++l) lp[l - 1] = xlevel_ptr[l];
    lp[max_level] = (uint32_t)kept.size();
    xlevel_ptr.swap(lp);
    return L;
}

// Streamed witness program: per level, ops sorted by kind / size so that the threads of an iteration do similar work,
// padded with no-ops to whole iterations of WITNESS_THREADS records; the LC terms of an iteration form one contiguous,
// 16-byte aligned block.  Every level is padded to whole rounds of `cluster` iterations, iteration k belongs to CTA
// k % cluster.  Returns per level the index of its first iteration and the number of non-empty ones.
std::vector<std::pair<size_t, size_t>> stream_levels(const Circuit& c, const std::vector<uint32_t>& coef_word, const Levelised& L,
                                                     bool coop_fpmul, uint32_t cluster, WitnessStream& S) {
    const std::vector<WOp>& xops = L.xops;
    const std::vector<uint32_t>& xlevel_ptr = L.xlevel_ptr;
    const uint32_t T = WITNESS_THREADS;
    std::vector<uint32_t>& packed = S.ops;         // 4 words per record
    std::vector<uint32_t>& terms = S.terms, &hdr = S.iter_hdr;   // 2 words per term / 4 per iteration header
    std::vector<uint32_t>& coop = S.coop;          // cooperative ops (two words each), grouped by iteration
    packed.reserve(4 * (c.ops.size() + (size_t)T * c.n_levels()));
    terms.reserve(2 * c.lc_var.size() + 16);
    auto lc_len = [&](uint32_t id) { return c.lc_ptr[id + 1] - c.lc_ptr[id]; };
    const uint32_t n_xlevels = xlevel_ptr.empty() ? 0 : (uint32_t)xlevel_ptr.size() - 1;
    std::vector<uint32_t> order;
    std::vector<std::pair<size_t, size_t>> level_iters;
    for (uint32_t lvl = 0; lvl < n_xlevels; ++lvl) {
        const uint32_t beg = xlevel_ptr[lvl], end = xlevel_ptr[lvl + 1];
        const size_t level_first_iter = hdr.size() / 4;
        order.clear();
        const uint32_t coop_first = (uint32_t)(coop.size() / 2);
        std::vector<uint32_t> pos_coop;                // after the level's other cooperative ops: adjacent, one warp each
        for (uint32_t i = beg; i < end; ++i) {
            if (xops[i].code == XOP_POS) { pos_coop.push_back(0xc0000000u | L.pos_aux_off[xops[i].a]); pos_coop.push_back(0); }
            else if (xops[i].code == XOP_SHA) { coop.push_back(L.sha_aux_off[xops[i].a]); coop.push_back(0); }
            else if (xops[i].code == XOP_RX) { coop.push_back(0x40000000u | L.rx_aux_off[xops[i].a]); coop.push_back(0); }
            else if (xops[i].code == OP_FPMUL && coop_fpmul) { coop.push_back(0x80000000u | xops[i].a); coop.push_back(xops[i].dst); }
            else order.push_back(i);
        }
        coop.insert(coop.end(), pos_coop.begin(), pos_coop.end());
        uint32_t coop_left = (uint32_t)(coop.size() / 2) - coop_first;   // attached to the level's first iteration
        // Sort key: kind, then the positions of the terms that need a product (coefficient other than +-1) in the
        // flattened [A | B | C] term list, then the term count.  Within an LC the product terms are emitted first
        // (addition commutes), so the ops of a warp take the product branch of eval_lcs in the same term slots -
        // or not at all: a warp only pays for a Montgomery product where some lane needs one.
        auto key = [&](uint32_t i) -> uint64_t {
            const WOp& o = xops[i];
            if (o.code == OP_FPMUL) return ~0ull;
            if (o.code == OP_INVZ) return 1ull << 62;
            if (o.code == OP_SHRAND) return 0;
            const uint32_t ids[3] = {o.a, o.b, o.c};
            const uint32_t n_lc = o.code == OP_QUAD ? 3 : 1;
            uint64_t mask = 0;
            uint32_t pos = 0;
            for (uint32_t q = 0; q < n_lc; ++q) {
                uint32_t heavy = 0;
                for (uint32_t k = c.lc_ptr[ids[q]]; k < c.lc_ptr[ids[q] + 1]; ++k) heavy += (coef_word[c.lc_coef[k]] >> 24) >= 2;
                for (uint32_t t = 0; t < heavy && pos + t < 48; ++t) mask |= 1ull << (pos + t);
                pos += lc_len(ids[q]);
            }
            return ((uint64_t)(o.code == OP_QUAD ? 2 : 1) << 60) | (mask << 8) | std::min<uint32_t>(pos, 255);
        };
        std::vector<std::pair<uint64_t, uint32_t>> keyed(order.size());
        for (size_t i = 0; i < order.size(); ++i) keyed[i] = {key(order[i]), order[i]};
        std::stable_sort(keyed.begin(), keyed.end(), [](const std::pair<uint64_t, uint32_t>& x, const std::pair<uint64_t, uint32_t>& y) { return x.first > y.first; });
        for (size_t i = 0; i < order.size(); ++i) order[i] = keyed[i].second;
        const size_t n_regular = order.size();
        S.level_ops.push_back((uint32_t)n_regular);
        for (size_t base = 0; base < std::max<size_t>(n_regular, coop_left ? 1 : 0); base += T) {
            const uint32_t first_term = (uint32_t)(terms.size() / 2);
            for (uint32_t t = 0; t < T; ++t) {
                uint32_t rec[4] = {0, WOP_NOP, 0, 0};
                if (base + t < n_regular) {
                    const WOp& o = xops[order[base + t]];
                    rec[0] = o.dst;
                    if (o.code == OP_LIN || o.code == OP_QUAD || o.code == OP_SHRLC) {
                        const uint32_t ids[3] = {o.a, o.b, o.c};
                        const uint32_t n_lc = o.code == OP_QUAD ? 3 : 1;
                        uint32_t n[3] = {0, 0, 0};
                        rec[2] = (uint32_t)(terms.size() / 2);
                        for (uint32_t q = 0; q < n_lc; ++q) {
                            n[q] = lc_len(ids[q]);
                            if (n[q] > 31) throw std::runtime_error("linear combination too long for the streamed witness program");
                            for (int pass = 0; pass < 2; ++pass)   // product terms first
                                for (uint32_t k = c.lc_ptr[ids[q]]; k < c.lc_ptr[ids[q] + 1]; ++k)
                                    if (((coef_word[c.lc_coef[k]] >> 24) >= 2) == (pass == 0)) { terms.push_back(c.lc_var[k]); terms.push_back(coef_word[c.lc_coef[k]]); }
                        }
                        rec[1] = o.code | (n[0] << 8) | (n[1] << 13) | (n[2] << 18);
                        if (o.code == OP_SHRLC) {
                            if (o.b > 0xffffu || o.c > 0xffffu) throw std::runtime_error("OP_SHRLC operand out of range");
                            rec[3] = o.b | (o.c << 16);
                        }
                    } else if (o.code == OP_SHRAND) {
                        if (o.b > 0xffffu || o.c > 0xffffu) throw std::runtime_error("OP_SHRAND operand out of range");
                        rec[1] = o.code; rec[2] = o.a; rec[3] = o.b | (o.c << 16);
                    } else {
                        rec[1] = o.code; rec[2] = o.a;
                    }
                }
                packed.insert(packed.end(), rec, rec + 4);
            }
            if ((terms.size() / 2) & 1) { terms.push_back(0); terms.push_back(0); }   // keep blocks 16-byte aligned
            hdr.push_back(first_term);
            hdr.push_back((uint32_t)(terms.size() / 2) - first_term);
            hdr.push_back(coop_first);
            hdr.push_back(coop_left);
            coop_left = 0;
            S.iter_info.push_back(packed[packed.size() - 4 * T + 1]);
            S.iter_info.push_back((uint32_t)std::min<size_t>(T, n_regular > base ? n_regular - base : 0));
            S.iter_info.push_back((uint32_t)(terms.size() / 2) - first_term);
        }
        // pad the level to whole rounds (empty iterations: no-op records, no terms)
        level_iters.emplace_back(level_first_iter, hdr.size() / 4 - level_first_iter);
        while (cluster > 1 && (hdr.size() / 4 - level_first_iter) % cluster != 0) {
            for (uint32_t t = 0; t < T; ++t) { const uint32_t rec[4] = {0, WOP_NOP, 0, 0}; packed.insert(packed.end(), rec, rec + 4); }
            hdr.push_back((uint32_t)(terms.size() / 2)); hdr.push_back(0); hdr.push_back((uint32_t)(coop.size() / 2)); hdr.push_back(0);
            S.iter_info.push_back(WOP_NOP); S.iter_info.push_back(0); S.iter_info.push_back(0);
        }
    }
    S.n_levels = n_xlevels;
    return level_iters;
}

void barrier_flags_and_sentinels(const std::vector<std::pair<size_t, size_t>>& level_iters, uint32_t cluster, WitnessStream& S) {
    std::vector<uint32_t>& hdr = S.iter_hdr;
    const uint32_t n_iters = (uint32_t)(hdr.size() / 4);
    // Cluster barrier flags (bit 31 of header word 3, on every iteration of a level's last round): needed when signals cross
    // CTAs - the level had more than one iteration (other CTAs wrote) or the next one has (other CTAs will read).  Runs of
    // one-iteration levels (the Poseidon rounds, the tails of the comparison chains) stay on CTA 0 with its own barrier.
    for (size_t l = 0; l < level_iters.size(); ++l) {
        const bool last = l + 1 == level_iters.size();
        if (!(level_iters[l].second > 1 || last || level_iters[l + 1].second > 1)) continue;
        const size_t end_iter = last ? n_iters : level_iters[l + 1].first;
        for (uint32_t q = 1; q <= cluster && end_iter >= level_iters[l].first + q; ++q) hdr[4 * (end_iter - q) + 3] |= 0x80000000u;
    }
    for (uint32_t q = 0; q < 2 * cluster; ++q) { hdr.push_back((uint32_t)(S.terms.size() / 2)); hdr.push_back(0); hdr.push_back(0); hdr.push_back(0); }   // sentinel headers
    if (S.ops.empty()) S.ops.resize(4 * WITNESS_THREADS, 0);
    for (int q = 0; q < 8; ++q) S.terms.push_back(0);
    if (S.aux.empty()) S.aux.push_back(0);
    if (S.coop.empty()) { S.coop.push_back(0); S.coop.push_back(0); }
    S.n_iters = n_iters;
    S.cluster = cluster;
}

}  // namespace

WitnessStream lower_witness_program(const Circuit& c, const std::vector<uint32_t>& coef_word, const LowerOptions& opt) {
    // the device's big-integer hint works on at most 20 limbs (witness.cu: fpmul_hint_dev); refuse larger FpMul
    // instances here instead of producing a witness that fails its constraints later
    for (const WOp& o : c.ops)
        if (o.code == OP_FPMUL && c.aux[o.a + 1] > 20) throw std::runtime_error("FpMul with k = " + std::to_string(c.aux[o.a + 1]) + " limbs exceeds the device hint's limit of 20");
    Levelised L = substitute_and_levelise(c, opt.native_sha && !c.sha_blocks.empty(), opt.native_regex && !c.regex_seeds.empty(),
                                          opt.native_poseidon && !c.poseidon_blocks.empty());
    WitnessStream S;
    const std::vector<std::pair<size_t, size_t>> level_iters = stream_levels(c, coef_word, L, opt.coop_fpmul, opt.cluster, S);
    S.aux = std::move(L.aux);
    barrier_flags_and_sentinels(level_iters, opt.cluster, S);
    return S;
}

}  // namespace zke
