// Lowering of the front end's levelised witness program (circuit.hpp) into the stream the witness kernel walks
// (witness.cu).  Host only: no device, no environment - the engine chooses the options (engine.cu) and uploads the result;
// zke_circuit_program_stats (capi_circuit.cpp) reports on the same lowering without a GPU.
#pragma once
#include "circuit.hpp"
#include <cstdint>
#include <vector>

namespace zke {

static const int WITNESS_THREADS = 512;

// Witness program resident in HBM (built once per circuit): a STREAM of fixed-size op records, one per thread and
// iteration.  The levelised program of the front-end is cut into iterations of WITNESS_THREADS ops (levels are padded
// with no-ops), so the kernel needs no level table and no LC pool indirection: iteration k, thread t executes
// ops[k * WITNESS_THREADS + t]; the LC terms of an iteration's ops are one contiguous block of `terms`, described by
// iter_hdr[k], which the CTA stages into shared memory one iteration ahead (cp.async) while it evaluates the current
// one.  Everything that does not depend on witness data is therefore prefetched; the only dependent memory round
// trip left in an iteration is the gather of the witness values themselves.
//   op record  : x = dst, y = code | nA << 8 | nB << 13 | nC << 18, z = operand (first term index / source variable /
//                aux offset), w = shift | nbits << 16 (OP_SHRAND)
//   term       : {variable, coefficient index}; blocks of an op are laid out [A | B | C]
static const uint32_t WOP_NOP = 15;

// coefficient words (lc_term.cuh) of an interned coefficient table: index | k << 16 | kind << 24
std::vector<uint32_t> coef_words(const std::vector<U256>& coefs);

struct LowerOptions {
    bool native_sha = true;      // one cooperative op per recorded Sha256compression instead of the gadget's own ops
    bool native_regex = true;    // one cooperative op per zk-regex instance seeds its state signals
    bool native_poseidon = true; // one cooperative op per recorded Poseidon instance instead of the gadget's own ops
    bool coop_fpmul = true;      // FpMul hints as cooperative ops (false: the sequential single-thread hint, a regular record)
    uint32_t cluster = 1;        // CTAs per email (1, 2, 4, 8): every level is padded to whole rounds of `cluster` iterations
};

struct WitnessStream {
    std::vector<uint32_t> ops;         // [n_iters][WITNESS_THREADS] records of 4 words
    std::vector<uint32_t> iter_hdr;    // [n_iters + 2 * cluster] headers of 4 words (the last 2 * cluster are sentinels): {first term
                                       // (even), term count (even), first cooperative op, their count | 1 << 31 on the iterations of a
                                       // level's last round (cluster > 1: barrier across the CTAs)}
    std::vector<uint32_t> terms;       // 2 words per term; an iteration's block is 16-byte aligned
    std::vector<uint32_t> aux;         // the circuit's aux table, then the tables of the cooperative ops
    std::vector<uint32_t> coop;        // cooperative ops of the iterations (executed by the whole CTA), two words each:
                                       // {offset into `aux`, 0}: native Sha256compression table ({n_desc, inputs[768],
                                       // desc[n_desc][2]}, circuit.hpp: ShaBlock); {1 << 30 | offset into `aux`, 0}: regex seed
                                       // (circuit.hpp: regex_flat image of one seed); {1 << 31 | offset into `aux`, dst}: FpMul hint;
                                       // {3 << 30 | offset into `aux`, 0}: native Poseidon (POSEIDON_AUX below) - the Poseidon ops of
                                       // an iteration are adjacent and run side by side, one warp each
    // native Poseidon in `aux`: per instance {t, r_p, offset of the width's constants, inputs[t - 1], slots[t + (8 + r_p) t 4]}
    // (slots: the signal of each lane's input copy, then per round and lane the signals of x^2, x^4, x^5 and the mix output;
    // 0 = the gadget created none), per width once, 8-word aligned: round constants [(8 + r_p) t] in standard form, then the
    // MDS matrix [t][t] times R (the coefficient form of lc_term.cuh: a Montgomery product with it gives the plain product)
    std::vector<uint32_t> iter_info;   // per iteration {first op's record word 1, live ops, terms} (diagnostics: ZKE_WITNESS_TRACE)
    std::vector<uint32_t> level_ops;   // per level: records that are not cooperative ops
    uint32_t n_iters = 0, n_levels = 0, cluster = 1;
};

WitnessStream lower_witness_program(const Circuit& c, const std::vector<uint32_t>& coef_word, const LowerOptions& opt);

}  // namespace zke
