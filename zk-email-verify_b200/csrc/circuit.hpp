// Circuit front-end: an R1CS + witness-program builder.
//
// The reference compiles `email-verifier.circom` with the circom compiler (un-vendored; CI pins v2.1.8 at
// /root/reference/.github/workflows/action.yml:29-33) into an .r1cs and a WASM witness calculator.  circom
// is not part of the reference tree, so this builder plays its role: templates (gadgets.cpp) call the
// builder the way circom templates declare signals and constraints, and the builder emits
//   * the R1CS (A, B, C as CSR over an interned coefficient table), and
//   * a levelised witness program: one op per signal, ops grouped by dependency depth so that a
//     device can evaluate a level in parallel and synchronise between levels.
//
// Semantics follow circom at optimisation level --O1 (the level the reference's docs recommend,
// /root/reference/docs/zk-email-docs/UsageGuide/README.md:60-66): every `<==` of a non-trivial
// expression produces a signal and a constraint; only `signal = signal` / `signal = constant`
// aliases are elided.  Linear constraints are stored as A = B = 0, C = expr (as circom does).
#pragma once
#include "ff_host.hpp"
#include <map>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace zke {

typedef uint32_t Var;
static const Var TEMP_BIT = 0x80000000u;  // builder-time tag of scratch slots (not part of the R1CS)

// Sparse linear combination over witness variables; variable 0 is the constant one.
struct LC {
    std::vector<std::pair<Var, Fr>> t;  // sorted by var, unique, non-zero coefficients

    LC() {}
    LC(Var v) { t.emplace_back(v, Fr::one()); }
    static LC var(Var v) { return LC(v); }
    static LC constant(const Fr& c) { LC r; if (!c.is_zero()) r.t.emplace_back(0, c); return r; }
    static LC constant_i(int64_t c) { return constant(Fr::from_i64(c)); }
    static LC term(Var v, const Fr& c) { LC r; if (!c.is_zero()) r.t.emplace_back(v, c); return r; }

    bool is_zero() const { return t.empty(); }
    bool is_const() const { return t.empty() || (t.size() == 1 && t[0].first == 0); }
    Fr const_value() const { return t.empty() ? Fr::zero() : t[0].second; }
    bool is_single_var(Var* v) const {
        if (t.size() == 1 && t[0].first != 0 && t[0].second == Fr::one()) { *v = t[0].first; return true; }
        return false;
    }
    LC operator+(const LC& o) const;
    LC operator-(const LC& o) const;
    LC operator*(const Fr& k) const;
    LC neg() const;
    LC& operator+=(const LC& o) { *this = *this + o; return *this; }
    LC& operator-=(const LC& o) { *this = *this - o; return *this; }
    // in-place "+= k * v" for accumulations that append increasing variables (fast path), falls back to merge
    void add_term(Var v, const Fr& k);
};
inline LC operator*(const Fr& k, const LC& a) { return a * k; }

enum OpCode : uint32_t {
    OP_LIN = 0,     // dst = lc[a]
    OP_QUAD = 1,    // dst = lc[a] * lc[b] + lc[c]
    OP_SHRAND = 2,  // dst = (val[a] >> b) & (2^c - 1)   (c == 0: no mask); a is a variable / scratch slot
    OP_INVZ = 3,    // dst = val[a] == 0 ? 0 : 1 / val[a]
    OP_FPMUL = 4,   // big-integer hint of FpMul: aux[a..] = {n, k, a_vars[k], b_vars[k], p_vars[k]};
                    // dst..dst+k-1 = q limbs, dst+k..dst+2k-1 = r limbs where a*b = q*p + r, 0 <= r < p
    OP_SHRLC = 5,   // dst = (lc[a] >> b) & (2^c - 1): OP_SHRAND fused with the OP_LIN that fed it through a scratch slot
                    // (finalize(); one dependency level less per bit decomposition of a sum - SHA-256 adders)
};
struct WOp {
    uint32_t code;
    Var dst;
    uint32_t a, b, c;
};

// One Sha256compression instance as the front-end built it (gadgets.cpp: sha256_compression): every signal the gadget
// creates is a bit of some 64-bit quantity of the compression (a sigma / Ch / Maj word, an AND of two rotations, one of
// the adder sums), so a device can produce all of them from ONE native compression instead of walking the gadget's
// ~320 dependency levels.  The witness program itself (Circuit::ops) is unchanged - the CPU oracle walks it - the
// record only lets the engine substitute the sub-program (witness_program.cpp).
struct ShaBlock {
    uint32_t var_begin = 0, var_end = 0;      // signals created by the gadget: [var_begin, var_end), one descriptor each
    uint32_t temp_begin = 0, temp_end = 0;    // scratch slots created by the gadget (absolute slot numbers after finalize)
    // 768 inputs: hin[256] (8 words, LSB first) then inp[512] (16 words, MSB first): a variable, or SHA_CONST0 / SHA_CONST1
    std::vector<uint32_t> inputs;
    std::vector<uint32_t> desc;               // 2 words per created signal: {variable, quantity << 8 | bit}
};
static const uint32_t SHA_CONST0 = 0xfffffffeu, SHA_CONST1 = 0xffffffffu;
// quantities: group * 64 + index (index = round / schedule step t, or the state word for SHA_Q_FS)
enum ShaQuantity : uint32_t {
    SHA_Q_S1MID = 0, SHA_Q_S1 = 1, SHA_Q_S0MID = 2, SHA_Q_S0 = 3, SHA_Q_WSUM = 4,                       // message schedule, t = 16..63
    SHA_Q_BS1MID = 5, SHA_Q_BS1 = 6, SHA_Q_CH = 7, SHA_Q_T1SUM = 8, SHA_Q_BS0MID = 9, SHA_Q_BS0 = 10,   // rounds, t = 0..63
    SHA_Q_MAJMID = 11, SHA_Q_MAJ = 12, SHA_Q_T2SUM = 13, SHA_Q_SUME = 14, SHA_Q_SUMA = 15,
    SHA_Q_FS = 16,                                                                                      // final sums, i = 0..7
    SHA_Q_GROUPS = 17
};

// One zk-regex instance in the zk-regex circuit shape (regex.cpp: regex_circuit): the state signals of position i only
// depend on the byte at i and the state signals of position i - 1 - a dependency chain as long as the message.  The set
// of live DFA states per position is a plain automaton run, so a device can produce every state SIGNAL of the instance at
// once ("seed" them) and the per-position gadgets (comparators, ANDs, ORs) of all positions then evaluate side by side.
// The witness program keeps all of its ops - the seeded signals are simply written twice with the same value, and the
// CPU oracle walks the program as it is (witness_program.cpp uses the record when it levelises the program).
struct RegexSeed {
    uint32_t n_states = 0;            // <= 255; more than 64 (mode 0) is the wide mode: a 256-bit live set
    std::vector<uint32_t> bytes;      // the variable holding message byte j (position j + 1 of the circuit; position 0 is the marker)
    std::vector<uint8_t> table;       // n_states x 256: destination of (source state, byte) or 0xff; byte 255 never fires
    uint64_t first_mask[4] = {1, 0, 0, 0};   // live states after the marker position (bit 0 = state 0, always live)
    std::vector<uint32_t> desc;       // 2 words per seeded signal: {variable, position << 8 | state}, position >= 1
    // mode 1 - the compact shape (regex.cpp: regex_circuit_compact): ONE state per position (the automaton of live-state
    // sets is deterministic, n_states <= 255, first_mask = the state after the marker), the chain runs through the `fire`
    // products: `group` gives the product that fires on (state, byte) (0xff: none, the next state is then 0), and a
    // descriptor {variable, position << 8 | product id} is 1 exactly when that product fires at that position.
    uint32_t mode = 0;
    std::vector<uint8_t> group;       // mode 1: n_states x 256
    bool wide() const { return mode == 0 && n_states > 64; }
};

void append_regex_seed(std::vector<uint32_t>& out, const RegexSeed& R);   // flat image (circuit.cpp)

// One Poseidon(t - 1) instance as the front end built it (poseidon.cpp: poseidon with a record): every signal the gadget
// creates is a lane of the permutation's state at some round - the copy of an input, x^2, x^4 or x^5 of the S-box, or the
// output of the mix - so a device can produce all of them from ONE native permutation instead of walking the gadget's
// ~4 dependency levels per round.  As for ShaBlock, the witness program keeps all of its ops (the CPU oracle walks them);
// the record only lets the engine substitute the sub-program (witness_program.cpp).
struct PoseidonBlock {
    uint32_t t = 0;                           // width: t - 1 inputs, state lane 0 starts at zero
    std::vector<uint32_t> inputs;             // t - 1 variables
    uint32_t var_begin = 0, var_end = 0;      // signals created by the gadget: [var_begin, var_end), one descriptor each
    uint32_t temp_begin = 0, temp_end = 0;    // scratch slots of its long mix sums (absolute slot numbers after finalize)
    std::vector<uint32_t> desc;               // 2 words per created signal: {variable, round << 16 | lane << 8 | kind}
};
enum PoseidonKind : uint32_t { POS_K_INPUT = 0, POS_K_X2 = 1, POS_K_X4 = 2, POS_K_X5 = 3, POS_K_MIX = 4 };
// (input copies carry round 0; x^k of round r is the S-box of the state after round r's constants; mix of round r is the
// state after round r)

struct SignalGroup {
    std::string name;
    uint32_t first;  // first witness index
    uint32_t count;
    int kind;        // 0 output, 1 public input, 2 private input
};

// Finalised, flat circuit description (what a device / an exporter consumes).
struct Circuit {
    std::string name;
    uint32_t n_vars = 0;       // witness length m (w[0] = 1)
    uint32_t n_temps = 0;      // scratch slots appended after the witness during evaluation
    uint32_t n_outputs = 0, n_pub_inputs = 0, n_prv_inputs = 0;
    uint32_t n_public() const { return n_outputs + n_pub_inputs; }   // "nPublic" of snarkjs
    uint32_t n_inputs() const { return n_pub_inputs + n_prv_inputs; }
    uint32_t n_constraints = 0;
    std::vector<SignalGroup> groups;

    std::vector<U256> coefs;   // interned coefficients, standard form; [0] = 1, [1] = r - 1 (i.e. -1)

    // R1CS rows in CSR form; entry = (var, coef index)
    std::vector<uint32_t> a_ptr, b_ptr, c_ptr;
    std::vector<uint32_t> a_var, a_coef, b_var, b_coef, c_var, c_coef;
    std::vector<uint16_t> scope_of_constraint;
    std::vector<std::string> scopes;

    // witness program, ops sorted by level; level_ptr has n_levels + 1 entries
    std::vector<WOp> ops;
    std::vector<uint32_t> level_ptr;
    std::vector<uint32_t> lc_ptr, lc_var, lc_coef;  // LC pool referenced by OP_LIN / OP_QUAD
    std::vector<uint32_t> aux;

    std::vector<ShaBlock> sha_blocks;   // Sha256compression instances eligible for native evaluation (may be empty)
    // flat image of sha_blocks: {n_blocks, then per block: var_begin, var_end, temp_begin, temp_end, n_desc, inputs[768],
    // desc[2 n_desc]} (built by finalize; ZKE_ARR_SHA_BLOCKS)
    std::vector<uint32_t> sha_flat;

    std::vector<RegexSeed> regex_seeds; // zk-regex instances whose state signals can be produced by an automaton run (may be empty)
    // flat image of regex_seeds: {n_seeds, then per seed: n_desc, n_bytes, n_states | wide << 30 | mode << 31, first_mask
    // lo, hi (wide: 8 words, the 256-bit mask from its low word up), bytes[n_bytes], table[n_states * 64] (4 bytes per word, little-endian), mode 1: group[n_states * 64], desc[2 n_desc]}
    // (built by finalize; ZKE_ARR_REGEX_SEEDS); the engine appends the same image to the program's aux table
    std::vector<uint32_t> regex_flat;

    std::vector<PoseidonBlock> poseidon_blocks;   // Poseidon instances eligible for native evaluation (may be empty)
    // flat image of poseidon_blocks: {n_blocks, then per block: t, var_begin, var_end, temp_begin, temp_end, n_desc,
    // inputs[t - 1], desc[2 n_desc]} (built by finalize; ZKE_ARR_POSEIDON_BLOCKS)
    std::vector<uint32_t> poseidon_flat;

    // Read from an iden3 `.r1cs` (r1cs.cpp): the constraint system alone.  The witness program above is empty, witnesses
    // come from elsewhere (circom's witness calculator); nLabels and the section-3 wire -> label map are kept so that the
    // file can be written back as it came (labels empty: the identity map, as for builder circuits).
    bool r1cs_only = false;
    uint64_t n_labels = 0;
    std::vector<uint64_t> labels;

    uint32_t n_levels() const { return level_ptr.empty() ? 0 : (uint32_t)level_ptr.size() - 1; }
    const SignalGroup* find_group(const std::string& n) const;
    uint32_t domain_log2() const;  // smallest k with 2^k >= n_constraints + n_public + 1
};

class Builder {
   public:
    explicit Builder(const std::string& name);

    // --- signal declaration (must precede any intermediate signal, mirrors circom's witness order:
    //     [1, outputs, public inputs, private inputs, intermediates], SURVEY A.8) ---
    std::vector<Var> declare_outputs(const std::string& name, uint32_t n);
    std::vector<Var> declare_inputs(const std::string& name, uint32_t n, bool is_public);

    // --- constraints / signals ---
    LC signal(const LC& e);                                   // `signal x <== e` for a linear e
    LC mul(const LC& a, const LC& b);                         // `signal x <== a*b`
    LC mul_add(const LC& a, const LC& b, const LC& c);        // `signal x <== a*b + c`
    void enforce_mul(const LC& a, const LC& b, const LC& c);  // a*b === c
    void enforce_eq(const LC& a, const LC& b);                // a === b (linear)
    void assign_output(Var out, const LC& e);                 // `out <== e` for a pre-declared output

    // --- hints (`<--` in circom): no constraint is added, the caller constrains the result ---
    Var fresh() { return new_var(); }
    Var source_of(const LC& e);                                // variable or scratch slot holding e
    Var hint_shrand(Var src, uint32_t shift, uint32_t nbits);  // (src >> shift) & (2^nbits - 1)
    Var hint_invz(Var src);
    Var hint_lin(const LC& e);                                 // a signal assigned (not constrained) to e
    Var hint_fpmul(uint32_t n, uint32_t k, const std::vector<Var>& a, const std::vector<Var>& b,
                   const std::vector<Var>& p);                 // returns base of q[k] ++ r[k]

    // scope tag recorded with every constraint (for "Assert Failed: <scope>" messages)
    void push_scope(const std::string& s);
    void pop_scope();

    bool materialize_linear = true;  // circom --O1 behaviour; false ~ --O2 (linear signals substituted)
    // 0 = zk-regex circuit shape (comparators per range, OR of transitions), 1 = compact shape (regex.cpp); the same
    // function of the input either way.  Default from ZKE_REGEX_STYLE; the named templates take it as a parameter.
    int regex_style = default_regex_style();
    static int default_regex_style();
    bool fuse_shrand = default_fuse_shrand();   // OP_SHRLC fusion in finalize() (ZKE_FUSED_SHRAND)
    static bool default_fuse_shrand();

    Circuit finalize();

    uint32_t num_vars() const { return next_var_; }
    uint32_t num_temps() const { return next_temp_; }
    void add_sha_block(ShaBlock&& blk) { c_.sha_blocks.push_back(std::move(blk)); }   // temp range as raw temp indices
    void add_regex_seed(RegexSeed&& sd) { c_.regex_seeds.push_back(std::move(sd)); }
    void add_poseidon_block(PoseidonBlock&& blk) { c_.poseidon_blocks.push_back(std::move(blk)); }   // temp range as raw temp indices
    uint32_t num_constraints() const { return (uint32_t)c_.scope_of_constraint.size(); }

   private:
    Var new_var();
    Var new_temp();
    uint32_t intern(const Fr& c);
    uint32_t add_prog_lc(const LC& e);
    void push_row(std::vector<uint32_t>& ptr, std::vector<uint32_t>& var, std::vector<uint32_t>& coef, const LC& e);
    void add_constraint(const LC& a, const LC& b, const LC& c);
    void add_op(uint32_t code, Var dst, uint32_t a, uint32_t b, uint32_t c);

    Circuit c_;
    uint32_t next_var_ = 1;
    uint32_t next_temp_ = 0;
    bool decl_closed_ = false;
    struct U256Hash {
        size_t operator()(const U256& x) const { return (size_t)(x.v[0] * 0x9E3779B97F4A7C15ull ^ x.v[1] * 31 ^ x.v[2] * 131 ^ x.v[3]); }
    };
    std::unordered_map<U256, uint32_t, U256Hash> coef_index_;
    std::vector<uint16_t> scope_stack_;
    std::map<std::string, uint16_t> scope_index_;
};

struct ScopeGuard {
    Builder& b;
    ScopeGuard(Builder& b_, const std::string& s) : b(b_) { b.push_scope(s); }
    ~ScopeGuard() { b.pop_scope(); }
};

}  // namespace zke
