// C ABI - circuit construction and introspection (host only).  See include/zkemail_b200.h.
#include "../../include/zkemail_b200.h"
#include "engine.hpp"
#include "gadgets.hpp"
#include "bigdiv.hpp"
#include "setup_host.hpp"
#include "witness_program.hpp"
#include <cstdio>
#include <cstring>

using namespace zke;
using namespace zke::gadgets;

namespace zke {
void set_err(char* err, size_t cap, const std::string& msg) {
    if (!err || cap == 0) return;
    size_t n = msg.size() < cap - 1 ? msg.size() : cap - 1;
    memcpy(err, msg.data(), n);
    err[n] = 0;
}
void random_bytes(void* out, size_t n) {
    FILE* f = fopen("/dev/urandom", "rb");
    if (!f) throw std::runtime_error("cannot open /dev/urandom");
    const bool got = fread(out, 1, n, f) == n;
    fclose(f);
    if (!got) throw std::runtime_error("short read from /dev/urandom");
}
void random_scalar(U256& out) {
    do {
        random_bytes(out.v, 32);
        out.v[3] &= 0x3FFFFFFFFFFFFFFFull;   // 254 bits, then rejection
    } while (u256_cmp(out, fr_params().p) >= 0);
}
}  // namespace zke

namespace {

LCVec inputs(Builder& b, const char* name, uint32_t n, bool pub = false) {
    std::vector<Var> v = b.declare_inputs(name, n, pub);
    LCVec o(n);
    for (uint32_t i = 0; i < n; ++i) o[i] = LC(v[i]);
    return o;
}
void outputs(Builder& b, const char* name, const LCVec& vals, const std::vector<Var>& outs) {
    (void)name;
    for (size_t i = 0; i < vals.size(); ++i) b.assign_output(outs[i], vals[i]);
}

// The `component main = X(params)` wrappers of /root/reference/packages/circuits/tests/test-circuits/*.circom
// (plus a few leaf templates) so that every template can be exercised on its own, as the reference's unit tests do.
Circuit build_named(const std::string& name, const std::vector<int64_t>& p) {
    auto need = [&](size_t n) { if (p.size() < n) throw std::runtime_error(name + ": expected " + std::to_string(n) + " template parameters"); };
    if (name == "EmailVerifier") {
        need(4);
        EmailVerifierParams ep;
        ep.max_headers_length = (uint32_t)p[0]; ep.max_body_length = (uint32_t)p[1]; ep.n = (uint32_t)p[2]; ep.k = (uint32_t)p[3];
        if (p.size() > 4) ep.ignore_body_hash_check = p[4] != 0;
        if (p.size() > 5) ep.enable_header_masking = p[5] != 0;
        if (p.size() > 6) ep.enable_body_masking = p[6] != 0;
        if (p.size() > 7) ep.remove_soft_line_breaks = p[7] != 0;
        if (p.size() > 8) ep.public_pubkey = p[8] != 0;
        if (p.size() > 9) ep.regex_style = (int)p[9];
        return build_email_verifier(ep);
    }
    if (name == "TwitterVerifier") {          // Proof-of-Twitter: EmailVerifier(H, Bd, n, k, 0) + body regex + packing + address
        need(4);
        EmailVerifierParams ep;
        ep.max_headers_length = (uint32_t)p[0]; ep.max_body_length = (uint32_t)p[1]; ep.n = (uint32_t)p[2]; ep.k = (uint32_t)p[3];
        ep.twitter = true;
        if (p.size() > 4) ep.regex_style = (int)p[4];
        return build_email_verifier(ep);
    }
    Builder b(name);
    ScopeGuard g(b, name);
    if (name == "Sha256Bytes") {              // test-circuits/sha-test.circom
        need(1);
        auto out = b.declare_outputs("out", 256);
        LCVec in = inputs(b, "paddedIn", (uint32_t)p[0]);
        LC len = inputs(b, "paddedInLength", 1)[0];
        outputs(b, "out", sha256_bytes(b, in, len), out);
    } else if (name == "Sha256BytesPartial") {
        need(1);
        auto out = b.declare_outputs("out", 256);
        LCVec in = inputs(b, "paddedIn", (uint32_t)p[0]);
        LC len = inputs(b, "paddedInLength", 1)[0];
        LCVec pre = inputs(b, "preHash", 32);
        outputs(b, "out", sha256_bytes_partial(b, in, len, pre), out);
    } else if (name == "RSAVerifier65537") {  // test-circuits/rsa-test.circom
        need(2);
        uint32_t n = (uint32_t)p[0], k = (uint32_t)p[1];
        LCVec msg = inputs(b, "message", k), sig = inputs(b, "signature", k), mod = inputs(b, "modulus", k);
        rsa_verifier65537(b, n, k, msg, sig, mod);
    } else if (name == "FpMul") {             // test-circuits/fp-mul-test.circom
        need(2);
        uint32_t n = (uint32_t)p[0], k = (uint32_t)p[1];
        auto out = b.declare_outputs("out", k);
        LCVec a = inputs(b, "a", k), bb = inputs(b, "b", k), pp = inputs(b, "p", k);
        outputs(b, "out", fp_mul(b, n, k, a, bb, pp), out);
    } else if (name == "Base64Lookup") {      // test-circuits/base64-test.circom
        auto out = b.declare_outputs("out", 1);
        LC in = inputs(b, "in", 1)[0];
        outputs(b, "out", {base64_lookup(b, in)}, out);
    } else if (name == "Base64Decode") {
        need(1);
        uint32_t bl = (uint32_t)p[0];
        auto out = b.declare_outputs("out", bl);
        LCVec in = inputs(b, "in", 4 * ((bl + 2) / 3));
        outputs(b, "out", base64_decode(b, bl, in), out);
    } else if (name == "PackBits") {          // test-circuits/pack-bits-test.circom
        need(2);
        uint32_t nb = (uint32_t)p[0], bpe = (uint32_t)p[1];
        auto out = b.declare_outputs("out", (nb + bpe - 1) / bpe);
        LCVec in = inputs(b, "in", nb);
        outputs(b, "out", pack_bits(b, in, bpe), out);
    } else if (name == "PackBytes") {         // utils/bytes.circom:28-60
        need(1);
        uint32_t n = (uint32_t)p[0];
        auto out = b.declare_outputs("out", (n + 30) / 31);
        LCVec in = inputs(b, "in", n);
        outputs(b, "out", pack_bytes(b, in), out);
    } else if (name == "PackRegexReveal") {   // utils/regex.circom:61-77
        need(2);
        uint32_t n = (uint32_t)p[0], r = (uint32_t)p[1];
        auto out = b.declare_outputs("out", (r + 30) / 31);
        LCVec in = inputs(b, "in", n);
        LC start = inputs(b, "startIndex", 1)[0];
        outputs(b, "out", pack_regex_reveal(b, in, start, r), out);
    } else if (name == "TwitterResetRegex") {
        need(1);
        uint32_t n = (uint32_t)p[0];
        auto out = b.declare_outputs("out", 1);
        auto rev = b.declare_outputs("reveal0", n);
        LCVec msg = inputs(b, "msg", n);
        if (p.size() > 1) b.regex_style = (int)p[1];
        LCVec r = twitter_reset_regex(b, msg);
        b.assign_output(out[0], r[0]);
        for (uint32_t i = 0; i < n; ++i) b.assign_output(rev[i], r[1 + i]);
    } else if (name == "SplitBytesToWords") { // test-circuits/split-bytes-to-words-test.circom
        need(3);
        auto out = b.declare_outputs("out", (uint32_t)p[2]);
        LCVec in = inputs(b, "in", (uint32_t)p[0]);
        outputs(b, "out", split_bytes_to_words(b, in, (uint32_t)p[1], (uint32_t)p[2]), out);
    } else if (name == "CheckSubstringMatch") {   // test-circuits/check-substring-match-test.circom
        need(1);
        auto out = b.declare_outputs("isMatch", 1);
        LCVec in = inputs(b, "in", (uint32_t)p[0]), sub = inputs(b, "substring", (uint32_t)p[0]);
        outputs(b, "isMatch", {check_substring_match(b, in, sub)}, out);
    } else if (name == "CountSubstringOccurrences") {   // test-circuits/count-substring-occurrences-test.circom
        need(2);
        auto out = b.declare_outputs("count", 1);
        LCVec in = inputs(b, "in", (uint32_t)p[0]), sub = inputs(b, "substring", (uint32_t)p[1]);
        outputs(b, "count", {count_substring_occurrences(b, in, sub)}, out);
    } else if (name == "RevealSubstring") {   // test-circuits/reveal-substring-test.circom
        need(3);
        auto out = b.declare_outputs("substring", (uint32_t)p[1]);
        LCVec in = inputs(b, "in", (uint32_t)p[0]);
        LC start = inputs(b, "substringStartIndex", 1)[0], len = inputs(b, "substringLength", 1)[0];
        outputs(b, "substring", reveal_substring(b, in, start, len, (uint32_t)p[1], p[2] != 0), out);
    } else if (name == "SelectSubArray") {
        need(2);
        auto out = b.declare_outputs("out", (uint32_t)p[1]);
        LCVec in = inputs(b, "in", (uint32_t)p[0]);
        LC start = inputs(b, "startIndex", 1)[0], len = inputs(b, "length", 1)[0];
        outputs(b, "out", select_sub_array(b, in, start, len, (uint32_t)p[1]), out);
    } else if (name == "CleanEmailAddress") { // test-circuits/clean-email-address-test.circom
        need(1);
        auto out = b.declare_outputs("isValid", 1);
        LCVec enc = inputs(b, "encoded", (uint32_t)p[0]), dec = inputs(b, "decoded", (uint32_t)p[0]);
        outputs(b, "isValid", {clean_email_address(b, enc, dec)}, out);
    } else if (name == "EmailNullifier") {    // helpers/email-nullifier.circom
        need(2);
        auto out = b.declare_outputs("out", 1);
        LCVec sig = inputs(b, "signature", (uint32_t)p[1]);
        outputs(b, "out", {email_nullifier(b, (uint32_t)p[0], sig)}, out);
    } else if (name == "ByteMask") {          // test-circuits/byte-mask-test.circom
        need(1);
        uint32_t n = (uint32_t)p[0];
        auto out = b.declare_outputs("out", n);
        LCVec in = inputs(b, "in", n), mask = inputs(b, "mask", n);
        outputs(b, "out", byte_mask(b, in, mask), out);
    } else if (name == "SelectRegexReveal") { // test-circuits/select-regex-reveal-test.circom
        need(2);
        uint32_t n = (uint32_t)p[0], r = (uint32_t)p[1];
        auto out = b.declare_outputs("out", r);
        LCVec in = inputs(b, "in", n);
        LC start = inputs(b, "startIndex", 1)[0];
        outputs(b, "out", select_regex_reveal(b, in, start, r), out);
    } else if (name == "BodyHashRegex") {
        need(1);
        uint32_t n = (uint32_t)p[0];
        auto out = b.declare_outputs("out", 1);
        auto rev = b.declare_outputs("reveal0", n);
        LCVec msg = inputs(b, "msg", n);
        if (p.size() > 1) b.regex_style = (int)p[1];
        LCVec r = body_hash_regex(b, msg);
        b.assign_output(out[0], r[0]);
        for (uint32_t i = 0; i < n; ++i) b.assign_output(rev[i], r[1 + i]);
    } else if (name == "PoseidonLarge") {
        need(2);
        auto out = b.declare_outputs("out", 1);
        LCVec in = inputs(b, "in", (uint32_t)p[1]);
        outputs(b, "out", {poseidon_large(b, (uint32_t)p[0], in)}, out);
    } else if (name == "Poseidon") {
        need(1);
        auto out = b.declare_outputs("out", 1);
        LCVec in = inputs(b, "inputs", (uint32_t)p[0]);
        outputs(b, "out", {poseidon(b, in)}, out);
    } else if (name == "PoseidonModular") {   // test-circuits/poseidon-modular-test.circom
        need(1);
        auto out = b.declare_outputs("out", 1);
        LCVec in = inputs(b, "in", (uint32_t)p[0]);
        outputs(b, "out", {poseidon_modular(b, in)}, out);
    } else if (name == "BinaryMerkleRoot") {
        need(1);
        if (p[0] < 1 || p[0] > 32) throw std::runtime_error("BinaryMerkleRoot: depth must be 1..32");
        auto out = b.declare_outputs("root", 1);
        LC leaf = inputs(b, "leaf", 1)[0], index = inputs(b, "index", 1)[0];
        LCVec sib = inputs(b, "siblings", (uint32_t)p[0]);
        outputs(b, "root", {binary_merkle_root(b, leaf, index, sib)}, out);
    } else if (name == "RemoveSoftLineBreaks") {   // test-circuits/remove-soft-line-breaks-test.circom
        need(1);
        auto out = b.declare_outputs("isValid", 1);
        LCVec enc = inputs(b, "encoded", (uint32_t)p[0]), dec = inputs(b, "decoded", (uint32_t)p[0]);
        outputs(b, "isValid", {remove_soft_line_breaks(b, enc, dec)}, out);
    } else if (name == "ItemAtIndex") {
        need(1);
        auto out = b.declare_outputs("out", 1);
        LCVec in = inputs(b, "in", (uint32_t)p[0]);
        LC idx = inputs(b, "index", 1)[0];
        outputs(b, "out", {item_at_index(b, in, idx)}, out);
    } else if (name == "VarShiftLeft") {
        need(2);
        auto out = b.declare_outputs("out", (uint32_t)p[1]);
        LCVec in = inputs(b, "in", (uint32_t)p[0]);
        LC sh = inputs(b, "shift", 1)[0];
        outputs(b, "out", var_shift_left(b, in, sh, (uint32_t)p[1]), out);
    } else if (name == "AssertZeroPadding") {
        need(1);
        LCVec in = inputs(b, "in", (uint32_t)p[0]);
        LC st = inputs(b, "startIndex", 1)[0];
        assert_zero_padding(b, in, st);
    } else if (name == "BigLessThan") {
        need(2);
        auto out = b.declare_outputs("out", 1);
        LCVec a = inputs(b, "a", (uint32_t)p[1]), bb = inputs(b, "b", (uint32_t)p[1]);
        outputs(b, "out", {big_less_than(b, (uint32_t)p[0], a, bb)}, out);
    } else if (name == "LessThan") {
        need(1);
        auto out = b.declare_outputs("out", 1);
        LCVec in = inputs(b, "in", 2);
        outputs(b, "out", {less_than(b, (uint32_t)p[0], in[0], in[1])}, out);
    } else if (name == "Num2Bits") {
        need(1);
        auto out = b.declare_outputs("out", (uint32_t)p[0]);
        LC in = inputs(b, "in", 1)[0];
        outputs(b, "out", num2bits(b, in, (uint32_t)p[0]), out);
    } else if (name == "Multiplier") {        // toy circuit for prover tests: out = a*b, public a
        auto out = b.declare_outputs("out", 1);
        LC a = inputs(b, "a", 1, true)[0];
        LC bb = inputs(b, "b", 1, false)[0];
        LC sq = b.mul(a, bb);
        LC cube = b.mul(sq, bb);
        outputs(b, "out", {cube + a}, out);
    } else {
        throw std::runtime_error("unknown template '" + name + "'");
    }
    return b.finalize();
}

}  // namespace

extern "C" {

zke_circuit* zke_circuit_build(const char* template_name, const int64_t* params, size_t n_params, char* err, size_t errcap) {
    try {
        std::vector<int64_t> p(params, params + n_params);
        zke_circuit* c = new zke_circuit();
        c->c = build_named(template_name ? template_name : "", p);
        return c;
    } catch (const std::exception& e) {
        set_err(err, errcap, e.what());
        return nullptr;
    }
}

zke_circuit* zke_circuit_build_regex(const char* const* parts, const uint8_t* is_public, size_t n_parts, uint32_t msg_len,
                                     char* err, size_t errcap) {
    try {
        if (!parts || !is_public || n_parts == 0) throw std::runtime_error("no regex parts given");
        if (msg_len == 0 || msg_len > (1u << 16)) throw std::runtime_error("msg_len out of range");
        std::vector<std::pair<std::string, bool>> pv;
        for (size_t i = 0; i < n_parts; ++i) {
            if (!parts[i]) throw std::runtime_error("null regex part");
            pv.emplace_back(parts[i], is_public[i] != 0);
        }
        Builder b("Regex");
        ScopeGuard g(b, "Regex");
        auto out = b.declare_outputs("out", 1);
        auto rev = b.declare_outputs("reveal0", msg_len);
        LCVec msg = inputs(b, "msg", msg_len);
        LCVec r = regex_match(b, "Regex", pv, msg);
        b.assign_output(out[0], r[0]);
        for (uint32_t i = 0; i < msg_len; ++i) b.assign_output(rev[i], r[1 + i]);
        zke_circuit* c = new zke_circuit();
        c->c = b.finalize();
        return c;
    } catch (const std::exception& e) {
        set_err(err, errcap, e.what());
        return nullptr;
    }
}

void zke_circuit_free(zke_circuit* c) { delete c; }

int zke_circuit_get_info(const zke_circuit* c, zke_circuit_info* o) {
    if (!c || !o) return -1;
    const Circuit& k = c->c;
    o->n_vars = k.n_vars; o->n_temps = k.n_temps;
    o->n_outputs = k.n_outputs; o->n_pub_inputs = k.n_pub_inputs; o->n_prv_inputs = k.n_prv_inputs;
    o->n_public = k.n_public(); o->n_constraints = k.n_constraints;
    o->n_levels = k.n_levels(); o->n_ops = (uint32_t)k.ops.size(); o->n_coefs = (uint32_t)k.coefs.size();
    o->domain_log2 = k.domain_log2(); o->n_groups = (uint32_t)k.groups.size();
    o->nnz_a = k.a_var.size(); o->nnz_b = k.b_var.size(); o->nnz_c = k.c_var.size();
    return 0;
}

int zke_circuit_group(const zke_circuit* c, uint32_t index, char* name, size_t namecap, uint32_t* first, uint32_t* count, int* kind) {
    if (!c || index >= c->c.groups.size()) return -1;
    const SignalGroup& g = c->c.groups[index];
    set_err(name, namecap, g.name);
    if (first) *first = g.first;
    if (count) *count = g.count;
    if (kind) *kind = g.kind;
    return 0;
}

int64_t zke_circuit_input_offset(const zke_circuit* c, const char* name, uint32_t* count) {
    if (!c || !name) return -1;
    const SignalGroup* g = c->c.find_group(name);
    if (!g || g->kind == 0) return -1;
    if (count) *count = g->count;
    return (int64_t)g->first - 1 - (int64_t)c->c.n_outputs;
}

const void* zke_circuit_array(const zke_circuit* c, int which, size_t* n) {
    if (!c) return nullptr;
    const Circuit& k = c->c;
    size_t dummy;
    if (!n) n = &dummy;
#define RET(vec) do { *n = (vec).size(); return (vec).data(); } while (0)
    switch (which) {
        case ZKE_ARR_COEFS: *n = k.coefs.size(); return k.coefs.data();
        case ZKE_ARR_A_PTR: RET(k.a_ptr); case ZKE_ARR_A_VAR: RET(k.a_var); case ZKE_ARR_A_COEF: RET(k.a_coef);
        case ZKE_ARR_B_PTR: RET(k.b_ptr); case ZKE_ARR_B_VAR: RET(k.b_var); case ZKE_ARR_B_COEF: RET(k.b_coef);
        case ZKE_ARR_C_PTR: RET(k.c_ptr); case ZKE_ARR_C_VAR: RET(k.c_var); case ZKE_ARR_C_COEF: RET(k.c_coef);
        case ZKE_ARR_OPS: *n = k.ops.size(); return k.ops.data();
        case ZKE_ARR_LEVEL_PTR: RET(k.level_ptr);
        case ZKE_ARR_LC_PTR: RET(k.lc_ptr); case ZKE_ARR_LC_VAR: RET(k.lc_var); case ZKE_ARR_LC_COEF: RET(k.lc_coef);
        case ZKE_ARR_AUX: RET(k.aux);
        case ZKE_ARR_SCOPE_OF_CONSTRAINT: RET(k.scope_of_constraint);
        case ZKE_ARR_SHA_BLOCKS: RET(k.sha_flat);
        case ZKE_ARR_REGEX_SEEDS: RET(k.regex_flat);
        case ZKE_ARR_POSEIDON_BLOCKS: RET(k.poseidon_flat);
        default: *n = 0; return nullptr;
    }
#undef RET
}

const char* zke_circuit_scope_name(const zke_circuit* c, uint32_t i) {
    if (!c || i >= c->c.scopes.size()) return nullptr;
    return c->c.scopes[i].c_str();
}

int zke_circuit_program_stats(const zke_circuit* c, int native_sha, int native_regex, int coop_fpmul, uint32_t cluster,
                              zke_program_stats* out, uint32_t* level_ops, size_t level_cap, char* err, size_t errcap) {
    const uint32_t flags = (native_sha ? ZKE_LOWER_NATIVE_SHA : 0u) | (native_regex ? ZKE_LOWER_NATIVE_REGEX : 0u) |
                           (coop_fpmul ? ZKE_LOWER_COOP_FPMUL : 0u) | ZKE_LOWER_NATIVE_POSEIDON;
    return zke_circuit_program_stats_ex(c, flags, cluster, out, level_ops, level_cap, err, errcap);
}

int zke_circuit_program_stats_ex(const zke_circuit* c, uint32_t flags, uint32_t cluster, zke_program_stats* out,
                                 uint32_t* level_ops, size_t level_cap, char* err, size_t errcap) {
    try {
        if (!c || !out) throw std::runtime_error("null argument");
        if (c->c.r1cs_only) throw std::runtime_error(R1CS_NO_PROGRAM);
        if (cluster != 1 && cluster != 2 && cluster != 4 && cluster != 8) throw std::runtime_error("cluster must be 1, 2, 4 or 8");
        if (flags & ~(uint32_t)ZKE_LOWER_ALL) throw std::runtime_error("unknown lowering flag");
        LowerOptions opt;
        opt.native_sha = (flags & ZKE_LOWER_NATIVE_SHA) != 0; opt.native_regex = (flags & ZKE_LOWER_NATIVE_REGEX) != 0;
        opt.coop_fpmul = (flags & ZKE_LOWER_COOP_FPMUL) != 0; opt.native_poseidon = (flags & ZKE_LOWER_NATIVE_POSEIDON) != 0;
        opt.cluster = cluster;
        const WitnessStream S = lower_witness_program(c->c, coef_words(c->c.coefs), opt);
        memset(out, 0, sizeof *out);
        out->n_levels = S.n_levels; out->n_iters = S.n_iters; out->cluster = S.cluster;
        for (uint32_t n : S.level_ops) out->n_ops_kept += n;
        for (uint32_t k = 0; k < S.n_iters; ++k) { out->n_coop_ops += S.iter_hdr[4 * k + 3] & 0x7fffffffu; out->n_terms += S.iter_info[3 * k + 2]; }
        uint64_t h = 0xcbf29ce484222325ull;    // FNV-1a
        auto eat = [&h](uint64_t v, int n_bytes) { for (int i = 0; i < n_bytes; ++i) { h ^= (v >> (8 * i)) & 0xff; h *= 0x100000001b3ull; } };
        for (const std::vector<uint32_t>* a : {&S.ops, &S.iter_hdr, &S.terms, &S.aux, &S.coop}) {
            eat(a->size(), 8);
            for (uint32_t w : *a) eat(w, 4);
        }
        out->digest = h;
        for (size_t l = 0; level_ops && l < S.level_ops.size() && l < level_cap; ++l) level_ops[l] = S.level_ops[l];
        return 0;
    } catch (const std::exception& e) {
        set_err(err, errcap, e.what());
        return -1;
    }
}

int zke_poseidon_hash(const uint8_t* inputs, size_t n, uint8_t* out) {
    if (!inputs || !out || n < 1 || n > 16) return -1;
    std::vector<Fr> in(n);
    for (size_t i = 0; i < n; ++i) {
        U256 x;
        memcpy(x.v, inputs + 32 * i, 32);
        if (u256_cmp(x, fr_params().p) >= 0) return -2;
        in[i] = Fr::from_u256(x);
    }
    const U256 h = gadgets::poseidon_hash(in).to_u256();
    memcpy(out, h.v, 32);
    return 0;
}

int zke_selftest_fpmul_hint(uint32_t n, uint32_t k, const uint8_t* a, const uint8_t* b, const uint8_t* p, uint8_t* q, uint8_t* r) {
    if (k > 32) return 1;
    return fpmul_hint_words(n, k, (const uint32_t*)a, (const uint32_t*)b, (const uint32_t*)p, (uint32_t*)q, (uint32_t*)r);
}

int zke_setup_toxic(uint64_t seed, uint8_t* out160) {
    if (!out160) return -1;
    Fr t[5];
    derive_toxic(seed, t);
    for (int i = 0; i < 5; ++i) { U256 x = t[i].to_u256(); memcpy(out160 + 32 * i, x.v, 32); }
    return 0;
}

const char* zke_version(void) { return "zkemail_b200 0.1 (sm_90a)"; }

}  // extern "C"
