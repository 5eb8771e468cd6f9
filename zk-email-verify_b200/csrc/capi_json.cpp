// C ABI - the JSON faces of the boundary: snarkjs-format vkey / proof / public signals, input JSON.
//   snarkjs.groth16.verify(vkey, publicSignals, proof)      -> zke_verify_json
//   snarkjs.groth16.fullProve(input, wasm, zkey)            -> zke_fullprove_json
//   snarkjs zkey export verificationkey                     -> zke_zkey_vkey_json
// JSON shapes follow /root/reference/packages/rust-verifier/tests/data/proof_of_twitter/{vkey,proof,public}.json and
// the CircuitInput type of /root/reference/packages/helpers/src/input-generators.ts:6-18.
#include "../../include/zkemail_b200.h"
#include "engine.hpp"
#include "ec_host.hpp"
#include "gadgets.hpp"
#include "aggregate_host.hpp"
#include <cstring>
#include <memory>
#include <random>

using namespace zke;

namespace {

struct JV {
    enum Type { NUL, BOOL, NUM, STR, ARR, OBJ } type = NUL;
    std::string s;    // STR / NUM text / BOOL
    std::vector<JV> arr;
    std::vector<std::pair<std::string, JV>> obj;
    const JV* get(const std::string& k) const {
        for (auto& kv : obj) if (kv.first == k) return &kv.second;
        return nullptr;
    }
};

struct JParser {
    const char* p;
    const char* end;
    explicit JParser(const char* s) : p(s), end(s + strlen(s)) {}
    void ws() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\r' || *p == '\t')) ++p; }
    [[noreturn]] void fail(const char* m) { throw std::runtime_error(std::string("JSON: ") + m); }
    JV parse() { ws(); JV v = value(); ws(); if (p != end) fail("trailing characters"); return v; }
    std::string str() {
        if (*p != '"') fail("expected string");
        ++p;
        std::string o;
        while (p < end && *p != '"') {
            if (*p == '\\') {
                ++p;
                if (p >= end) fail("bad escape");
                switch (*p) {
                    case 'n': o.push_back('\n'); break;
                    case 'r': o.push_back('\r'); break;
                    case 't': o.push_back('\t'); break;
                    case 'b': o.push_back('\b'); break;
                    case 'f': o.push_back('\f'); break;
                    case 'u': {
                        if (end - p < 5) fail("bad \\u escape");
                        unsigned cp = 0;
                        for (int i = 1; i <= 4; ++i) {
                            char c = p[i];
                            cp = cp * 16 + (c >= '0' && c <= '9' ? c - '0' : (c | 32) >= 'a' && (c | 32) <= 'f' ? (c | 32) - 'a' + 10 : 99);
                        }
                        p += 4;
                        if (cp < 0x80) o.push_back((char)cp);
                        else if (cp < 0x800) { o.push_back((char)(0xC0 | (cp >> 6))); o.push_back((char)(0x80 | (cp & 0x3F))); }
                        else { o.push_back((char)(0xE0 | (cp >> 12))); o.push_back((char)(0x80 | ((cp >> 6) & 0x3F))); o.push_back((char)(0x80 | (cp & 0x3F))); }
                        break;
                    }
                    default: o.push_back(*p); break;
                }
                ++p;
            } else o.push_back(*p++);
        }
        if (p >= end) fail("unterminated string");
        ++p;
        return o;
    }
    JV value() {
        ws();
        if (p >= end) fail("unexpected end");
        JV v;
        if (*p == '{') {
            v.type = JV::OBJ; ++p; ws();
            if (*p == '}') { ++p; return v; }
            for (;;) {
                ws();
                std::string k = str();
                ws();
                if (*p != ':') fail("expected ':'");
                ++p;
                v.obj.emplace_back(k, value());
                ws();
                if (*p == ',') { ++p; continue; }
                if (*p == '}') { ++p; break; }
                fail("expected ',' or '}'");
            }
        } else if (*p == '[') {
            v.type = JV::ARR; ++p; ws();
            if (*p == ']') { ++p; return v; }
            for (;;) {
                v.arr.push_back(value());
                ws();
                if (*p == ',') { ++p; continue; }
                if (*p == ']') { ++p; break; }
                fail("expected ',' or ']'");
            }
        } else if (*p == '"') {
            v.type = JV::STR; v.s = str();
        } else if (!strncmp(p, "true", 4)) { v.type = JV::BOOL; v.s = "true"; p += 4; }
        else if (!strncmp(p, "false", 5)) { v.type = JV::BOOL; v.s = "false"; p += 5; }
        else if (!strncmp(p, "null", 4)) { v.type = JV::NUL; p += 4; }
        else {
            v.type = JV::NUM;
            const char* b = p;
            while (p < end && (strchr("+-0123456789.eE", *p))) ++p;
            if (b == p) fail("unexpected character");
            v.s.assign(b, p);
        }
        return v;
    }
};

U256 dec_of(const JV& v) {
    if (v.type != JV::STR && v.type != JV::NUM) throw std::runtime_error("expected a decimal string");
    return u256_from_dec(v.s);
}
Fq fq_of(const JV& v) {
    U256 x = dec_of(v);
    if (u256_cmp(x, fq_params().p) >= 0) throw std::runtime_error("coordinate not reduced");
    return Fq::from_u256(x);
}
G1AffineH g1_of(const JV& v) {
    if (v.type != JV::ARR || v.arr.size() < 2) throw std::runtime_error("bad G1 point");
    if (v.arr.size() >= 3 && dec_of(v.arr[2]).is_zero()) return G1AffineH::inf();
    return G1AffineH{fq_of(v.arr[0]), fq_of(v.arr[1])};
}
G2AffineH g2_of(const JV& v) {
    if (v.type != JV::ARR || v.arr.size() < 2 || v.arr[0].arr.size() != 2 || v.arr[1].arr.size() != 2) throw std::runtime_error("bad G2 point");
    if (v.arr.size() >= 3 && v.arr[2].arr.size() == 2 && dec_of(v.arr[2].arr[0]).is_zero() && dec_of(v.arr[2].arr[1]).is_zero())
        return G2AffineH::inf();
    // pi_b[0][0] -> x.c0, pi_b[0][1] -> x.c1 (/root/reference/packages/rust-verifier/src/verifier_utils.rs:73-83)
    return G2AffineH{Fq2{fq_of(v.arr[0].arr[0]), fq_of(v.arr[0].arr[1])}, Fq2{fq_of(v.arr[1].arr[0]), fq_of(v.arr[1].arr[1])}};
}
const JV& need(const JV& o, const char* k) {
    const JV* v = o.get(k);
    if (!v) throw std::runtime_error(std::string("missing key '") + k + "'");
    return *v;
}

std::string dec(const Fq& x) { return u256_to_dec(x.to_u256()); }
std::string g1_json(const G1AffineH& p) {
    if (p.is_inf()) return "[\"0\",\"1\",\"0\"]";
    return "[\"" + dec(p.x) + "\",\"" + dec(p.y) + "\",\"1\"]";
}
std::string g2_json(const G2AffineH& p) {
    if (p.is_inf()) return "[[\"0\",\"0\"],[\"1\",\"0\"],[\"0\",\"0\"]]";
    return "[[\"" + dec(p.x.c0) + "\",\"" + dec(p.x.c1) + "\"],[\"" + dec(p.y.c0) + "\",\"" + dec(p.y.c1) + "\"],[\"1\",\"0\"]]";
}
Fq fq_le(const uint8_t* b) { U256 x; memcpy(x.v, b, 32); return Fq::from_u256(x); }

int copy_out(const std::string& s, char* out, size_t* len) {
    if (!len) return -1;
    size_t cap = *len;
    *len = s.size() + 1;
    if (!out || cap < s.size() + 1) return -2;
    memcpy(out, s.c_str(), s.size() + 1);
    return 0;
}

void flatten_values(const JV& v, std::vector<U256>& out) {
    if (v.type == JV::ARR) { for (auto& e : v.arr) flatten_values(e, out); return; }
    if (v.type != JV::STR && v.type != JV::NUM) throw std::runtime_error("input values must be decimal strings or numbers");
    // snarkjs reduces inputs modulo the field; negative numbers are accepted as p - |x|
    std::string t = v.s;
    bool neg = !t.empty() && t[0] == '-';
    if (neg) t = t.substr(1);
    U256 x = u256_from_dec(t);
    while (u256_cmp(x, fr_params().p) >= 0) u256_sub(x, x, fr_params().p);
    if (neg && !x.is_zero()) u256_sub(x, fr_params().p, x);
    out.push_back(x);
}

// ---- email app spec (zke_circuit_build_app) ----
void only_keys(const JV& o, const std::string& field, std::initializer_list<const char*> keys) {
    if (o.type != JV::OBJ) throw std::runtime_error(field + ": expected an object");
    for (auto& kv : o.obj) {
        bool known = false;
        for (const char* k : keys) known = known || kv.first == k;
        if (!known) throw std::runtime_error(field + ": unknown key '" + kv.first + "'");
    }
}
bool bool_of(const JV& o, const char* key, bool dflt, const std::string& field) {
    const JV* v = o.get(key);
    if (!v) return dflt;
    if (v->type == JV::BOOL) return v->s == "true";
    if (v->type == JV::NUM && (v->s == "0" || v->s == "1")) return v->s == "1";
    throw std::runtime_error(field + key + ": expected true or false");
}
uint32_t uint_of(const JV& v, const std::string& field) {
    if (v.type != JV::NUM || v.s.empty() || v.s.size() > 9 || v.s.find_first_not_of("0123456789") != std::string::npos)
        throw std::runtime_error(field + ": expected a non-negative integer");
    return (uint32_t)std::stoul(v.s);
}
std::string str_of(const JV& o, const char* key, const std::string& field) {
    const JV* v = o.get(key);
    if (!v) throw std::runtime_error(field + key + ": missing");
    if (v->type != JV::STR) throw std::runtime_error(field + key + ": expected a string");
    return v->s;
}
const JV* array_of(const JV& o, const char* key) {
    const JV* v = o.get(key);
    if (v && v->type != JV::ARR) throw std::runtime_error(std::string(key) + ": expected an array");
    return v;
}

// a packed external input is ceil(maxLength / 31) public inputs, each a row of the verifier's IC: 64 KiB is 2,115 of them
const uint32_t MAX_EXTERNAL_BYTES = 1u << 16;

gadgets::AppSpec app_spec_of(const JV& s) {
    only_keys(s, "spec", {"maxHeadersLength", "maxBodyLength", "n", "k", "ignoreBodyHashCheck", "enableHeaderMasking",
                          "enableBodyMasking", "removeSoftLineBreaks", "publicPubkey", "regexStyle", "exposeHeaderHash",
                          "regexes", "externalInputs", "emailNullifier", "shaPrecomputeSelector", "keyRegistryDepth",
                          "keyDomain"});
    gadgets::AppSpec a;
    gadgets::EmailVerifierParams& ev = a.ev;
    if (const JV* v = s.get("maxHeadersLength")) ev.max_headers_length = uint_of(*v, "maxHeadersLength");
    if (const JV* v = s.get("maxBodyLength")) ev.max_body_length = uint_of(*v, "maxBodyLength");
    if (const JV* v = s.get("n")) ev.n = uint_of(*v, "n");
    if (const JV* v = s.get("k")) ev.k = uint_of(*v, "k");
    if (ev.max_headers_length > (1u << 20) || ev.max_body_length > (1u << 20)) throw std::runtime_error("maxHeadersLength / maxBodyLength: at most 2^20");
    if (ev.k > 64) throw std::runtime_error("k: at most 64");
    ev.ignore_body_hash_check = bool_of(s, "ignoreBodyHashCheck", false, "");
    ev.enable_header_masking = bool_of(s, "enableHeaderMasking", false, "");
    ev.enable_body_masking = bool_of(s, "enableBodyMasking", false, "");
    ev.remove_soft_line_breaks = bool_of(s, "removeSoftLineBreaks", false, "");
    ev.public_pubkey = bool_of(s, "publicPubkey", false, "");
    if (const JV* v = s.get("regexStyle")) {
        const uint32_t st = uint_of(*v, "regexStyle");
        if (st > 1) throw std::runtime_error("regexStyle: 0 (zk-regex shape) or 1 (compact shape)");
        ev.regex_style = (int)st;
    }
    if (const JV* v = s.get("shaPrecomputeSelector"))   // input generation only (generate_app_inputs)
        if (v->type != JV::STR && v->type != JV::NUL) throw std::runtime_error("shaPrecomputeSelector: expected a string");
    a.expose_header_hash = bool_of(s, "exposeHeaderHash", true, "");
    a.email_nullifier = bool_of(s, "emailNullifier", false, "");
    if (const JV* v = s.get("keyRegistryDepth")) {
        a.key_registry_depth = uint_of(*v, "keyRegistryDepth");
        if (a.key_registry_depth > 32) throw std::runtime_error("keyRegistryDepth: at most 32, not " + v->s);
    }
    if (s.get("keyDomain")) {
        a.key_domain = str_of(s, "keyDomain", "");
        if (a.key_domain.empty()) throw std::runtime_error("keyDomain: empty name");
    }
    if (const JV* rs = array_of(s, "regexes")) {
        for (size_t r = 0; r < rs->arr.size(); ++r) {
            const JV& e = rs->arr[r];
            const std::string f = "regexes[" + std::to_string(r) + "].";
            only_keys(e, "regexes[" + std::to_string(r) + "]", {"name", "location", "parts"});
            gadgets::AppRegex rx;
            rx.name = str_of(e, "name", f);
            const std::string loc = str_of(e, "location", f);
            if (loc != "header" && loc != "body") throw std::runtime_error(f + "location: '" + loc + "' is neither \"header\" nor \"body\"");
            rx.body = loc == "body";
            const JV* parts = e.get("parts");
            if (!parts || parts->type != JV::ARR) throw std::runtime_error(f + "parts: expected an array");
            for (size_t i = 0; i < parts->arr.size(); ++i) {
                const JV& pt = parts->arr[i];
                const std::string pf = f + "parts[" + std::to_string(i) + "]";
                only_keys(pt, pf, {"regexDef", "isPublic", "maxLength", "reveal", "salt"});
                gadgets::AppRegexPart part;
                part.regex = str_of(pt, "regexDef", pf + ".");
                part.is_public = bool_of(pt, "isPublic", false, pf + ".");
                if (const JV* ml = pt.get("maxLength")) part.max_length = uint_of(*ml, pf + ".maxLength");
                if (pt.get("reveal")) {
                    const std::string rv = str_of(pt, "reveal", pf + ".");
                    if (rv == "bytes") part.reveal = gadgets::REVEAL_BYTES;
                    else if (rv == "hash") part.reveal = gadgets::REVEAL_HASH;
                    else if (rv == "commit") part.reveal = gadgets::REVEAL_COMMIT;
                    else throw std::runtime_error(pf + ".reveal: '" + rv + "' is none of \"bytes\", \"hash\", \"commit\"");
                    part.reveal_given = true;
                }
                if (pt.get("salt")) {
                    part.salt = str_of(pt, "salt", pf + ".");
                    if (part.salt.empty()) throw std::runtime_error(pf + ".salt: empty name");
                }
                rx.parts.push_back(part);
            }
            a.regexes.push_back(rx);
        }
    }
    if (const JV* es = array_of(s, "externalInputs")) {
        for (size_t i = 0; i < es->arr.size(); ++i) {
            const std::string f = "externalInputs[" + std::to_string(i) + "]";
            only_keys(es->arr[i], f, {"name", "maxLength", "isPublic"});
            gadgets::AppExternalInput ei;
            ei.name = str_of(es->arr[i], "name", f + ".");
            ei.is_public = bool_of(es->arr[i], "isPublic", true, f + ".");
            if (const JV* ml = es->arr[i].get("maxLength")) {
                ei.max_length = uint_of(*ml, f + ".maxLength");
                if (ei.max_length == 0) throw std::runtime_error(f + ".maxLength: must be positive (leave it out for one field element)");
                if (ei.max_length > MAX_EXTERNAL_BYTES)
                    throw std::runtime_error(f + ".maxLength: at most " + std::to_string(MAX_EXTERNAL_BYTES) + " bytes");
            }
            a.external_inputs.push_back(ei);
        }
    }
    return a;
}

}  // namespace

VerifyingKey zke::vkey_from_json(const char* json) {
    JV vk = JParser(json).parse();
    const JV* prot = vk.get("protocol");
    if (prot && prot->s != "groth16") throw std::runtime_error("vkey protocol is not groth16");
    VerifyingKey k;
    k.alpha1 = g1_of(need(vk, "vk_alpha_1"));
    k.beta2 = g2_of(need(vk, "vk_beta_2"));
    k.gamma2 = g2_of(need(vk, "vk_gamma_2"));
    k.delta2 = g2_of(need(vk, "vk_delta_2"));
    for (auto& p : need(vk, "IC").arr) k.ic.push_back(g1_of(p));
    if (k.ic.empty()) throw std::runtime_error("vkey has no IC");
    return k;
}

agg::AggVk zke::agg::agg_vk_from_json(const char* json) {
    JV o = JParser(json).parse();
    const JV* prot = o.get("protocol");
    if (!prot || prot->s != "snarkpack") throw std::runtime_error("aggregation key protocol is not snarkpack");
    AggVk k;
    k.g = g1_of(need(o, "g")); k.g_a = g1_of(need(o, "g_a")); k.g_b = g1_of(need(o, "g_b"));
    k.h = g2_of(need(o, "h")); k.h_a = g2_of(need(o, "h_a")); k.h_b = g2_of(need(o, "h_b"));
    return k;
}

std::string zke::agg::agg_vk_to_json(const AggVk& k) {
    return "{\"protocol\":\"snarkpack\",\"curve\":\"bn128\",\"g\":" + g1_json(k.g) + ",\"h\":" + g2_json(k.h) +
           ",\"g_a\":" + g1_json(k.g_a) + ",\"g_b\":" + g1_json(k.g_b) + ",\"h_a\":" + g2_json(k.h_a) + ",\"h_b\":" + g2_json(k.h_b) + "}";
}

extern "C" {

int zke_verify_json(const char* vkey_json, const char* public_json, const char* proof_json, char* err, size_t errcap) {
    try {
        if (!vkey_json || !public_json || !proof_json) throw std::runtime_error("null argument");
        JV vk = JParser(vkey_json).parse(), pub = JParser(public_json).parse(), pr = JParser(proof_json).parse();
        const JV* prot = vk.get("protocol");
        if (prot && prot->s != "groth16") throw std::runtime_error("vkey protocol is not groth16");
        const JV* pprot = pr.get("protocol");
        if (pprot && pprot->s != "groth16") throw std::runtime_error("proof protocol is not groth16");
        VerifyingKey k;
        k.alpha1 = g1_of(need(vk, "vk_alpha_1"));
        k.beta2 = g2_of(need(vk, "vk_beta_2"));
        k.gamma2 = g2_of(need(vk, "vk_gamma_2"));
        k.delta2 = g2_of(need(vk, "vk_delta_2"));
        for (auto& p : need(vk, "IC").arr) k.ic.push_back(g1_of(p));
        Proof proof;
        proof.a = g1_of(need(pr, "pi_a"));
        proof.b = g2_of(need(pr, "pi_b"));
        proof.c = g1_of(need(pr, "pi_c"));
        std::vector<U256> publics;
        if (pub.type != JV::ARR) throw std::runtime_error("public signals must be an array");
        for (auto& s : pub.arr) publics.push_back(dec_of(s));
        return groth16_verify(k, publics, proof) ? 1 : 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

/* n proofs under one verification key: one randomised product of pairings (pairing_host.cpp: groth16_verify_batch); if it
 * fails the proofs are checked one by one so that ok[i] names the offenders.  Returns the number of valid proofs. */
int zke_verify_batch_json(const char* vkey_json, const char* publics_json, const char* proofs_json, const uint8_t* rand16,
                          uint8_t* ok, char* err, size_t errcap) {
    try {
        if (!vkey_json || !publics_json || !proofs_json) throw std::runtime_error("null argument");
        JV vk = JParser(vkey_json).parse(), pubs = JParser(publics_json).parse(), prs = JParser(proofs_json).parse();
        const JV* prot = vk.get("protocol");
        if (prot && prot->s != "groth16") throw std::runtime_error("vkey protocol is not groth16");
        if (pubs.type != JV::ARR || prs.type != JV::ARR || pubs.arr.size() != prs.arr.size())
            throw std::runtime_error("public signals and proofs must be arrays of the same length");
        VerifyingKey k;
        k.alpha1 = g1_of(need(vk, "vk_alpha_1"));
        k.beta2 = g2_of(need(vk, "vk_beta_2"));
        k.gamma2 = g2_of(need(vk, "vk_gamma_2"));
        k.delta2 = g2_of(need(vk, "vk_delta_2"));
        for (auto& p : need(vk, "IC").arr) k.ic.push_back(g1_of(p));
        if (k.ic.empty()) throw std::runtime_error("vkey has no IC");
        const size_t n = prs.arr.size();
        std::vector<Proof> proofs(n);
        std::vector<std::vector<U256>> publics(n);
        std::vector<U256> rnd(n);
        std::random_device rd;
        for (size_t i = 0; i < n; ++i) {
            const JV& pr = prs.arr[i];
            const JV* pprot = pr.get("protocol");
            if (pprot && pprot->s != "groth16") throw std::runtime_error("proof protocol is not groth16");
            proofs[i].a = g1_of(need(pr, "pi_a"));
            proofs[i].b = g2_of(need(pr, "pi_b"));
            proofs[i].c = g1_of(need(pr, "pi_c"));
            if (pubs.arr[i].type != JV::ARR) throw std::runtime_error("public signals must be an array per proof");
            for (auto& s : pubs.arr[i].arr) publics[i].push_back(dec_of(s));
            U256 r = {{0, 0, 0, 0}};
            if (rand16) memcpy(r.v, rand16 + 16 * i, 16);
            else { r.v[0] = ((uint64_t)rd() << 32) | rd(); r.v[1] = ((uint64_t)rd() << 32) | rd(); }
            if (r.is_zero()) r.v[0] = 1;
            rnd[i] = r;
        }
        int valid = 0;
        if (groth16_verify_batch(k, publics, proofs, rnd)) {
            for (size_t i = 0; i < n; ++i) if (ok) ok[i] = 1;
            valid = (int)n;
        } else {
            for (size_t i = 0; i < n; ++i) {
                const bool good = groth16_verify(k, publics[i], proofs[i]);
                if (ok) ok[i] = good ? 1 : 0;
                valid += good ? 1 : 0;
            }
        }
        return valid;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

/* e(alpha_1, beta_2) in snarkjs' vk_alphabeta_12 layout; points and result in standard form, little-endian */
int zke_pairing_alphabeta(const uint8_t* alpha64, const uint8_t* beta128, uint8_t* out384) {
    try {
        if (!alpha64 || !beta128 || !out384) return -1;
        for (int i = 0; i < 6; ++i) {
            U256 v;
            memcpy(v.v, (i < 2 ? alpha64 : beta128 - 64) + 32 * i, 32);
            if (u256_cmp(v, fq_params().p) >= 0) return -1;
        }
        G1AffineH a{fq_le(alpha64), fq_le(alpha64 + 32)};
        G2AffineH b{Fq2{fq_le(beta128), fq_le(beta128 + 32)}, Fq2{fq_le(beta128 + 64), fq_le(beta128 + 96)}};
        if (!g1_on_curve(a) || !g2_on_curve(b) || !g2_in_subgroup(b)) return -1;
        U256 ab[12];
        pairing_alphabeta(a, b, ab);
        for (int i = 0; i < 12; ++i) memcpy(out384 + 32 * i, ab[i].v, 32);
        return 0;
    } catch (const std::exception&) { return -1; }
}

/* proofs as produced by zke_prove: 8 x 32 bytes; publics: n_public x 32 bytes -> snarkjs proof.json / public.json */
int zke_proof_to_json(const uint8_t* proof256, const uint8_t* publics, uint32_t n_public, char* proof_json, size_t* proof_len,
                      char* public_json, size_t* public_len) {
    try {
        G1AffineH a{fq_le(proof256), fq_le(proof256 + 32)}, c{fq_le(proof256 + 192), fq_le(proof256 + 224)};
        G2AffineH b{Fq2{fq_le(proof256 + 64), fq_le(proof256 + 96)}, Fq2{fq_le(proof256 + 128), fq_le(proof256 + 160)}};
        std::string pj = "{\"pi_a\":" + g1_json(a) + ",\"pi_b\":" + g2_json(b) + ",\"pi_c\":" + g1_json(c) +
                         ",\"protocol\":\"groth16\",\"curve\":\"bn128\"}";
        std::string sj = "[";
        for (uint32_t i = 0; i < n_public; ++i) {
            U256 x; memcpy(x.v, publics + 32 * i, 32);
            sj += (i ? ",\"" : "\"") + u256_to_dec(x) + "\"";
        }
        sj += "]";
        int r1 = copy_out(pj, proof_json, proof_len), r2 = copy_out(sj, public_json, public_len);
        return r1 ? r1 : r2;
    } catch (const std::exception&) { return -1; }
}

int zke_zkey_vkey_json(const zke_zkey* z, char* out, size_t* len) {
    try {
        if (!z) return -1;
        uint32_t n_public = 0;
        zke_zkey_info(z, nullptr, &n_public, nullptr);
        auto g1sec = [&](int sec, size_t n) {
            std::vector<uint8_t> buf(64 * n);
            if (zke_zkey_section(z, sec, buf.data(), buf.size()) < 0) throw std::runtime_error("section read failed");
            std::vector<G1AffineH> pts(n);
            for (size_t i = 0; i < n; ++i) pts[i] = G1AffineH{fq_le(&buf[64 * i]), fq_le(&buf[64 * i + 32])};
            return pts;
        };
        auto g2sec = [&](int sec) {
            uint8_t buf[128];
            if (zke_zkey_section(z, sec, buf, sizeof buf) < 0) throw std::runtime_error("section read failed");
            return G2AffineH{Fq2{fq_le(buf), fq_le(buf + 32)}, Fq2{fq_le(buf + 64), fq_le(buf + 96)}};
        };
        std::string s = "{\"protocol\":\"groth16\",\"curve\":\"bn128\",\"nPublic\":" + std::to_string(n_public);
        s += ",\"vk_alpha_1\":" + g1_json(g1sec(ZKE_SEC_ALPHA1, 1)[0]);
        s += ",\"vk_beta_2\":" + g2_json(g2sec(ZKE_SEC_BETA2));
        s += ",\"vk_gamma_2\":" + g2_json(g2sec(ZKE_SEC_GAMMA2));
        s += ",\"vk_delta_2\":" + g2_json(g2sec(ZKE_SEC_DELTA2));
        {
            U256 ab[12];
            pairing_alphabeta(g1sec(ZKE_SEC_ALPHA1, 1)[0], g2sec(ZKE_SEC_BETA2), ab);
            s += ",\"vk_alphabeta_12\":[";
            for (int i = 0; i < 2; ++i) {
                s += i ? ",[" : "[";
                for (int j = 0; j < 3; ++j)
                    s += std::string(j ? "," : "") + "[\"" + u256_to_dec(ab[(i * 3 + j) * 2]) + "\",\"" + u256_to_dec(ab[(i * 3 + j) * 2 + 1]) + "\"]";
                s += "]";
            }
            s += "]";
        }
        s += ",\"IC\":[";
        auto ic = g1sec(ZKE_SEC_IC, n_public + 1);
        for (size_t i = 0; i < ic.size(); ++i) s += (i ? "," : "") + g1_json(ic[i]);
        s += "]}";
        return copy_out(s, out, len);
    } catch (const std::exception&) { return -1; }
}

zke_circuit* zke_circuit_build_app(const char* spec_json, char* err, size_t errcap) {
    try {
        if (!spec_json) throw std::runtime_error("null spec");
        const gadgets::AppSpec spec = app_spec_of(JParser(spec_json).parse());
        zke_circuit* c = new zke_circuit();
        try { c->c = gadgets::build_email_app(spec); } catch (...) { delete c; throw; }
        return c;
    } catch (const std::exception& e) {
        set_err(err, errcap, e.what());
        return nullptr;
    }
}

/* snarkjs input JSON -> packed [n_inputs][32] vector in witness order.  Mirrors circom_runtime's checks:
 * unknown signal, wrong number of values, missing signal. */
int zke_pack_inputs_json(const zke_circuit* c, const char* input_json, uint8_t* out, size_t cap, char* err, size_t errcap) {
    try {
        if (!c || !input_json || !out) throw std::runtime_error("null argument");
        const Circuit& k = c->c;
        if (k.r1cs_only) throw std::runtime_error(R1CS_NO_PROGRAM);
        const size_t n_in = k.n_inputs();
        if (cap < 32 * n_in) throw std::runtime_error("output buffer too small");
        JV in = JParser(input_json).parse();
        if (in.type != JV::OBJ) throw std::runtime_error("input must be a JSON object");
        std::vector<uint8_t> seen(k.groups.size(), 0);
        for (auto& kv : in.obj) {
            const SignalGroup* g = k.find_group(kv.first);
            if (!g || g->kind == 0) throw std::runtime_error("Signal not found: " + kv.first);
            std::vector<U256> vals;
            flatten_values(kv.second, vals);
            if (vals.size() != g->count)
                throw std::runtime_error(std::string(vals.size() > g->count ? "Too many" : "Not enough") + " values for input signal " + kv.first);
            for (size_t i = 0; i < vals.size(); ++i) memcpy(out + 32 * (g->first - 1 - k.n_outputs + i), vals[i].v, 32);
            seen[g - k.groups.data()] = 1;
        }
        for (size_t i = 0; i < k.groups.size(); ++i)
            if (k.groups[i].kind != 0 && !seen[i]) throw std::runtime_error("Not all inputs have been set. Missing: " + k.groups[i].name);
        return 0;
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

int zke_fullprove_json(zke_ctx* x, const zke_circuit* c, const char* input_json, char* proof_json, size_t* proof_len,
                       char* public_json, size_t* public_len, char* err, size_t errcap) {
    try {
        if (!x || !c) throw std::runtime_error("null argument");
        const Circuit& k = c->c;
        if (k.r1cs_only) throw std::runtime_error(R1CS_NO_PROGRAM);
        std::vector<uint8_t> packed(32 * (size_t)std::max(1u, k.n_inputs()));
        int rc = zke_pack_inputs_json(c, input_json, packed.data(), packed.size(), err, errcap);
        if (rc) return rc;
        uint8_t proof[256];
        std::vector<uint8_t> pub(32 * (size_t)std::max(1u, k.n_public()));
        int32_t status = -1;
        rc = zke_fullprove(x, packed.data(), 1, nullptr, proof, pub.data(), &status, err, errcap);
        if (rc) return rc;
        return zke_proof_to_json(proof, pub.data(), k.n_public(), proof_json, proof_len, public_json, public_len);
    } catch (const std::exception& e) { set_err(err, errcap, e.what()); return -1; }
}

}  // extern "C"
