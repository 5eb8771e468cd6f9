// C ABI - circom's constraint system: the iden3 `.r1cs` reader and writer (host only).  See include/zkemail_b200.h.
//
// `circom --r1cs` writes the file that `snarkjs r1cs info` and `snarkjs groth16 setup` read
// (/root/reference/docs/zk-email-docs/UsageGuide/README.md, steps 3-5).  Layout (SURVEY 8(b), iden3_binfile.py), all
// little-endian, sections in any order:
//   container : "r1cs", u32 version = 1, u32 nSections, then {u32 type, u64 size, payload} per section
//   1 header  : u32 n8, prime[n8], u32 nWires, nPubOut, nPubIn, nPrvIn, u64 nLabels, u32 nConstraints
//   2 constraints: per constraint A, B, C as {u32 nTerms, (u32 wire, coef[n8]) x nTerms}, coefficients standard form
//   3 wire -> label map: u64 per wire (optional)
//   4, 5 custom gates (PLONK only; refused)
// The circuit read here has the constraint system and nothing else: an empty witness program, no named signal groups.
#include "../../include/zkemail_b200.h"
#include "engine.hpp"
#include "binfile.hpp"
#include <cstring>
#include <memory>
#include <unordered_map>

using namespace zke;

namespace {

const size_t R1CS_HEADER_BYTES = 4 + 32 + 4 * 4 + 8 + 4;

// BLS12-381's scalar field modulus: the other prime circom compiles for, named in the refusal
const U256 BLS12_381_R = {{0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull}};

struct U256Hash {
    size_t operator()(const U256& x) const { return (size_t)(x.v[0] * 0x9E3779B97F4A7C15ull ^ x.v[1] * 31 ^ x.v[2] * 131 ^ x.v[3]); }
};

bool is_pow2(const U256& v) {
    int bits = 0;
    for (int i = 0; i < 4; ++i) bits += __builtin_popcountll(v.v[i]);
    return bits == 1;
}

Circuit read_r1cs(const uint8_t* b, size_t len) {
    if (!b || len < 12 || memcmp(b, "r1cs", 4) != 0) throw std::runtime_error("not an .r1cs file (bad magic)");
    if (rd32(b + 4) != 1) throw std::runtime_error(".r1cs version " + std::to_string(rd32(b + 4)) + " is not supported (expected 1)");
    SecView sec[4];
    for (const BinSection& s : binfile_sections(b, len, ".r1cs")) {
        if (s.type == 4 || s.type == 5) throw std::runtime_error(".r1cs section " + std::to_string(s.type) + ": custom gates (PLONK) are not supported");
        if (s.type < 1 || s.type > 3) continue;
        if (sec[s.type].p) throw std::runtime_error(".r1cs section " + std::to_string(s.type) + " appears twice");
        sec[s.type] = s.view;
    }
    if (!sec[1].p) throw std::runtime_error(".r1cs section 1 (header) is missing");
    if (!sec[2].p) throw std::runtime_error(".r1cs section 2 (constraints) is missing");

    // ---- header
    const uint8_t* h = sec[1].p;
    if (sec[1].n < 4) throw std::runtime_error("truncated .r1cs header (section 1 has " + std::to_string(sec[1].n) + " bytes)");
    const uint32_t n8 = rd32(h);
    if (n8 != 32) throw std::runtime_error(".r1cs field elements have " + std::to_string(n8) + " bytes, expected 32 (BN254)");
    if (sec[1].n != R1CS_HEADER_BYTES)
        throw std::runtime_error((sec[1].n < R1CS_HEADER_BYTES ? "truncated .r1cs header: section 1 has " : ".r1cs header: section 1 has ") +
                                 std::to_string(sec[1].n) + " bytes, expected " + std::to_string(R1CS_HEADER_BYTES));
    U256 prime;
    memcpy(prime.v, h + 4, 32);
    if (prime == BLS12_381_R) throw std::runtime_error(".r1cs is over the BLS12-381 scalar field; only BN254 is supported");
    if (!(prime == fr_params().p)) throw std::runtime_error(".r1cs prime is not the BN254 scalar field modulus r");
    Circuit c;
    c.name = "r1cs";
    c.r1cs_only = true;
    c.n_vars = rd32(h + 36);
    c.n_outputs = rd32(h + 40); c.n_pub_inputs = rd32(h + 44); c.n_prv_inputs = rd32(h + 48);
    c.n_labels = rd64(h + 52);
    c.n_constraints = rd32(h + 60);
    const uint64_t declared = 1ull + c.n_outputs + c.n_pub_inputs + c.n_prv_inputs;
    if (declared > c.n_vars)
        throw std::runtime_error(".r1cs header: 1 + nPubOut + nPubIn + nPrvIn = " + std::to_string(declared) + " exceeds nWires = " + std::to_string(c.n_vars));
    const uint64_t rows = (uint64_t)c.n_constraints + c.n_public() + 1;
    if (rows > (1ull << 28))
        throw std::runtime_error(".r1cs header: nConstraints + nPublic + 1 = " + std::to_string(rows) + " exceeds the largest domain, 2^28");
    if (sec[3].p && sec[3].n != 8 * (size_t)c.n_vars)
        throw std::runtime_error(".r1cs section 3 (labels) has " + std::to_string(sec[3].n) + " bytes, expected 8 * nWires = " + std::to_string(8 * (size_t)c.n_vars));

    // ---- constraints, in file order; coefficients interned in order of appearance after 1 and r - 1
    const uint8_t* p = sec[2].p;
    const size_t n2 = sec[2].n;
    if (n2 / 12 < c.n_constraints) throw std::runtime_error("truncated .r1cs: section 2 is too short for " + std::to_string(c.n_constraints) + " constraints");
    std::unordered_map<U256, uint32_t, U256Hash> index;
    U256 minus_one;
    u256_sub(minus_one, fr_params().p, U256{{1, 0, 0, 0}});
    c.coefs = {U256{{1, 0, 0, 0}}, minus_one};
    index.emplace(c.coefs[0], 0u);
    index.emplace(c.coefs[1], 1u);
    std::vector<uint32_t>* ptrs[3] = {&c.a_ptr, &c.b_ptr, &c.c_ptr};
    std::vector<uint32_t>* vars[3] = {&c.a_var, &c.b_var, &c.c_var};
    std::vector<uint32_t>* cfs[3] = {&c.a_coef, &c.b_coef, &c.c_coef};
    for (int m = 0; m < 3; ++m) { ptrs[m]->reserve((size_t)c.n_constraints + 1); ptrs[m]->push_back(0); }
    size_t pos = 0;
    uint32_t last_id = 0;
    U256 last = c.coefs[0];
    for (uint32_t row = 0; row < c.n_constraints; ++row) {
        for (int m = 0; m < 3; ++m) {
            if (n2 - pos < 4) throw std::runtime_error("truncated .r1cs: section 2 ends inside constraint " + std::to_string(row));
            const uint32_t n_terms = rd32(p + pos);
            pos += 4;
            if ((n2 - pos) / 36 < n_terms) throw std::runtime_error("truncated .r1cs: section 2 ends inside constraint " + std::to_string(row));
            if (vars[m]->size() + n_terms > 0xffffffffull) throw std::runtime_error(".r1cs has more than 2^32 terms in one matrix");
            for (uint32_t t = 0; t < n_terms; ++t, pos += 36) {
                const uint32_t wire = rd32(p + pos);
                if (wire >= c.n_vars)
                    throw std::runtime_error(".r1cs constraint " + std::to_string(row) + ": wire " + std::to_string(wire) + " is out of range (nWires = " + std::to_string(c.n_vars) + ")");
                U256 v;
                memcpy(v.v, p + pos + 4, 32);
                if (!(v == last)) {
                    auto it = index.find(v);
                    if (it == index.end()) {
                        if (u256_cmp(v, fr_params().p) >= 0) throw std::runtime_error(".r1cs constraint " + std::to_string(row) + ": coefficient is not below r");
                        it = index.emplace(v, (uint32_t)c.coefs.size()).first;
                        c.coefs.push_back(v);
                    }
                    last = v;
                    last_id = it->second;
                }
                vars[m]->push_back(wire);
                cfs[m]->push_back(last_id);
            }
            ptrs[m]->push_back((uint32_t)vars[m]->size());
        }
    }
    if (pos != n2) throw std::runtime_error("trailing bytes in .r1cs section 2: " + std::to_string(n2 - pos) + " after the last constraint");
    if (c.coefs.size() >= (1u << 24)) throw std::runtime_error(".r1cs has more than 2^24 distinct coefficients");

    // Powers of two (+-2^k) right after 1 and r - 1, so that they get the small table indices the engine's shift
    // shortcut needs (witness_program.cpp: coef_words); every other coefficient after them, each group in order of appearance.
    {
        std::vector<uint32_t> order = {0, 1};
        for (int pass = 0; pass < 2; ++pass)
            for (uint32_t i = 2; i < (uint32_t)c.coefs.size(); ++i) {
                U256 neg;
                u256_sub(neg, fr_params().p, c.coefs[i]);
                const bool p2 = !c.coefs[i].is_zero() && (is_pow2(c.coefs[i]) || is_pow2(neg));
                if (p2 == (pass == 0)) order.push_back(i);
            }
        std::vector<uint32_t> remap(order.size());
        std::vector<U256> coefs(order.size());
        for (uint32_t k = 0; k < (uint32_t)order.size(); ++k) { remap[order[k]] = k; coefs[k] = c.coefs[order[k]]; }
        c.coefs.swap(coefs);
        for (int m = 0; m < 3; ++m) for (uint32_t& id : *cfs[m]) id = remap[id];
    }
    c.scopes = {"r1cs"};
    c.scope_of_constraint.assign(c.n_constraints, 0);
    if (sec[3].p) {
        c.labels.resize(c.n_vars);
        if (c.n_vars) memcpy(c.labels.data(), sec[3].p, 8 * (size_t)c.n_vars);
    }
    return c;
}

// The `.r1cs` image of a circuit: sections 1, 2, 3 in that order, the kept labels or the identity map.
int64_t write_r1cs(const Circuit& c, uint8_t* out, size_t cap) {
    const std::vector<uint32_t>* ptrs[3] = {&c.a_ptr, &c.b_ptr, &c.c_ptr};
    const std::vector<uint32_t>* vars[3] = {&c.a_var, &c.b_var, &c.c_var};
    const std::vector<uint32_t>* cfs[3] = {&c.a_coef, &c.b_coef, &c.c_coef};
    size_t body = 12 * (size_t)c.n_constraints;
    for (int m = 0; m < 3; ++m) body += 36 * (size_t)(*ptrs[m])[c.n_constraints];
    const size_t total = 12 + (12 + R1CS_HEADER_BYTES) + (12 + body) + (12 + 8 * (size_t)c.n_vars);
    if (!out) return (int64_t)total;
    if (cap < total) return -2;
    BinWriter w{out};
    w.header("r1cs", 1, 3);
    w.section(1, R1CS_HEADER_BYTES);
    w.u32(32); w.bytes(fr_params().p.v, 32);
    w.u32(c.n_vars); w.u32(c.n_outputs); w.u32(c.n_pub_inputs); w.u32(c.n_prv_inputs);
    w.u64(c.r1cs_only ? c.n_labels : c.n_vars);
    w.u32(c.n_constraints);
    w.section(2, body);
    for (uint32_t row = 0; row < c.n_constraints; ++row)
        for (int m = 0; m < 3; ++m) {
            const uint32_t beg = (*ptrs[m])[row], end = (*ptrs[m])[row + 1];
            w.u32(end - beg);
            for (uint32_t k = beg; k < end; ++k) { w.u32((*vars[m])[k]); w.bytes(c.coefs[(*cfs[m])[k]].v, 32); }
        }
    w.section(3, 8 * (size_t)c.n_vars);
    if (!c.labels.empty()) w.bytes(c.labels.data(), 8 * (size_t)c.n_vars);
    else for (uint32_t i = 0; i < c.n_vars; ++i) w.u64(i);
    return (int64_t)(w.p - out);
}

}  // namespace

extern "C" {

zke_circuit* zke_circuit_from_r1cs(const void* r1cs, size_t len, char* err, size_t errcap) {
    try {
        std::unique_ptr<zke_circuit> c(new zke_circuit());
        c->c = read_r1cs((const uint8_t*)r1cs, len);
        return c.release();
    } catch (const std::exception& e) {
        set_err(err, errcap, e.what());
        return nullptr;
    }
}

int64_t zke_circuit_write_r1cs(const zke_circuit* c, uint8_t* out, size_t cap) {
    if (!c) return -1;
    try { return write_r1cs(c->c, out, cap); }
    catch (const std::exception&) { return -3; }
}

}  // extern "C"
