#include "circuit.hpp"
#include <cstdlib>
#include <algorithm>
#include <stdexcept>

namespace zke {

// ---------------------------------------------------------------- LC
LC LC::operator+(const LC& o) const {
    if (o.t.empty()) return *this;
    if (t.empty()) return o;
    LC r;
    r.t.reserve(t.size() + o.t.size());
    size_t i = 0, j = 0;
    while (i < t.size() && j < o.t.size()) {
        if (t[i].first < o.t[j].first) r.t.push_back(t[i++]);
        else if (t[i].first > o.t[j].first) r.t.push_back(o.t[j++]);
        else {
            Fr s = t[i].second + o.t[j].second;
            if (!s.is_zero()) r.t.emplace_back(t[i].first, s);
            ++i; ++j;
        }
    }
    for (; i < t.size(); ++i) r.t.push_back(t[i]);
    for (; j < o.t.size(); ++j) r.t.push_back(o.t[j]);
    return r;
}
LC LC::neg() const {
    LC r = *this;
    for (auto& p : r.t) p.second = p.second.neg();
    return r;
}
LC LC::operator-(const LC& o) const { return *this + o.neg(); }
LC LC::operator*(const Fr& k) const {
    LC r;
    if (k.is_zero()) return r;
    r.t.reserve(t.size());
    for (auto& p : t) r.t.emplace_back(p.first, p.second * k);
    return r;
}
void LC::add_term(Var v, const Fr& k) {
    if (k.is_zero()) return;
    if (t.empty() || t.back().first < v) { t.emplace_back(v, k); return; }
    *this = *this + LC::term(v, k);
}

// ---------------------------------------------------------------- Circuit
const SignalGroup* Circuit::find_group(const std::string& n) const {
    for (auto& g : groups) if (g.name == n) return &g;
    return nullptr;
}
uint32_t Circuit::domain_log2() const {
    uint64_t need = (uint64_t)n_constraints + n_public() + 1;
    uint32_t k = 1;
    while ((1ull << k) < need) ++k;
    return k;
}

// ---------------------------------------------------------------- Builder
static const size_t LC_FANIN = 8;   // longer program LCs are split into a tree of scratch partial sums

Builder::Builder(const std::string& name) {
    c_.name = name;
    c_.a_ptr.push_back(0); c_.b_ptr.push_back(0); c_.c_ptr.push_back(0);
    c_.lc_ptr.push_back(0);
    intern(Fr::one());        // coefficient 0 = +1
    intern(Fr::one().neg());  // coefficient 1 = -1
    push_scope("main");
}

Var Builder::new_var() {
    decl_closed_ = true;
    if (next_var_ >= TEMP_BIT - 1) throw std::runtime_error("too many signals");
    return next_var_++;
}
Var Builder::new_temp() { return TEMP_BIT | next_temp_++; }

std::vector<Var> Builder::declare_outputs(const std::string& name, uint32_t n) {
    if (decl_closed_ || c_.n_pub_inputs || c_.n_prv_inputs) throw std::runtime_error("outputs must be declared first");
    SignalGroup g{name, next_var_, n, 0};
    c_.groups.push_back(g);
    std::vector<Var> v(n);
    for (uint32_t i = 0; i < n; ++i) v[i] = next_var_++;
    c_.n_outputs += n;
    return v;
}
std::vector<Var> Builder::declare_inputs(const std::string& name, uint32_t n, bool is_public) {
    if (decl_closed_) throw std::runtime_error("inputs must be declared before intermediate signals");
    if (is_public && c_.n_prv_inputs) throw std::runtime_error("public inputs must precede private inputs");
    SignalGroup g{name, next_var_, n, is_public ? 1 : 2};
    c_.groups.push_back(g);
    std::vector<Var> v(n);
    for (uint32_t i = 0; i < n; ++i) v[i] = next_var_++;
    (is_public ? c_.n_pub_inputs : c_.n_prv_inputs) += n;
    return v;
}

uint32_t Builder::intern(const Fr& c) {
    U256 s = c.to_u256();
    auto it = coef_index_.find(s);
    if (it != coef_index_.end()) return it->second;
    uint32_t idx = (uint32_t)c_.coefs.size();
    c_.coefs.push_back(s);
    coef_index_.emplace(s, idx);
    return idx;
}

void Builder::push_row(std::vector<uint32_t>& ptr, std::vector<uint32_t>& var, std::vector<uint32_t>& coef, const LC& e) {
    static const Fr ONE = Fr::one();
    static const Fr MONE = Fr::one().neg();
    for (auto& p : e.t) {
        var.push_back(p.first);
        coef.push_back(p.second == ONE ? 0u : (p.second == MONE ? 1u : intern(p.second)));
    }
    ptr.push_back((uint32_t)var.size());
}

uint32_t Builder::add_prog_lc(const LC& e) {
    if (e.t.size() > LC_FANIN) {
        // split into partial sums held in scratch slots (one extra level per factor of LC_FANIN)
        LC top;
        for (size_t i = 0; i < e.t.size(); i += LC_FANIN) {
            LC part;
            part.t.assign(e.t.begin() + i, e.t.begin() + std::min(e.t.size(), i + LC_FANIN));
            Var tmp = new_temp();
            uint32_t id = add_prog_lc(part);
            add_op(OP_LIN, tmp, id, 0, 0);
            top.t.emplace_back(tmp, Fr::one());
        }
        return add_prog_lc(top);
    }
    push_row(c_.lc_ptr, c_.lc_var, c_.lc_coef, e);
    return (uint32_t)c_.lc_ptr.size() - 2;
}

void Builder::add_op(uint32_t code, Var dst, uint32_t a, uint32_t b, uint32_t c) { c_.ops.push_back(WOp{code, dst, a, b, c}); }

void Builder::add_constraint(const LC& a, const LC& b, const LC& c) {
    for (const LC* e : {&a, &b, &c})
        for (auto& p : e->t)
            if (p.first & TEMP_BIT) throw std::runtime_error("scratch slot used in a constraint");
    push_row(c_.a_ptr, c_.a_var, c_.a_coef, a);
    push_row(c_.b_ptr, c_.b_var, c_.b_coef, b);
    push_row(c_.c_ptr, c_.c_var, c_.c_coef, c);
    c_.scope_of_constraint.push_back(scope_stack_.back());
}

void Builder::push_scope(const std::string& s) {
    auto it = scope_index_.find(s);
    uint16_t id;
    if (it == scope_index_.end()) {
        id = (uint16_t)c_.scopes.size();
        c_.scopes.push_back(s);
        scope_index_[s] = id;
    } else id = it->second;
    scope_stack_.push_back(id);
}
void Builder::pop_scope() { scope_stack_.pop_back(); }

LC Builder::signal(const LC& e) {
    Var v;
    if (e.is_const() || e.is_single_var(&v) || !materialize_linear) return e;
    Var x = new_var();
    add_op(OP_LIN, x, add_prog_lc(e), 0, 0);
    add_constraint(LC(), LC(), e - LC(x));
    return LC(x);
}

LC Builder::mul(const LC& a, const LC& b) { return mul_add(a, b, LC()); }

LC Builder::mul_add(const LC& a, const LC& b, const LC& c) {
    if (a.is_const()) return signal(b * a.const_value() + c);
    if (b.is_const()) return signal(a * b.const_value() + c);
    Var x = new_var();
    uint32_t ia = add_prog_lc(a), ib = add_prog_lc(b), ic = add_prog_lc(c);
    add_op(OP_QUAD, x, ia, ib, ic);
    add_constraint(a, b, LC(x) - c);
    return LC(x);
}

void Builder::enforce_mul(const LC& a, const LC& b, const LC& c) {
    if (a.is_const()) { enforce_eq(b * a.const_value(), c); return; }
    if (b.is_const()) { enforce_eq(a * b.const_value(), c); return; }
    add_constraint(a, b, c);
}

void Builder::enforce_eq(const LC& a, const LC& b) {
    LC d = a - b;
    if (d.is_zero()) return;
    if (d.is_const()) throw std::runtime_error("constraint is a non-zero constant (circuit can never be satisfied)");
    add_constraint(LC(), LC(), d);
}

void Builder::assign_output(Var out, const LC& e) {
    add_op(OP_LIN, out, add_prog_lc(e), 0, 0);
    add_constraint(LC(), LC(), e - LC(out));
}

Var Builder::source_of(const LC& e) {
    Var v;
    if (e.is_single_var(&v)) return v;
    Var t = new_temp();
    add_op(OP_LIN, t, add_prog_lc(e), 0, 0);
    return t;
}
Var Builder::hint_shrand(Var src, uint32_t shift, uint32_t nbits) {
    Var x = new_var();
    add_op(OP_SHRAND, x, src, shift, nbits);
    return x;
}
Var Builder::hint_invz(Var src) {
    Var x = new_var();
    add_op(OP_INVZ, x, src, 0, 0);
    return x;
}
Var Builder::hint_lin(const LC& e) {
    Var x = new_var();
    add_op(OP_LIN, x, add_prog_lc(e), 0, 0);
    return x;
}
Var Builder::hint_fpmul(uint32_t n, uint32_t k, const std::vector<Var>& a, const std::vector<Var>& b,
                        const std::vector<Var>& p) {
    if (a.size() != k || b.size() != k || p.size() != k) throw std::runtime_error("hint_fpmul: bad operand sizes");
    uint32_t off = (uint32_t)c_.aux.size();
    c_.aux.push_back(n);
    c_.aux.push_back(k);
    for (Var v : a) c_.aux.push_back(v);
    for (Var v : b) c_.aux.push_back(v);
    for (Var v : p) c_.aux.push_back(v);
    Var base = new_var();
    for (uint32_t i = 1; i < 2 * k; ++i) new_var();
    add_op(OP_FPMUL, base, off, 0, 0);
    return base;
}

int Builder::default_regex_style() {
    const char* e = getenv("ZKE_REGEX_STYLE");
    return e && atoi(e) == 1 ? 1 : 0;
}

bool Builder::default_fuse_shrand() {
    const char* e = getenv("ZKE_FUSED_SHRAND");
    return e ? atoi(e) != 0 : true;
}

// flat image of one RegexSeed (circuit.hpp); also what the engine appends to the device program's aux table
void append_regex_seed(std::vector<uint32_t>& out, const RegexSeed& R) {
    out.insert(out.end(), {(uint32_t)(R.desc.size() / 2), (uint32_t)R.bytes.size(), R.n_states | ((uint32_t)R.wide() << 30) | (R.mode << 31)});
    for (int q = 0; q < (R.wide() ? 4 : 1); ++q) out.insert(out.end(), {(uint32_t)R.first_mask[q], (uint32_t)(R.first_mask[q] >> 32)});
    out.insert(out.end(), R.bytes.begin(), R.bytes.end());
    auto pack = [&](const std::vector<uint8_t>& t) {
        for (uint32_t q = 0; q < R.n_states * 64; ++q) {
            uint32_t wd = 0;
            for (int k = 0; k < 4; ++k) wd |= (uint32_t)t[4 * (size_t)q + k] << (8 * k);
            out.push_back(wd);
        }
    };
    pack(R.table);
    if (R.mode == 1) pack(R.group);
    out.insert(out.end(), R.desc.begin(), R.desc.end());
}

Circuit Builder::finalize() {
    Circuit& c = c_;
    c.n_vars = next_var_;
    c.n_temps = next_temp_;
    c.n_constraints = (uint32_t)c.scope_of_constraint.size();
    const uint32_t m = c.n_vars;
    auto remap = [m](uint32_t& v) { if (v & TEMP_BIT) v = m + (v & ~TEMP_BIT); };
    for (auto& v : c.lc_var) remap(v);
    for (auto& op : c.ops) {
        remap(op.dst);
        if (op.code == OP_SHRAND || op.code == OP_INVZ) remap(op.a);
    }
    // (aux holds only real variables: hint_fpmul operands are witness signals)
    for (auto& blk : c.sha_blocks) { blk.temp_begin += m; blk.temp_end += m; }   // raw temp indices -> slot numbers
    c.sha_flat.clear();
    c.sha_flat.push_back((uint32_t)c.sha_blocks.size());
    for (auto& blk : c.sha_blocks) {
        c.sha_flat.insert(c.sha_flat.end(), {blk.var_begin, blk.var_end, blk.temp_begin, blk.temp_end, (uint32_t)(blk.desc.size() / 2)});
        c.sha_flat.insert(c.sha_flat.end(), blk.inputs.begin(), blk.inputs.end());
        c.sha_flat.insert(c.sha_flat.end(), blk.desc.begin(), blk.desc.end());
    }

    c.regex_flat.clear();
    c.regex_flat.push_back((uint32_t)c.regex_seeds.size());
    for (auto& R : c.regex_seeds) {
        append_regex_seed(c.regex_flat, R);
    }

    for (auto& blk : c.poseidon_blocks) { blk.temp_begin += m; blk.temp_end += m; }
    c.poseidon_flat.clear();
    c.poseidon_flat.push_back((uint32_t)c.poseidon_blocks.size());
    for (auto& blk : c.poseidon_blocks) {
        c.poseidon_flat.insert(c.poseidon_flat.end(), {blk.t, blk.var_begin, blk.var_end, blk.temp_begin, blk.temp_end, (uint32_t)(blk.desc.size() / 2)});
        c.poseidon_flat.insert(c.poseidon_flat.end(), blk.inputs.begin(), blk.inputs.end());
        c.poseidon_flat.insert(c.poseidon_flat.end(), blk.desc.begin(), blk.desc.end());
    }

    // Fuse "scratch <- LC; bits <- (scratch >> k) & mask" into OP_SHRLC when the scratch slot feeds nothing else:
    // the shift ops then sit one dependency level earlier (13.9 k -> 10.8 k levels for the default EmailVerifier).
    // ZKE_FUSED_SHRAND=0 keeps the two-op form (GPU witness == oracle verified in both forms).
    if (fuse_shrand) {
        const uint32_t total_slots = m + c.n_temps;
        std::vector<uint32_t> lc_uses(total_slots, 0), shr_uses(total_slots, 0), other_uses(total_slots, 0);
        std::vector<int64_t> producer(total_slots, -1);
        for (uint32_t v : c.lc_var) lc_uses[v]++;
        for (size_t i = 0; i < c.ops.size(); ++i) {
            const WOp& op = c.ops[i];
            if (op.code == OP_LIN && op.dst >= m) producer[op.dst] = (int64_t)i;
            if (op.code == OP_SHRAND) shr_uses[op.a]++;
            if (op.code == OP_INVZ) other_uses[op.a]++;
        }
        std::vector<uint8_t> dead(c.ops.size(), 0);
        for (auto& op : c.ops) {
            if (op.code != OP_SHRAND || op.a < m) continue;
            const int64_t pi = producer[op.a];
            if (pi < 0 || lc_uses[op.a] != 0 || other_uses[op.a] != 0) continue;
            dead[pi] = 1;                       // every consumer of the slot is an OP_SHRAND, all of them get rewritten
            op.code = OP_SHRLC;
            op.a = c.ops[pi].a;                 // the LC the scratch slot held
        }
        std::vector<WOp> live;
        live.reserve(c.ops.size());
        for (size_t i = 0; i < c.ops.size(); ++i) if (!dead[i]) live.push_back(c.ops[i]);
        c.ops.swap(live);
    }

    // levelise
    const uint32_t total = m + c.n_temps;
    std::vector<uint32_t> level(total, 0);
    std::vector<uint8_t> defined(total, 0);
    defined[0] = 1;
    for (auto& g : c.groups)
        if (g.kind != 0) for (uint32_t i = 0; i < g.count; ++i) defined[g.first + i] = 1;
    std::vector<uint32_t> op_level(c.ops.size());
    uint32_t max_level = 0;
    auto lc_level = [&](uint32_t id) {
        uint32_t l = 0;
        for (uint32_t k = c.lc_ptr[id]; k < c.lc_ptr[id + 1]; ++k) {
            uint32_t v = c.lc_var[k];
            if (!defined[v]) throw std::runtime_error("witness program reads an unassigned signal");
            l = std::max(l, level[v]);
        }
        return l;
    };
    for (size_t i = 0; i < c.ops.size(); ++i) {
        const WOp& op = c.ops[i];
        uint32_t l = 0, ndst = 1;
        switch (op.code) {
            case OP_LIN: l = lc_level(op.a); break;
            case OP_SHRLC: l = lc_level(op.a); break;
            case OP_QUAD: l = std::max(lc_level(op.a), std::max(lc_level(op.b), lc_level(op.c))); break;
            case OP_SHRAND:
            case OP_INVZ:
                if (!defined[op.a]) throw std::runtime_error("hint reads an unassigned signal");
                l = level[op.a];
                break;
            case OP_FPMUL: {
                uint32_t k = c.aux[op.a + 1];
                for (uint32_t j = 0; j < 3 * k; ++j) {
                    uint32_t v = c.aux[op.a + 2 + j];
                    if (!defined[v]) throw std::runtime_error("fpmul hint reads an unassigned signal");
                    l = std::max(l, level[v]);
                }
                ndst = 2 * k;
                break;
            }
            default: throw std::runtime_error("bad opcode");
        }
        l += 1;
        for (uint32_t j = 0; j < ndst; ++j) {
            if (defined[op.dst + j]) throw std::runtime_error("signal assigned twice");
            defined[op.dst + j] = 1;
            level[op.dst + j] = l;
        }
        op_level[i] = l;
        max_level = std::max(max_level, l);
    }
    for (uint32_t v = 0; v < m; ++v)
        if (!defined[v]) throw std::runtime_error("signal " + std::to_string(v) + " is never assigned");

    // stable counting sort of ops by level (levels are 1-based; level_ptr[l-1]..level_ptr[l])
    c.level_ptr.assign(max_level + 1, 0);
    for (uint32_t l : op_level) c.level_ptr[l]++;
    {
        uint32_t run = 0;
        for (uint32_t l = 1; l <= max_level; ++l) { uint32_t n = c.level_ptr[l]; c.level_ptr[l] = run; run += n; }
        c.level_ptr[0] = 0;
    }
    std::vector<WOp> sorted(c.ops.size());
    {
        std::vector<uint32_t> cursor(c.level_ptr.begin(), c.level_ptr.end());
        for (size_t i = 0; i < c.ops.size(); ++i) sorted[cursor[op_level[i]]++] = c.ops[i];
        // shift: level l (1-based) occupies [level_ptr[l], next); re-express as 0-based array with n_levels+1 entries
        std::vector<uint32_t> lp(max_level + 1);
        for (uint32_t l = 1; l <= max_level; ++l) lp[l - 1] = c.level_ptr[l];
        lp[max_level] = (uint32_t)c.ops.size();
        c.level_ptr.swap(lp);
    }
    c.ops.swap(sorted);
    // Within a level the ops are independent: order them by opcode and by the amount of work (LC terms) so that the
    // 32 lanes of a warp of the device interpreter execute the same case with similar trip counts.
    auto op_cost = [&](const WOp& o) -> uint32_t {
        auto len = [&](uint32_t id) { return c.lc_ptr[id + 1] - c.lc_ptr[id]; };
        if (o.code == OP_LIN || o.code == OP_SHRLC) return len(o.a);
        if (o.code == OP_QUAD) return len(o.a) + len(o.b) + len(o.c);
        return 0;
    };
    for (uint32_t l = 0; l + 1 < c.level_ptr.size(); ++l) {
        auto beg = c.ops.begin() + c.level_ptr[l], end = c.ops.begin() + c.level_ptr[l + 1];
        std::stable_sort(beg, end, [&](const WOp& x, const WOp& y) {
            if (x.code != y.code) return x.code < y.code;
            return op_cost(x) < op_cost(y);
        });
    }
    return std::move(c_);
}

}  // namespace zke
