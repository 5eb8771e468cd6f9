// Regex -> DFA -> constraint generator for the DKIM body-hash regex.
//
// The reference includes `@zk-email/zk-regex-circom/circuits/common/body_hash_regex.circom` (un-vendored,
// v2.3.2, /root/reference/yarn.lock:2794-2799; call site /root/reference/packages/circuits/email-verifier.circom:5,126),
// a circom file generated from the decomposed regex
//     (\r\n|^)dkim-signature:   ([a-z]+=[^;]+; )+bh=   [a-zA-Z0-9+/=]+ (public)   ;
// by a Rust tool.  Neither the tool nor its output is in the reference tree, so this file restates the
// construction: Thompson NFA per part (char transitions tagged public/private), subset construction to a
// DFA, then the zk-regex circuit shape: the input is prefixed with byte 255 (the `^` marker), state 0 is
// live at every position (unanchored search), states[i+1][s] is the OR over incoming transitions of
// (states[i][src] AND in[i] in class), out = OR_i states[i][accept], and reveal[i] = in[i] wherever a
// transition of the public part fires (contract in SURVEY A.6).  regex_match_reveals gives every public part a reveal
// array of its own (the edges of public part p carry tag bit p); the other entry points OR all public parts into reveal0.
//
// Builder::regex_style = 1 emits the same function of the input (same `out`, same `reveal0`) in a different circuit
// shape ("compact", regex_circuit_compact below): character classes from nibble one-hots of a single bit decomposition per
// byte instead of one 9-bit comparator per range end, and the live-state set itself as ONE one-hot state of the automaton
// of live sets, so that a position costs one multiplication level and no OR gates.  ~3x fewer constraints.
#include "gadgets.hpp"
#include <algorithm>
#include <array>
#include <bitset>
#include <map>
#include <set>
#include <stdexcept>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <tuple>

namespace zke {
namespace gadgets {

namespace {

typedef std::bitset<256> CharSet;

struct NfaEdge { int to; CharSet cs; bool eps; uint32_t pub; };   // pub: bit set of the public parts the edge belongs to
struct Nfa {
    std::vector<std::vector<NfaEdge>> adj;
    int new_state() { adj.emplace_back(); return (int)adj.size() - 1; }
    void eps(int a, int b) { adj[a].push_back(NfaEdge{b, CharSet(), true, 0}); }
    void chr(int a, int b, const CharSet& cs, uint32_t pub) { adj[a].push_back(NfaEdge{b, cs, false, pub}); }
};
struct Frag { int s, e; };

// Recursive-descent parser for the subset: | concatenation ( ) + * ? [..] [^..] escapes ^ literals
struct Parser {
    const std::string& re;
    size_t pos = 0;
    Nfa& nfa;
    uint32_t pub;
    Parser(const std::string& r, Nfa& n, uint32_t p) : re(r), nfa(n), pub(p) {}

    bool more() const { return pos < re.size(); }
    char peek() const { return re[pos]; }

    static CharSet escape_class(char c) {
        CharSet cs;
        switch (c) {
            case 'r': cs.set('\r'); break;
            case 'n': cs.set('\n'); break;
            case 't': cs.set('\t'); break;
            case 'w':
                for (int x = 'a'; x <= 'z'; ++x) cs.set(x);
                for (int x = 'A'; x <= 'Z'; ++x) cs.set(x);
                for (int x = '0'; x <= '9'; ++x) cs.set(x);
                cs.set('_');
                break;
            case 'd': for (int x = '0'; x <= '9'; ++x) cs.set(x); break;
            case 's': cs.set(' '); cs.set('\t'); cs.set('\r'); cs.set('\n'); break;
            default: cs.set((unsigned char)c); break;
        }
        return cs;
    }

    CharSet parse_class(bool& neg) {  // after '['
        CharSet cs;
        neg = false;
        if (more() && peek() == '^') { neg = true; ++pos; }
        bool first = true;
        while (more() && (peek() != ']' || first)) {
            first = false;
            CharSet lo_set;
            int lo = -1;
            if (peek() == '\\') {
                ++pos;
                if (!more()) throw std::runtime_error("regex: dangling escape");
                lo_set = escape_class(re[pos++]);
                if (lo_set.count() == 1) for (int x = 0; x < 256; ++x) if (lo_set.test(x)) lo = x;
            } else {
                lo = (unsigned char)re[pos++];
                lo_set.set(lo);
            }
            if (lo >= 0 && pos + 1 < re.size() && re[pos] == '-' && re[pos + 1] != ']') {
                ++pos;
                int hi = (unsigned char)re[pos++];
                if (hi < lo) throw std::runtime_error("regex: bad range");
                for (int x = lo; x <= hi; ++x) cs.set(x);
            } else cs |= lo_set;
        }
        if (!more()) throw std::runtime_error("regex: unterminated class");
        ++pos;  // ']'
        if (neg) {
            // complement within ASCII; bytes >= 0x80 are handled as well-formed UTF-8 sequences by utf8_fragment()
            cs.flip();
            for (int x = 128; x < 256; ++x) cs.reset(x);
        }
        return cs;
    }

    static CharSet byte_range(int lo, int hi) { CharSet cs; for (int x = lo; x <= hi; ++x) cs.set(x); return cs; }

    // zk-regex treats negated classes and '.' as "one well-formed UTF-8 code point" (Unicode table 3-7):
    // every non-ASCII code point is outside any ASCII exclusion list, so all multi-byte sequences match.
    void utf8_fragment(int s, int e) {
        const CharSet cont = byte_range(0x80, 0xBF);
        auto chain = [&](const CharSet& lead, std::vector<CharSet> rest) {
            int cur = nfa.new_state();
            nfa.chr(s, cur, lead, pub);
            for (size_t i = 0; i < rest.size(); ++i) {
                int nx = (i + 1 == rest.size()) ? e : nfa.new_state();
                nfa.chr(cur, nx, rest[i], pub);
                cur = nx;
            }
        };
        chain(byte_range(0xC2, 0xDF), {cont});
        chain(byte_range(0xE0, 0xE0), {byte_range(0xA0, 0xBF), cont});
        chain(byte_range(0xE1, 0xEC), {cont, cont});
        chain(byte_range(0xED, 0xED), {byte_range(0x80, 0x9F), cont});
        chain(byte_range(0xEE, 0xEF), {cont, cont});
        chain(byte_range(0xF0, 0xF0), {byte_range(0x90, 0xBF), cont, cont});
        chain(byte_range(0xF1, 0xF3), {cont, cont, cont});
        chain(byte_range(0xF4, 0xF4), {byte_range(0x80, 0x8F), cont, cont});
    }

    Frag parse_atom() {
        char c = re[pos++];
        if (c == '(') {
            Frag f = parse_alt();
            if (!more() || re[pos] != ')') throw std::runtime_error("regex: missing ')'");
            ++pos;
            return f;
        }
        CharSet cs;
        bool utf8 = false;
        if (c == '[') cs = parse_class(utf8);
        else if (c == '\\') { if (!more()) throw std::runtime_error("regex: dangling escape"); cs = escape_class(re[pos++]); }
        else if (c == '^') cs.set(255);
        else if (c == '.') { for (int x = 0; x < 128; ++x) cs.set(x); utf8 = true; }
        else cs.set((unsigned char)c);
        int s = nfa.new_state(), e = nfa.new_state();
        nfa.chr(s, e, cs, pub);
        if (utf8) utf8_fragment(s, e);
        return Frag{s, e};
    }

    Frag parse_repeat() {
        Frag f = parse_atom();
        while (more() && (peek() == '+' || peek() == '*' || peek() == '?')) {
            char q = re[pos++];
            int s = nfa.new_state(), e = nfa.new_state();
            nfa.eps(s, f.s);
            nfa.eps(f.e, e);
            if (q == '+' || q == '*') nfa.eps(f.e, f.s);
            if (q == '*' || q == '?') nfa.eps(s, e);
            f = Frag{s, e};
        }
        return f;
    }

    Frag parse_concat() {
        int s = nfa.new_state();
        int cur = s;
        while (more() && peek() != '|' && peek() != ')') {
            Frag f = parse_repeat();
            nfa.eps(cur, f.s);
            cur = f.e;
        }
        return Frag{s, cur};
    }

    Frag parse_alt() {
        Frag f = parse_concat();
        if (!(more() && peek() == '|')) return f;
        int s = nfa.new_state(), e = nfa.new_state();
        nfa.eps(s, f.s); nfa.eps(f.e, e);
        while (more() && peek() == '|') {
            ++pos;
            Frag g = parse_concat();
            nfa.eps(s, g.s); nfa.eps(g.e, e);
        }
        return Frag{s, e};
    }
};

struct DfaTransition { int src, dst; CharSet cs; uint32_t pub; };
struct Dfa {
    int n_states = 0;
    std::vector<bool> accept;
    std::vector<DfaTransition> trans;   // grouped by (src, dst, pub)
};

// per_part = false: every public part carries tag 1 (one reveal array for all of them); true: public part p carries tag
// 1 << p, so that each public part gets a reveal array of its own
Dfa build_dfa(const std::vector<std::pair<std::string, bool>>& parts, bool per_part = false) {
    Nfa nfa;
    int start = nfa.new_state();
    int cur = start;
    uint32_t n_public = 0;
    for (auto& pr : parts) {
        uint32_t tag = 0;
        if (pr.second) {
            if (per_part && n_public >= 32) throw std::runtime_error("regex: more than 32 public parts");
            tag = per_part ? 1u << n_public : 1u;
            ++n_public;
        }
        Parser ps(pr.first, nfa, tag);
        Frag f = ps.parse_alt();
        if (ps.more()) throw std::runtime_error("regex: trailing characters");
        nfa.eps(cur, f.s);
        cur = f.e;
    }
    const int nfa_accept = cur;
    auto closure = [&](std::set<int> s) {
        std::vector<int> stack(s.begin(), s.end());
        while (!stack.empty()) {
            int u = stack.back(); stack.pop_back();
            for (auto& e : nfa.adj[u]) if (e.eps && !s.count(e.to)) { s.insert(e.to); stack.push_back(e.to); }
        }
        return s;
    };
    std::map<std::set<int>, int> index;
    std::vector<std::set<int>> sets;
    Dfa d;
    auto get = [&](const std::set<int>& s) {
        auto it = index.find(s);
        if (it != index.end()) return it->second;
        int id = (int)sets.size();
        index[s] = id; sets.push_back(s);
        return id;
    };
    get(closure({start}));
    std::map<std::tuple<int, int, uint32_t>, CharSet> grouped;
    for (size_t si = 0; si < sets.size(); ++si) {
        for (int c = 0; c < 256; ++c) {
            std::set<int> tgt;
            uint32_t pub = 0;
            for (int u : sets[si])
                for (auto& e : nfa.adj[u])
                    if (!e.eps && e.cs.test(c)) { tgt.insert(e.to); pub |= e.pub; }
            if (tgt.empty()) continue;
            int ti = get(closure(tgt));
            grouped[std::make_tuple((int)si, ti, pub)].set(c);
        }
    }
    d.n_states = (int)sets.size();
    d.accept.resize(d.n_states);
    for (int i = 0; i < d.n_states; ++i) d.accept[i] = sets[i].count(nfa_accept) > 0;
    for (auto& kv : grouped) d.trans.push_back(DfaTransition{std::get<0>(kv.first), std::get<1>(kv.first), kv.second, std::get<2>(kv.first)});
    return d;
}

// constraint for "in is in [lo, hi]" (bytes); in is assumed to be a byte (range-checked elsewhere, as in zk-regex)
LC range_match(Builder& b, const LC& in, int lo, int hi) {
    if (lo == hi) return is_equal(b, in, LC::constant(Fr::from_u64(lo)));
    if (lo == 0) return less_than(b, 8, in, LC::constant(Fr::from_u64(hi + 1)));
    if (hi == 255) return greater_than(b, 8, in, LC::constant(Fr::from_u64(lo - 1)));
    LC lt = less_than(b, 8, in, LC::constant(Fr::from_u64(hi + 1)));
    LC gt = greater_than(b, 8, in, LC::constant(Fr::from_u64(lo - 1)));
    return gate_and(b, gt, lt);
}

}  // namespace

// out = [match, reveal of tag bit 0 (msg.size()), reveal of tag bit 1, ...]: n_reveal arrays (regex_match_reveals)
static LCVec regex_circuit(Builder& b, const Dfa& dfa, const LCVec& msg, uint32_t n_reveal = 1) {
    const int S = dfa.n_states;
    const size_t num_bytes = msg.size() + 1;
    if (dfa.accept[0]) throw std::runtime_error("regex: matches the empty string");

    // decompose every transition's class into maximal byte ranges once
    std::vector<std::vector<std::pair<int, int>>> ranges(dfa.trans.size());
    for (size_t k = 0; k < dfa.trans.size(); ++k) {
        const CharSet& cs = dfa.trans[k].cs;
        for (int c = 0; c < 256;) {
            if (!cs.test(c)) { ++c; continue; }
            int e = c;
            while (e + 1 < 256 && cs.test(e + 1)) ++e;
            ranges[k].emplace_back(c, e);
            c = e + 1;
        }
    }
    std::vector<std::vector<int>> incoming(S);
    for (size_t k = 0; k < dfa.trans.size(); ++k) incoming[dfa.trans[k].dst].push_back((int)k);

    const LC one = LC::constant(Fr::one());
    LCVec states(S);                       // states[i][*]
    states[0] = one;
    LCVec accept_flags;
    LCVec out(1 + n_reveal * msg.size());
    // record for the device's automaton run (circuit.hpp: RegexSeed): possible when every message byte is a plain signal;
    // more than 64 states take the wide live set (256 bits), the uint8 table caps the DFA at 255 states
    RegexSeed seed;
    bool seedable = S <= 255 && msg.size() < (1u << 24);
    for (size_t j = 0; j < msg.size() && seedable; ++j) {
        Var v;
        if (msg[j].is_single_var(&v)) seed.bytes.push_back(v); else seedable = false;
    }
    if (seedable) {
        seed.n_states = (uint32_t)S;
        seed.table.assign((size_t)S * 256, 0xff);
        for (size_t k = 0; k < dfa.trans.size(); ++k) {
            const DfaTransition& t = dfa.trans[k];
            for (int c = 0; c < 255; ++c) if (t.cs.test(c)) seed.table[(size_t)t.src * 256 + c] = (uint8_t)t.dst;
            if (t.src == 0 && t.cs.test(255)) seed.first_mask[t.dst >> 6] |= 1ull << (t.dst & 63);   // the marker byte: only state 0 is live before it
        }
    }
    for (size_t i = 0; i < num_bytes; ++i) {
        const bool is_marker = (i == 0);
        const LC in = is_marker ? LC::constant(Fr::from_u64(255)) : msg[i - 1];
        std::map<std::pair<int, int>, LC> range_cache;
        std::vector<LC> fire(dfa.trans.size());
        for (size_t k = 0; k < dfa.trans.size(); ++k) {
            const DfaTransition& t = dfa.trans[k];
            if (t.src != 0 && states[t.src].is_zero()) continue;    // source state statically dead at this position
            LC m;
            if (is_marker) {
                if (t.cs.test(255)) m = one;
            } else {
                for (auto& r : ranges[k]) {
                    if (r.first == 255) continue;                   // the marker byte never occurs inside the message
                    int hi = std::min(r.second, 254);
                    auto key = std::make_pair(r.first, hi);
                    auto it = range_cache.find(key);
                    if (it == range_cache.end()) it = range_cache.emplace(key, range_match(b, in, r.first, hi)).first;
                    m += it->second;
                }
            }
            if (m.is_zero()) continue;
            fire[k] = (t.src == 0) ? m : gate_and(b, states[t.src], m);
        }
        LCVec next(S);
        next[0] = one;
        for (int s = 1; s < S; ++s) {
            LCVec ins;
            for (int k : incoming[s]) if (!fire[k].is_zero()) ins.push_back(fire[k]);
            if (!ins.empty()) next[s] = multi_or(b, ins);
        }
        for (uint32_t p = 0; p < n_reveal && !is_marker; ++p) {
            LCVec pubs;
            for (size_t k = 0; k < dfa.trans.size(); ++k) if ((dfa.trans[k].pub >> p & 1) && !fire[k].is_zero()) pubs.push_back(fire[k]);
            out[p * msg.size() + i] = pubs.empty() ? LC() : b.mul(in, multi_or(b, pubs));   // reveal_p[i-1] <== in[i] * is_reveal
        }
        states.swap(next);
        if (seedable && !is_marker)
            for (int s = 1; s < S; ++s) {
                Var v;
                if (states[s].is_single_var(&v)) { seed.desc.push_back(v); seed.desc.push_back(((uint32_t)i << 8) | (uint32_t)s); }
            }
        for (int s = 1; s < S; ++s) if (dfa.accept[s] && !states[s].is_zero()) accept_flags.push_back(states[s]);
    }
    if (accept_flags.empty()) throw std::runtime_error("regex: accept state unreachable for this length");
    out[0] = multi_or(b, accept_flags);
    if (seedable && !seed.desc.empty()) b.add_regex_seed(std::move(seed));
    return out;
}

// ------------------------------------------------------------------------------------------------ compact shape
namespace {

// The zk-regex shape keeps DFA state 0 live at every position, i.e. it runs one DFA thread per start position and the set
// of live threads is what moves from byte to byte.  That set is itself the state of a deterministic automaton: from the
// live set L and byte c the next set is {0} u {delta(s, c) : s in L}.  PowerDfa lists the reachable live sets (index 0 =
// {0}), their transitions on bytes 0..254 (byte 255 is the `^` marker and matches nothing inside the message), whether a
// public edge is taken by some thread, and whether the set holds an accepting DFA state.
struct PowerDfa {
    struct Tr { int src, dst; CharSet cs; uint32_t pub; };
    std::vector<std::vector<int>> members;
    std::vector<bool> accept;
    std::vector<Tr> trans;            // only transitions with dst != 0 ("every thread died" needs no product)
    int after_marker = 0;             // live set after the 255 marker byte
};

PowerDfa build_power(const Dfa& dfa) {
    const int S = dfa.n_states;
    std::vector<std::array<int, 256>> delta(S);        // dst * 2 + (pub != 0), or -1
    std::vector<std::array<uint32_t, 256>> pubs(S);    // public-part tags of the edge
    for (auto& row : delta) row.fill(-1);
    for (auto& t : dfa.trans)
        for (int c = 0; c < 256; ++c) if (t.cs.test(c)) { delta[t.src][c] = t.dst * 2 + (t.pub ? 1 : 0); pubs[t.src][c] = t.pub; }
    PowerDfa pd;
    std::map<std::vector<int>, int> index;
    auto get = [&](std::vector<int> set) {
        std::sort(set.begin(), set.end());
        set.erase(std::unique(set.begin(), set.end()), set.end());
        auto it = index.find(set);
        if (it != index.end()) return it->second;
        if (pd.members.size() >= 4096) throw std::runtime_error("regex: too many live-state sets for the compact circuit shape");
        int id = (int)pd.members.size();
        index[set] = id;
        pd.members.push_back(set);
        return id;
    };
    auto step = [&](const std::vector<int>& from, int c, uint32_t& pub) {
        std::vector<int> to{0};
        pub = 0;
        for (int s : from) if (delta[s][c] >= 0) { to.push_back(delta[s][c] >> 1); pub |= pubs[s][c]; }
        return to;
    };
    get({0});
    uint32_t dummy;
    pd.after_marker = get(step({0}, 255, dummy));
    std::map<std::tuple<int, int, uint32_t>, CharSet> grouped;
    for (size_t li = 0; li < pd.members.size(); ++li) {
        for (int c = 0; c < 255; ++c) {
            uint32_t pub;
            const std::vector<int> from = pd.members[li];      // copy: get() may grow pd.members
            int ti = get(step(from, c, pub));
            if (ti != 0) grouped[std::make_tuple((int)li, ti, pub)].set(c);
        }
    }
    pd.accept.resize(pd.members.size());
    for (size_t li = 0; li < pd.members.size(); ++li) {
        bool a = false;
        for (int s : pd.members[li]) a = a || dfa.accept[s];
        pd.accept[li] = a;
    }
    for (auto& kv : grouped) pd.trans.push_back(PowerDfa::Tr{std::get<0>(kv.first), std::get<1>(kv.first), kv.second, std::get<2>(kv.first)});
    return pd;
}

// One-hot indicators of the two nibbles of a byte: 8 booleanity rows + 1 sum row (this IS the byte range check),
// 2 + 15 products per nibble.
struct ByteOneHot { LC lo[16], hi[16]; };

ByteOneHot byte_one_hot(Builder& b, const LC& in) {
    ScopeGuard g(b, "ByteOneHot");
    const LC one = LC::constant(Fr::one());
    LCVec bits = num2bits(b, in, 8);
    ByteOneHot r;
    for (int half = 0; half < 2; ++half) {
        const LC* q = &bits[4 * half];
        LC* out = half ? r.hi : r.lo;
        LC p11 = b.mul(q[0], q[1]), r11 = b.mul(q[2], q[3]);
        const LC p[4] = {one - q[0] - q[1] + p11, q[0] - p11, q[1] - p11, p11};      // index = q0 + 2 q1
        const LC t[4] = {one - q[2] - q[3] + r11, q[2] - r11, q[3] - r11, r11};      // index = q2 + 2 q3
        LC sum;
        for (int j = 0; j < 15; ++j) { out[j] = b.mul(p[j & 3], t[j >> 2]); sum += out[j]; }
        out[15] = one - sum;
    }
    return r;
}

// [byte in cs] as a linear combination of products (hi-nibble set) x (lo-nibble set); products are shared per position
LC class_match(Builder& b, const ByteOneHot& oh, const CharSet& cs, std::map<std::pair<uint32_t, uint32_t>, LC>& cache) {
    std::map<uint32_t, uint32_t> by_mask;        // lo-nibble mask -> set of hi nibbles that have exactly this mask
    for (int h = 0; h < 16; ++h) {
        uint32_t mask = 0;
        for (int l = 0; l < 16; ++l) if (16 * h + l != 255 && cs.test(16 * h + l)) mask |= 1u << l;
        if (mask) by_mask[mask] |= 1u << h;
    }
    LC m;
    for (auto& kv : by_mask) {
        LC hs;
        for (int h = 0; h < 16; ++h) if (kv.second >> h & 1) hs += oh.hi[h];
        if (kv.first == 0xffffu) { m += hs; continue; }
        auto key = std::make_pair(kv.second, kv.first);
        auto it = cache.find(key);
        if (it == cache.end()) {
            LC ls;
            for (int l = 0; l < 16; ++l) if (kv.first >> l & 1) ls += oh.lo[l];
            it = cache.emplace(key, b.mul(hs, ls)).first;
        }
        m += it->second;
    }
    return m;
}

LCVec regex_circuit_compact(Builder& b, const Dfa& dfa, const LCVec& msg, uint32_t n_reveal = 1) {
    if (dfa.accept[0]) throw std::runtime_error("regex: matches the empty string");
    const PowerDfa pd = build_power(dfa);
    const int S = (int)pd.members.size();
    if (getenv("ZKE_REGEX_DEBUG")) {
        std::set<std::tuple<int, uint32_t, std::string>> groups;
        std::set<std::string> classes;
        for (auto& t : pd.trans) { groups.insert(std::make_tuple(t.dst, t.pub, t.cs.to_string())); classes.insert(t.cs.to_string()); }
        fprintf(stderr, "regex compact: %d DFA states, %d live sets, %zu transitions, %zu (dst, pub, class) groups, %zu classes\n",
                dfa.n_states, S, pd.trans.size(), groups.size(), classes.size());
    }
    const LC one = LC::constant(Fr::one());
    LCVec states(S);                       // exactly one of them is 1 at every position
    states[pd.after_marker] = one;
    LC accepted;                           // number of positions at which an accepting DFA state is live
    auto count_accepts = [&]() { for (int s = 0; s < S; ++s) if (pd.accept[s] && !states[s].is_zero()) accepted += states[s]; };
    count_accepts();
    LCVec out(1 + n_reveal * msg.size());
    // record for the device's automaton run (circuit.hpp: RegexSeed, mode 1): the chain runs through the `fire` products
    RegexSeed seed;
    std::map<std::tuple<int, uint32_t, std::string>, int> gid;           // (dst, public, class) -> product id, the same at every position
    for (auto& t : pd.trans) gid.emplace(std::make_tuple(t.dst, t.pub, t.cs.to_string()), (int)gid.size());
    bool seedable = S <= 255 && gid.size() <= 254 && msg.size() < (1u << 24);
    for (size_t j = 0; j < msg.size() && seedable; ++j) {
        Var v;
        if (msg[j].is_single_var(&v)) seed.bytes.push_back(v); else seedable = false;
    }
    if (seedable) {
        seed.mode = 1;
        seed.n_states = (uint32_t)S;
        seed.first_mask[0] = (uint64_t)pd.after_marker;
        seed.table.assign((size_t)S * 256, 0xff);
        seed.group.assign((size_t)S * 256, 0xff);
        for (auto& t : pd.trans) {
            const int g = gid[std::make_tuple(t.dst, t.pub, t.cs.to_string())];
            for (int c = 0; c < 256; ++c) if (t.cs.test(c)) { seed.table[(size_t)t.src * 256 + c] = (uint8_t)t.dst; seed.group[(size_t)t.src * 256 + c] = (uint8_t)g; }
        }
    }
    for (size_t i = 0; i < msg.size(); ++i) {
        const ByteOneHot oh = byte_one_hot(b, msg[i]);
        std::map<std::pair<uint32_t, uint32_t>, LC> cache;
        LCVec next(S), reveal(n_reveal);
        LC moved;
        // transitions that enter the same live set on the same class (and agree on `public`) share one product: the
        // states are one-hot, so the sum of their sources is itself 0 / 1
        std::map<std::tuple<int, uint32_t, std::string>, std::pair<LC, const CharSet*>> groups;
        for (auto& t : pd.trans) {
            if (states[t.src].is_zero()) continue;                   // live set statically unreachable at this position
            auto& gr = groups[std::make_tuple(t.dst, t.pub, t.cs.to_string())];
            gr.first += states[t.src];
            gr.second = &t.cs;
        }
        for (auto& kv : groups) {
            LC m = class_match(b, oh, *kv.second.second, cache);
            if (m.is_zero()) continue;
            const LC& src = kv.second.first;
            LC fire;
            {
                ScopeGuard g(b, "AND");
                fire = src.is_const() ? m * src.const_value() : b.mul(src, m);
            }
            Var fv;
            if (seedable && fire.is_single_var(&fv)) { seed.desc.push_back(fv); seed.desc.push_back((uint32_t)((i + 1) << 8) | (uint32_t)gid[kv.first]); }
            next[std::get<0>(kv.first)] += fire;
            moved += fire;
            for (uint32_t p = 0; p < n_reveal; ++p) if (std::get<1>(kv.first) >> p & 1) reveal[p] += fire;
        }
        next[0] = one - moved;                                       // no transition fired: only the fresh thread is live
        for (uint32_t p = 0; p < n_reveal; ++p)                       // reveal_p[i] <== in[i] * is_reveal
            out[1 + p * msg.size() + i] = reveal[p].is_zero() ? LC() : b.mul(msg[i], reveal[p]);
        states.swap(next);
        count_accepts();
    }
    if (accepted.is_zero()) throw std::runtime_error("regex: accept state unreachable for this length");
    out[0] = b.signal(one - is_zero(b, accepted));
    if (seedable && !seed.desc.empty()) b.add_regex_seed(std::move(seed));
    return out;
}

}  // namespace

LCVec body_hash_regex(Builder& b, const LCVec& msg) {
    ScopeGuard g(b, "BodyHashRegex");
    static const Dfa dfa = build_dfa({
        {"(\r\n|^)dkim-signature:", false},
        {"([a-z]+=[^;]+; )+bh=", false},
        {"[a-zA-Z0-9+/=]+", true},
        {";", false},
    });
    return b.regex_style ? regex_circuit_compact(b, dfa, msg) : regex_circuit(b, dfa, msg);
}

LCVec regex_match(Builder& b, const std::string& scope, const std::vector<std::pair<std::string, bool>>& parts, const LCVec& msg) {
    ScopeGuard g(b, scope.c_str());
    const Dfa dfa = build_dfa(parts);
    return b.regex_style ? regex_circuit_compact(b, dfa, msg) : regex_circuit(b, dfa, msg);
}

LCVec regex_match_reveals(Builder& b, const std::string& scope, const std::vector<std::pair<std::string, bool>>& parts, const LCVec& msg) {
    ScopeGuard g(b, scope.c_str());
    uint32_t n_public = 0;
    for (auto& p : parts) n_public += p.second ? 1 : 0;
    const Dfa dfa = build_dfa(parts, true);
    return b.regex_style ? regex_circuit_compact(b, dfa, msg, n_public) : regex_circuit(b, dfa, msg, n_public);
}

LCVec twitter_reset_regex(Builder& b, const LCVec& msg) {
    ScopeGuard g(b, "TwitterResetRegex");
    static const Dfa dfa = build_dfa({
        {"email was meant for @", false},
        {"[a-zA-Z0-9_]+", true},
    });
    return b.regex_style ? regex_circuit_compact(b, dfa, msg) : regex_circuit(b, dfa, msg);
}

}  // namespace gadgets
}  // namespace zke
