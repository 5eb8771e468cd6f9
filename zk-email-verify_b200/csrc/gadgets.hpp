// Template library: restatement of the circom templates on the EmailVerifier path.
// Every function cites the template it follows.  Paths are relative to /root/reference/packages/circuits/.
// circomlib 2.0.5 (un-vendored, pinned at /root/reference/yarn.lock:3619-3621) templates are restated
// from their published definitions; their call sites in the reference are cited.
#pragma once
#include "circuit.hpp"

namespace zke {
namespace gadgets {

typedef std::vector<LC> LCVec;

// ---- circomlib bitify / comparators / gates -------------------------------------------------
LCVec num2bits(Builder& b, const LC& in, uint32_t n);          // Num2Bits(n)        (sha.circom:27, rsa.circom:28)
LC bits2num(Builder& b, const LCVec& bits);                    // Bits2Num(n)        (email-verifier.circom:77)
LC is_zero(Builder& b, const LC& in);                          // IsZero()           (rsa.circom:154)
LC is_equal(Builder& b, const LC& x, const LC& y);             // IsEqual()          (utils/array.circom:28)
LC less_than(Builder& b, uint32_t n, const LC& x, const LC& y);     // LessThan(n)   (utils/array.circom:158)
LC greater_than(Builder& b, uint32_t n, const LC& x, const LC& y);  // GreaterThan(n) (utils/regex.circom:37)
LC less_eq_than(Builder& b, uint32_t n, const LC& x, const LC& y);  // LessEqThan(n) (lib/sha.circom:126)
LC gate_and(Builder& b, const LC& x, const LC& y);             // AND()              (lib/bigint.circom:39)
LC gate_or(Builder& b, const LC& x, const LC& y);              // OR()               (lib/bigint.circom:41)
LC multi_or(Builder& b, const LCVec& in);                      // 1 - IsZero(sum)    (zk-regex MultiOR)

// ---- circomlib sha256 ------------------------------------------------------------------------
// Sha256compression(): hin 8 words LSB-first, inp 512 bits MSB-first per word, out MSB-first per word.
LCVec sha256_compression(Builder& b, const LCVec& hin, const LCVec& inp);   // (lib/sha.circom:158,247)
LCVec sha256_iv_bits();                                                     // H(0..7), LSB-first per word (sha.circom:146-153)

// ---- circomlib poseidon ------------------------------------------------------------------------
// record: inputs are signals, and the instance gets a PoseidonBlock (circuit.hpp) for native evaluation
LC poseidon(Builder& b, const LCVec& inputs, bool record = false);          // Poseidon(n) (utils/hash.circom:38)
struct PoseidonParams {
    int t, r_f, r_p;
    std::vector<Fr> rc;                  // (r_f + r_p) * t round constants, round-major
    std::vector<std::vector<Fr>> mds;    // t x t
};
const PoseidonParams& poseidon_params(int t);                               // t = 2..17
// host-side Poseidon permutation on field elements (used by tests and by the helpers mirror)
Fr poseidon_hash(const std::vector<Fr>& inputs);

// ---- utils/ ----------------------------------------------------------------------------------
uint32_t log2_ceil(uint64_t a);                                             // utils/functions.circom:7-17
LC calculate_total(Builder& b, const LCVec& nums);                          // utils/array.circom:51-64
LC item_at_index(Builder& b, const LCVec& in, const LC& index);             // utils/array.circom:16-43
LCVec var_shift_left(Builder& b, const LCVec& in, const LC& shift, uint32_t max_out_len);  // utils/array.circom:111-141
void assert_zero_padding(Builder& b, const LCVec& in, const LC& start_index);              // utils/array.circom:149-164
LCVec pack_bits(Builder& b, const LCVec& in, uint32_t bits_per_element);    // utils/bytes.circom:194-210
LCVec byte_mask(Builder& b, const LCVec& in, const LCVec& mask);            // utils/bytes.circom:173-185
LCVec pack_bytes(Builder& b, const LCVec& in);                              // utils/bytes.circom:28-60 (31 bytes per field element, little-endian)
LCVec pack_regex_reveal(Builder& b, const LCVec& in, const LC& start_index, uint32_t max_reveal_len);  // utils/regex.circom:61-77
LCVec split_bytes_to_words(Builder& b, const LCVec& in, uint32_t n, uint32_t k);          // utils/bytes.circom:125-149
LCVec select_sub_array(Builder& b, const LCVec& in, const LC& start_index, const LC& length, uint32_t max_sub_len);  // utils/array.circom:78-98
LC check_substring_match(Builder& b, const LCVec& in, const LCVec& substring);             // utils/array.circom:193-217
LC count_substring_occurrences(Builder& b, const LCVec& in, const LCVec& substring);       // utils/array.circom:226-253
LCVec reveal_substring(Builder& b, const LCVec& in, const LC& start_index, const LC& length, uint32_t max_substring_len,
                       bool check_uniqueness);                                             // helpers/reveal-substring.circom:13-49
LC clean_email_address(Builder& b, const LCVec& encoded, const LCVec& decoded);            // utils/email.circom:16-139 (returns isValid)
LC email_nullifier(Builder& b, uint32_t bits_per_chunk, const LCVec& signature);           // helpers/email-nullifier.circom:14-23
LCVec select_regex_reveal(Builder& b, const LCVec& in, const LC& start_index, uint32_t max_reveal_len);  // utils/regex.circom:17-52
LC poseidon_large(Builder& b, uint32_t bits_per_chunk, const LCVec& in);    // utils/hash.circom:15-39
LC poseidon_modular(Builder& b, const LCVec& in, bool record = false);      // utils/hash.circom:49-83
LC remove_soft_line_breaks(Builder& b, const LCVec& encoded, const LCVec& decoded);   // helpers/remove-soft-line-breaks.circom:14-126 (returns isValid)
// root of a binary Poseidon(2) Merkle tree of depth siblings.size() (1..32) from a leaf, its index (bit l set: the node at
// level l is a right child; index < 2^depth is enforced) and the authentication path; each node hash is recorded
LC binary_merkle_root(Builder& b, const LC& leaf, const LC& index, const LCVec& siblings);
// a registry leaf bound to a domain: Poseidon(2)([Poseidon(9)(words zero-padded to 9), key_hash]), words = the packed
// domain (at most 9, PackBytes of at most 255 bytes); both hashes are recorded
LC domain_key_leaf(Builder& b, const LCVec& words, const LC& key_hash);

// ---- lib/ ------------------------------------------------------------------------------------
LCVec sha256_general(Builder& b, const LCVec& padded_in_bits, const LC& padded_in_length_bits,
                     const LCVec* pre_hash_bits);                           // lib/sha.circom:89-203, 212-292
LCVec sha256_bytes(Builder& b, const LCVec& padded_in, const LC& padded_in_length);        // lib/sha.circom:17-38
LCVec sha256_bytes_partial(Builder& b, const LCVec& padded_in, const LC& padded_in_length,
                           const LCVec& pre_hash);                          // lib/sha.circom:47-80
LC big_less_than(Builder& b, uint32_t n, const LCVec& x, const LCVec& y);   // lib/bigint.circom:16-60
void check_carry_to_zero(Builder& b, uint32_t n, uint32_t m, const LCVec& in);             // lib/bigint.circom:69-94
LCVec fp_mul(Builder& b, uint32_t n, uint32_t k, const LCVec& x, const LCVec& y, const LCVec& p);  // lib/fp.circom:16-81
LCVec fp_pow65537_mod(Builder& b, uint32_t n, uint32_t k, const LCVec& base, const LCVec& modulus);  // lib/rsa.circom:57-92
LCVec rsa_pad(Builder& b, uint32_t n, uint32_t k, const LCVec& modulus, const LCVec& message);     // lib/rsa.circom:101-181
void rsa_verifier65537(Builder& b, uint32_t n, uint32_t k, const LCVec& message, const LCVec& signature,
                       const LCVec& modulus);                               // lib/rsa.circom:13-46
LC base64_lookup(Builder& b, const LC& in);                                 // lib/base64.circom:71-128
LCVec base64_decode(Builder& b, uint32_t byte_length, const LCVec& in);     // lib/base64.circom:14-64

// ---- @zk-email/zk-regex-circom body_hash_regex (un-vendored; call site email-verifier.circom:126) ----
// out[0] = match flag, out[1..] = reveal bytes (msg[i] inside the bh= value, else 0)
LCVec body_hash_regex(Builder& b, const LCVec& msg);
// zk-regex circuit of an arbitrary decomposed regex: parts = {(regex, is_public)...}; same output layout
LCVec regex_match(Builder& b, const std::string& scope, const std::vector<std::pair<std::string, bool>>& parts, const LCVec& msg);
// `email was meant for @(\w+)` with the user name public - the body regex of the Proof-of-Twitter circuit
// (selector string: docs/zk-email-docs/UsageGuide/README.md:84; the circuit itself is not in the reference tree)
LCVec twitter_reset_regex(Builder& b, const LCVec& msg);

// ---- email-verifier.circom:42-174 ------------------------------------------------------------
struct EmailVerifierParams {
    uint32_t max_headers_length = 1024, max_body_length = 1536, n = 121, k = 17;
    bool ignore_body_hash_check = false, enable_header_masking = false, enable_body_masking = false;
    bool remove_soft_line_breaks = false;
    bool public_pubkey = false;   // `component main { public [pubkey] }` as in tests/test-circuits/email-verifier-test.circom:5
    // Proof-of-Twitter wrapper (BASELINE configs[3]; public signals as in packages/rust-verifier/tests/data/
    // proof_of_twitter/public.json: [pubkeyHash, twitterUsername, address]): EmailVerifier as a sub-component whose
    // shaHi / shaLo stay internal, plus the body regex, PackRegexReveal(maxBodyLength, 21) and a public `address` input
    bool twitter = false;
    int regex_style = -1;         // -1: Builder default (ZKE_REGEX_STYLE); 0 zk-regex shape; 1 compact shape (regex.cpp)
};
Circuit build_email_verifier(const EmailVerifierParams& p, bool materialize_linear = true);

// zk-regex circuit with one reveal array per public part: out = [match, reveal of public part 0 (msg.size()), reveal of
// public part 1, ...] (regex_match ORs every public part into one reveal array)
LCVec regex_match_reveals(Builder& b, const std::string& scope, const std::vector<std::pair<std::string, bool>>& parts, const LCVec& msg);

// ---- email app circuits: EmailVerifier + the app's regexes, revealed substrings and public inputs ----------------------
// The circuit a zk-email app writes by hand (docs/zk-email-docs/UsageGuide/README.md: write the regex, wrap EmailVerifier,
// reveal what it matched), built from a description.  TwitterVerifier is the app {body regex twitterUsername, external
// input address, exposeHeaderHash = false}; EmailVerifier is the app with nothing added.
// reveal (public parts): the packed bytes as outputs (PackRegexReveal), one output PoseidonModular(packed bytes) (hash), or
// one output Poseidon(2)([that hash, salt]) with `salt` a private one-element external input (commit)
enum AppReveal { REVEAL_BYTES = 0, REVEAL_HASH = 1, REVEAL_COMMIT = 2 };
struct AppRegexPart {
    std::string regex;
    bool is_public = false;
    uint32_t max_length = 0;           // public parts
    int reveal = REVEAL_BYTES;
    bool reveal_given = false;         // the spec named a reveal (refused on a part that is not public)
    std::string salt;                  // REVEAL_COMMIT: the external input holding the salt
};
struct AppRegex {
    std::string name;
    bool body = false;                 // search emailBody (decodedEmailBodyIn with removeSoftLineBreaks), else emailHeader
    std::vector<AppRegexPart> parts;
    std::string scope;                 // scope of its constraints (default: name)
};
struct AppExternalInput {
    std::string name;
    uint32_t max_length = 0;           // 0: one field element, else PackBytes layout
    bool is_public = true;             // private inputs follow the start indices of the public parts
};
struct AppSpec {
    EmailVerifierParams ev;            // ev.twitter is ignored
    bool expose_header_hash = true;
    std::vector<AppRegex> regexes;
    std::vector<AppExternalInput> external_inputs;
    bool email_nullifier = false;
    std::string scope = "EmailApp";    // scope of everything after pubkeyHash
    // 1..32: pubkeyHash stays private and is proven a leaf of a Merkle registry of keys; the output registryRoot takes
    // its place, the private inputs registryIndex and registrySiblings[depth] come last.  0: no registry
    uint32_t key_registry_depth = 0;
    // with a registry: the output name of a public header regex part (maxLength <= 255) whose matched bytes D bind the
    // leaf to a domain, leaf = domain_key_leaf(D's packed words, pubkeyHash).  Empty: the leaf is pubkeyHash
    std::string key_domain;
};
Circuit build_email_app(const AppSpec& spec, bool materialize_linear = true);

}  // namespace gadgets
}  // namespace zke
