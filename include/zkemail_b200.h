/*
 * zkemail_b200.h - C ABI of the H100-native EmailVerifier witness + Groth16 proving engine.
 *
 * This is the drop-in boundary (SURVEY.md section 8(b)).  It replaces, for the EmailVerifier path, what the
 * reference reaches through
 *     snarkjs.groth16.fullProve(input, wasm, zkey)   /root/reference/packages/helpers/src/chunked-zkey.ts:80-84
 *     snarkjs.groth16.verify(vkey, publicSignals, proof)   /root/reference/packages/helpers/src/chunked-zkey.ts:101
 * and, at test time, the circom_tester verbs
 *     wasm_tester(circuit) / calculateWitness / checkConstraints / assertOut
 *                                                 /root/reference/packages/circuits/tests/email-verifier.test.ts:21-44,204
 *
 * Conventions
 *   - Field elements cross the ABI as 32-byte little-endian integers in standard (non-Montgomery) form,
 *     the same image as a `.wtns` entry (SURVEY 8(b), data formats).
 *   - All buffers are caller-owned host memory; contexts own device memory.  No torch / C++ types.
 *   - Return codes: 0 ok; > 0 per-item failure (e.g. a witness that violates a constraint: the message
 *     contains "Assert Failed", the string the reference's tests match, email-verifier.test.ts:78);
 *     < 0 fatal (bad arguments, CUDA failure, library built without a device).
 *   - `err`/`errcap`: optional message buffer, always NUL-terminated when errcap > 0.
 */
#ifndef ZKEMAIL_B200_H
#define ZKEMAIL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct zke_circuit zke_circuit; /* R1CS + levelised witness program (the ".r1cs + .wasm" pair) */
typedef struct zke_zkey zke_zkey;       /* Groth16 proving + verification key (the ".zkey")           */
typedef struct zke_ctx zke_ctx;         /* circuit + zkey resident on one GPU, with work buffers       */

#define ZKE_FR_BYTES 32

/* ---------------------------------------------------------------------------------------------------
 * Circuits.  Replaces "circom file -> r1cs + witness calculator" (wasm_tester(...) in
 * /root/reference/packages/circuits/tests/email-verifier.test.ts:21-31).
 * `template_name` is a template of /root/reference/packages/circuits (e.g. "EmailVerifier", "Sha256Bytes",
 * "RSAVerifier65537", "FpMul", "Base64Lookup", ...); `params` are its circom template parameters in order.
 * For "EmailVerifier": {maxHeadersLength, maxBodyLength, n, k, ignoreBodyHashCheck, enableHeaderMasking,
 * enableBodyMasking, removeSoftLineBreaks, publicPubkey(0/1: `component main { public [pubkey] }`)}.
 * ------------------------------------------------------------------------------------------------- */
zke_circuit* zke_circuit_build(const char* template_name, const int64_t* params, size_t n_params,
                               char* err, size_t errcap);
/* zk-regex circuit of an arbitrary decomposed regex (the generator behind BodyHashRegex; un-vendored
 * @zk-email/zk-regex-circom, call site /root/reference/packages/circuits/email-verifier.circom:5,126):
 * `parts[i]` is a regex fragment, `is_public[i]` != 0 marks the fragment whose matched bytes are revealed.
 * Signals: input msg[msg_len], outputs out (match flag) and reveal0[msg_len]. */
zke_circuit* zke_circuit_build_regex(const char* const* parts, const uint8_t* is_public, size_t n_parts, uint32_t msg_len,
                                     char* err, size_t errcap);
/* An email app circuit from a JSON spec (the "write the regex, wrap EmailVerifier, reveal what it matched" recipe of the
 * zk-email usage guide): the EmailVerifier body with its flags (maxHeadersLength,
 * maxBodyLength, n, k, ignoreBodyHashCheck, enableHeaderMasking, enableBodyMasking, removeSoftLineBreaks, publicPubkey,
 * regexStyle) plus exposeHeaderHash (default true: shaHi / shaLo are outputs), then per entry of `regexes` ({name,
 * location: "header" | "body", parts: [{regexDef, isPublic, maxLength}]}) a regex that must match and, per public part, a
 * PackRegexReveal output (`name`, or `name0`, `name1`, ... for several public parts) with its private index input
 * (`nameIndex` / `name0Index`, ...); `externalInputs` ([{name, maxLength?}]) are public inputs, one field element or
 * ceil(maxLength / 31) packed ones; `emailNullifier` adds the EmailNullifier output.  `keyRegistryDepth` d (1..32; 0 or
 * absent: no registry) hides the signing key: pubkeyHash stays private and is proven a leaf of a Poseidon(2) Merkle tree
 * of depth d (zke_merkle_build), whose root `registryRoot` is published in pubkeyHash's place; the private inputs
 * registryIndex and registrySiblings[d] come last.  It is refused with publicPubkey, and the three names are then
 * reserved.  `keyDomain` (with keyRegistryDepth) names the output of a public header regex part of maxLength <= 255
 * whose matched bytes D bind the leaf to a domain: the leaf is Poseidon(2)([Poseidon(9)(D's packed words, zero-padded to
 * 9), pubkeyHash]) (zke_domain_key_leaves) instead of pubkeyHash; it adds no signal.  Signal order: outputs (pubkeyHash or registryRoot, shaHi, shaLo, masks, regex outputs, emailNullifier),
 * public inputs (external inputs, pubkey if public), the EmailVerifier inputs, the index inputs, private external inputs,
 * then registryIndex and registrySiblings.  A malformed spec is refused with a message naming the field. */
zke_circuit* zke_circuit_build_app(const char* spec_json, char* err, size_t errcap);
void zke_circuit_free(zke_circuit* c);
/* circom's constraint system: an iden3 `.r1cs` image (what `circom --r1cs` writes and `snarkjs r1cs info` / `snarkjs groth16
 * setup` read, /root/reference/docs/zk-email-docs/UsageGuide/README.md steps 3-5; layout in r1cs.cpp), BN254 only.  The
 * circuit holds the constraints in file order (duplicate wires and zero coefficients kept) and no witness program:
 * zke_witness, zke_fullprove, zke_fullprove_submit, zke_upload_inputs, zke_pack_inputs_json and zke_fullprove_json refuse
 * it, witnesses come in through zke_load_witness / zke_wtns_prove.  Key setup, contributions, key checks and proving take
 * it like any other circuit.  The image may be a memory-mapped file; nothing of it is kept. */
zke_circuit* zke_circuit_from_r1cs(const void* r1cs, size_t len, char* err, size_t errcap);
/* The circuit as an `.r1cs` image (sections 1, 2, 3; the labels read with the circuit, else the identity map).  out == NULL:
 * returns the size needed; -2 if cap is too small; < 0 on error. */
int64_t zke_circuit_write_r1cs(const zke_circuit* c, uint8_t* out, size_t cap);

typedef struct zke_circuit_info {
    uint32_t n_vars;        /* witness length m, w[0] = 1 */
    uint32_t n_temps;       /* scratch slots used by the witness program (not part of the witness) */
    uint32_t n_outputs, n_pub_inputs, n_prv_inputs;
    uint32_t n_public;      /* snarkjs nPublic = n_outputs + n_pub_inputs */
    uint32_t n_constraints;
    uint32_t n_levels;      /* dependency depth of the witness program */
    uint32_t n_ops;
    uint32_t n_coefs;
    uint32_t domain_log2;   /* Groth16 evaluation domain: 2^domain_log2 >= n_constraints + n_public + 1 */
    uint32_t n_groups;      /* named signal groups (outputs and inputs) */
    uint64_t nnz_a, nnz_b, nnz_c;
} zke_circuit_info;
int zke_circuit_get_info(const zke_circuit* c, zke_circuit_info* out);

/* Named signals (the .sym role for main's inputs/outputs; circom_tester assertOut / snarkjs input JSON keys).
 * kind: 0 output, 1 public input, 2 private input.  `first` is the witness index of element 0. */
int zke_circuit_group(const zke_circuit* c, uint32_t index, char* name, size_t namecap,
                      uint32_t* first, uint32_t* count, int* kind);
/* Index (into the packed input vector, i.e. witness index - 1 - n_outputs) of a named input; < 0 if absent. */
int64_t zke_circuit_input_offset(const zke_circuit* c, const char* name, uint32_t* count);

/* Raw read-only views of the flat circuit arrays (for exporters and for the test oracle).  `which`: */
enum {
    ZKE_ARR_COEFS = 0,      /* uint8[n_coefs][32]  interned coefficients, standard form, LE            */
    ZKE_ARR_A_PTR = 1, ZKE_ARR_A_VAR = 2, ZKE_ARR_A_COEF = 3,     /* uint32 CSR of matrix A            */
    ZKE_ARR_B_PTR = 4, ZKE_ARR_B_VAR = 5, ZKE_ARR_B_COEF = 6,
    ZKE_ARR_C_PTR = 7, ZKE_ARR_C_VAR = 8, ZKE_ARR_C_COEF = 9,
    ZKE_ARR_OPS = 10,       /* uint32[n_ops][5] = {code, dst, a, b, c}, sorted by level               */
    ZKE_ARR_LEVEL_PTR = 11, /* uint32[n_levels + 1]                                                   */
    ZKE_ARR_LC_PTR = 12, ZKE_ARR_LC_VAR = 13, ZKE_ARR_LC_COEF = 14, /* LC pool of the witness program */
    ZKE_ARR_AUX = 15,       /* uint32 operands of OP_FPMUL                                            */
    ZKE_ARR_SCOPE_OF_CONSTRAINT = 16, /* uint16[n_constraints]                                        */
    ZKE_ARR_SHA_BLOCKS = 17, /* uint32: {n_blocks, per block: var_begin, var_end, temp_begin, temp_end, n_desc,
                               inputs[768], desc[n_desc][2] = {signal, quantity << 8 | bit}} - the Sha256compression
                               instances the engine evaluates natively (one compression instead of ~320 levels)  */
    ZKE_ARR_REGEX_SEEDS = 18,/* uint32: {n_seeds, per seed: n_desc, n_bytes, n_states | wide << 30 | mode << 31,
                               first_mask lo, hi (wide = zk-regex shape with 65..255 states: 8 words, the 256-bit live set
                               from its low word up), bytes[n_bytes] (signal of message byte j), table[n_states * 64] (destination state of
                               (source, byte), 0xff = none, 4 per word), mode 1 (compact shape): group[n_states * 64] (the
                               product that fires), desc[n_desc][2] = {signal, position << 8 | state or product}} - the
                               regex instances whose chained signals the engine seeds with one automaton run      */
    ZKE_ARR_POSEIDON_BLOCKS = 19 /* uint32: {n_blocks, per block: t, var_begin, var_end, temp_begin, temp_end, n_desc,
                               inputs[t - 1], desc[n_desc][2] = {signal, round << 16 | lane << 8 | kind}}, kind 0 input copy,
                               1 x^2, 2 x^4, 3 x^5 (the S-box of round `round`), 4 mix output of round `round` - the Poseidon
                               instances of hashed and committed app outputs, which the engine evaluates natively (one
                               permutation instead of ~4 levels per round)                                          */
};
const void* zke_circuit_array(const zke_circuit* c, int which, size_t* n_elems);
const char* zke_circuit_scope_name(const zke_circuit* c, uint32_t scope_index);

/* What the engine's lowering of the witness program builds for this circuit (the stream the witness kernel walks: the native
 * SHA-256 and regex-seeding substitutions, levels cut into iterations of 512 records and padded to rounds of `cluster`
 * iterations), computed on the host - no device needed.  zke_ctx_open lowers with the same code; its options come from
 * ZKE_NATIVE_SHA, ZKE_NATIVE_REGEX, ZKE_COOP_FPMUL, ZKE_NATIVE_POSEIDON (default 1 each) and ZKE_WITNESS_CLUSTER (default: chosen from max_batch).
 * cluster: 1, 2, 4 or 8.  level_ops (optional, may be NULL): the first min(n_levels, level_cap) entries receive the number of
 * records of each level that are not cooperative ops.  A circuit read from an `.r1cs` has no program: an error.
 * Returns 0, or non-zero with a message in err. */
typedef struct zke_program_stats {
    uint32_t n_levels;      /* dependency depth after the substitutions */
    uint32_t n_iters;       /* iterations of 512 records, padding iterations included */
    uint32_t n_ops_kept;    /* records that are not cooperative ops (the sum of level_ops) */
    uint32_t n_coop_ops;    /* cooperative ops: native SHA-256 blocks, regex seeds, FpMul hints */
    uint32_t n_terms;       /* linear-combination terms of the stream, alignment padding included */
    uint32_t cluster;
    uint64_t digest;        /* 64-bit FNV-1a over the stream's five arrays (op records, iteration headers, terms, aux table,
                               cooperative ops, in that order): per array its word count as 8 little-endian bytes, then its
                               32-bit words as 4 little-endian bytes each */
} zke_program_stats;
int zke_circuit_program_stats(const zke_circuit* c, int native_sha, int native_regex, int coop_fpmul, uint32_t cluster,
                              zke_program_stats* out, uint32_t* level_ops, size_t level_cap, char* err, size_t errcap);
/* The same with every lowering option as a flag (zke_circuit_program_stats lowers with native Poseidon on).  The engine's
 * native Poseidon follows ZKE_NATIVE_POSEIDON (default 1). */
enum {
    ZKE_LOWER_NATIVE_SHA = 1, ZKE_LOWER_NATIVE_REGEX = 2, ZKE_LOWER_COOP_FPMUL = 4, ZKE_LOWER_NATIVE_POSEIDON = 8,
    ZKE_LOWER_ALL = 15
};
int zke_circuit_program_stats_ex(const zke_circuit* c, uint32_t flags, uint32_t cluster, zke_program_stats* out,
                                 uint32_t* level_ops, size_t level_cap, char* err, size_t errcap);

/* Poseidon(n) of n = 1..16 field elements (32-byte little-endian, each below r) into out[32]: circomlib's parameters, the
 * permutation the circuits constrain (the `poseidon` of @zk-email/helpers).  Returns 0, -1 for a bad n or pointer, -2 for an
 * input not below r. */
int zke_poseidon_hash(const uint8_t* inputs, size_t n, uint8_t* out);

/* Merkle registry of DKIM keys, on the GPU (registry.cu).  Field elements are 32-byte little-endian.  Without a device
 * these return the library's "no CUDA device available (this library has no CPU fallback)" error; argument refusals
 * come first.  Each returns < 0 with a message in err on a refusal.
 * zke_poseidon_batch: out[count][32] = Poseidon(width)(inputs[i][0..width-1]) for width 1..16, the values of
 *   zke_poseidon_hash; an input not below r is refused, naming its instance.  Returns 0.
 * zke_pubkey_hashes: the pubkeyHash of each of `count` RSA moduli (modulus_bytes each, little-endian): k limbs of n
 *   bits, merged in pairs as PoseidonLarge does, through Poseidon(ceil(k / 2)).  Refuses k outside 17..32, 2n >= 251
 *   and a modulus >= 2^(n k).  Returns 0.
 * zke_domain_key_leaves: the domain-bound leaf of each of `count` (domain, modulus) pairs, Poseidon(2)([domainHash,
 *   pubkeyHash]) with domainHash = Poseidon(9) of the domain's 9 packed words (PackBytes(D, 255)).  `domains` holds
 *   count rows of 255 bytes: the name, lower-case ASCII without a trailing dot, then zero padding.  Refuses what
 *   zke_pubkey_hashes refuses, and an empty row, a zero byte inside the name, a byte >= 0x80 or in A-Z, and a trailing
 *   dot, naming the first such row.  Returns 0.
 * zke_merkle_build: every level of the tree of depth 1..32 over count <= 2^depth leaves (below r), node hash
 *   H(l, r) = Poseidon(2)([l, r]).  Level l holds ceil(count / 2^l) nodes, a missing right child at level l is
 *   zeros[l] (zeros[0] = 0, zeros[l + 1] = H(zeros[l], zeros[l])); levels are written one after the other from the
 *   leaves (level 0) to the root.  Returns the bytes written, the size needed when levels == NULL, -2 if cap is too small.
 * zke_registry_open: the tree of zke_merkle_build (same refusals and messages), kept resident on `device` for in-place
 *   updates; NULL with a message in err on a refusal.  A handle is used by one host thread at a time.
 * zke_registry_update: sets leaf indices[i] to leaves[i] for i < k.  An index below the count replaces a leaf (a leaf of
 *   0 revokes it: zeros[0] = 0, so revoking the last leaves gives the root of the tree without them); indices at or above
 *   the count append and must be exactly count .. count + a - 1, in any order.  Refuses a leaf not below r (naming its
 *   position in the update), a duplicate index, a gap and a count above 2^depth, all before any device write: a
 *   refused update leaves the tree unchanged.  Rehashes only the ancestors of the updated leaves, so every level equals
 *   zke_merkle_build's over the resulting leaves.  k = 0 does nothing.  Returns 0.
 * zke_registry_nodes: out[k][32] = node indices[i] of level levels[i] (level 0 = the leaves), zeros[level] past the
 *   level's size; refuses level > depth and index >= 2^(depth - level).  Authentication paths are the nodes
 *   (l, (i >> l) ^ 1) for l < depth.  Returns 0.
 * zke_registry_levels: every level, in zke_merkle_build's layout and size rules (the size needed when out == NULL, -2
 *   if cap is too small).
 * zke_registry_count: the number of leaves (0 for NULL).  zke_registry_close frees the handle (NULL is ignored).
 * zke_registry_device_ms: device time of the calling thread's last successful call above (CUDA events around its kernels,
 *   around the copy for zke_registry_levels). */
typedef struct zke_registry zke_registry;     /* a registry tree resident on one GPU */
int zke_poseidon_batch(const uint8_t* inputs, uint32_t width, size_t count, int device, uint8_t* out, char* err, size_t errcap);
int zke_pubkey_hashes(const uint8_t* moduli, size_t count, uint32_t modulus_bytes, uint32_t n, uint32_t k, int device,
                      uint8_t* out, char* err, size_t errcap);
int zke_domain_key_leaves(const uint8_t* moduli, size_t count, uint32_t modulus_bytes, uint32_t n, uint32_t k,
                          const uint8_t* domains, int device, uint8_t* out, char* err, size_t errcap);
int64_t zke_merkle_build(const uint8_t* leaves, size_t count, uint32_t depth, int device, uint8_t* levels, size_t cap,
                         char* err, size_t errcap);
zke_registry* zke_registry_open(const uint8_t* leaves, size_t count, uint32_t depth, int device, char* err, size_t errcap);
int zke_registry_update(zke_registry* r, const uint64_t* indices, const uint8_t* leaves, size_t k, char* err, size_t errcap);
int zke_registry_nodes(zke_registry* r, const uint32_t* levels, const uint64_t* indices, size_t k, uint8_t* out,
                       char* err, size_t errcap);
int64_t zke_registry_levels(zke_registry* r, uint8_t* out, size_t cap, char* err, size_t errcap);
uint64_t zke_registry_count(const zke_registry* r);
void zke_registry_close(zke_registry* r);
double zke_registry_device_ms(void);


/* ---------------------------------------------------------------------------------------------------
 * Proving key.  zke_setup() is a TOY trusted setup (`snarkjs groth16 setup` role,
 * /root/reference/docs/zk-email-docs/UsageGuide/README.md:139-153): tau, alpha, beta, gamma, delta are derived
 * from `seed`, i.e. the toxic waste is known - benchmark / test keys only.  The field side runs on the host, the
 * ~5m + N fixed-base scalar multiplications on GPU `device`; the key stays resident on that GPU.
 * ------------------------------------------------------------------------------------------------- */
zke_zkey* zke_setup(const zke_circuit* c, uint64_t seed, int device, char* err, size_t errcap);
/* Real proving keys: an iden3 `.zkey` (Groth16, BN254) as produced by `snarkjs groth16 setup` / `zkey contribute` -
 * the third argument of snarkjs.groth16.fullProve(input, wasm, zkey)
 * (/root/reference/packages/helpers/src/chunked-zkey.ts:80-84) and the first of `snarkjs groth16 prove zkey wtns`
 * (/root/reference/docs/zk-email-docs/UsageGuide/README.md:139-195).  Sections 2-9 are validated (field moduli, every
 * point on its curve) and made resident on GPU `device`: points as they are stored (affine, Montgomery), the A / B
 * coefficient matrices of section 4 as CSR, the H points with their fixed-base table.
 * zke_zkey_load_chunks takes the fork's chunked form: chunk i holds section i + 1, i.e. the files `${name}.zkeyb` ..
 * `${name}.zkeyk` (chunked-zkey.ts:9,35-37); n_chunks >= 9 (section 10, the contribution log, is not needed). */
zke_zkey* zke_zkey_load(const void* zkey_bytes, size_t len, int device, char* err, size_t errcap);
zke_zkey* zke_zkey_load_chunks(const void* const* chunks, const size_t* lens, size_t n_chunks, int device, char* err, size_t errcap);
/* Writes the key as a `.zkey` file image.  `c` supplies the coefficient section for keys made by zke_setup (pass NULL
 * for loaded keys, which carry their own).  out == NULL: returns the size needed; < 0 on error. */
int64_t zke_zkey_write(const zke_zkey* z, const zke_circuit* c, uint8_t* out, size_t cap);
/* 1 if the key came from zke_setup (toxic waste known - anyone can forge proofs for it), 0 for a loaded key. */
int zke_zkey_is_toy(const zke_zkey* z);
void zke_zkey_free(zke_zkey* z);
int zke_zkey_info(const zke_zkey* z, uint32_t* n_vars, uint32_t* n_public, uint32_t* domain_log2);
/* zkey sections (iden3 .zkey numbering where one exists: 3 IC, 5 A, 6 B1, 7 B2, 8 C/"L", 9 H; header points apart). */
enum {
    ZKE_SEC_ALPHA1 = 101, ZKE_SEC_BETA1 = 102, ZKE_SEC_DELTA1 = 103,
    ZKE_SEC_BETA2 = 104, ZKE_SEC_GAMMA2 = 105, ZKE_SEC_DELTA2 = 106,
    ZKE_SEC_IC = 3, ZKE_SEC_A = 5, ZKE_SEC_B1 = 6, ZKE_SEC_B2 = 7, ZKE_SEC_C = 8, ZKE_SEC_H = 9
};
/* Copies a section to host memory as affine points, standard-form LE coordinates (G1 64 bytes: x,y;
 * G2 128 bytes: x.c0,x.c1,y.c0,y.c1; infinity = zeros).  Returns the number of points (with out == NULL: just the
 * count), < 0 on error.  Sections A/B1/B2/C have n_vars entries (C is infinity for the public signals). */
int64_t zke_zkey_section(const zke_zkey* z, int section, uint8_t* out, size_t cap);

/* ---------------------------------------------------------------------------------------------------
 * Keys from a Powers-of-Tau file (`snarkjs groth16 setup` / `zkey new`, then `zkey contribute`; the route of
 * /root/reference/docs/zk-email-docs/UsageGuide/README.md:149-180), for this engine's own R1CS.
 * ------------------------------------------------------------------------------------------------- */
/* A prepared phase-2 `.ptau` image (layout in setup.cu) -> key with gamma = delta = 1 on GPU `device`: the sums of
 * Lagrange-basis points of every signal, computed on the GPU.  The file must hold the Lagrange bases of size 2^(domain_log2 + 1);
 * every point used is validated.  Such a key reports zke_zkey_is_toy = 1 (anyone can forge proofs while delta = 1) until
 * zke_zkey_contribute is applied. */
zke_zkey* zke_zkey_from_ptau(const zke_circuit* c, const void* ptau, size_t len, int device, char* err, size_t errcap);
/* Host-only structure check of a `.ptau` image (magic, modulus, every section size against its power and, with c != NULL,
 * that it is large enough for c): power, and per section type < 16 its payload offset and size in the file (0 if absent). */
int zke_ptau_info(const zke_circuit* c, const void* ptau, size_t len, uint32_t* power, uint64_t* offsets16, uint64_t* sizes16,
                  char* err, size_t errcap);
/* Wall time of this thread's last zke_zkey_from_ptau: host part (parse, transpose) and device part (upload, sums, H table). */
int zke_zkey_from_ptau_timing(double* host_ms, double* gpu_ms);
/* Phase-2 contribution with secret s (32 bytes LE, 1 < s < r): a NEW key with delta1, delta2 times s and the C ("L") and H
 * points times s^-1; everything else copied.  Not a snarkjs transcript: the result can be contributed to again here, not by
 * snarkjs.  A contribution to a zke_zkey_from_ptau key makes it a real key (is_toy 0); one to a zke_setup key stays a toy. */
zke_zkey* zke_zkey_contribute(const zke_zkey* prev, const uint8_t* secret32, char* err, size_t errcap);
/* The ratio check of `snarkjs zkey verify`: 1 if `next` follows from `prev` by contributions (header, IC, A, B1, B2 and the
 * coefficient matrices identical; e(delta1', G2) == e(G1, delta2'); e(X', delta2') == e(X, delta2) for X a random 128-bit
 * combination of the L and H points, weights derived from rand16, or /dev/urandom when NULL), 0 if not with the reason in
 * err, < 0 on errors.  Both keys must live on one device. */
int zke_zkey_check_contribution(const zke_zkey* prev, const zke_zkey* next, const uint8_t* rand16, char* err, size_t errcap);
/* TOY prepared `.ptau` image from KNOWN tau, alpha, beta (3 x 32 bytes LE, in [1, r)) - tests and measurement only, like
 * zke_setup.  out == NULL: returns the size needed; -2 if cap is too small; < 0 on error. */
int64_t zke_ptau_toy(uint32_t power, const uint8_t* tau_alpha_beta96, int device, uint8_t* out, size_t cap, char* err, size_t errcap);

/* Phase 1 of the Powers-of-Tau ceremony (ptau.cu).  An UNPREPARED image holds sections 1-7, a PREPARED one also 12-15.
 * Every writer returns the bytes written, the size needed when out == NULL, -2 if cap is too small, -1 on error.
 * `snarkjs powersoftau new`: unprepared image of `power` (in [1, 28]) with every point the generator.  Host only. */
int64_t zke_ptau_new(uint32_t power, uint8_t* out, size_t cap, char* err, size_t errcap);
/* `snarkjs powersoftau contribute` with secrets (tau, alpha, beta) (3 x 32 bytes LE, each in [2, r); NULL: drawn from
 * /dev/urandom): tauG1[i], tauG2[i] times tau^i, alphaTauG1[i] times alpha tau^i, betaTauG1[i] times beta tau^i, betaG2
 * times beta.  Input points are validated on the device.  The output is unprepared; sections 1 and 7 are copied byte for
 * byte and the contribution is not recorded in section 7 (no snarkjs transcript).  receipt384 (may be NULL) receives
 * [tau]_2, [alpha]_2, [beta]_2, the public part of the contribution that zke_ptau_verify checks. */
int64_t zke_ptau_contribute(const void* ptau, size_t len, const uint8_t* secrets96, int device, uint8_t* out, size_t cap, uint8_t* receipt384,
                            char* err, size_t errcap);
/* `snarkjs powersoftau prepare phase2`: an unprepared image plus sections 12-15, the Lagrange bases of the domains 1, 2, ...,
 * 2^power computed by inverse transforms of curve points on the device.  A power whose largest transform does not fit in
 * the device's free memory is refused before anything is allocated. */
int64_t zke_ptau_prepare(const void* ptau, size_t len, int device, uint8_t* out, size_t cap, char* err, size_t errcap);
/* Wall time of this thread's last zke_ptau_prepare: the three G1 families and the G2 family. */
int zke_ptau_prepare_timing(double* g1_ms, double* g2_ms);
/* The algebraic part of `snarkjs powersoftau verify` on an unprepared or prepared image: points valid (G2 in the order-r
 * subgroup), generators at index 0, consecutive powers of one tau in every family, the Lagrange sections (if present) the
 * bases of the powers and, with prev and receipt384 (both or neither), that the file is prev's after the contribution the
 * receipt describes.  Weights derived from rand16 (NULL: /dev/urandom).  1 ok, 0 rejected with the reason in err, < 0 on error. */
int zke_ptau_verify(const void* ptau, size_t len, const void* prev, size_t prev_len, const uint8_t* receipt384, const uint8_t* rand16,
                    int device, char* err, size_t errcap);

/* ---------------------------------------------------------------------------------------------------
 * Contexts: circuit (+ optional proving key) resident on one GPU with work buffers for `max_batch` emails.
 * One host thread per context (or external locking).  All calls are synchronous at the ABI.
 * ------------------------------------------------------------------------------------------------- */
/* `c` may be NULL when the key was loaded from a `.zkey`: such a context proves externally computed witnesses
 * (zke_load_witness / zke_wtns_prove + zke_prove) from the key's own coefficient matrices.  With a circuit read from an
 * `.r1cs` and a key that carries coefficient matrices (loaded from a `.zkey`, or made by zke_zkey_from_ptau), the key's A and
 * B must equal the circuit's as linear forms ("zkey does not belong to this circuit: A row i differs" otherwise). */
zke_ctx* zke_ctx_open(const zke_circuit* c, const zke_zkey* zkey_or_null, int device, uint32_t max_batch,
                      char* err, size_t errcap);
void zke_ctx_close(zke_ctx* x);
void* zke_ctx_stream(const zke_ctx* x);      /* the cudaStream_t all of the context's work is enqueued on */
uint64_t zke_kernel_launches(void);          /* kernels launched by this library since it was loaded */

/* Copies a batch of packed inputs into the context's device buffer; a later zke_witness / zke_fullprove call with
 * inputs == NULL uses them (lets a benchmark start its timed region with the inputs already resident in HBM). */
int zke_upload_inputs(zke_ctx* x, const uint8_t* inputs, size_t batch, char* err, size_t errcap);

/* Optional per-stage device timing (CUDA events on the context's stream, accumulated over calls). */
enum {
    ZKE_STAGE_WITNESS = 0,        /* witness kernel, whole batch                                   */
    ZKE_STAGE_MATVEC = 1,         /* <A,w>, <B,w>, constraint check, per email                     */
    ZKE_STAGE_NTT = 2,            /* hadamard + 3 inverse + 3 forward NTTs + quotient, per email   */
    ZKE_STAGE_MSM_A = 3, ZKE_STAGE_MSM_B1 = 4, ZKE_STAGE_MSM_C = 5,
    ZKE_STAGE_MSM_H = 6,          /* whole H multi-exponentiation (N full-width scalars)           */
    ZKE_STAGE_MSM_H_BUCKETS = 7,  /* its bucket-accumulation kernel alone (the dominant kernel)    */
    ZKE_STAGE_MSM_B2 = 8,
    ZKE_N_STAGES = 9
};
/* Number of concurrent proving lanes (streams) used by zke_prove, 1..allocated (default min(8, max_batch), or the
 * ZKE_LANES environment variable at zke_ctx_open).  Returns the value in effect.  Profiling forces one lane. */
int zke_ctx_set_lanes(zke_ctx* x, int n);
int zke_ctx_profile(zke_ctx* x, int enable);                       /* enabling also clears the accumulators */
int zke_ctx_profile_get(const zke_ctx* x, double* ms_out, uint64_t* count_out);  /* arrays of ZKE_N_STAGES */

/* calculateWitness + checkConstraints for a batch (circom_tester verbs; witness step of fullProve).
 * inputs: [batch][n_inputs][32] in witness order (see zke_circuit_input_offset), or NULL to use the inputs made
 * resident by zke_upload_inputs.  wtns_out (optional):
 * [batch][n_vars][32], the `.wtns` payload.  status (optional): per email, -1 = satisfied, else the index of
 * the first violated constraint.  Returns the number of failing emails (message: "Assert Failed: ..."). */
int zke_witness(zke_ctx* x, const uint8_t* inputs, size_t batch, uint8_t* wtns_out, int32_t* status,
                char* err, size_t errcap);
/* Makes host witnesses resident (snarkjs `groth16 prove zkey wtns` entry). */
int zke_load_witness(zke_ctx* x, const uint8_t* wtns, size_t batch, char* err, size_t errcap);
/* `snarkjs wtns check` (/root/reference/docs/zk-email-docs/UsageGuide/README.md step 6) for the first `batch` witnesses made
 * resident by zke_load_witness (or zke_witness): every constraint of the circuit, one kernel launch.  Needs the circuit (a
 * context opened from a `.zkey` alone has no C matrix); works without a key.  status (optional) and the return value as for
 * zke_witness: the number of failing witnesses, per witness -1 or the first violated constraint ("Assert Failed: ..."). */
int zke_check_witness(zke_ctx* x, size_t batch, int32_t* status, char* err, size_t errcap);
/* Groth16 prove for the resident witnesses (snarkjs.groth16.prove).  rs (optional): [batch][2][32] fixed blinding
 * scalars r, s (parity tests); NULL draws them from /dev/urandom.  proofs_out: [batch][8][32] =
 * A.x, A.y, B.x.c0, B.x.c1, B.y.c0, B.y.c1, C.x, C.y (standard form, LE).  publics_out: [batch][n_public][32]. */
int zke_prove(zke_ctx* x, size_t batch, const uint8_t* rs, uint8_t* proofs_out, uint8_t* publics_out,
              int32_t* status, char* err, size_t errcap);
/* witness + prove in one call with host buffers (snarkjs.groth16.fullProve,
 * /root/reference/packages/helpers/src/chunked-zkey.ts:80-84). */
int zke_fullprove(zke_ctx* x, const uint8_t* inputs, size_t batch, const uint8_t* rs, uint8_t* proofs_out,
                  uint8_t* publics_out, int32_t* status, char* err, size_t errcap);

/* Pipelined form of zke_fullprove: _submit enqueues the H2D copy, the witness kernel and all proving kernels of one
 * batch and returns; _collect waits for the oldest submitted batch, finishes its proofs on the host and returns them.
 * Up to two batches may be in flight, so the (latency-bound) witness kernel of batch k + 1 runs under the proving
 * kernels of batch k.  zke_fullprove == submit + collect.  Returns as zke_fullprove. */
int zke_fullprove_submit(zke_ctx* x, const uint8_t* inputs, size_t batch, const uint8_t* rs, char* err, size_t errcap);
int zke_fullprove_collect(zke_ctx* x, uint8_t* proofs_out, uint8_t* publics_out, int32_t* status, char* err, size_t errcap);
/* `snarkjs groth16 prove <zkey> <wtns>` (/root/reference/docs/zk-email-docs/UsageGuide/README.md:139-195): one iden3
 * `.wtns` file image in, proof + public signals out. */
int zke_wtns_prove(zke_ctx* x, const void* wtns_bytes, size_t len, const uint8_t* rs, uint8_t* proof_out, uint8_t* publics_out,
                   char* err, size_t errcap);

/* ---------------------------------------------------------------------------------------------------
 * One proof across 2, 4 or 8 GPUs (SURVEY 8(e)(ii); BASELINE configs[3] "sharded MSM", configs[4] "NCCL-sharded MSM+NTT").
 * Every GPU (one process each) opens a context with the key and loads the same witness (zke_witness / zke_load_witness,
 * batch 1); then, in lock step:
 *     zke_shard_begin   mat-vec for the rows of this GPU's column range + the cross-block inverse NTT stages
 *     [exchange 1]      all-to-all "columns -> rows" on the three vectors of zke_shard_vector (caller: NCCL / torch.distributed)
 *     zke_shard_mid     block-local inverse stages, coset shift, block-local forward stages on this GPU's row block
 *     [exchange 2]      all-to-all "rows -> columns"
 *     zke_shard_end     cross-block forward stages, a o b - c on the column range (this GPU's H scalars), the five
 *                       multi-exponentiations over this GPU's share of the points -> ZKE_SHARD_PARTIAL_BYTES
 *     [all-gather]      of the partial blocks
 *     zke_shard_combine (host only) adds the partial points and assembles the proof: bit-identical to the 1-GPU proof.
 * Layout of the vectors: element i of the N = 2^domain_log2 evaluation vector at byte offset 32 i; block g = elements
 * [g M, (g + 1) M) with M = N / world; GPU r owns row block r and the columns [r M / world, (r + 1) M / world) of
 * every block.  Exchange 1 sends (block g, columns of r) to GPU g; exchange 2 is its inverse.
 * ------------------------------------------------------------------------------------------------- */
#define ZKE_SHARD_PARTIAL_BYTES 388   /* A, B1, C, H (G1: x, y) + B2 (G2: x.c0, x.c1, y.c0, y.c1), standard form LE, + u32 first bad row */
int zke_shard_begin(zke_ctx* x, int rank, int world, char* err, size_t errcap);
void* zke_shard_vector(zke_ctx* x, int which /* 0 a, 1 b, 2 c */, size_t* n_elems);   /* device pointer, 32 bytes per element */
int zke_shard_mid(zke_ctx* x, char* err, size_t errcap);
int zke_shard_end(zke_ctx* x, uint8_t* partial_out, uint8_t* publics_out, char* err, size_t errcap);
int zke_shard_combine(const zke_zkey* z, const uint8_t* partials, int world, const uint8_t* rs, uint8_t* proof_out, int32_t* status,
                      char* err, size_t errcap);
/* the same with the five key points it needs given directly: alpha_1, beta_1, delta_1 (64 bytes each), beta_2, delta_2
 * (128 bytes each), standard form LE - no GPU-resident key required (a coordinator process can combine) */
int zke_shard_combine_raw(const uint8_t* key_points, const uint8_t* partials, int world, const uint8_t* rs, uint8_t* proof_out,
                          int32_t* status, char* err, size_t errcap);

/* ---------------------------------------------------------------------------------------------------
 * JSON faces of the boundary (snarkjs file formats; shapes as in
 * /root/reference/packages/rust-verifier/tests/data/proof_of_twitter/{vkey,proof,public}.json).
 * String outputs: pass the buffer capacity in *len; on return *len = bytes needed incl. NUL (rc -2 if too small).
 * ------------------------------------------------------------------------------------------------- */
/* snarkjs.groth16.verify(vkey, publicSignals, proof): 1 valid, 0 invalid, < 0 malformed input.  Host only. */
int zke_verify_json(const char* vkey_json, const char* public_json, const char* proof_json, char* err, size_t errcap);
/* The same check for n proofs under ONE verification key (SURVEY.md 8(f) rank 4, "batch Groth16 verification"; the reference
 * verifies one proof per call: chunked-zkey.ts:93-105, rust-verifier/src/verifier_utils.rs:20): a random linear combination
 * turns the 4n pairings into n + 3 Miller loops and one final exponentiation.  publics_json: array of n public-signal
 * arrays, proofs_json: array of n proof objects; rand16: n x 16 bytes of caller randomness the provers cannot predict
 * (NULL: std::random_device); ok (may be NULL): ok[i] = 1 / 0 - when the combined check fails the proofs are verified one
 * by one to name the offenders.  Returns the number of valid proofs, < 0 on malformed input.  Host only. */
int zke_verify_batch_json(const char* vkey_json, const char* publics_json, const char* proofs_json, const uint8_t* rand16,
                          uint8_t* ok, char* err, size_t errcap);
/* ---------------------------------------------------------------------------------------------------
 * Batch verification on the GPU: snarkjs.groth16.verify(vkey, publicSignals, proof)
 * (/root/reference/packages/helpers/src/chunked-zkey.ts:101) for n proofs under one key per call, with the verdicts of
 * zke_verify_batch_json.  The proofs are validated in parallel (coordinates below q, points on their curves, B in the
 * order-r subgroup, n_public signals below r); then ONE randomised product of n + 3 Miller loops and one final
 * exponentiation checks them all; if a proof is malformed or that check fails, every proof is verified on its own.
 * ------------------------------------------------------------------------------------------------- */
typedef struct zke_verifier zke_verifier;
/* vkey.json in; validates the key (points on their curves, G2 points in the subgroup), precomputes the Miller-loop lines
 * of beta_2, gamma_2, delta_2 and e(alpha, beta), and keeps them on GPU `device`.  NULL + message for an invalid key. */
zke_verifier* zke_verifier_open(const char* vkey_json, int device, char* err, size_t errcap);
void zke_verifier_close(zke_verifier* v);
/* proofs: [n][8][32] in zke_prove's layout (an all-zero point is the point at infinity); publics: [n][n_public][32]
 * (n_public = number of IC points - 1), standard form LE; rand16: n x 16 bytes of caller randomness the provers cannot
 * predict, or NULL (/dev/urandom); a zero weight counts as 1.  ok (may be NULL): ok[i] = 1 / 0.
 * Returns the number of valid proofs, < 0 on a fatal error. */
int zke_verifier_batch(zke_verifier* v, size_t n, const uint8_t* proofs, const uint8_t* publics, const uint8_t* rand16,
                       uint8_t* ok, char* err, size_t errcap);
/* ---- Proof aggregation (SnarkPack; DESIGN.md "Proof aggregation") -------------------------------------------------
 * n Groth16 proofs under one key (n a power of two from 2 to 8192) -> one proof of zke_agg_bytes(n) = 3008 + 3968 log2 n
 * bytes that the host checks with O(log n) pairings.  The SRS holds the powers of two independent taus a and b, read
 * from the tauG1 / tauG2 sections of two `.ptau` files of power >= log2(n_max) + 1 (prepared or not; points checked on
 * GPU `device`; both must start from the same generators). */
typedef struct zke_agg_srs zke_agg_srs;
zke_agg_srs* zke_agg_srs_from_ptau(const void* ptau_a, size_t len_a, const void* ptau_b, size_t len_b, uint32_t n_max, int device,
                                   char* err, size_t errcap);
void zke_agg_srs_free(zke_agg_srs* s);
uint32_t zke_agg_srs_n_max(const zke_agg_srs* s);
/* The verifier key {"protocol":"snarkpack", g, h, g_a, g_b, h_a, h_b} (snarkjs point encoding); *len in/out as
 * zke_zkey_vkey_json (-2: buffer too small, *len = bytes needed). */
int zke_agg_vk_json(const zke_agg_srs* s, char* out, size_t* len);
/* Bytes of an aggregate of n proofs; 0 for an n that cannot be aggregated. */
size_t zke_agg_bytes(size_t n);
/* proofs: [n][8][32] and publics: [n][n_public][32] in zke_prove's layout; vkey_json: snarkjs vkey.json.  Writes
 * zke_agg_bytes(n) bytes to `out` and returns that count, < 0 on a refusal (n, SRS size, a proof point off its curve or
 * outside its subgroup, a public signal not below r) with the reason in err. */
int64_t zke_aggregate(zke_agg_srs* s, const char* vkey_json, size_t n, const uint8_t* proofs, const uint8_t* publics, uint8_t* out,
                      size_t cap, char* err, size_t errcap);
/* Host only: 1 if `agg` proves n valid proofs under vkey_json for these public signals ([n][n_public][32]), 0 if not,
 * < 0 on malformed input (n, lengths, unreduced coordinates, points off their curves or outside their subgroups). */
int zke_agg_verify(const char* agg_vk_json, const char* vkey_json, size_t n, const uint8_t* publics, const uint8_t* agg, size_t agg_len,
                   char* err, size_t errcap);
/* Diagnostic: e(P_i, Q_i) for n pairs on GPU `device`, in zke_pairing_alphabeta's output layout (g1: [n][64],
 * g2: [n][128], out: [n][384]; standard form LE).  Points must be on their curves (< 0 otherwise). */
int zke_selftest_pairing_gpu(int device, size_t n, const uint8_t* g1, const uint8_t* g2, uint8_t* out, char* err, size_t errcap);
/* `snarkjs zkey export verificationkey`, incl. vk_alphabeta_12 = e(alpha_1, beta_2) in snarkjs' Fq12 tower layout
 * (/root/reference/packages/rust-verifier/tests/data/proof_of_twitter/vkey.json:43). */
int zke_zkey_vkey_json(const zke_zkey* z, char* out, size_t* len);
/* e(alpha_1, beta_2) as snarkjs exports it: 12 x 32 bytes = vk_alphabeta_12[i][j][k] flattened, standard form LE.
 * alpha: x, y; beta: x.c0, x.c1, y.c0, y.c1 (standard form LE).  Host only. */
int zke_pairing_alphabeta(const uint8_t* alpha64, const uint8_t* beta128, uint8_t* out384);
/* zke_prove output -> proof.json / public.json */
int zke_proof_to_json(const uint8_t* proof256, const uint8_t* publics, uint32_t n_public, char* proof_json, size_t* proof_len,
                      char* public_json, size_t* public_len);
/* input.json ({signal: decimal string | number | nested arrays}) -> packed inputs in witness order */
int zke_pack_inputs_json(const zke_circuit* c, const char* input_json, uint8_t* out, size_t cap, char* err, size_t errcap);
/* snarkjs.groth16.fullProve(input, wasm, zkey) for one email: JSON in, proof.json + public.json out */
int zke_fullprove_json(zke_ctx* x, const zke_circuit* c, const char* input_json, char* proof_json, size_t* proof_len,
                       char* public_json, size_t* public_len, char* err, size_t errcap);
/* Diagnostic: the FpMul big-integer hint evaluated on the host with the same code the witness kernel runs
 * (a, b, p: k limbs of 32 bytes LE; q, r out likewise). */
/* Diagnostic: the toxic waste (tau, alpha, beta, gamma, delta; 5 x 32 bytes LE) zke_setup derives from `seed` -
 * lets a test rebuild the same key independently.  It exists precisely because the setup is a toy. */
int zke_setup_toxic(uint64_t seed, uint8_t* out160);
int zke_selftest_fpmul_hint(uint32_t n, uint32_t k, const uint8_t* a, const uint8_t* b, const uint8_t* p, uint8_t* q, uint8_t* r);

/* Library / device introspection.  zke_device_count() returns 0 when no CUDA device is usable;
 * every compute entry point then fails with a negative code (no CPU fallback exists). */
int zke_device_count(void);
const char* zke_version(void);

#ifdef __cplusplus
}
#endif
#endif /* ZKEMAIL_B200_H */
