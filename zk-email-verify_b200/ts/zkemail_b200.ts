// TypeScript host shim (UNRUN: node is not present in the build image).  Drop-in for the two snarkjs verbs the
// reference uses in packages/helpers/src/chunked-zkey.ts:80-84,101, backed by the C ABI of include/zkemail_b200.h.
// See INTEGRATION.md.
import koffi from 'koffi';

const lib = koffi.load(process.env.ZKEMAIL_B200_LIB ?? 'libzkemail_b200.so');
const zke_circuit_build = lib.func('void* zke_circuit_build(const char*, const int64_t*, size_t, char*, size_t)');
const zke_circuit_build_app = lib.func('void* zke_circuit_build_app(const char*, char*, size_t)');   // app circuit from a JSON spec
const zke_setup = lib.func('void* zke_setup(void*, uint64_t, int, char*, size_t)');
const zke_zkey_load = lib.func('void* zke_zkey_load(const void*, size_t, int, char*, size_t)');
const zke_zkey_load_chunks = lib.func('void* zke_zkey_load_chunks(const void**, const size_t*, size_t, int, char*, size_t)');
const zke_zkey_is_toy = lib.func('int zke_zkey_is_toy(void*)');
const zke_ctx_open = lib.func('void* zke_ctx_open(void*, void*, int, uint32_t, char*, size_t)');
const zke_zkey_vkey_json = lib.func('int zke_zkey_vkey_json(void*, char*, size_t*)');
const zke_fullprove_json = lib.func('int zke_fullprove_json(void*, void*, const char*, char*, size_t*, char*, size_t*, char*, size_t)');
const zke_verify_json = lib.func('int zke_verify_json(const char*, const char*, const char*, char*, size_t)');
const zke_verify_batch_json = lib.func('int zke_verify_batch_json(const char*, const char*, const char*, const uint8_t*, uint8_t*, char*, size_t)');

const zke_agg_srs_from_ptau = lib.func('void* zke_agg_srs_from_ptau(const void*, size_t, const void*, size_t, uint32_t, int, char*, size_t)');
const zke_agg_vk_json = lib.func('int zke_agg_vk_json(void*, char*, size_t*)');
const zke_agg_bytes = lib.func('size_t zke_agg_bytes(size_t)');
const zke_aggregate = lib.func('int64_t zke_aggregate(void*, const char*, size_t, const uint8_t*, const uint8_t*, uint8_t*, size_t, char*, size_t)');
const zke_agg_verify = lib.func('int zke_agg_verify(const char*, const char*, size_t, const uint8_t*, const uint8_t*, size_t, char*, size_t)');

const zke_poseidon_hash = lib.func('int zke_poseidon_hash(const uint8_t*, size_t, uint8_t*)');
const zke_poseidon_batch = lib.func('int zke_poseidon_batch(const uint8_t*, uint32_t, size_t, int, uint8_t*, char*, size_t)');
const zke_pubkey_hashes = lib.func('int zke_pubkey_hashes(const uint8_t*, size_t, uint32_t, uint32_t, uint32_t, int, uint8_t*, char*, size_t)');
const zke_domain_key_leaves = lib.func('int zke_domain_key_leaves(const uint8_t*, size_t, uint32_t, uint32_t, uint32_t, const uint8_t*, int, uint8_t*, char*, size_t)');
const zke_merkle_build = lib.func('int64_t zke_merkle_build(const uint8_t*, size_t, uint32_t, int, uint8_t*, size_t, char*, size_t)');
const zke_registry_open = lib.func('void* zke_registry_open(const uint8_t*, size_t, uint32_t, int, char*, size_t)');
const zke_registry_update = lib.func('int zke_registry_update(void*, const uint64_t*, const uint8_t*, size_t, char*, size_t)');
const zke_registry_nodes = lib.func('int zke_registry_nodes(void*, const uint32_t*, const uint64_t*, size_t, uint8_t*, char*, size_t)');
const zke_registry_count = lib.func('uint64_t zke_registry_count(void*)');
const zke_registry_close = lib.func('void zke_registry_close(void*)');

const cstr = (b: Buffer) => b.toString('utf8', 0, b.indexOf(0));
type Entry = { circuit: unknown; zkey: unknown; ctx: unknown };
const registry = new Map<string, Entry>();

/**
 * Plays the role of downloadProofFiles + uncompress (chunked-zkey.ts:35-37, 59-74): makes `${circuitName}.zkey`
 * resident on a GPU.  `zkeyChunks` are the contents of `${circuitName}.zkeyb` .. `.zkeyk` (the fork's per-section
 * files, chunked-zkey.ts:9) or a single whole `.zkey`; they are parsed and validated by zke_zkey_load[_chunks].
 * The circuit's witness program replaces `${circuitName}.wasm`.
 */
export function registerEmailVerifier(circuitName: string, params: number[], zkeyChunks: Buffer[], device = 0): void {
  const err = Buffer.alloc(4096);
  const circuit = zke_circuit_build('EmailVerifier', BigInt64Array.from(params.map(BigInt)), params.length, err, err.length);
  if (!circuit) throw new Error(cstr(err));
  const zkey = zkeyChunks.length === 1
    ? zke_zkey_load(zkeyChunks[0], zkeyChunks[0].length, device, err, err.length)
    : zke_zkey_load_chunks(zkeyChunks, BigUint64Array.from(zkeyChunks.map((c) => BigInt(c.length))), zkeyChunks.length, device, err, err.length);
  if (!zkey) throw new Error(cstr(err));
  const ctx = zke_ctx_open(circuit, zkey, device, 1, err, err.length);
  if (!ctx) throw new Error(cstr(err));
  registry.set(circuitName, { circuit, zkey, ctx });
}

/** registerEmailVerifier for an app circuit built from its spec (Circuit.from_spec in Python; layout at zke_circuit_build_app). */
export function registerEmailApp(circuitName: string, spec: object | string, zkeyChunks: Buffer[], device = 0): void {
  const err = Buffer.alloc(4096);
  const circuit = zke_circuit_build_app(typeof spec === 'string' ? spec : JSON.stringify(spec), err, err.length);
  if (!circuit) throw new Error(cstr(err));
  const zkey = zkeyChunks.length === 1
    ? zke_zkey_load(zkeyChunks[0], zkeyChunks[0].length, device, err, err.length)
    : zke_zkey_load_chunks(zkeyChunks, BigUint64Array.from(zkeyChunks.map((c) => BigInt(c.length))), zkeyChunks.length, device, err, err.length);
  if (!zkey) throw new Error(cstr(err));
  const ctx = zke_ctx_open(circuit, zkey, device, 1, err, err.length);
  if (!ctx) throw new Error(cstr(err));
  registry.set(circuitName, { circuit, zkey, ctx });
}

/** Tests and benchmarks only: a key from the seeded TOY setup (known toxic waste - proofs under it are forgeable). */
export function registerEmailVerifierWithToyKey(circuitName: string, params: number[], seed: number, device = 0): void {
  const err = Buffer.alloc(4096);
  const circuit = zke_circuit_build('EmailVerifier', BigInt64Array.from(params.map(BigInt)), params.length, err, err.length);
  if (!circuit) throw new Error(cstr(err));
  const zkey = zke_setup(circuit, BigInt(seed), device, err, err.length);
  if (!zkey || zke_zkey_is_toy(zkey) !== 1) throw new Error(cstr(err));
  const ctx = zke_ctx_open(circuit, zkey, device, 1, err, err.length);
  if (!ctx) throw new Error(cstr(err));
  registry.set(circuitName, { circuit, zkey, ctx });
}

export function exportVerificationKey(circuitName: string): object {
  const e = registry.get(circuitName);
  if (!e) throw new Error(`unknown circuit ${circuitName}`);
  const len = [1 << 20];
  const buf = Buffer.alloc(len[0]);
  if (zke_zkey_vkey_json(e.zkey, buf, len) !== 0) throw new Error('vkey export failed');
  return JSON.parse(cstr(buf));
}

export const groth16 = {
  /** snarkjs.groth16.fullProve(input, wasmFile, zkeyFileName) */
  async fullProve(input: object, _wasmFile: string, zkeyFileName: string) {
    const e = registry.get(zkeyFileName.replace(/\.zkey$/, ''));
    if (!e) throw new Error(`Error downloading ${zkeyFileName} after 3 retries`);
    const proof = Buffer.alloc(4096), pub = Buffer.alloc(1 << 16), err = Buffer.alloc(4096);
    const pl = [proof.length], sl = [pub.length];
    const rc = zke_fullprove_json(e.ctx, e.circuit, JSON.stringify(input), proof, pl, pub, sl, err, err.length);
    if (rc !== 0) throw new Error(cstr(err));
    return { proof: JSON.parse(cstr(proof)), publicSignals: JSON.parse(cstr(pub)) };
  },
  /** snarkjs.groth16.verify(vkey, publicSignals, proof) */
  async verify(vkey: object, publicSignals: string[], proof: object): Promise<boolean> {
    const err = Buffer.alloc(4096);
    const rc = zke_verify_json(JSON.stringify(vkey), JSON.stringify(publicSignals), JSON.stringify(proof), err, err.length);
    if (rc < 0) throw new Error(cstr(err));
    return rc === 1;
  },
  /** n proofs under one key with one randomised product of pairings; per-proof verdicts (not in snarkjs) */
  async verifyBatch(vkey: object, publicSignals: string[][], proofs: object[]): Promise<boolean[]> {
    const err = Buffer.alloc(4096), ok = Buffer.alloc(proofs.length);
    const rand = require('crypto').randomBytes(16 * proofs.length);
    const rc = zke_verify_batch_json(JSON.stringify(vkey), JSON.stringify(publicSignals), JSON.stringify(proofs), rand, ok, err, err.length);
    if (rc < 0) throw new Error(cstr(err));
    return Array.from(ok).map((b) => b === 1);
  },
};

/** Proof aggregation (SnarkPack, not in snarkjs): n proofs under one key -> one O(log n) proof.  `proofs` / `publics` are
 * zke_prove's binary layouts ([n][8][32], [n][nPublic][32]); the SRS comes from two `.ptau` files with independent taus. */
export const aggregation = {
  srsFromPtau(ptauA: Buffer, ptauB: Buffer, nMax: number, device = 0): { srs: unknown; vk: object } {
    const err = Buffer.alloc(4096);
    const srs = zke_agg_srs_from_ptau(ptauA, ptauA.length, ptauB, ptauB.length, nMax, device, err, err.length);
    if (!srs) throw new Error(cstr(err));
    const buf = Buffer.alloc(4096), len = [buf.length];
    if (zke_agg_vk_json(srs, buf, len) !== 0) throw new Error('zke_agg_vk_json failed');
    return { srs, vk: JSON.parse(cstr(buf)) };
  },
  aggregate(srs: unknown, vkey: object, n: number, proofs: Buffer, publics: Buffer): Buffer {
    const out = Buffer.alloc(Number(zke_agg_bytes(n)) || 1), err = Buffer.alloc(4096);
    const rc = zke_aggregate(srs, JSON.stringify(vkey), n, proofs, publics, out, out.length, err, err.length);
    if (rc < 0) throw new Error(cstr(err));
    return out.subarray(0, Number(rc));
  },
  verify(aggVk: object, vkey: object, n: number, publics: Buffer, agg: Buffer): boolean {
    const err = Buffer.alloc(4096);
    const rc = zke_agg_verify(JSON.stringify(aggVk), JSON.stringify(vkey), n, publics, agg, agg.length, err, err.length);
    if (rc < 0) throw new Error(cstr(err));
    return rc === 1;
  },
};

/** Poseidon hashes of packages/helpers/src/hash.ts on the library's host permutation (zke_poseidon_hash), synchronous:
 *  what a hashed (`"reveal": "hash"`) or committed (`"reveal": "commit"`) app output holds. */
const R = 21888242871839275222246405745257275088548364400416034343698204186575808495617n;
const le32 = (x: bigint) => { const b = Buffer.alloc(32); let v = ((x % R) + R) % R; for (let i = 0; i < 32; i++) { b[i] = Number(v & 0xffn); v >>= 8n; } return b; };
export function poseidon(inputs: bigint[]): bigint {
  if (inputs.length < 1 || inputs.length > 16) throw new Error(`Poseidon takes 1 to 16 inputs, not ${inputs.length}`);
  const out = Buffer.alloc(32);
  if (zke_poseidon_hash(Buffer.concat(inputs.map(le32)), inputs.length, out) !== 0) throw new Error('zke_poseidon_hash failed');
  let v = 0n;
  for (let i = 31; i >= 0; i--) v = (v << 8n) | BigInt(out[i]);
  return v;
}
export function poseidonLarge(input: bigint, numChunks: number, bitsPerChunk: number): bigint {
  const mask = (1n << BigInt(bitsPerChunk)) - 1n;
  return poseidon(Array.from({ length: numChunks }, (_, i) => (input >> BigInt(i * bitsPerChunk)) & mask));
}
export function poseidonModular(inputs: bigint[]): bigint {
  let out: bigint | null = null;
  for (let start = 0; start < inputs.length; start += 16) {
    const h = poseidon(inputs.slice(start, start + 16));
    out = out === null ? h : poseidon([out, h]);
  }
  if (out === null) throw new Error('No inputs provided');
  return out;
}

/** The key registry on the GPU (zke_poseidon_batch, zke_pubkey_hashes, zke_merkle_build): field elements as bigints. */
const fromLe32 = (b: Buffer, i: number) => {
  let x = 0n;
  for (let j = 31; j >= 0; --j) x = (x << 8n) | BigInt(b[32 * i + j]);
  return x;
};
const toLe = (x: bigint, n: number) => {
  const b = Buffer.alloc(n);
  for (let j = 0; j < n; ++j) { b[j] = Number(x & 0xffn); x >>= 8n; }
  return b;
};
export function poseidonBatch(rows: bigint[][], device = 0): bigint[] {
  if (rows.length === 0) return [];
  const out = Buffer.alloc(32 * rows.length), err = Buffer.alloc(4096);
  const data = Buffer.concat(rows.flat().map((x) => toLe(((x % R) + R) % R, 32)));
  if (zke_poseidon_batch(data, rows[0].length, rows.length, device, out, err, err.length) !== 0) throw new Error(cstr(err));
  return rows.map((_, i) => fromLe32(out, i));
}
export function pubkeyHashes(moduli: bigint[], n = 121, k = 17, device = 0): bigint[] {
  if (moduli.length === 0) return [];
  const bytes = Math.ceil((n * k) / 8);
  const out = Buffer.alloc(32 * moduli.length), err = Buffer.alloc(4096);
  if (zke_pubkey_hashes(Buffer.concat(moduli.map((m) => toLe(m, bytes))), moduli.length, bytes, n, k, device, out, err, err.length) !== 0)
    throw new Error(cstr(err));
  return moduli.map((_, i) => fromLe32(out, i));
}
/** A domain in canonical form: ASCII (A-labels for international names), lower case, no trailing dot, 1..255 bytes. */
const canonicalDomain = (domain: string): Buffer => {
  if (!/^[\x01-\x7f]*$/.test(domain)) throw new Error(`domain ${domain} is not ASCII: give an international name in its A-label (xn--) form`);
  let d = domain.toLowerCase();
  if (d.endsWith('.')) d = d.slice(0, -1);
  if (d.length < 1 || d.length > 255) throw new Error(`domain ${d} has ${d.length} bytes; a domain has 1 to 255`);
  return Buffer.from(d, 'ascii');
};
/** PoseidonModular(PackBytes(domain, 255)): one Poseidon(9), the domain half of a domain-bound registry leaf. */
export function domainHash(domain: string): bigint {
  const row = Buffer.alloc(255);
  canonicalDomain(domain).copy(row);
  return poseidon(Array.from({ length: 9 }, (_, i) => {
    let x = 0n;
    for (let j = 30; j >= 0; --j) x = (x << 8n) | BigInt(31 * i + j < 255 ? row[31 * i + j] : 0);
    return x;
  }));
}
/** Domain-bound leaves Poseidon(2)([domainHash(domain), pubkeyHash(modulus)]) of (domain, modulus) pairs on the GPU:
 *  the leaves of a registry for specs with "keyDomain". */
export function domainKeyLeaves(pairs: [string, bigint][], n = 121, k = 17, device = 0): bigint[] {
  if (pairs.length === 0) return [];
  const bytes = Math.ceil((n * k) / 8);
  const rows = Buffer.concat(pairs.map(([d]) => { const row = Buffer.alloc(255); canonicalDomain(d).copy(row); return row; }));
  const out = Buffer.alloc(32 * pairs.length), err = Buffer.alloc(4096);
  if (zke_domain_key_leaves(Buffer.concat(pairs.map(([, m]) => toLe(m, bytes))), pairs.length, bytes, n, k, rows, device, out, err, err.length) !== 0)
    throw new Error(cstr(err));
  return pairs.map((_, i) => fromLe32(out, i));
}
/** Every level of the registry tree, leaves first, root last. */
export function merkleBuild(leaves: bigint[], depth: number, device = 0): bigint[][] {
  const err = Buffer.alloc(4096), data = Buffer.concat(leaves.map((x) => toLe(x, 32)));
  const need = Number(zke_merkle_build(data, leaves.length, depth, device, null, 0, err, err.length));
  if (need < 0) throw new Error(cstr(err));
  const buf = Buffer.alloc(need);
  if (Number(zke_merkle_build(data, leaves.length, depth, device, buf, need, err, err.length)) !== need) throw new Error(cstr(err));
  const levels: bigint[][] = [];
  for (let l = 0, pos = 0; l <= depth; ++l) {
    const size = Math.ceil(leaves.length / 2 ** l);
    levels.push(Array.from({ length: size }, (_, i) => fromLe32(buf, pos + i)));
    pos += size;
  }
  return levels;
}

/** A registry tree resident on one GPU (zke_registry_*), updated in place: only the ancestors of changed leaves are
 *  rehashed.  Leaves are field elements (pubkeyHashes, domainKeyLeaves).  One caller at a time; close() frees it. */
export class Registry {
  private h: unknown;
  constructor(leaves: bigint[], readonly depth: number, device = 0) {
    const err = Buffer.alloc(4096);
    this.h = zke_registry_open(Buffer.concat(leaves.map((x) => toLe(x, 32))), leaves.length, depth, device, err, err.length);
    if (!this.h) throw new Error(cstr(err));
  }
  get count(): number { return Number(zke_registry_count(this.h)); }
  /** Replace (leaf 0 revokes) and append: indices from `count` on must be count, count + 1, ... in any order. */
  update(changes: [number, bigint][]): void {
    if (changes.length === 0) return;
    const err = Buffer.alloc(4096);
    const rc = zke_registry_update(this.h, BigUint64Array.from(changes.map(([i]) => BigInt(i))),
      Buffer.concat(changes.map(([, x]) => toLe(x, 32))), changes.length, err, err.length);
    if (rc !== 0) throw new Error(cstr(err));
  }
  /** Appends after the last leaf; returns the new indices. */
  append(leaves: bigint[]): number[] {
    const first = this.count, idx = leaves.map((_, j) => first + j);
    this.update(idx.map((i, j) => [i, leaves[j]]));
    return idx;
  }
  private nodes(levels: number[], indices: number[]): bigint[] {
    const out = Buffer.alloc(32 * levels.length), err = Buffer.alloc(4096);
    if (zke_registry_nodes(this.h, Uint32Array.from(levels), BigUint64Array.from(indices.map(BigInt)), levels.length, out, err, err.length) !== 0)
      throw new Error(cstr(err));
    return levels.map((_, i) => fromLe32(out, i));
  }
  /** The circuit's registryIndex and registrySiblings for leaf i. */
  path(i: number): { index: number; siblings: bigint[] } {
    if (!(i >= 0 && i < this.count)) throw new Error(`leaf ${i} is not in a registry of ${this.count} keys`);
    const levels = Array.from({ length: this.depth }, (_, l) => l);
    return { index: i, siblings: this.nodes(levels, levels.map((l) => Number((BigInt(i) >> BigInt(l)) ^ 1n))) };
  }
  get root(): bigint { return this.nodes([this.depth], [0])[0]; }
  close(): void { if (this.h) zke_registry_close(this.h); this.h = null; }
}
