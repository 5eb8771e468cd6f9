"""ctypes binding of the C ABI declared in include/zkemail_b200.h.

The shared library is the product: it holds the circuit front-end, the CUDA kernels and the Groth16 engine.
There is no Python or CPU fallback - if the library is missing this module raises at import time, and every
compute entry point fails when no CUDA device is present.
"""
from __future__ import annotations
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get(
    "ZKEMAIL_B200_LIB", os.path.normpath(os.path.join(_HERE, "..", "..", "lib", "libzkemail_b200.so"))
)
if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found - build it first (python -c 'import __graft_entry__ as g; g.build()' "
        "or make -C zk-email-verify_b200/csrc); there is no fallback implementation"
    )
lib = ctypes.CDLL(LIB_PATH)

c_void_p, c_char_p, c_size_t = ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t
c_u32, c_u64, c_i64, c_int = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int64, ctypes.c_int
ERRCAP = 4096


class CircuitInfo(ctypes.Structure):
    _fields_ = [(n, c_u32) for n in (
        "n_vars", "n_temps", "n_outputs", "n_pub_inputs", "n_prv_inputs", "n_public", "n_constraints",
        "n_levels", "n_ops", "n_coefs", "domain_log2", "n_groups")] + [(n, c_u64) for n in ("nnz_a", "nnz_b", "nnz_c")]


class ProgramStats(ctypes.Structure):
    _fields_ = [(n, c_u32) for n in ("n_levels", "n_iters", "n_ops_kept", "n_coop_ops", "n_terms", "cluster")] + [("digest", c_u64)]


def _sig(name, restype, argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = argtypes
    return fn


zke_circuit_build = _sig("zke_circuit_build", c_void_p, [c_char_p, ctypes.POINTER(c_i64), c_size_t, c_char_p, c_size_t])
zke_circuit_free = _sig("zke_circuit_free", None, [c_void_p])
zke_circuit_build_app = _sig("zke_circuit_build_app", c_void_p, [c_char_p, c_char_p, c_size_t])
zke_circuit_from_r1cs = _sig("zke_circuit_from_r1cs", c_void_p, [c_void_p, c_size_t, c_char_p, c_size_t])
zke_circuit_write_r1cs = _sig("zke_circuit_write_r1cs", c_i64, [c_void_p, c_void_p, c_size_t])
zke_circuit_get_info = _sig("zke_circuit_get_info", c_int, [c_void_p, ctypes.POINTER(CircuitInfo)])
zke_circuit_group = _sig("zke_circuit_group", c_int, [c_void_p, c_u32, c_char_p, c_size_t, ctypes.POINTER(c_u32),
                                                       ctypes.POINTER(c_u32), ctypes.POINTER(c_int)])
zke_circuit_input_offset = _sig("zke_circuit_input_offset", c_i64, [c_void_p, c_char_p, ctypes.POINTER(c_u32)])
zke_circuit_array = _sig("zke_circuit_array", c_void_p, [c_void_p, c_int, ctypes.POINTER(c_size_t)])
zke_circuit_scope_name = _sig("zke_circuit_scope_name", c_char_p, [c_void_p, c_u32])
zke_circuit_program_stats = _sig("zke_circuit_program_stats", c_int, [c_void_p, c_int, c_int, c_int, c_u32, ctypes.POINTER(ProgramStats),
                                                                      ctypes.POINTER(c_u32), c_size_t, c_char_p, c_size_t])
zke_circuit_program_stats_ex = _sig("zke_circuit_program_stats_ex", c_int, [c_void_p, c_u32, c_u32, ctypes.POINTER(ProgramStats),
                                                                            ctypes.POINTER(c_u32), c_size_t, c_char_p, c_size_t])
LOWER_NATIVE_SHA, LOWER_NATIVE_REGEX, LOWER_COOP_FPMUL, LOWER_NATIVE_POSEIDON = 1, 2, 4, 8
zke_poseidon_hash = _sig("zke_poseidon_hash", c_int, [c_char_p, c_size_t, c_char_p])
zke_poseidon_batch = _sig("zke_poseidon_batch", c_int, [c_char_p, c_u32, c_size_t, c_int, c_void_p, c_char_p, c_size_t])
zke_pubkey_hashes = _sig("zke_pubkey_hashes", c_int, [c_char_p, c_size_t, c_u32, c_u32, c_u32, c_int, c_void_p, c_char_p, c_size_t])
zke_domain_key_leaves = _sig("zke_domain_key_leaves", c_int, [c_char_p, c_size_t, c_u32, c_u32, c_u32, c_char_p, c_int, c_void_p,
                                                               c_char_p, c_size_t])
zke_merkle_build = _sig("zke_merkle_build", c_i64, [c_char_p, c_size_t, c_u32, c_int, c_void_p, c_size_t, c_char_p, c_size_t])
zke_registry_open = _sig("zke_registry_open", c_void_p, [c_char_p, c_size_t, c_u32, c_int, c_char_p, c_size_t])
zke_registry_update = _sig("zke_registry_update", c_int, [c_void_p, c_void_p, c_char_p, c_size_t, c_char_p, c_size_t])
zke_registry_nodes = _sig("zke_registry_nodes", c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_char_p, c_size_t])
zke_registry_levels = _sig("zke_registry_levels", c_i64, [c_void_p, c_void_p, c_size_t, c_char_p, c_size_t])
zke_registry_count = _sig("zke_registry_count", c_u64, [c_void_p])
zke_registry_close = _sig("zke_registry_close", None, [c_void_p])
zke_registry_device_ms = _sig("zke_registry_device_ms", ctypes.c_double, [])
zke_device_count = _sig("zke_device_count", c_int, [])
zke_version = _sig("zke_version", c_char_p, [])

# array selectors (enum in the header)
(ARR_COEFS, ARR_A_PTR, ARR_A_VAR, ARR_A_COEF, ARR_B_PTR, ARR_B_VAR, ARR_B_COEF, ARR_C_PTR, ARR_C_VAR, ARR_C_COEF,
 ARR_OPS, ARR_LEVEL_PTR, ARR_LC_PTR, ARR_LC_VAR, ARR_LC_COEF, ARR_AUX, ARR_SCOPE_OF_CONSTRAINT) = range(17)
ARR_SHA_BLOCKS = 17
ARR_REGEX_SEEDS = 18
ARR_POSEIDON_BLOCKS = 19


class ZkeError(RuntimeError):
    pass

# ---- engine (needs a CUDA device) -----------------------------------------------------------------------
c_u8p = ctypes.POINTER(ctypes.c_uint8)
c_i32p = ctypes.POINTER(ctypes.c_int32)
zke_setup = _sig("zke_setup", c_void_p, [c_void_p, c_u64, c_int, c_char_p, c_size_t])
zke_zkey_free = _sig("zke_zkey_free", None, [c_void_p])
zke_zkey_load = _sig("zke_zkey_load", c_void_p, [c_void_p, c_size_t, c_int, c_char_p, c_size_t])
zke_zkey_load_chunks = _sig("zke_zkey_load_chunks", c_void_p, [ctypes.POINTER(c_void_p), ctypes.POINTER(c_size_t), c_size_t, c_int, c_char_p, c_size_t])
zke_zkey_write = _sig("zke_zkey_write", c_i64, [c_void_p, c_void_p, c_void_p, c_size_t])
zke_zkey_is_toy = _sig("zke_zkey_is_toy", c_int, [c_void_p])
zke_circuit_build_regex = _sig("zke_circuit_build_regex", c_void_p, [ctypes.POINTER(c_char_p), c_char_p, c_size_t, c_u32, c_char_p, c_size_t])
zke_fullprove_submit = _sig("zke_fullprove_submit", c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_char_p, c_size_t])
zke_fullprove_collect = _sig("zke_fullprove_collect", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_wtns_prove = _sig("zke_wtns_prove", c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_pairing_alphabeta = _sig("zke_pairing_alphabeta", c_int, [c_void_p, c_void_p, c_void_p])
zke_zkey_info = _sig("zke_zkey_info", c_int, [c_void_p, ctypes.POINTER(c_u32), ctypes.POINTER(c_u32), ctypes.POINTER(c_u32)])
zke_zkey_section = _sig("zke_zkey_section", c_i64, [c_void_p, c_int, c_void_p, c_size_t])
zke_ctx_open = _sig("zke_ctx_open", c_void_p, [c_void_p, c_void_p, c_int, c_u32, c_char_p, c_size_t])
zke_ctx_close = _sig("zke_ctx_close", None, [c_void_p])
zke_ctx_stream = _sig("zke_ctx_stream", c_void_p, [c_void_p])
zke_kernel_launches = _sig("zke_kernel_launches", c_u64, [])
zke_witness = _sig("zke_witness", c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_char_p, c_size_t])
zke_load_witness = _sig("zke_load_witness", c_int, [c_void_p, c_void_p, c_size_t, c_char_p, c_size_t])
zke_check_witness = _sig("zke_check_witness", c_int, [c_void_p, c_size_t, c_void_p, c_char_p, c_size_t])
zke_prove = _sig("zke_prove", c_int, [c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_fullprove = _sig("zke_fullprove", c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_verify_json = _sig("zke_verify_json", c_int, [c_char_p, c_char_p, c_char_p, c_char_p, c_size_t])
zke_verify_batch_json = _sig("zke_verify_batch_json", c_int, [c_char_p, c_char_p, c_char_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_verifier_open = _sig("zke_verifier_open", c_void_p, [c_char_p, c_int, c_char_p, c_size_t])
zke_verifier_close = _sig("zke_verifier_close", None, [c_void_p])
zke_verifier_batch = _sig("zke_verifier_batch", c_int, [c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_selftest_pairing_gpu = _sig("zke_selftest_pairing_gpu", c_int, [c_int, c_size_t, c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_zkey_vkey_json = _sig("zke_zkey_vkey_json", c_int, [c_void_p, c_char_p, ctypes.POINTER(c_size_t)])
zke_proof_to_json = _sig("zke_proof_to_json", c_int, [c_void_p, c_void_p, c_u32, c_char_p, ctypes.POINTER(c_size_t), c_char_p, ctypes.POINTER(c_size_t)])
zke_pack_inputs_json = _sig("zke_pack_inputs_json", c_int, [c_void_p, c_char_p, c_void_p, c_size_t, c_char_p, c_size_t])
zke_fullprove_json = _sig("zke_fullprove_json", c_int, [c_void_p, c_void_p, c_char_p, c_char_p, ctypes.POINTER(c_size_t), c_char_p,
                                                        ctypes.POINTER(c_size_t), c_char_p, c_size_t])
zke_upload_inputs = _sig("zke_upload_inputs", c_int, [c_void_p, c_void_p, c_size_t, c_char_p, c_size_t])
zke_ctx_set_lanes = _sig("zke_ctx_set_lanes", c_int, [c_void_p, c_int])
zke_ctx_profile = _sig("zke_ctx_profile", c_int, [c_void_p, c_int])
zke_ctx_profile_get = _sig("zke_ctx_profile_get", c_int, [c_void_p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(c_u64)])
STAGES = ("witness", "matvec", "ntt", "msm_a", "msm_b1", "msm_c", "msm_h", "msm_h_buckets", "msm_b2")
zke_setup_toxic = _sig("zke_setup_toxic", c_int, [c_u64, c_void_p])
zke_zkey_from_ptau = _sig("zke_zkey_from_ptau", c_void_p, [c_void_p, c_void_p, c_size_t, c_int, c_char_p, c_size_t])
zke_ptau_info = _sig("zke_ptau_info", c_int, [c_void_p, c_void_p, c_size_t, ctypes.POINTER(c_u32), ctypes.POINTER(c_u64),
                                              ctypes.POINTER(c_u64), c_char_p, c_size_t])
zke_zkey_from_ptau_timing = _sig("zke_zkey_from_ptau_timing", c_int, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)])
zke_zkey_contribute = _sig("zke_zkey_contribute", c_void_p, [c_void_p, c_void_p, c_char_p, c_size_t])
zke_zkey_check_contribution = _sig("zke_zkey_check_contribution", c_int, [c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_ptau_toy = _sig("zke_ptau_toy", c_i64, [c_u32, c_void_p, c_int, c_void_p, c_size_t, c_char_p, c_size_t])
zke_ptau_new = _sig("zke_ptau_new", c_i64, [c_u32, c_void_p, c_size_t, c_char_p, c_size_t])
zke_ptau_contribute = _sig("zke_ptau_contribute", c_i64, [c_void_p, c_size_t, c_void_p, c_int, c_void_p, c_size_t, c_void_p, c_char_p, c_size_t])
zke_ptau_prepare = _sig("zke_ptau_prepare", c_i64, [c_void_p, c_size_t, c_int, c_void_p, c_size_t, c_char_p, c_size_t])
zke_ptau_prepare_timing = _sig("zke_ptau_prepare_timing", c_int, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)])
zke_ptau_verify = _sig("zke_ptau_verify", c_int, [c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_void_p, c_int, c_char_p, c_size_t])
zke_agg_srs_from_ptau = _sig("zke_agg_srs_from_ptau", c_void_p, [c_void_p, c_size_t, c_void_p, c_size_t, c_u32, c_int, c_char_p, c_size_t])
zke_agg_srs_free = _sig("zke_agg_srs_free", None, [c_void_p])
zke_agg_srs_n_max = _sig("zke_agg_srs_n_max", c_u32, [c_void_p])
zke_agg_vk_json = _sig("zke_agg_vk_json", c_int, [c_void_p, c_char_p, ctypes.POINTER(c_size_t)])
zke_agg_bytes = _sig("zke_agg_bytes", c_size_t, [c_size_t])
zke_aggregate = _sig("zke_aggregate", c_i64, [c_void_p, c_char_p, c_size_t, c_void_p, c_void_p, c_void_p, c_size_t, c_char_p, c_size_t])
zke_agg_verify = _sig("zke_agg_verify", c_int, [c_char_p, c_char_p, c_size_t, c_void_p, c_void_p, c_size_t, c_char_p, c_size_t])
zke_selftest_fpmul_hint =_sig("zke_selftest_fpmul_hint", c_int, [c_u32, c_u32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p])

(SEC_ALPHA1, SEC_BETA1, SEC_DELTA1, SEC_BETA2, SEC_GAMMA2, SEC_DELTA2) = (101, 102, 103, 104, 105, 106)
(SEC_IC, SEC_A, SEC_B1, SEC_B2, SEC_C, SEC_H) = (3, 5, 6, 7, 8, 9)

SHARD_PARTIAL_BYTES = 388
zke_shard_begin = _sig("zke_shard_begin", c_int, [c_void_p, c_int, c_int, c_char_p, c_size_t])
zke_shard_vector = _sig("zke_shard_vector", c_void_p, [c_void_p, c_int, ctypes.POINTER(c_size_t)])
zke_shard_mid = _sig("zke_shard_mid", c_int, [c_void_p, c_char_p, c_size_t])
zke_shard_end = _sig("zke_shard_end", c_int, [c_void_p, c_void_p, c_void_p, c_char_p, c_size_t])
zke_shard_combine = _sig("zke_shard_combine", c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, ctypes.POINTER(ctypes.c_int32), c_char_p, c_size_t])
zke_shard_combine_raw = _sig("zke_shard_combine_raw", c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, ctypes.POINTER(ctypes.c_int32), c_char_p, c_size_t])
