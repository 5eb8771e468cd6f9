"""H100-native host package mirroring the @zk-email/helpers surface for the EmailVerifier path
(/root/reference/packages/helpers/src/index.ts:1-4)."""
from .circuit import Circuit, FR_MODULUS, r1cs_info  # noqa: F401
from .constants import *  # noqa: F401,F403
from .binary_format import (bigint_to_chunked_bytes, bytes_to_bigint, int64_to_bytes, int8_to_bytes,  # noqa: F401
                            to_circom_bigint_bytes, uint8array_to_char_array)
from .sha_utils import generate_partial_sha, partial_sha, sha256_pad, sha_hash  # noqa: F401
from .dkim import DKIMVerificationResult, verify_dkim_signature  # noqa: F401
from .input_generators import (generate_circuit_inputs, generate_email_verifier_inputs,  # noqa: F401
                               generate_twitter_verifier_inputs_from_dkim_result,
                               generate_email_verifier_inputs_from_dkim_result)
from .app import decode_app_outputs, expected_app_output, generate_app_inputs  # noqa: F401
from . import hash  # noqa: F401,E402
from .registry import KeyRegistry  # noqa: F401,E402
from .engine import AssertFailed, Context, Verifier, Zkey, device_count, proof_to_json, verify, verify_batch  # noqa: F401
from .engine import ptau_info, ptau_toy, verify_zkey  # noqa: F401
from .engine import ptau_contribute, ptau_new, ptau_prepare, ptau_report, verify_ptau  # noqa: F401
from .aggregate import AggSrs, aggregate, verify_aggregate  # noqa: F401
from .chunked_zkey import (generate_proof, verify_proof, register_circuit, register_zkey_files, generateProof, verifyProof,  # noqa: F401
                           InsecureKeyError)
from . import synthetic  # noqa: F401,E402
from . import iden3_binfile  # noqa: F401,E402
from . import verifier_args  # noqa: F401,E402
