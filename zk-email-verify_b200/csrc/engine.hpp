// Internal definitions behind the opaque C-ABI handles (include/zkemail_b200.h).
#pragma once
#include "circuit.hpp"
#include <string>

namespace zke {
void set_err(char* err, size_t cap, const std::string& msg);
void random_bytes(void* out, size_t n);   // from /dev/urandom
void random_scalar(U256& out);   // uniform in [0, r), from /dev/urandom
// the refusal of every entry point that needs a witness program, for a circuit read from an `.r1cs`
constexpr const char* R1CS_NO_PROGRAM =
    "this circuit was read from an .r1cs: it has no witness program (load witnesses with zke_load_witness / zke_wtns_prove)";
}

struct zke_circuit {
    zke::Circuit c;
};

// per-email result block: the MSM result blocks (msm.cuh: 64 XYZZ slots each) of A, B1, C, H (G1, 128-byte slots)
// followed by B2 (G2, 256-byte slots), then the first-violated-constraint word
enum ZkeResBlock { RES_A = 0, RES_B1 = 1, RES_C = 2, RES_H = 3, RES_B2 = 4 };   // block b at b * ZKE_RES_G1_BLOCK
#define ZKE_RES_G1_BLOCK (64 * 128)
#define ZKE_RES_G2_BLOCK (64 * 256)
#define ZKE_RES_FLAG_OFF (4 * ZKE_RES_G1_BLOCK + ZKE_RES_G2_BLOCK)
#define ZKE_RESULT_STRIDE (ZKE_RES_FLAG_OFF + 256)
#define ZKE_MAX_LANES 16
