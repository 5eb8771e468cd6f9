// Device-side data structures and kernel launchers shared by the .cu files.
#pragma once
#include "ec.cuh"
#include "witness_program.hpp"
#include <cstddef>
#include <cstdint>

namespace zke {
namespace dev {

using zke::WITNESS_THREADS;   // witness_program.hpp: the stream's formats and constants
using zke::WOP_NOP;
static const uint32_t WITNESS_TERM_BUF = 8192;   // LC terms staged in shared memory per iteration (x 2 buffers x 8 B)

// number of kernels launched by this library since load (reported by bench.py as gpu_launches)
extern unsigned long long g_kernel_launches;
#define ZKE_COUNT_LAUNCH(n) (::zke::dev::g_kernel_launches += (n))

// SMs of the current device (132 on an H100 SXM): grid-stride and persistent kernels are sized in multiples of it
inline int sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
        return 132;
    return n;
}

// Witness program resident in HBM (built once per circuit): the stream of witness_program.hpp, which gives the formats.
struct DevProgram {
    const uint4* ops;            // [n_iters][WITNESS_THREADS]
    const uint4* iter_hdr;       // [n_iters + 2 * cluster]
    const uint32_t* coop;        // cooperative ops of the iterations (executed by the whole CTA), two words each
    const uint2* terms;
    const uint32_t* aux;
    const uint8_t* coef_r;       // [n_coefs][32]: coefficient * R mod r  (Montgomery-scaled: (cR) (x) w = c*w)
    const uint8_t* small_inv;    // [n_small_inv][32]: x^-1 mod r in standard form, entry 0 unused
    uint32_t n_small_inv;
    uint32_t n_iters, n_ops, n_vars, n_temps, n_outputs, n_inputs;
    uint32_t cluster;            // CTAs per email (thread-block cluster): iteration k belongs to CTA k % cluster, every level is
                                 // padded to whole rounds of `cluster` iterations (1: one CTA walks all of them)
    unsigned long long* trace;   // optional (diagnostics): clock64() of CTA 0 after every iteration
};

// R1CS matrices resident in HBM.
struct DevR1cs {
    const uint32_t *a_ptr, *b_ptr, *c_ptr;
    const uint2 *a_terms, *b_terms, *c_terms;   // {var, coefficient word (lc_term.cuh)}
    const uint8_t* coef_r;                      // same table as DevProgram::coef_r
    uint32_t n_constraints, n_public, n_vars;
};

void upload_field_constants();

cudaError_t configure_witness_kernel();   // once per device, before the first launch_witness on it
void launch_witness(const DevProgram& P, uint8_t* w_all, size_t stride_elems, const uint8_t* inputs, uint32_t batch, cudaStream_t st);

// circom's `===` check for a batch of witnesses in one launch, nothing stored: first_bad[e] (initialised to 0xffffffff by the
// caller) = smallest row of email e with <A,w><B,w> != <C,w>
void launch_check_rows(const DevR1cs& R, const uint8_t* w_all, size_t stride_elems, uint32_t batch, uint32_t* first_bad, cudaStream_t st);

// a[i] = <A_i, w>, b[i] = <B_i, w> in Montgomery form for i < n_constraints, the n_public + 1 extra rows of the
// Groth16 QAP (a = w_j, b = 0), zero padding up to n; also checks <A,w><B,w> = <C,w> and atomically records the
// smallest violated row in *first_bad (initialised to 0xffffffff by the caller).
// c_out (optional): a_i * b_i in Montgomery form (fused Hadamard product).  R1CS term words use the encoding of
// lc_term.cuh.
// flag[0] = 1 if any of the n 32-byte values is >= r, flag[1] = 1 if some witness (stride_elems apart) has w[0] != 1
void launch_check_witness(const uint8_t* w_all, size_t stride_elems, uint32_t n_vars, uint32_t batch, uint32_t* flag, cudaStream_t st);

// map (optional): thread t handles row ((t >> log_cols) << log_m) + col0 + (t & (2^log_cols - 1)) instead of row t - the
// rows of the column range one GPU holds when a proof is sharded (n = number of threads = rows handled).
struct RowMap { int log_cols = -1, log_m = 0; uint32_t col0 = 0; };
void launch_build_ab(const DevR1cs& R, const uint8_t* w, uint8_t* a_out, uint8_t* b_out, uint8_t* c_out, uint32_t n, uint32_t* first_bad, cudaStream_t st,
                     const RowMap* map = nullptr);

}  // namespace dev
}  // namespace zke
