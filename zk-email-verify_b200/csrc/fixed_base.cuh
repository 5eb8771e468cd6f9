#pragma once
#include "ec.cuh"
namespace zke {
namespace dev {
// out_affine[i] = scalars[i] * G for the generator whose window table is `table` (see fixed_base.cu).
// scratch_xyzz must hold n XYZZ points.
template <class F>
void fixed_base_batch(const uint8_t* table, const uint8_t* scalars, uint32_t n, uint8_t* scratch_xyzz, uint8_t* out_affine, cudaStream_t st);
// out_affine[i] = 2^k * in_affine[i]; scratch_xyzz must hold n XYZZ points (builds the window levels of a fixed-base table)
template <class F>
void xyzz_to_affine_batch(const uint8_t* in_xyzz, uint32_t n, uint8_t* out_affine, cudaStream_t st);
template <class F>
void scale_pow2_batch(const uint8_t* in_affine, uint32_t n, int k, uint8_t* scratch_xyzz, uint8_t* out_affine, cudaStream_t st);
}  // namespace dev
}  // namespace zke
