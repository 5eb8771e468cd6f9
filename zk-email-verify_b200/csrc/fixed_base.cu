// Fixed-base scalar multiplication batches for the trusted setup: out[i] = scalars[i] * G with G the G1 or G2
// generator, via a table of 32 x 256 window multiples (8-bit windows) built on the host.  Not on the proving path.
#include "device_engine.cuh"
#include "fixed_base.cuh"

namespace zke {
namespace dev {

static const int TO_AFFINE_BATCH = 8;

// table[(w * 256 + d)] = d * 2^(8 w) * G  (affine, Montgomery; d = 0 is the point at infinity)
template <class F>
__global__ void __launch_bounds__(128)
fixed_base_kernel(const uint8_t* __restrict__ table, const uint8_t* __restrict__ scalars, uint32_t n, uint8_t* out_xyzz) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s = Fr::load(scalars + 32ull * i);
    XYZZ<F> acc = XYZZ<F>::inf();
    for (int w = 0; w < 32; ++w) {
        const uint32_t d = (s.v[w >> 2] >> (8 * (w & 3))) & 0xff;
        if (d) acc.madd(Affine<F>::load(table + sizeof(Affine<F>) * (size_t)(w * 256 + d)), false);
    }
    acc.store(out_xyzz + sizeof(XYZZ<F>) * (size_t)i);
}

template <class F>
__global__ void __launch_bounds__(128)
xyzz_to_affine_kernel(const uint8_t* __restrict__ in_xyzz, uint32_t n, uint8_t* out_affine) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t beg = t * TO_AFFINE_BATCH;
    if (beg >= n) return;
    const uint32_t cnt = min((uint32_t)TO_AFFINE_BATCH, n - beg);
    // Montgomery's trick on u_i = zz_i * zzz_i
    F prefix[TO_AFFINE_BATCH];
    F acc = F::one();
    for (uint32_t k = 0; k < cnt; ++k) {
        XYZZ<F> p = XYZZ<F>::load(in_xyzz + sizeof(XYZZ<F>) * (size_t)(beg + k));
        prefix[k] = acc;
        if (!p.is_inf()) acc = acc * (p.zz * p.zzz);
    }
    F inv = acc.inv();
    for (uint32_t k = cnt; k-- > 0;) {
        XYZZ<F> p = XYZZ<F>::load(in_xyzz + sizeof(XYZZ<F>) * (size_t)(beg + k));
        Affine<F> a;
        if (p.is_inf()) { a.x = F::zero(); a.y = F::zero(); }
        else {
            F u_inv = inv * prefix[k];          // 1 / (zz zzz)
            inv = inv * (p.zz * p.zzz);
            a.x = p.x * (u_inv * p.zzz);        // x / zz
            a.y = p.y * (u_inv * p.zz);         // y / zzz
        }
        a.store(out_affine + sizeof(Affine<F>) * (size_t)(beg + k));
    }
}

// out[i] = 2^k * in[i]  (affine in, XYZZ out)
template <class F>
__global__ void __launch_bounds__(128)
scale_pow2_kernel(const uint8_t* __restrict__ in_affine, uint32_t n, int k, uint8_t* out_xyzz) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    XYZZ<F> p = XYZZ<F>::from_affine(Affine<F>::load(in_affine + sizeof(Affine<F>) * (size_t)i));
    for (int j = 0; j < k; ++j) p.dbl();
    p.store(out_xyzz + sizeof(XYZZ<F>) * (size_t)i);
}

template <class F>
void scale_pow2_batch(const uint8_t* in_affine, uint32_t n, int k, uint8_t* scratch_xyzz, uint8_t* out_affine, cudaStream_t st) {
    if (!n) return;
    scale_pow2_kernel<F><<<(n + 127) / 128, 128, 0, st>>>(in_affine, n, k, scratch_xyzz);
    const uint32_t threads = (n + TO_AFFINE_BATCH - 1) / TO_AFFINE_BATCH;
    xyzz_to_affine_kernel<F><<<(threads + 127) / 128, 128, 0, st>>>(scratch_xyzz, n, out_affine);
    ZKE_COUNT_LAUNCH(2);
}
template void scale_pow2_batch<Fq>(const uint8_t*, uint32_t, int, uint8_t*, uint8_t*, cudaStream_t);

template <class F>
void fixed_base_batch(const uint8_t* table, const uint8_t* scalars, uint32_t n, uint8_t* scratch_xyzz, uint8_t* out_affine, cudaStream_t st) {
    if (!n) return;
    fixed_base_kernel<F><<<(n + 127) / 128, 128, 0, st>>>(table, scalars, n, scratch_xyzz);
    const uint32_t threads = (n + TO_AFFINE_BATCH - 1) / TO_AFFINE_BATCH;
    xyzz_to_affine_kernel<F><<<(threads + 127) / 128, 128, 0, st>>>(scratch_xyzz, n, out_affine);
    ZKE_COUNT_LAUNCH(2);
}
template void fixed_base_batch<Fq>(const uint8_t*, const uint8_t*, uint32_t, uint8_t*, uint8_t*, cudaStream_t);
template void fixed_base_batch<Fq2>(const uint8_t*, const uint8_t*, uint32_t, uint8_t*, uint8_t*, cudaStream_t);

template <class F>
void xyzz_to_affine_batch(const uint8_t* in_xyzz, uint32_t n, uint8_t* out_affine, cudaStream_t st) {
    if (!n) return;
    const uint32_t threads = (n + TO_AFFINE_BATCH - 1) / TO_AFFINE_BATCH;
    xyzz_to_affine_kernel<F><<<(threads + 127) / 128, 128, 0, st>>>(in_xyzz, n, out_affine);
    ZKE_COUNT_LAUNCH(1);
}
template void xyzz_to_affine_batch<Fq>(const uint8_t*, uint32_t, uint8_t*, cudaStream_t);
template void xyzz_to_affine_batch<Fq2>(const uint8_t*, uint32_t, uint8_t*, cudaStream_t);

}  // namespace dev
}  // namespace zke

namespace zke { namespace dev { ZKE_DEFINE_CONSTANT_UPLOAD(upload_constants_fixed_base) } }
