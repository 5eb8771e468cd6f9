// CPU harness for zk-email-verify_b200/csrc/ec_ntt.cuh under ZKE_FF_EMULATE (tests/test_ec_ntt_emulation.py): the per-point
// scaling and the point transform, run thread by thread as the kernels of ptau.cu launch them, with the affine
// conversion between stages done here point by point.
#define ZKE_FF_EMULATE
#include "ec_ntt.cuh"
#include <cstring>
#include <vector>
using namespace zke::dev;

template <class F>
static void to_affine(const uint8_t* in_xyzz, uint32_t n, uint8_t* out_affine) {
    for (uint32_t i = 0; i < n; ++i) {
        const XYZZ<F> p = XYZZ<F>::load(in_xyzz + sizeof(XYZZ<F>) * i);
        Affine<F> a;
        if (p.is_inf()) { a.x = F::zero(); a.y = F::zero(); }
        else { a.x = p.x * p.zz.inv(); a.y = p.y * p.zzz.inv(); }
        a.store(out_affine + sizeof(Affine<F>) * i);
    }
}

template <class F>
static void scale(uint32_t n, const uint8_t* in_affine, const uint32_t* scalars, uint8_t* out_affine) {
    std::vector<uint8_t> x((size_t)n * sizeof(XYZZ<F>));
    for (uint32_t i = 0; i < n; ++i) scale_point_each<F>(in_affine, scalars, 1, 0, i, x.data());
    to_affine<F>(x.data(), n, out_affine);
}

// out = n^-1 sum_j omega^(-ij) in[j], n = 2^log_n; tw: omega_n^-j (j < n/2) in standard form, n_inv: 1/n in standard form
template <class F>
static void transform(int log_n, const uint8_t* in_affine, const uint32_t* tw, const uint32_t* n_inv, uint8_t* out_affine) {
    const uint32_t n = 1u << log_n;
    std::vector<uint8_t> x((size_t)n * sizeof(XYZZ<F>));
    for (uint32_t i = 0; i < n; ++i) scale_point_each<F>(in_affine, n_inv, 0, log_n, i, x.data());
    to_affine<F>(x.data(), n, out_affine);
    for (uint32_t m = 1; m < n; m <<= 1) {
        for (uint32_t t = 0; t < n / 2; ++t) point_butterfly<F>(out_affine, m, tw, n / (2 * m), t, x.data());
        to_affine<F>(x.data(), n, out_affine);
    }
}

extern "C" {
void en_set_consts(const uint32_t* mod, const uint32_t* r, const uint32_t* r2, uint32_t inv) {
    memcpy(FQ_C.mod, mod, 32); memcpy(FQ_C.r, r, 32); memcpy(FQ_C.r2, r2, 32); FQ_C.inv = inv;
}
void en_scale(int g2, uint32_t n, const uint8_t* in_affine, const uint32_t* scalars, uint8_t* out_affine) {
    if (g2) scale<Fq2>(n, in_affine, scalars, out_affine);
    else scale<Fq>(n, in_affine, scalars, out_affine);
}
void en_transform(int g2, int log_n, const uint8_t* in_affine, const uint32_t* tw, const uint32_t* n_inv, uint8_t* out_affine) {
    if (g2) transform<Fq2>(log_n, in_affine, tw, n_inv, out_affine);
    else transform<Fq>(log_n, in_affine, tw, n_inv, out_affine);
}
}
