// Host-side CUDA plumbing shared by the engine's translation unit (engine.cu with setup.cu and ptau.cu) and the
// verifier's (verify.cu): error checks, a device buffer, and device selection with the field constants of every TU.
#pragma once
#include "ff.cuh"
#include "ff_host.hpp"
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#define CUDA_OK(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " #expr); } while (0)

// launch-configuration errors are not sticky: pick them up right after the launches of a stage
#define CHECK_LAUNCH() CUDA_OK(cudaGetLastError())

namespace zke {

struct DevBuf {
    uint8_t* p = nullptr;
    size_t bytes = 0;
    DevBuf() {}
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    void alloc(size_t n) { release(); if (n) { CUDA_OK(cudaMalloc(&p, n)); bytes = n; } }
    // grow-only: allocates only when n exceeds the current size (the contents are not kept then)
    uint8_t* reserve(size_t n) { if (n > bytes) alloc(n); return p; }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    template <class T> void upload(const std::vector<T>& v) {
        alloc(v.size() * sizeof(T));
        if (!v.empty()) CUDA_OK(cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    }
};

inline void fill_consts(dev::FieldConsts& c, const FieldParams& p) {
    memcpy(c.mod, p.p.v, 32); memcpy(c.r, p.r.v, 32); memcpy(c.r2, p.r2.v, 32);
    c.inv = (uint32_t)p.inv;
    U256 zero = {{0, 0, 0, 0}}, n;
    u256_sub(n, zero, p.p);          // 2^256 - p
    memcpy(c.nmod, n.v, 32);
}

// Makes `device` current and uploads the field constants of every translation unit to it (engine.cu)
void select_device(int device);

}  // namespace zke
