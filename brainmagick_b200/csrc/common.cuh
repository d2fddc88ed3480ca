// Shared device/host helpers for the brainmagick_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>

namespace bm {

// ---- error plumbing (C-ABI returns an int, message kept for bm_last_error()) -------------------
extern thread_local char g_last_error[512];
extern int g_debug_flags;               // bm_set_debug_flags(): experiment switches (none defined: every kernel ignores them)
extern long long* g_debug_buf;           // bm_set_debug_buffer(): device scratch for cycle counters (no kernel records any)
extern unsigned long long g_launches;   // kernels launched by this library since load (bm_launch_count())
inline int set_error(int code, const char* fmt, const char* a = "", const char* b = "") {
    snprintf(g_last_error, sizeof(g_last_error), fmt, a, b);
    return code;
}
#define BM_CHECK_ARG(cond)                                                                          \
    do {                                                                                            \
        if (!(cond)) return ::bm::set_error(2, "%s: invalid argument: %s", __func__, #cond);        \
    } while (0)
#define BM_CHECK_LAUNCH()                                                                           \
    do {                                                                                            \
        cudaError_t e_ = cudaGetLastError();                                                        \
        ++::bm::g_launches;                                                                         \
        if (e_ != cudaSuccess) return ::bm::set_error(3, "%s: launch failed: %s", __func__, cudaGetErrorString(e_)); \
    } while (0)
#define BM_CUDA(call)                                                                               \
    do {                                                                                            \
        cudaError_t e_ = (call);                                                                    \
        if (e_ != cudaSuccess) return ::bm::set_error(3, "%s: %s", #call, cudaGetErrorString(e_));  \
    } while (0)

// ---- math ---------------------------------------------------------------------------------------
// erf-GELU (nn.GELU() default; bm/models/simpleconv.py:85-86, bm/models/common.py:120) and its derivative, branch-free:
// Phi(z) = erfc(-z/sqrt2)/2 with the Chebyshev-fitted complementary error function of Numerical Recipes (erfcc):
//     erfc(x) = t exp(-x^2 + P(t)),  t = 1/(1 + x/2),  x >= 0        fractional error < 1.2e-7 EVERYWHERE, so the tails keep
// their relative accuracy (measured in fp32 over [-9, 9]: <= 7e-6 relative at |z| > 8, ~1e-7 elsewhere).  erff() + expf()
// cost about twice the instructions and made the HBM-bound BatchNorm/GELU kernels ALU-bound.
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void gelu_parts(float z, float& cdf, float& pdf) {
    const float ax = fabsf(z) * 0.70710678118654752440f;
    const float t = rcp_approx(fmaf(0.5f, ax, 1.0f));            // MUFU.RCP (1 ulp); __frcp_rn branches on special cases
    float poly = fmaf(t, 0.17087277f, -0.82215223f);
    poly = fmaf(t, poly, 1.48851587f);
    poly = fmaf(t, poly, -1.13520398f);
    poly = fmaf(t, poly, 0.27886807f);
    poly = fmaf(t, poly, -0.18628806f);
    poly = fmaf(t, poly, 0.09678418f);
    poly = fmaf(t, poly, 0.37409196f);
    poly = fmaf(t, poly, 1.00002368f);
    poly = fmaf(t, poly, -1.26551223f);
    const float half_erfc = 0.5f * t * __expf(fmaf(-ax, ax, poly));       // Phi(-|z|)
    cdf = z >= 0.f ? 1.0f - half_erfc : half_erfc;
    pdf = 0.39894228040143267794f * __expf(-0.5f * z * z);
}
__device__ __forceinline__ float gelu_f(float z) {
    float cdf, pdf;
    gelu_parts(z, cdf, pdf);
    return z * cdf;
}
// d/dz GELU(z) = Phi(z) + z * phi(z)
__device__ __forceinline__ float gelu_grad_f(float z) {
    float cdf, pdf;
    gelu_parts(z, cdf, pdf);
    return fmaf(z, pdf, cdf);
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// for the HBM-bound GLU backward (MUFU.EX2 + MUFU.RCP instead of the IEEE division and expf).  __expf's error, 2 +
// floor(|1.173 x|) ulp, reaches the result scaled by 1 - sigmoid(x), and 1 + e and rcp.approx add one rounding and 1 ulp:
// about 4 ulp for x >= 0, but up to (4 + floor(1.173 |x|)) ulp for x < 0 (~40 ulp at x = -30)
__device__ __forceinline__ float sigmoid_fast(float x) { return rcp_approx(1.0f + __expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

inline int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 148;
    }
    return n;
}

inline bool aligned16(const void* a, const void* b = nullptr, const void* c = nullptr) {
    return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) == 0;
}

inline int ew_grid(long long total, int block = 256, int per_thread = 1) {
    long long g = (total / per_thread + block - 1) / block;
    long long cap = (long long)num_sms() * 16;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace bm
