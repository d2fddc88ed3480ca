// The conv of tc_convp.cuh with the weights given as TWO FP16 PIECES of a power-of-two-scaled copy (w*s = hi + lo, 11 + 11
// significant bits, s from the tensor's largest magnitude: bm_amax + bm_f16_split / bm_tc_weight_split_f16).  The pieces
// are summed back on load (~22 significant bits, the pieces' precision) and the GEMM runs on the same 3xTF32 engine; x_amax is accepted for the ABI and
// not needed.  The epilogue can also report max |output| (amax_out) for the conv that consumes the tensor next.
#pragma once
#include <cuda_fp16.h>
#include "tc_convp.cuh"

namespace bm {
namespace tc {

// ---- operand preparation ---------------------------------------------------------------------------------------------
// largest |x| of a tensor into `cell` (a float whose bits compare like an unsigned integer because it is non-negative);
// NaNs are ignored by fmaxf, +-inf gives inf (=> scale 1: the conv then propagates the non-finite values like fp32 would)
__global__ void __launch_bounds__(256) amax_kernel(const float* __restrict__ x, long long n, unsigned int* __restrict__ cell) {
    float m = 0.f;
    const long long n4 = n >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(x4 + i);
        m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
    }
    if (blockIdx.x == 0)
        for (long long i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(x[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float wm[8];
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) m = fmaxf(m, wm[w]);
        if (m > 0.f) atomicMax(cell, __float_as_uint(m));
    }
}
// src * scale(amax) -> fp16 hi and lo copies (same element order)
__global__ void __launch_bounds__(256) f16_split_kernel(const float* __restrict__ src, long long n,
                                                        const float* __restrict__ amax, __half* __restrict__ hi,
                                                        __half* __restrict__ lo) {
    const float s = f16_scale_of(__ldg(amax));
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = src[i] * s;
        const __half h = __float2half_rn(v);
        hi[i] = h;
        lo[i] = __float2half_rn(v - __half2float(h));
    }
}

// W[o][i][j] (nn.Conv1d layout) * scale(amax) -> fp16 hi / lo pieces in the K-major layouts of bm_tc_weight_split:
//   forward operand F[j][o][i], data-gradient operand G[j][i][o]; either pair may be NULL.  One launch per layer and step
//   instead of re-layout + two splits.
__global__ void __launch_bounds__(256) weight_split_f16_kernel(const float* __restrict__ W, const float* __restrict__ amax,
                                                               __half* __restrict__ f_hi, __half* __restrict__ f_lo,
                                                               __half* __restrict__ g_hi, __half* __restrict__ g_lo, int O, int I,
                                                               int Kw) {
    const float s = f16_scale_of(__ldg(amax));
    const long long total = (long long)O * I * Kw;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(idx % Kw);
        const long long oi = idx / Kw;
        const int i = (int)(oi % I), o = (int)(oi / I);
        const float v = W[idx] * s;
        const __half h = __float2half_rn(v);
        const __half l = __float2half_rn(v - __half2float(h));
        const long long fi = ((long long)j * O + o) * I + i, gi = ((long long)j * I + i) * O + o;
        if (f_hi) { f_hi[fi] = h; f_lo[fi] = l; }
        if (g_hi) { g_hi[gi] = h; g_lo[gi] = l; }
    }
}

struct ConvHPArgs {
    ConvPPArgs c;                    // c.w_raw unused
    const float* x_amax; const void* w_hi; const void* w_lo; const float* w_amax;
    float* out_amax;                 // nullable (zeroed by the caller)
};

inline int launch_conv_hp(const ConvHPArgs& h, cudaStream_t st) {
    const ConvPPArgs& a = h.c;
    const int nh = conv_pp_pick_nh(a.Ntot, a.glu);
    if (nh == 0 || nh % 32 != 0) return set_error(2, "%s: unsupported N%s", __func__);
    const int ntn = a.glu ? (a.Ntot / 2) / nh : a.Ntot / (2 * nh);
    if (a.stats && (a.glu || a.out_tmajor || a.act || a.accumulate || ntn != 1))
        return set_error(2, "%s: statistics need a plain single-N-tile conv%s", __func__);
    if (a.glu && (a.act || a.out_tmajor || a.aux || a.accumulate)) return set_error(2, "%s: GLU excludes the other epilogues%s", __func__);
    if (a.out_tmajor && (a.act || a.accumulate)) return set_error(2, "%s: channel-major output is a plain store%s", __func__);
    if (a.act && a.accumulate) return set_error(2, "%s: accumulate excludes the activation%s", __func__);
    ConvOp o = conv_pp_op(a);
    o.passes = 3;                    // the fp16-piece entry points have no single-pass form
    o.w = nullptr;
    o.w_hi = reinterpret_cast<const __half*>(h.w_hi); o.w_lo = reinterpret_cast<const __half*>(h.w_lo); o.w_amax = h.w_amax;
    o.out_amax = reinterpret_cast<unsigned int*>(h.out_amax);
    return launch_conv_op(o, st, __func__);
}

inline int launch_amax(const float* x, long long n, float* cell, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(cell, 0, 4, st);
    if (e != cudaSuccess) return set_error(3, "%s: memset: %s", __func__, cudaGetErrorString(e));
    long long blocks = (n / 4 + 255) / 256;
    const long long cap = (long long)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    amax_kernel<<<(int)blocks, 256, 0, st>>>(x, n, reinterpret_cast<unsigned int*>(cell));
    ++g_launches;
    e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: launch failed: %s", __func__, cudaGetErrorString(e));
    return 0;
}
inline int launch_f16_split(const float* src, long long n, const float* amax, void* hi, void* lo, cudaStream_t st) {
    f16_split_kernel<<<ew_grid(n), 256, 0, st>>>(src, n, amax, reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo));
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: launch failed: %s", __func__, cudaGetErrorString(e));
    return 0;
}

}  // namespace tc
}  // namespace bm
