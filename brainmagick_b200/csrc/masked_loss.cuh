// Masked regression losses (bm/losses.py:11-26, L1Loss / L2Loss): mean |e - o| or mean (e - o)^2 over the entries where
// the broadcast mask is True, and their gradients, without a host read of the True count.
//
// Operands: est and out are [B, C, T] with t-stride 1 and any (b, c) strides and element offset (the solver's time crop
// estimate[..., limit:] is read in place); mask is bytes read through its own (b, c, t) strides (0 where it broadcasts).
// A row is one (b, c); it is walked in chunks of 4 time steps, through float4 loads when both row starts are 16-byte
// aligned and scalar loads otherwise.
//
//   masked_loss_partials_kernel  fixed grid (ml_blocks: shape and SM count); CTA k owns rows [k*rows/n, (k+1)*rows/n) and
//                                stores its fp64 (sum, count) -- each thread's chunks in a fixed order, then a fixed tree
//   masked_loss_finalize_kernel  one CTA: the partials in a fixed tree -> loss = sum / N, inv_n = 1 / N (fp32)
//   masked_loss_bwd_kernel       d_est = s(e - o) * g * inv_n where the mask is True, else 0 (s = sign for L1, 2x for L2);
//                                d_out = -d_est; contiguous [B, C, T] outputs, float4 stores when T % 4 == 0 and both
//                                outputs are 16-byte aligned
// No atomics anywhere: the loss and the gradients are bitwise repeatable.
#pragma once
#include "common.cuh"

namespace bm {

constexpr int ML_THREADS = 256;
constexpr int ML_FINAL_THREADS = 512;

enum MaskedLossKind { ML_L1 = 0, ML_L2 = 1 };

struct MlOperands {
    const float* est;
    long long e_sb, e_sc;
    const float* out;
    long long o_sb, o_sc;
    const unsigned char* mask;
    long long m_sb, m_sc, m_st;
    int C, T;
};

// CTAs of the partials kernel: two per SM, never more than there are rows
inline int ml_blocks(long long rows) {
    long long n = 2ll * num_sms();
    if (n > rows) n = rows;
    return n < 1 ? 1 : (int)n;
}

// Reads the up to 4 elements of chunk k of row r: e[i], o[i] and the mask bits; returns the number of valid elements
__device__ __forceinline__ int ml_load_chunk(const MlOperands& p, long long r, int k, float (&e)[4], float (&o)[4],
                                             bool (&m)[4]) {
    const int b = (int)(r / p.C), c = (int)(r - (long long)b * p.C);
    const float* er = p.est + b * p.e_sb + c * p.e_sc;
    const float* orow = p.out + b * p.o_sb + c * p.o_sc;
    const unsigned char* mr = p.mask + b * p.m_sb + c * p.m_sc;
    const int t0 = 4 * k;
    const int n = min(4, p.T - t0);
    const bool vec = n == 4 && ((reinterpret_cast<uintptr_t>(er) | reinterpret_cast<uintptr_t>(orow)) & 15) == 0;
    if (vec) {
        const float4 ev = __ldg(reinterpret_cast<const float4*>(er + t0));
        const float4 ov = __ldg(reinterpret_cast<const float4*>(orow + t0));
        e[0] = ev.x; e[1] = ev.y; e[2] = ev.z; e[3] = ev.w;
        o[0] = ov.x; o[1] = ov.y; o[2] = ov.z; o[3] = ov.w;
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            e[i] = i < n ? __ldg(er + t0 + i) : 0.f;
            o[i] = i < n ? __ldg(orow + t0 + i) : 0.f;
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) m[i] = i < n && __ldg(mr + (t0 + i) * p.m_st) != 0;
    return n;
}

// fixed-order CTA reduction of (sum, count); the result is valid in thread 0
__device__ __forceinline__ void ml_block_sum(double& s, double& n) {
    __shared__ double ss[32], sn[32];
    s = warp_sum_d(s);
    n = warp_sum_d(n);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if ((threadIdx.x & 31) == 0) { ss[w] = s; sn[w] = n; }
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < nw ? ss[threadIdx.x] : 0.0;
        n = threadIdx.x < nw ? sn[threadIdx.x] : 0.0;
        s = warp_sum_d(s);
        n = warp_sum_d(n);
    }
}

template <int KIND>
__global__ void __launch_bounds__(ML_THREADS) masked_loss_partials_kernel(MlOperands p, long long rows,
                                                                         double* __restrict__ part) {
    const long long r0 = rows * blockIdx.x / gridDim.x, r1 = rows * (blockIdx.x + 1) / gridDim.x;
    const int nch = (p.T + 3) >> 2;
    const long long chunks = (r1 - r0) * nch;
    double s = 0.0, cnt = 0.0;
    for (long long j = threadIdx.x; j < chunks; j += ML_THREADS) {
        const long long rr = j / nch;
        float e[4], o[4];
        bool m[4];
        ml_load_chunk(p, r0 + rr, (int)(j - rr * nch), e, o, m);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (!m[i]) continue;
            const float d = e[i] - o[i];                       // fp32, as torch forms the difference
            s += KIND == ML_L1 ? (double)fabsf(d) : (double)d * (double)d;
            cnt += 1.0;
        }
    }
    ml_block_sum(s, cnt);
    if (threadIdx.x == 0) {
        part[2 * blockIdx.x] = s;
        part[2 * blockIdx.x + 1] = cnt;
    }
}

// loss = sum / N and inv_n = 1 / N; N = 0 gives loss NaN (0 / 0, torch's mean of nothing) and inv_n inf, which the
// backward never multiplies into a value (every entry is then masked out)
__global__ void __launch_bounds__(ML_FINAL_THREADS) masked_loss_finalize_kernel(const double* __restrict__ part, int n,
                                                                               float* __restrict__ loss,
                                                                               float* __restrict__ inv_n) {
    double s = 0.0, cnt = 0.0;
    for (int i = threadIdx.x; i < n; i += ML_FINAL_THREADS) {
        s += part[2 * i];
        cnt += part[2 * i + 1];
    }
    ml_block_sum(s, cnt);
    if (threadIdx.x == 0) {
        loss[0] = (float)(s / cnt);
        inv_n[0] = (float)(1.0 / cnt);
    }
}

template <int KIND>
__global__ void __launch_bounds__(ML_THREADS) masked_loss_bwd_kernel(MlOperands p, long long rows,
                                                                    const float* __restrict__ g,
                                                                    const float* __restrict__ inv_n,
                                                                    float* __restrict__ d_est, float* __restrict__ d_out,
                                                                    bool vec_out) {
    // L1: sign(d) * (g / N), sign(0) = sign(NaN) = 0 as torch's sgn; L2: d * (2 g / N), as torch's mse_loss backward
    const float scale = (KIND == ML_L1 ? 1.f : 2.f) * (__ldg(g) * __ldg(inv_n));
    const int nch = (p.T + 3) >> 2;
    const long long chunks = rows * nch;
    for (long long j = blockIdx.x * (long long)ML_THREADS + threadIdx.x; j < chunks; j += (long long)gridDim.x * ML_THREADS) {
        const long long r = j / nch;
        const int k = (int)(j - r * nch);
        float e[4], o[4], v[4], w[4];
        bool m[4];
        const int n = ml_load_chunk(p, r, k, e, o, m);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float d = e[i] - o[i];
            const float f = (KIND == ML_L1 ? (float)((d > 0.f) - (d < 0.f)) : d) * scale;
            v[i] = m[i] ? f : 0.f;                             // a select: a masked-out NaN or inf stays out
            w[i] = m[i] ? -f : 0.f;
        }
        const long long at = r * p.T + 4 * k;
        if (vec_out && n == 4) {
            if (d_est) *reinterpret_cast<float4*>(d_est + at) = make_float4(v[0], v[1], v[2], v[3]);
            if (d_out) *reinterpret_cast<float4*>(d_out + at) = make_float4(w[0], w[1], w[2], w[3]);
        } else {
            for (int i = 0; i < n; ++i) {
                if (d_est) d_est[at + i] = v[i];
                if (d_out) d_out[at + i] = w[i];
            }
        }
    }
}

}  // namespace bm
