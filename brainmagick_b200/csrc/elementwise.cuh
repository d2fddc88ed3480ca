// HBM-bound kernels of the FP32-FMA layers: BatchNorm finalize, column reductions and the column-stationary GLU backward.
// Templates only: front_api.cu and convseq_api.cu both include this header.
// Activations are channels-last [B, T, C] inside the encoder (rows = B*T), so a warp always walks
// contiguous channels; per-channel parameters are read through the read-only path.
#pragma once
#include "common.cuh"

namespace bm {

// ------------------------------------------------------------------------------------------------
// BatchNorm1d statistics (common.py:118-120); the layer epilogue that applies them is in convseq.cuh
// ------------------------------------------------------------------------------------------------
// stats[0:C] = sum y, stats[C:2C] = sum y^2 (fp64) over n = B*T rows  ->  mean, invstd (biased var),
// running stats update with the unbiased variance (momentum), as nn.BatchNorm1d in training mode.
// COUNTED: n is read from stats[2C] on the device (a SyncBatchNorm group's row count, all-reduced with the sums).
// batches (nullable): the layer's num_batches_tracked, already incremented for this batch; momentum is then torch's
// cumulative-average factor 1 / num_batches_tracked (momentum=None), computed here so that the host never reads the count.
template <bool COUNTED = false>
__global__ void bn_finalize_kernel(const double* __restrict__ stats, double n, float eps, float momentum,
                                   const long long* __restrict__ batches, float* running_mean, float* running_var,
                                   float* __restrict__ mean, float* __restrict__ invstd, int C) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    if (COUNTED) n = stats[2 * C];
    if (batches) momentum = (float)(1.0 / (double)*batches);
    double m = stats[c] / n;
    double var = stats[C + c] / n - m * m;
    if (var < 0) var = 0;
    mean[c] = (float)m;
    invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
    if (running_mean) {
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
        double unb = n > 1 ? var * n / (n - 1) : var;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
    }
}

// ------------------------------------------------------------------------------------------------
// bias gradients
// ------------------------------------------------------------------------------------------------
// out[c] += sum_r X[r][c]   (channels-last rows); out must be zeroed by the caller
// DET (here and in the column reductions below): out is a [gridDim.x][C] partials buffer, the block stores its row
template <bool DET = false>
__global__ void colsum_cl_kernel(const float* __restrict__ X, float* __restrict__ out, long long rows, int C,
                                 int rows_per_block) {
    int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = min(rows, r0 + rows_per_block);
    float s = 0.f;
#pragma unroll 4
    for (long long r = r0; r < r1; ++r) s += X[r * C + c];
    if (DET) out[(long long)blockIdx.x * C + c] = s;
    else atomicAdd(out + c, s);
}

// out[c] += sum_r X[r*ld + c]   (rows with a leading dimension ld >= C)
template <bool DET = false>
__global__ void colsum_strided_kernel(const float* __restrict__ X, float* __restrict__ out, long long rows, int C,
                                      int ld, int rows_per_block) {
    int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = min(rows, r0 + rows_per_block);
    float s = 0.f;
#pragma unroll 4
    for (long long r = r0; r < r1; ++r) s += X[r * ld + c];
    if (DET) out[(long long)blockIdx.x * C + c] = s;
    else atomicAdd(out + c, s);
}

// stats[c] += sum_r X[r][c], stats[C+c] += sum_r X[r][c]^2   (fp64 atomics; BatchNorm batch statistics)
// The per-thread sums are fp64 too: bn_finalize_kernel takes the variance as E[y^2] - E[y]^2, and fp32 partial sums of
// squares would lose it to rounding once a channel's mean is ~100x its standard deviation.
// DET: stats is a [gridDim.x][2C] partials buffer
template <bool DET = false>
__global__ void col_stats_kernel(const float* __restrict__ X, double* __restrict__ stats, long long rows, int C,
                                 int rows_per_block) {
    int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = min(rows, r0 + rows_per_block);
    double s = 0.0, q = 0.0;
#pragma unroll 4
    for (long long r = r0; r < r1; ++r) {
        const double v = X[r * C + c];
        s += v;
        q = fma(v, v, q);
    }
    if (DET) {
        stats[(long long)blockIdx.x * 2 * C + c] = s;
        stats[(long long)blockIdx.x * 2 * C + C + c] = q;
        return;
    }
    atomicAdd(stats + c, s);
    atomicAdd(stats + C + c, q);
}

// out[n] += sum_{z,t} X[z][n][t]  (channel-major [Z,N,T]); one warp per (z, n) row
// DET: out is a [Z][N] partials buffer that receives each row's sum
template <bool DET = false>
__global__ void rowsum_cm_kernel(const float* __restrict__ X, float* __restrict__ out, int Z, int N, int T) {
    long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= (long long)Z * N) return;
    const float* x = X + row * T;
    float s = 0.f;
    for (int t = lane; t < T; t += 32) s += x[t];
    s = warp_sum(s);
    if (lane == 0) {
        if (DET) out[row] = s;
        else atomicAdd(out + (int)(row % N), s);
    }
}

// ------------------------------------------------------------------------------------------------
// Column-stationary kernels (channels-last rows, C % 4 == 0, C/4 <= 256: GLU backward here, the layer epilogue in convseq.cuh):
// block = (C/4, RY) threads; thread (cx, ry) owns columns 4cx..4cx+3 for the rows ry, ry+RY, ... of the block's row range, so
// the per-column parameters live in registers (no i % C, no parameter reloads, no fp64 divisions per element) and every
// warp-level access is a contiguous row piece.  Rows are unrolled by 4 for memory-level parallelism.
// ------------------------------------------------------------------------------------------------
constexpr int CS_ROWS_PER_BLOCK = 96, CS_U = 4;       // rows per block; rows per thread whose loads are issued together

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4s(const float* p) { return __ldcs(reinterpret_cast<const float4*>(p)); }   // streamed once

// max |.| of what a block has just written -> ONE atomicMax per block on `cell` (the bits of a non-negative float order like
// unsigned integers).  The consumer is the F16-pipe conv (bm_tc_conv1d_f16), which scales its operand by a power of two from it:
// fusing the reduction here saves bm_amax's extra pass over the tensor.  Every thread of the block must call.
__device__ __forceinline__ float amax4(float m, const float4& o) {
    return fmaxf(fmaxf(m, fmaxf(fabsf(o.x), fabsf(o.y))), fmaxf(fabsf(o.z), fabsf(o.w)));
}
__device__ __forceinline__ void block_amax_commit(float m, unsigned int* cell) {
    __shared__ float warp_max[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y;
    if ((tid & 31) == 0) warp_max[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < (nthr + 31) / 32; ++w) m = fmaxf(m, warp_max[w]);
        if (m > 0.f) atomicMax(cell, __float_as_uint(m));
    }
}

// GLU backward, column-stationary (H % 4 == 0, H/4 <= 256): thread (cx, ry) owns a-columns 4cx.. and the matching gate columns;
// optionally accumulates the bias gradient of the GLU convolution, dbias[c] = sum_rows dh[row][c] (2H columns), from the values
// it has just produced (shared-memory combine over the row lanes, one fp32 atomic per column per block; zeroed by the caller).
// DET: dbias is a [gridDim.x][2H] partials buffer, the block stores its row.
template <bool DET = false>
__global__ void __launch_bounds__(320, 2)
glu_bwd_cs_kernel(const float* __restrict__ g, const float* __restrict__ h, float* __restrict__ dh, float* __restrict__ dbias,
                  long long rows, int H, unsigned int* __restrict__ amax) {
    extern __shared__ float red[];                       // [RY][2H]
    const int c = threadIdx.x * 4, RY = blockDim.y;
    const long long r0 = (long long)blockIdx.x * CS_ROWS_PER_BLOCK;
    const long long r1 = min(rows, r0 + CS_ROWS_PER_BLOCK);
    float4 sa = make_float4(0.f, 0.f, 0.f, 0.f), sb = sa;
    float am = 0.f;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)CS_U * RY) {
        float4 av[CS_U], bv[CS_U], gv[CS_U];
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) { av[k] = ld4s(h + rr * 2 * H + c); bv[k] = ld4s(h + rr * 2 * H + H + c); gv[k] = ld4s(g + rr * H + c); }
        }
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) {
                const float4 a = av[k], b = bv[k], gg = gv[k];
                float4 da, db;
                float s;
                s = sigmoid_fast(b.x); da.x = gg.x * s; db.x = gg.x * a.x * s * (1.f - s);
                s = sigmoid_fast(b.y); da.y = gg.y * s; db.y = gg.y * a.y * s * (1.f - s);
                s = sigmoid_fast(b.z); da.z = gg.z * s; db.z = gg.z * a.z * s * (1.f - s);
                s = sigmoid_fast(b.w); da.w = gg.w * s; db.w = gg.w * a.w * s * (1.f - s);
                *reinterpret_cast<float4*>(dh + rr * 2 * H + c) = da;
                *reinterpret_cast<float4*>(dh + rr * 2 * H + H + c) = db;
                sa.x += da.x; sa.y += da.y; sa.z += da.z; sa.w += da.w;
                sb.x += db.x; sb.y += db.y; sb.z += db.z; sb.w += db.w;
                am = amax4(amax4(am, da), db);
            }
        }
    }
    if (amax) block_amax_commit(am, amax);
    if (!dbias) return;
    float* mine = red + (size_t)threadIdx.y * 2 * H;
    *reinterpret_cast<float4*>(mine + c) = sa;
    *reinterpret_cast<float4*>(mine + H + c) = sb;
    __syncthreads();
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y;
    for (int i = tid; i < 2 * H; i += nthr) {
        float acc = 0.f;
        for (int ry = 0; ry < RY; ++ry) acc += red[(size_t)ry * 2 * H + i];
        if (DET) dbias[(long long)blockIdx.x * 2 * H + i] = acc;
        else atomicAdd(dbias + i, acc);
    }
}

// out[c] = sum_{r < n} part[r][c] in the order r = 0, 1, ..., n-1: the fixed-order second half of every deterministic column
// reduction above (T = double where the atomic form accumulates in fp64, float where it accumulates in fp32)
template <class T>
__global__ void reduce_rows_kernel(const T* __restrict__ part, long long n, int W, T* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= W) return;
    T s = 0;
    for (long long r = 0; r < n; ++r) s += part[r * W + c];
    out[c] = s;
}


}  // namespace bm
