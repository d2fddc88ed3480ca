// Pre-model batch preparation (SURVEY.md 8(f) row 2): the per-recording affine of BatchScaler._transform
// (bm/norm.py:239-275), the clamp / peak detection of ScaleReject (bm/norm.py:325-341) and the offset crop of
// Solver._process_batch (bm/solver.py:262-274) as ONE pass over the batch.
//
// HBM-bound: algorithmic traffic = 4 B read + 4 B written per kept element, nothing else (the [R, C] tables stay in
// L1/L2).  One warp owns one (sample, channel) row of T contiguous floats, so every access is a coalesced 128 B line;
// the arithmetic is two separately rounded fp32 operations (subtract, IEEE divide), bit-identical to torch's CPU result.
#pragma once
#include "common.cuh"

namespace bm {

constexpr int PREP_ILP = 8;

// x [B, C, T] -> y [B, C, T_out] = op(x[..., t0 : t0 + T_out]);  op = (x - center[slot[b]][c]) / scale[slot[b]][c]
// (or x * scale + center when `inverse`), then clamp to +-limit when `clip`.
// peak_bits[b] = max over the WHOLE sample (all T, like the reference, which rejects before it crops) of |op(x)|, as
// the bit pattern of a non-negative float (monotonic as unsigned -> plain atomicMax, order independent).
// With `clip` the peak can never exceed the limit (and without `peak_bits` nobody asks), so the cropped-away samples are
// not even read.
__global__ void scale_clamp_crop_kernel(const float* __restrict__ x, const int* __restrict__ slot,
                                        const float* __restrict__ center, const float* __restrict__ scale, int B,
                                        int C, int T, int t0, int T_out, float limit, int clip, int inverse,
                                        float* __restrict__ y, unsigned* __restrict__ peak_bits) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    const long long n_rows = (long long)B * C;
    const bool window_only = clip || peak_bits == nullptr;      // nothing outside the kept window can matter
    const int t_lo = window_only ? t0 : 0, t_hi = window_only ? t0 + T_out : T;
    for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < n_rows; row += warps) {
        const int b = (int)(row / C), c = (int)(row - (long long)b * C);
        const int s = slot ? slot[b] : 0;
        // a recording the scaler was never fitted on (the reference raises KeyError, norm.py:256): poison the sample with
        // NaN instead of reading outside the table; Solver._process_batch asserts finiteness right after (solver.py:256)
        const bool known = s >= 0;
        const float ctr = known ? center[(long long)s * C + c] : __int_as_float(0x7fc00000);
        const float scl = known ? scale[(long long)s * C + c] : 1.f;
        const float* xr = x + row * T;
        float* yr = y + row * T_out;
        float peak = 0.f;
        // 8 independent 128 B loads in flight per warp before the first use (a row is ~11 such lines)
        for (int base = t_lo; base < t_hi; base += 32 * PREP_ILP) {
            float v[PREP_ILP];
#pragma unroll
            for (int i = 0; i < PREP_ILP; ++i) {
                const int t = base + i * 32 + lane;
                v[i] = t < t_hi ? xr[t] : 0.f;
            }
#pragma unroll
            for (int i = 0; i < PREP_ILP; ++i) {
                const int t = base + i * 32 + lane;
                float w = inverse ? __fadd_rn(__fmul_rn(v[i], scl), ctr) : __fdiv_rn(__fsub_rn(v[i], ctr), scl);
                if (clip) w = w < -limit ? -limit : (w > limit ? limit : w);     // NaN stays NaN, like Tensor.clamp_
                if (t < t_hi) {
                    peak = fmaxf(peak, fabsf(w));
                    if (t >= t0 && t < t0 + T_out) yr[t - t0] = w;
                }
            }
        }
        if (peak_bits) {
            peak = warp_max(peak);
            if (lane == 0) atomicMax(peak_bits + b, __float_as_uint(peak));
        }
    }
}

// reject[b] = peak[b] > limit  ||  (mask != NULL && the sample's features mask is empty)        (norm.py:334-337)
// keep_rows = the kept sample indices in order, n_keep[0] = how many; one block, B is a batch size.
__global__ void reject_compact_kernel(const unsigned* __restrict__ peak_bits, const unsigned char* __restrict__ mask,
                                      long long mask_elems, float limit, int B, unsigned char* __restrict__ keep,
                                      int* __restrict__ keep_rows, int* __restrict__ n_keep) {
    __shared__ int s_keep[1024];
    __shared__ int s_base;
    if (threadIdx.x == 0) s_base = 0;
    for (int b0 = 0; b0 < B; b0 += blockDim.x) {
        const int b = b0 + threadIdx.x;
        int k = 0;
        if (b < B) {
            k = !(__uint_as_float(peak_bits[b]) > limit);
            if (k && mask) {
                bool any = false;
                const unsigned char* m = mask + (long long)b * mask_elems;
                for (long long i = 0; i < mask_elems && !any; ++i) any = m[i] != 0;
                k = any;
            }
            keep[b] = (unsigned char)k;
        }
        s_keep[threadIdx.x] = k;
        __syncthreads();
        if (threadIdx.x == 0) {             // B <= a few thousand: a serial scan of one block's flags is negligible
            int base = s_base;
            for (int i = 0; i < blockDim.x && b0 + i < B; ++i)
                if (s_keep[i]) keep_rows[base++] = b0 + i;
            s_base = base;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) n_keep[0] = s_base;
}

// y[i][:] = x[rows[i]][:]   (batch[keep], norm.py:340) -- only launched when something was rejected
__global__ void gather_rows_kernel(const float* __restrict__ x, const int* __restrict__ rows, int n_rows,
                                   long long row_elems, float* __restrict__ y) {
    const long long total = (long long)n_rows * row_elems;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / row_elems, e = i - r * row_elems;
        y[i] = x[(long long)rows[r] * row_elems + e];
    }
}

// y[rows[i]][:] = x[i][:], the inverse of gather_rows_kernel: a batch written into free rows of the negative pool's
// device storage (the rows must be distinct)
__global__ void scatter_rows_kernel(const float* __restrict__ x, const int* __restrict__ rows, int n_rows,
                                    long long row_elems, float* __restrict__ y) {
    const long long total = (long long)n_rows * row_elems;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / row_elems, e = i - r * row_elems;
        y[(long long)rows[r] * row_elems + e] = x[i];
    }
}

// y[b][c][t] = x[b][c][t] * mask[c]   (simpleconv.py:200-203: `subsample_meg_channels` zeroes the sensors not drawn)
__global__ void channel_mask_kernel(const float* __restrict__ x, const float* __restrict__ mask, float* __restrict__ y,
                                    int C, int T, long long total) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)((i / T) % C);
        y[i] = x[i] * mask[c];
    }
}

// in [Z][N][T] -> out [Z][T][N]   (32x32 tiles through shared memory, both sides coalesced)
__global__ void transpose_nt_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int T, int ld_out,
                                    int n_store) {
    // n_store = N: plain transpose; n_store = ld_out > N: the pad columns [N, ld_out) are written as zeros
    __shared__ float tile[32][33];
    const long long zoff = (long long)blockIdx.z * N * T;
    const long long zout = (long long)blockIdx.z * T * ld_out;
    int t = blockIdx.x * 32 + threadIdx.x;
#pragma unroll
    for (int i = threadIdx.y; i < 32; i += 8) {
        int n = blockIdx.y * 32 + i;
        tile[i][threadIdx.x] = (n < N && t < T) ? in[zoff + (long long)n * T + t] : 0.f;
    }
    __syncthreads();
    int n = blockIdx.y * 32 + threadIdx.x;
#pragma unroll
    for (int i = threadIdx.y; i < 32; i += 8) {
        int tt = blockIdx.x * 32 + i;
        if (n < n_store && tt < T) out[zout + (long long)tt * ld_out + n] = tile[threadIdx.x][i];
    }
}

// ------------------------------------------------------------------------------------------------
// ClipLoss's `assert mask.all()` (bm/losses.py:110) without a host read: status <- code (if still 0) when any of the n
// bytes of `mask` is 0.  `vec`: mask is 16-byte aligned, read as uint4 (the last n % 16 bytes one by one).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool has_zero_byte(unsigned w) { return ((w - 0x01010101u) & ~w & 0x80808080u) != 0u; }

__global__ void check_all_true_kernel(const unsigned char* __restrict__ mask, long long n, bool vec, int code,
                                      int* __restrict__ status) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    bool bad = false;
    long long tail = 0;
    if (vec) {
        const long long nv = n >> 4;
        const uint4* m4 = reinterpret_cast<const uint4*>(mask);
        for (long long i = tid; i < nv; i += stride) {
            const uint4 w = __ldg(m4 + i);
            bad |= has_zero_byte(w.x) | has_zero_byte(w.y) | has_zero_byte(w.z) | has_zero_byte(w.w);
        }
        tail = nv << 4;
    }
    for (long long i = tail + tid; i < n; i += stride) bad |= mask[i] == 0;
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicCAS(status, 0, code);
}

}  // namespace bm
