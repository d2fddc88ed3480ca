// HBM-bound kernels of the hot path: everything that is not a contraction.
// Activations are channels-last [B, T, C] inside the encoder (rows = B*T), so a warp always walks
// contiguous channels; per-channel parameters are read through the read-only path.
#pragma once
#include "common.cuh"

namespace bm {

// ------------------------------------------------------------------------------------------------
// K1 pieces: Fourier embedding of sensor positions and the masked softmax (common.py:254-271,339-357)
// ------------------------------------------------------------------------------------------------
// emb[rc][k*n+l] = cos(loc), emb[rc][P/2 + k*n+l] = sin(loc), loc = (x+margin)*f[k] + (y+margin)*f[l]
// `freq` is the table 2*pi*arange(n)/(1+2*margin) built by the host with the reference's own op order, and
// the products/sum are rounded separately (no FMA contraction) so that `loc` is bit-identical to torch's.
__global__ void fourier_emb_kernel(const float* __restrict__ pos, const float* __restrict__ freq, float margin,
                                   int RC, int n, float* __restrict__ emb) {
    const int P2 = n * n;
    long long total = (long long)RC * P2;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        int rc = (int)(idx / P2);
        int kl = (int)(idx - (long long)rc * P2);
        int k = kl / n, l = kl - k * n;
        float x = __fadd_rn(pos[2 * rc], margin), y = __fadd_rn(pos[2 * rc + 1], margin);
        float loc = __fadd_rn(__fmul_rn(x, freq[k]), __fmul_rn(y, freq[l]));
        float s, c;
        sincosf(loc, &s, &c);
        emb[(long long)rc * 2 * P2 + kl] = c;
        emb[(long long)rc * 2 * P2 + P2 + kl] = s;
    }
}

// in-place softmax over c of scores[r][o][:] with -inf on invalid (pos == INVALID) and banned sensors
// (||pos - centre|| <= radius, training only).  One warp per (r, o) row.
__global__ void masked_softmax_kernel(float* __restrict__ w, const float* __restrict__ pos,
                                      const float* __restrict__ centre, float radius, float invalid, int R, int O,
                                      int C) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= R * O) return;
    int r = row / O;
    float* s = w + (long long)row * C;
    const float* pr = pos + (long long)r * C * 2;
    float cx = 0.f, cy = 0.f;
    if (centre) { cx = centre[0]; cy = centre[1]; }
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) {
        float x = pr[2 * c], y = pr[2 * c + 1];
        bool masked = (x == invalid) && (y == invalid);
        if (centre) {
            float dx = x - cx, dy = y - cy;
            masked = masked || (sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) <= radius);
        }
        float v = masked ? -INFINITY : s[c];
        s[c] = v;
        mx = fmaxf(mx, v);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) {
        float e = expf(s[c] - mx);
        s[c] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    float inv = 1.f / sum;
    for (int c = lane; c < C; c += 32) s[c] *= inv;
}

// dscore = w * (dw - sum_c w*dw)   (softmax backward, one warp per row)
__global__ void softmax_bwd_kernel(const float* __restrict__ w, const float* __restrict__ dw,
                                   float* __restrict__ ds, int rows, int C) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* wr = w + (long long)row * C;
    const float* dr = dw + (long long)row * C;
    float dot = 0.f;
    for (int c = lane; c < C; c += 32) dot += wr[c] * dr[c];
    dot = warp_sum(dot);
    for (int c = lane; c < C; c += 32) ds[(long long)row * C + c] = wr[c] * (dr[c] - dot);
}

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

// eval mode: mean = running_mean, invstd = 1/sqrt(running_var + eps)
__global__ void bn_eval_stats_kernel(const float* __restrict__ rm, const float* __restrict__ rv, float eps,
                                     float* __restrict__ mean, float* __restrict__ invstd, int C) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    mean[c] = rm[c];
    invstd[c] = 1.f / sqrtf(rv[c] + eps);
}

// ------------------------------------------------------------------------------------------------
// GLU backward (common.py:133-138): h = [a | b] per row (2H columns), out = a*sigmoid(b)
// ------------------------------------------------------------------------------------------------
__global__ void glu_bwd_kernel(const float* __restrict__ g, const float* __restrict__ h, float* __restrict__ dh,
                               long long rows, int H) {
    long long total = rows * H;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        long long r = i / H;
        int c = (int)(i - r * H);
        float a = h[r * 2 * H + c], b = h[r * 2 * H + H + c];
        float s = sigmoid_f(b);
        float gg = g[i];
        dh[r * 2 * H + c] = gg * s;
        dh[r * 2 * H + H + c] = gg * a * s * (1.f - s);
    }
}

// dh = dq * GELU'(h)   (head, simpleconv.py:185-189)
__global__ void gelu_bwd_kernel(const float* __restrict__ dq, const float* __restrict__ h, float* __restrict__ dh,
                                long long total) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x)
        dh[i] = dq[i] * gelu_grad_f(h[i]);
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
// conv weight re-layout: W[o][i][j] -> Wf[j][i][o] (forward B operand) and Wb[j][o][i] (data-gradient B operand)
// ------------------------------------------------------------------------------------------------
__global__ void weight_prep_kernel(const float* __restrict__ W, float* __restrict__ Wf, float* __restrict__ Wb,
                                   int O, int I, int Kw) {
    long long total = (long long)O * I * Kw;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        int j = (int)(idx % Kw);
        long long oi = idx / Kw;
        int i = (int)(oi % I), o = (int)(oi / I);
        float v = W[idx];
        if (Wf) Wf[((long long)j * I + i) * O + o] = v;
        if (Wb) Wb[((long long)j * O + o) * I + i] = v;
    }
}

// ------------------------------------------------------------------------------------------------
// ClipLoss pieces (losses.py:91-114)
// ------------------------------------------------------------------------------------------------
// ss[o] += sum_k cand[o][k]^2 (fp64 atomics; grid = (rows, splits)).  With one split, every slot receives exactly one add
// onto its zero: the deterministic form.
__device__ __forceinline__ void row_sumsq_row(const float* __restrict__ x, double* __restrict__ ss, long long K) {
    __shared__ double red[32];
    long long chunk = (K + gridDim.y - 1) / gridDim.y;
    long long k0 = (long long)blockIdx.y * chunk, k1 = min(K, k0 + chunk);
    float s = 0.f;
    double acc = 0.0;
    int cnt = 0;
    for (long long k = k0 + threadIdx.x; k < k1; k += blockDim.x) {
        float v = x[k];
        s = fmaf(v, v, s);
        if (++cnt == 64) { acc += (double)s; s = 0.f; cnt = 0; }
    }
    acc += (double)s;
    acc = warp_sum_d(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
        v = warp_sum_d(v);
        if (threadIdx.x == 0) atomicAdd(ss + blockIdx.x, v);
    }
}
__global__ void row_sumsq_kernel(const float* __restrict__ X, double* __restrict__ ss, long long K) {
    row_sumsq_row(X + (long long)blockIdx.x * K, ss, K);
}
// the same over pooled candidates: row o is X[o] for o < Bb (the batch), else arena[slots[o - Bb]] (the negative pool)
__global__ void row_sumsq_pooled_kernel(const float* __restrict__ X, int Bb, const float* __restrict__ arena,
                                        const int* __restrict__ slots, double* __restrict__ ss, long long K) {
    const int o = blockIdx.x;
    row_sumsq_row(o < Bb ? X + (long long)o * K : arena + (long long)slots[o - Bb] * K, ss, K);
}

// inv_norm[o] = 1 / (1e-8 + sqrt(ss[o]))    (losses.py:91)
__global__ void inv_norm_kernel(const double* __restrict__ ss, float* __restrict__ inv, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) inv[i] = 1.f / (1e-8f + (float)sqrt(ss[i]));
}

// per row b: lse, row_loss[b] = lse - s[b][b+off]; optional probs = softmax(s)   (one block per row)
__global__ void clip_ce_rows_kernel(const float* __restrict__ scores, int Bn, int Bc, int target_offset,
                                    float* __restrict__ row_loss, float* __restrict__ probs) {
    __shared__ float red[32];
    __shared__ float bcast;
    int b = blockIdx.x;
    const float* s = scores + (long long)b * Bc;
    float mx = -INFINITY;
    for (int o = threadIdx.x; o < Bc; o += blockDim.x) mx = fmaxf(mx, s[o]);
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : -INFINITY;
        v = warp_max(v);
        if (threadIdx.x == 0) bcast = v;
    }
    __syncthreads();
    mx = bcast;
    __syncthreads();
    float sum = 0.f;
    for (int o = threadIdx.x; o < Bc; o += blockDim.x) sum += expf(s[o] - mx);
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) bcast = v;
    }
    __syncthreads();
    sum = bcast;
    if (row_loss && threadIdx.x == 0) row_loss[b] = (logf(sum) + mx) - s[b + target_offset];
    if (probs) {
        float inv = 1.f / sum;
        for (int o = threadIdx.x; o < Bc; o += blockDim.x) probs[(long long)b * Bc + o] = expf(s[o] - mx) * inv;
    }
}

// loss = mean(row_loss)  (single block, deterministic order)
__global__ void mean_kernel(const float* __restrict__ x, int n, float* __restrict__ out) {
    __shared__ double red[32];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += (double)x[i];
    s = warp_sum_d(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
        v = warp_sum_d(v);
        if (threadIdx.x == 0) out[0] = (float)(v / n);
    }
}

// G[b][o] = gout * (softmax(s)[b][o] - [o == b+off]) / Bn * inv_norm[o]    (A.6 of SURVEY.md)
// transposed != 0: G is written as [Bc][Bn] (the dY operand layout of the tensor-core dE GEMM)
__global__ void clip_ce_bwd_kernel(const float* __restrict__ probs, const float* __restrict__ inv_norm,
                                   const float* __restrict__ gout, int Bn, int Bc, int target_offset,
                                   float* __restrict__ G, int transposed) {
    long long total = (long long)Bn * Bc;
    float gs = gout[0] / (float)Bn;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        int b = (int)(i / Bc), o = (int)(i - (long long)b * Bc);
        float p = probs[i] - (o == b + target_offset ? 1.f : 0.f);
        float v = gs * p * inv_norm[o];
        if (transposed) G[(long long)o * Bn + b] = v;
        else G[i] = v;
    }
}

// clip_ce_bwd_kernel's G [Bn][Bc] in rows of ld >= Bc floats, the columns Bc..ld-1 zero (the pooled backward's GEMM reads
// G in float4 steps along the candidates)
__global__ void clip_ce_bwd_padded_kernel(const float* __restrict__ probs, const float* __restrict__ inv_norm,
                                          const float* __restrict__ gout, int Bn, int Bc, int ld, int target_offset,
                                          float* __restrict__ G) {
    long long total = (long long)Bn * ld;
    float gs = gout[0] / (float)Bn;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        int b = (int)(i / ld), o = (int)(i - (long long)b * ld);
        float v = 0.f;
        if (o < Bc) {
            float p = probs[(long long)b * Bc + o] - (o == b + target_offset ? 1.f : 0.f);
            v = gs * p * inv_norm[o];
        }
        G[i] = v;
    }
}

// G[b][o] = dscores[b][o] * inv_norm[o]: the same G for an arbitrary upstream gradient of the scores (get_scores backward);
// transposed as in clip_ce_bwd_kernel
__global__ void clip_scores_grad_kernel(const float* __restrict__ dscores, const float* __restrict__ inv_norm, int Bn, int Bc,
                                        float* __restrict__ G, int transposed) {
    long long total = (long long)Bn * Bc;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        int b = (int)(i / Bc), o = (int)(i - (long long)b * Bc);
        float v = dscores[i] * inv_norm[o];
        if (transposed) G[(long long)o * Bn + b] = v;
        else G[i] = v;
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
// float4 versions (C % 4 == 0, 16-byte aligned rows): one thread owns 4 consecutive channels
// ------------------------------------------------------------------------------------------------
__global__ void glu_bwd_v4_kernel(const float4* __restrict__ g, const float4* __restrict__ h, float4* __restrict__ dh,
                                  long long rows, int H) {
    const int H4 = H >> 2;
    long long total = rows * H4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / H4;
        const int c4 = (int)(i - r * H4);
        const float4 a = h[r * 2 * H4 + c4], b = h[r * 2 * H4 + H4 + c4], gg = g[i];
        float4 da, db;
        float s;
        s = sigmoid_f(b.x); da.x = gg.x * s; db.x = gg.x * a.x * s * (1.f - s);
        s = sigmoid_f(b.y); da.y = gg.y * s; db.y = gg.y * a.y * s * (1.f - s);
        s = sigmoid_f(b.z); da.z = gg.z * s; db.z = gg.z * a.z * s * (1.f - s);
        s = sigmoid_f(b.w); da.w = gg.w * s; db.w = gg.w * a.w * s * (1.f - s);
        dh[r * 2 * H4 + c4] = da;
        dh[r * 2 * H4 + H4 + c4] = db;
    }
}

__global__ void gelu_bwd_v4_kernel(const float4* __restrict__ dq, const float4* __restrict__ h, float4* __restrict__ dh,
                                   long long total4) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4;
         i += (long long)gridDim.x * blockDim.x) {
        const float4 d = dq[i], x = h[i];
        dh[i] = make_float4(d.x * gelu_grad_f(x.x), d.y * gelu_grad_f(x.y), d.z * gelu_grad_f(x.z), d.w * gelu_grad_f(x.w));
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
