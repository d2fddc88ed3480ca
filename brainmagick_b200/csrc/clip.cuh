// ClipLoss pieces beside the score GEMMs (clip_api.cu): candidate norms, the row cross-entropy, the score gradient G that
// the backward GEMMs contract, and the candidate-side correction.
#pragma once
#include "common.cuh"

namespace bm {

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

// ---- ClipLoss, gradient w.r.t. the candidates -----------------------------------------------------------------
// scores[b][o] = inv_o <e_b, c_o>, inv_o = 1/(1e-8 + ||c_o||)   (losses.py:91-94).  With G = dL/d<e_b, c_o> (the matrix
// clip_ce_bwd_kernel builds), dL/dc_o = sum_b G[b][o] e_b  -  coef_o c_o,
//   coef_o = (sum_b G[b][o] scores[b][o]) / ||c_o||      (the derivative of inv_o; 0 for a zero candidate, as autograd's
//                                                          norm backward defines it)
__global__ void clip_cand_coef_kernel(const float* __restrict__ G, const float* __restrict__ scores,
                                      const float* __restrict__ inv_norm, int Bn, int Bc, float* __restrict__ coef) {
    int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= Bc) return;
    float acc = 0.f;
    for (int b = 0; b < Bn; ++b) acc = fmaf(G[(long long)b * Bc + o], scores[(long long)b * Bc + o], acc);
    float norm = 1.f / inv_norm[o] - 1e-8f;
    coef[o] = norm > 0.f ? acc / norm : 0.f;
}

// dcand[o][k] -= coef[o] * cand[o][k]
__global__ void clip_cand_correct_kernel(const float* __restrict__ cand, const float* __restrict__ coef, long long KT,
                                         long long total, float* __restrict__ dcand) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int o = (int)(i / KT);
        dcand[i] = fmaf(-coef[o], cand[i], dcand[i]);
    }
}

}  // namespace bm
