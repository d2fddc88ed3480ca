// Layer epilogues of a stand-alone ConvSequence (bm/models/common.py:79-151) outside the clip_conv family -- the
// DeepMel feature model (bm/models/features.py:15-35; conf/feature_model/deep_mel.yaml) uses LeakyReLU(0) and leaves its
// last layer without BatchNorm / activation -- and the candidate-side gradient of ClipLoss that a trainable feature model
// needs (bm/losses.py:91-94 differentiated w.r.t. `candidates`).
//
// HBM-bound elementwise / column-reduction kernels over channels-last rows [rows, C]; the BatchNorm+GELU case of the
// brain encoder keeps its own tuned kernels in elementwise.cuh.
#pragma once
#include "common.cuh"

namespace bm {

enum { ACT_GELU = 0, ACT_LRELU = 1, ACT_NONE = 2 };

__device__ __forceinline__ float act_f(int act, float z, float slope) {
    if (act == ACT_GELU) return gelu_f(z);
    if (act == ACT_LRELU) return z > 0.f ? z : z * slope;          // nn.LeakyReLU (common.py:95)
    return z;
}
__device__ __forceinline__ float act_grad_f(int act, float z, float slope) {
    if (act == ACT_GELU) return gelu_grad_f(z);
    if (act == ACT_LRELU) return z > 0.f ? 1.f : slope;
    return 1.f;
}

// x_new = act(bn(y)) (+ x_old);  bn(y) = (y - mean) * invstd * gamma + beta, or y itself when mean == NULL
__global__ void bn_act_skip_fwd_kernel(const float* __restrict__ y, const float* __restrict__ mean,
                                       const float* __restrict__ invstd, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, const float* __restrict__ x_old,
                                       float* __restrict__ x_new, long long total, int C, int act, float slope) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        float z = y[i];
        if (mean) {
            const int c = (int)(i % C);
            z = (z - mean[c]) * invstd[c] * gamma[c] + beta[c];
        }
        float a = act_f(act, z, slope);
        x_new[i] = x_old ? a + x_old[i] : a;
    }
}

// backward pass 1 (BatchNorm only): sums[c] += sum dz, sums[C+c] += sum dz*yhat  with dz = g * act'(z)
// DET: sums is a [gridDim.x][2C] partials buffer, the block stores its row
template <bool DET = false>
__global__ void bn_act_bwd_reduce_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                         const float* __restrict__ mean, const float* __restrict__ invstd,
                                         const float* __restrict__ gamma, const float* __restrict__ beta,
                                         double* __restrict__ sums, long long rows, int C, int rows_per_block, int act,
                                         float slope) {
    int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = min(rows, r0 + rows_per_block);
    float mu = mean[c], is = invstd[c], ga = gamma[c], be = beta[c];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll 4
    for (long long r = r0; r < r1; ++r) {
        float yh = (y[r * C + c] - mu) * is;
        float dz = g[r * C + c] * act_grad_f(act, yh * ga + be, slope);
        s1 += dz;
        s2 += dz * yh;
    }
    if (DET) {
        sums[(long long)blockIdx.x * 2 * C + c] = (double)s1;
        sums[(long long)blockIdx.x * 2 * C + C + c] = (double)s2;
        return;
    }
    atomicAdd(sums + c, (double)s1);
    atomicAdd(sums + C + c, (double)s2);
}

// backward pass 2: dy = gamma*invstd*(dz - mean(dz) - yhat*mean(dz*yhat))   (training BatchNorm)
//                  dy = gamma*invstd*dz                                      (eval BatchNorm: use_batch_stats = 0)
//                  dy = g * act'(y)                                          (no BatchNorm: mean == NULL)
// COUNTED: n is read from sums[2C] on the device (a SyncBatchNorm group's row count, all-reduced with the sums)
template <bool COUNTED = false>
__global__ void bn_act_bwd_apply_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                        const float* __restrict__ mean, const float* __restrict__ invstd,
                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                        const double* __restrict__ sums, double n, int use_batch_stats,
                                        float* __restrict__ dy, long long total, int C, int act, float slope) {
    if (COUNTED) n = sums[2 * C];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        if (!mean) {
            dy[i] = g[i] * act_grad_f(act, y[i], slope);
            continue;
        }
        const int c = (int)(i % C);
        const float is = invstd[c], ga = gamma[c];
        const float yh = (y[i] - mean[c]) * is;
        const float dz = g[i] * act_grad_f(act, yh * ga + beta[c], slope);
        float v = dz;
        if (use_batch_stats) v = dz - (float)(sums[c] / n) - yh * (float)(sums[C + c] / n);
        dy[i] = ga * is * v;
    }
}

// ---- Residual gain: LayerScale and post_skip (common.py:65-76,126-130) ------------------------------------------------
// branch = act(bn(y)) (act(y) without BatchNorm), x_new = post[c] * ((boost * scale[c]) * branch) (+ x_old), in the
// reference's operation order; a NULL gain is 1.
__device__ __forceinline__ float gain_f(const float* __restrict__ scale, float boost, const float* __restrict__ post, int c,
                                        float v) {
    if (scale) v = (boost * scale[c]) * v;
    if (post) v = post[c] * v;
    return v;
}

__global__ void act_gain_skip_fwd_kernel(const float* __restrict__ y, const float* __restrict__ mean,
                                         const float* __restrict__ invstd, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, const float* __restrict__ x_old,
                                         float* __restrict__ x_new, long long total, int C, int act, float slope,
                                         const float* __restrict__ scale, float boost, const float* __restrict__ post) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        float z = y[i];
        if (mean) z = (z - mean[c]) * invstd[c] * gamma[c] + beta[c];
        const float a = gain_f(scale, boost, post, c, act_f(act, z, slope));
        x_new[i] = x_old ? a + x_old[i] : a;
    }
}

// backward pass 1: per column, fp64 per thread, sums[c] += sum dz, sums[C+c] += sum dz*yhat (BatchNorm only; dz = gain(g) *
// act'(z)) and sums[2C+c] += sum g*branch (the gains' common reduction; branch recomputed from y).
// DET: sums is a [gridDim.x][3C] partials buffer, the block stores its row
template <bool DET = false>
__global__ void act_gain_bwd_reduce_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                           const float* __restrict__ mean, const float* __restrict__ invstd,
                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                           double* __restrict__ sums, long long rows, int C, int rows_per_block, int act,
                                           float slope, const float* __restrict__ scale, float boost,
                                           const float* __restrict__ post) {
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    const long long r1 = min(rows, r0 + rows_per_block);
    float mu = 0.f, is = 1.f, ga = 1.f, be = 0.f;
    if (mean) { mu = mean[c]; is = invstd[c]; ga = gamma[c]; be = beta[c]; }
    double s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll 4
    for (long long r = r0; r < r1; ++r) {
        const float gv = g[r * C + c], yv = y[r * C + c];
        const float yh = mean ? (yv - mu) * is : yv;
        const float z = mean ? yh * ga + be : yv;
        s3 = fma((double)gv, (double)act_f(act, z, slope), s3);
        if (mean) {
            const double dz = gain_f(scale, boost, post, c, gv) * act_grad_f(act, z, slope);
            s1 += dz;
            s2 = fma(dz, (double)yh, s2);
        }
    }
    if (DET) {
        double* row = sums + (long long)blockIdx.x * 3 * C;
        row[c] = s1;
        row[C + c] = s2;
        row[2 * C + c] = s3;
        return;
    }
    if (mean) {
        atomicAdd(sums + c, s1);
        atomicAdd(sums + C + c, s2);
    }
    atomicAdd(sums + 2 * C + c, s3);
}

// dbeta = sums[c], dgamma = sums[C+c]; with S = sums[2C+c] = sum g*branch: dscale = boost*post*S, dpost = (boost*scale)*S.
// Every output is nullable.
__global__ void act_gain_param_grad_kernel(const double* __restrict__ sums, int C, const float* __restrict__ scale, float boost,
                                           const float* __restrict__ post, float* __restrict__ dgamma,
                                           float* __restrict__ dbeta, float* __restrict__ dscale, float* __restrict__ dpost) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    if (dbeta) dbeta[c] = (float)sums[c];
    if (dgamma) dgamma[c] = (float)sums[C + c];
    const double S = sums[2 * C + c];
    if (dscale) dscale[c] = (float)((double)boost * (post ? (double)post[c] : 1.0) * S);
    if (dpost) dpost[c] = (float)((scale ? (double)(boost * scale[c]) : 1.0) * S);
}

// backward pass 2 with gb = gain(g): dy = gamma*invstd*(dz - mean(dz) - yhat*mean(dz*yhat)), dz = gb*act'(z) (training
// BatchNorm); dy = gamma*invstd*dz (eval: use_batch_stats = 0); dy = gb*act'(y) (no BatchNorm: mean == NULL)
__global__ void act_gain_bwd_apply_kernel(const float* __restrict__ g, const float* __restrict__ y,
                                          const float* __restrict__ mean, const float* __restrict__ invstd,
                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                          const double* __restrict__ sums, double n, int use_batch_stats,
                                          float* __restrict__ dy, long long total, int C, int act, float slope,
                                          const float* __restrict__ scale, float boost, const float* __restrict__ post) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const float gb = gain_f(scale, boost, post, c, g[i]);
        if (!mean) {
            dy[i] = gb * act_grad_f(act, y[i], slope);
            continue;
        }
        const float is = invstd[c], ga = gamma[c];
        const float yh = (y[i] - mean[c]) * is;
        const float dz = gb * act_grad_f(act, yh * ga + beta[c], slope);
        float v = dz;
        if (use_batch_stats) v = dz - (float)(sums[c] / n) - yh * (float)(sums[C + c] / n);
        dy[i] = ga * is * v;
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
