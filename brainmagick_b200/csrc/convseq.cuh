// The ConvSequence layer epilogue (bm/models/common.py:65-76,79-151) of every convolution layer -- SimpleConv's encoder,
// the stand-alone ConvSequence and the DeepMel feature model (bm/models/features.py:15-35) -- and the other elementwise
// kernels of the FP32-FMA layers (convseq_api.cu): BatchNorm eval statistics, GLU and GELU backward, conv weight re-layout.
//
// Epilogue over channels-last rows [rows, C]: branch = act(bn(y)) with bn(y) = ((y - mean) * invstd) * gamma + beta (or y
// itself without a BatchNorm), x_new = post[c] * ((boost * scale[c]) * branch) (+ x_old) with the residual gains (LayerScale,
// post_skip) each optional.  Its backward is a column reduction -- sums (sum dz, sum dz*yhat) for the BatchNorm, dz =
// gain(g) * act'(z), and S = sum g*branch for the gains -- followed by an elementwise apply pass.  The activation, the
// BatchNorm's presence and the gains' presence are template parameters.  Two forms of each kernel, chosen by shape and
// alignment alone:
//   - column-stationary (C % 4 == 0, C/4 <= 256, 16-byte aligned operands): the per-column operands live in registers;
//   - generic (any shape): one thread per element, or per 4 elements through float4 accesses where C % 4 == 0 and the
//     operands are aligned (one thread per column in the reduction).
#pragma once
#include "elementwise.cuh"

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

// ---- column-stationary kernels --------------------------------------------------------------------------------------------
// block = (C/4, RY) threads; thread (cx, ry) owns columns 4cx..4cx+3 for the rows ry, ry+RY, ... of the block's
// CS_ROWS_PER_BLOCK rows, so the per-column operands live in registers (no i % C, no parameter reloads, no fp64 divisions per
// element) and every warp-level access is a contiguous row piece.  Rows are unrolled by CS_U for memory-level parallelism.
// ACT: the activation; BN: a BatchNorm in front of it (mean .. beta read), else z = y; GAIN: scale / post given (a NULL one
// is 1).

// the gains of columns c..c+3: ks = boost * scale, kp = post (1 where NULL; multiplying by 1 is exact)
__device__ __forceinline__ void gain_cols(const float* __restrict__ scale, float boost, const float* __restrict__ post, int c,
                                          float4& ks, float4& kp) {
    ks = kp = make_float4(1.f, 1.f, 1.f, 1.f);
    if (scale) {
        const float4 s = ld4(scale + c);
        ks = make_float4(boost * s.x, boost * s.y, boost * s.z, boost * s.w);
    }
    if (post) kp = ld4(post + c);
}

// one element of the forward: gain(act(bn(y))), in the reference's operation order
template <int ACT, bool BN, bool GAIN>
__device__ __forceinline__ float epi_fwd1(float y, float mu, float is, float ga, float be, float ks, float kp, float slope) {
    const float a = act_f(ACT, BN ? fmaf((y - mu) * is, ga, be) : y, slope);
    return GAIN ? kp * (ks * a) : a;
}

// one element of the apply pass: kk*(dz - m1 - yhat*m2) with kk = gamma*invstd (BN), else gain(g) * act'(y)
template <int ACT, bool BN, bool GAIN>
__device__ __forceinline__ float epi_apply1(float y, float g, float mu, float is, float ga, float be, float ks, float kp,
                                            float kk, float m1, float m2, float slope) {
    const float gb = GAIN ? kp * (ks * g) : g;
    if (!BN) return gb * act_grad_f(ACT, y, slope);
    const float yh = (y - mu) * is;
    return kk * (gb * act_grad_f(ACT, fmaf(yh, ga, be), slope) - m1 - yh * m2);
}

// x_new = gain(act(bn(y))) (+ x_old); amax: see block_amax_commit
template <int ACT, bool BN, bool GAIN>
__global__ void __launch_bounds__(320, 2)
epi_fwd_cs_kernel(const float* __restrict__ y, const float* __restrict__ mean, const float* __restrict__ invstd,
                  const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ x_old,
                  float* __restrict__ x_new, long long rows, int C, unsigned int* __restrict__ amax, float slope,
                  const float* __restrict__ scale, float boost, const float* __restrict__ post) {
    const int c = threadIdx.x * 4, RY = blockDim.y;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 mu = BN ? ld4(mean + c) : zero, is = BN ? ld4(invstd + c) : zero, ga = BN ? ld4(gamma + c) : zero,
                 be = BN ? ld4(beta + c) : zero;
    float4 ks, kp;
    if (GAIN) gain_cols(scale, boost, post, c, ks, kp);
    const long long r0 = (long long)blockIdx.x * CS_ROWS_PER_BLOCK;
    const long long r1 = min(rows, r0 + CS_ROWS_PER_BLOCK);
    float am = 0.f;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)CS_U * RY) {
        float4 v[CS_U], u[CS_U];
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) {
                v[k] = ld4s(y + rr * C + c);
                if (x_old) u[k] = ld4(x_old + rr * C + c);
            }
        }
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) {
                float4 o;
                o.x = epi_fwd1<ACT, BN, GAIN>(v[k].x, mu.x, is.x, ga.x, be.x, ks.x, kp.x, slope);
                o.y = epi_fwd1<ACT, BN, GAIN>(v[k].y, mu.y, is.y, ga.y, be.y, ks.y, kp.y, slope);
                o.z = epi_fwd1<ACT, BN, GAIN>(v[k].z, mu.z, is.z, ga.z, be.z, ks.z, kp.z, slope);
                o.w = epi_fwd1<ACT, BN, GAIN>(v[k].w, mu.w, is.w, ga.w, be.w, ks.w, kp.w, slope);
                if (x_old) { o.x += u[k].x; o.y += u[k].y; o.z += u[k].z; o.w += u[k].w; }
                *reinterpret_cast<float4*>(x_new + rr * C + c) = o;
                am = amax4(am, o);
            }
        }
    }
    if (amax) block_amax_commit(am, amax);
}

// backward pass 1: sums [NS*C] = (sum dz, sum dz*yhat[, S = sum g*branch]) (the BatchNorm sums stay 0 without BN); fp32 per
// thread, combined over the block's RY row lanes in shared memory, ONE fp64 atomic per sum and column per block (DET: sums is a
// [gridDim.x][NS*C] partials buffer, the block stores its row)
template <int ACT, bool BN, bool GAIN, bool DET = false>
__global__ void __launch_bounds__(320, 2)
epi_bwd_reduce_cs_kernel(const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ mean,
                         const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                         double* __restrict__ sums, long long rows, int C, float slope, const float* __restrict__ scale,
                         float boost, const float* __restrict__ post) {
    constexpr int NS = GAIN ? 3 : 2;                     // sums per column
    extern __shared__ float red[];                       // [RY][NS][C]
    const int c = threadIdx.x * 4, RY = blockDim.y;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 mu = BN ? ld4(mean + c) : zero, is = BN ? ld4(invstd + c) : zero, ga = BN ? ld4(gamma + c) : zero,
                 be = BN ? ld4(beta + c) : zero;
    float4 ks, kp;
    if (GAIN) gain_cols(scale, boost, post, c, ks, kp);
    const long long r0 = (long long)blockIdx.x * CS_ROWS_PER_BLOCK;
    const long long r1 = min(rows, r0 + CS_ROWS_PER_BLOCK);
    float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1, s3 = s1;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)CS_U * RY) {
        float4 yv[CS_U], gv[CS_U];
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) { yv[k] = ld4(y + rr * C + c); gv[k] = ld4(g + rr * C + c); }
        }
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) {
                // per column: s1 += dz, s2 += dz*yhat (BN), s3 += g*branch (GAIN).  Expanded in place: a helper taking the
                // sums by reference changes how the compiler assigns their registers.
                float yh, pre, dz;
#define EPI_RED1(X)                                                                                                           \
    yh = (yv[k].X - mu.X) * is.X;                                                                                             \
    pre = BN ? fmaf(yh, ga.X, be.X) : yv[k].X;                                                                                \
    if (BN) {                                                                                                                 \
        dz = (GAIN ? kp.X * (ks.X * gv[k].X) : gv[k].X) * act_grad_f(ACT, pre, slope);                                        \
        s1.X += dz;                                                                                                           \
        s2.X = fmaf(dz, yh, s2.X);                                                                                            \
    }                                                                                                                         \
    if (GAIN) s3.X = fmaf(gv[k].X, act_f(ACT, pre, slope), s3.X);
                EPI_RED1(x) EPI_RED1(y) EPI_RED1(z) EPI_RED1(w)
#undef EPI_RED1
            }
        }
    }
    float* mine = red + (size_t)threadIdx.y * NS * C;
    *reinterpret_cast<float4*>(mine + c) = s1;
    *reinterpret_cast<float4*>(mine + C + c) = s2;
    if (GAIN) *reinterpret_cast<float4*>(mine + 2 * C + c) = s3;
    __syncthreads();
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y;
    for (int i = tid; i < NS * C; i += nthr) {
        double acc = 0.0;
        for (int ry = 0; ry < RY; ++ry) acc += (double)red[(size_t)ry * NS * C + i];
        if (DET) sums[(long long)blockIdx.x * NS * C + i] = acc;
        else atomicAdd(sums + i, acc);
    }
}

// backward pass 2: dy = gamma*invstd*(dz - mean(dz) - yhat*mean(dz*yhat)); the two means come as dbeta/n and dgamma/n
// (written by epi_param_grad_kernel from the fp64 sums); eval mode (use_batch_stats = 0): dy = gamma*invstd*dz; without
// BN: dy = gain(g) * act'(y).
// COUNTED: the two sums are rounded from `sums` [2C + 1] here and rn = (float)(1 / sums[2C]) -- the same bits as the
// float sums of epi_param_grad_kernel and the host's (float)(1.0 / (double)rows) for the same row count.
template <int ACT, bool BN, bool GAIN, bool COUNTED = false>
__global__ void __launch_bounds__(320, 2)
epi_bwd_apply_cs_kernel(const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ mean,
                        const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                        const float* __restrict__ dgamma, const float* __restrict__ dbeta, const double* __restrict__ sums,
                        float rn, int use_batch_stats, float* __restrict__ dy, long long rows, int C,
                        unsigned int* __restrict__ amax, float slope, const float* __restrict__ scale, float boost,
                        const float* __restrict__ post) {
    const int c = threadIdx.x * 4, RY = blockDim.y;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 mu = BN ? ld4(mean + c) : zero, is = BN ? ld4(invstd + c) : zero, ga = BN ? ld4(gamma + c) : zero,
                 be = BN ? ld4(beta + c) : zero;
    float4 ks, kp;
    if (GAIN) gain_cols(scale, boost, post, c, ks, kp);
    float am = 0.f;
    float4 m1 = zero, m2 = zero;
    if (BN && use_batch_stats) {
        float4 db, dg;
        if (COUNTED) {
            rn = (float)(1.0 / sums[2 * C]);
            db = make_float4((float)sums[c], (float)sums[c + 1], (float)sums[c + 2], (float)sums[c + 3]);
            dg = make_float4((float)sums[C + c], (float)sums[C + c + 1], (float)sums[C + c + 2], (float)sums[C + c + 3]);
        } else {
            db = ld4(dbeta + c);
            dg = ld4(dgamma + c);
        }
        m1 = make_float4(db.x * rn, db.y * rn, db.z * rn, db.w * rn);
        m2 = make_float4(dg.x * rn, dg.y * rn, dg.z * rn, dg.w * rn);
    }
    const float4 kk = make_float4(ga.x * is.x, ga.y * is.y, ga.z * is.z, ga.w * is.w);
    const long long r0 = (long long)blockIdx.x * CS_ROWS_PER_BLOCK;
    const long long r1 = min(rows, r0 + CS_ROWS_PER_BLOCK);
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)CS_U * RY) {
        float4 yv[CS_U], gv[CS_U];
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) { yv[k] = ld4s(y + rr * C + c); gv[k] = ld4s(g + rr * C + c); }
        }
#pragma unroll
        for (int k = 0; k < CS_U; ++k) {
            const long long rr = r + (long long)k * RY;
            if (rr < r1) {
                float4 o;
                o.x = epi_apply1<ACT, BN, GAIN>(yv[k].x, gv[k].x, mu.x, is.x, ga.x, be.x, ks.x, kp.x, kk.x, m1.x, m2.x, slope);
                o.y = epi_apply1<ACT, BN, GAIN>(yv[k].y, gv[k].y, mu.y, is.y, ga.y, be.y, ks.y, kp.y, kk.y, m1.y, m2.y, slope);
                o.z = epi_apply1<ACT, BN, GAIN>(yv[k].z, gv[k].z, mu.z, is.z, ga.z, be.z, ks.z, kp.z, kk.z, m1.z, m2.z, slope);
                o.w = epi_apply1<ACT, BN, GAIN>(yv[k].w, gv[k].w, mu.w, is.w, ga.w, be.w, ks.w, kp.w, kk.w, m1.w, m2.w, slope);
                *reinterpret_cast<float4*>(dy + rr * C + c) = o;
                am = amax4(am, o);
            }
        }
    }
    if (amax) block_amax_commit(am, amax);
}

// ---- generic kernels ------------------------------------------------------------------------------------------------------
// One thread per element (per column in the reduction), the same template parameters and expressions; a NULL gain is 1.
__device__ __forceinline__ float gain_f(const float* __restrict__ scale, float boost, const float* __restrict__ post, int c,
                                        float v) {
    if (scale) v = (boost * scale[c]) * v;
    if (post) v = post[c] * v;
    return v;
}

// VEC = 4 (C % 4 == 0, 16-byte aligned operands): a thread owns 4 consecutive elements of a row, through float4 loads/stores
template <int ACT, bool BN, bool GAIN, int VEC>
__global__ void epi_fwd_kernel(const float* __restrict__ y, const float* __restrict__ mean, const float* __restrict__ invstd,
                               const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ x_old,
                               float* __restrict__ x_new, long long total, int C, float slope, const float* __restrict__ scale,
                               float boost, const float* __restrict__ post) {
    for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * VEC; i < total;
         i += (long long)gridDim.x * blockDim.x * VEC) {
        const int c = (int)(i % C);
        float v[VEC], o[VEC];
        if (VEC == 4) {
            const float4 t = ld4(y + i);
            v[0] = t.x; v[1 % VEC] = t.y; v[2 % VEC] = t.z; v[3 % VEC] = t.w;
            if (x_old) {
                const float4 u = ld4(x_old + i);
                o[0] = u.x; o[1 % VEC] = u.y; o[2 % VEC] = u.z; o[3 % VEC] = u.w;
            }
        } else {
            v[0] = y[i];
            if (x_old) o[0] = x_old[i];
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            float z = v[j];
            if (BN) z = (z - mean[c + j]) * invstd[c + j] * gamma[c + j] + beta[c + j];
            float a = act_f(ACT, z, slope);
            if (GAIN) a = gain_f(scale, boost, post, c + j, a);
            v[j] = x_old ? a + o[j] : a;
        }
        if (VEC == 4) *reinterpret_cast<float4*>(x_new + i) = make_float4(v[0], v[1 % VEC], v[2 % VEC], v[3 % VEC]);
        else x_new[i] = v[0];
    }
}

// backward pass 1, one thread per column: the sums of epi_bwd_reduce_cs_kernel, fp32 per thread
// DET: sums is a [gridDim.x][NS*C] partials buffer, the block stores its row
template <int ACT, bool BN, bool GAIN, bool DET = false>
__global__ void epi_bwd_reduce_kernel(const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ mean,
                                      const float* __restrict__ invstd, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, double* __restrict__ sums, long long rows, int C,
                                      int rows_per_block, float slope, const float* __restrict__ scale, float boost,
                                      const float* __restrict__ post) {
    constexpr int NS = GAIN ? 3 : 2;
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    const long long r1 = min(rows, r0 + rows_per_block);
    float mu = 0.f, is = 1.f, ga = 1.f, be = 0.f;
    if (BN) { mu = mean[c]; is = invstd[c]; ga = gamma[c]; be = beta[c]; }
    float s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll 4
    for (long long r = r0; r < r1; ++r) {
        const float yh = (y[r * C + c] - mu) * is;
        const float z = BN ? yh * ga + be : y[r * C + c];
        if (BN) {
            const float gv = g[r * C + c];
            const float dz = (GAIN ? gain_f(scale, boost, post, c, gv) : gv) * act_grad_f(ACT, z, slope);
            s1 += dz;
            s2 += dz * yh;
        }
        if (GAIN) s3 = fmaf(g[r * C + c], act_f(ACT, z, slope), s3);
    }
    if (DET) {
        double* row = sums + (long long)blockIdx.x * NS * C;
        row[c] = (double)s1;
        row[C + c] = (double)s2;
        if (GAIN) row[2 * C + c] = (double)s3;
        return;
    }
    if (BN) {
        atomicAdd(sums + c, (double)s1);
        atomicAdd(sums + C + c, (double)s2);
    }
    if (GAIN) atomicAdd(sums + 2 * C + c, (double)s3);
}

// dbeta = sums[c], dgamma = sums[C+c]; with S = sums[2C+c]: dscale = boost*post*S, dpost = (boost*scale)*S.  Every output is
// nullable (sums [2C] suffices without dscale / dpost).
__global__ void epi_param_grad_kernel(const double* __restrict__ sums, int C, const float* __restrict__ scale, float boost,
                                      const float* __restrict__ post, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                      float* __restrict__ dscale, float* __restrict__ dpost) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    if (dbeta) dbeta[c] = (float)sums[c];
    if (dgamma) dgamma[c] = (float)sums[C + c];
    if (!dscale && !dpost) return;
    const double S = sums[2 * C + c];
    if (dscale) dscale[c] = (float)((double)boost * (post ? (double)post[c] : 1.0) * S);
    if (dpost) dpost[c] = (float)((scale ? (double)(boost * scale[c]) : 1.0) * S);
}

// backward pass 2 with gb = gain(g): dy = gamma*invstd*(dz - mean(dz) - yhat*mean(dz*yhat)), dz = gb*act'(z) (training
// BatchNorm); dy = gamma*invstd*dz (eval: use_batch_stats = 0); dy = gb*act'(y) (no BatchNorm).  VEC as in epi_fwd_kernel.
// VEC = 4 subtracts the two means unconditionally (0 in eval mode), which lets the compiler fuse dz's product into the
// subtraction; VEC = 1 does not.  Each form keeps the bits of the BatchNorm + GELU kernel of its shapes (float4 / scalar).
// COUNTED: n is read from sums[2C] on the device (a SyncBatchNorm group's row count, all-reduced with the sums)
template <int ACT, bool BN, bool GAIN, int VEC, bool COUNTED = false>
__global__ void epi_bwd_apply_kernel(const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ mean,
                                     const float* __restrict__ invstd, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, const double* __restrict__ sums, double n,
                                     int use_batch_stats, float* __restrict__ dy, long long total, int C, float slope,
                                     const float* __restrict__ scale, float boost, const float* __restrict__ post) {
    if (COUNTED) n = sums[2 * C];
    for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * VEC; i < total;
         i += (long long)gridDim.x * blockDim.x * VEC) {
        const int c0 = (int)(i % C);
        float yv[VEC], gv[VEC], o[VEC];
        if (VEC == 4) {
            const float4 t = ld4(y + i), u = ld4(g + i);
            yv[0] = t.x; yv[1 % VEC] = t.y; yv[2 % VEC] = t.z; yv[3 % VEC] = t.w;
            gv[0] = u.x; gv[1 % VEC] = u.y; gv[2 % VEC] = u.z; gv[3 % VEC] = u.w;
        } else {
            yv[0] = y[i];
            gv[0] = g[i];
        }
        float m1[VEC], m2[VEC];                          // VEC = 4: the batch means, 0 in eval mode
        float mu[VEC], is4[VEC], ga4[VEC], be[VEC];      // VEC = 4: the BatchNorm operands of the 4 columns
#pragma unroll
        for (int j = 0; j < VEC; ++j) m1[j] = m2[j] = 0.f;
        if (VEC == 4 && BN) {
            const float4 a = ld4(mean + c0), b = ld4(invstd + c0), d = ld4(gamma + c0), e = ld4(beta + c0);
            mu[0] = a.x; mu[1 % VEC] = a.y; mu[2 % VEC] = a.z; mu[3 % VEC] = a.w;
            is4[0] = b.x; is4[1 % VEC] = b.y; is4[2 % VEC] = b.z; is4[3 % VEC] = b.w;
            ga4[0] = d.x; ga4[1 % VEC] = d.y; ga4[2 % VEC] = d.z; ga4[3 % VEC] = d.w;
            be[0] = e.x; be[1 % VEC] = e.y; be[2 % VEC] = e.z; be[3 % VEC] = e.w;
        }
        if (VEC == 4 && BN && use_batch_stats) {
#pragma unroll
            for (int j = 0; j < VEC; ++j) { m1[j] = (float)(sums[c0 + j] / n); m2[j] = (float)(sums[C + c0 + j] / n); }
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            const int c = c0 + j;
            const float gb = GAIN ? gain_f(scale, boost, post, c, gv[j]) : gv[j];
            if (!BN) {
                o[j] = gb * act_grad_f(ACT, yv[j], slope);
                continue;
            }
            const float is = VEC == 4 ? is4[j] : invstd[c], ga = VEC == 4 ? ga4[j] : gamma[c];
            const float yh = (yv[j] - (VEC == 4 ? mu[j] : mean[c])) * is;
            const float dz = gb * act_grad_f(ACT, yh * ga + (VEC == 4 ? be[j] : beta[c]), slope);
            if (VEC == 4) {
                o[j] = ga * is * (dz - m1[j] - yh * m2[j]);
            } else {
                float v = dz;
                if (use_batch_stats) v = dz - (float)(sums[c] / n) - yh * (float)(sums[C + c] / n);
                o[j] = ga * is * v;
            }
        }
        if (VEC == 4) *reinterpret_cast<float4*>(dy + i) = make_float4(o[0], o[1 % VEC], o[2 % VEC], o[3 % VEC]);
        else dy[i] = o[0];
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

}  // namespace bm
