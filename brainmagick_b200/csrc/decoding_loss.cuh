// FeatureDecodingLoss (bm/losses.py:117-173): over the features of a builder, in order, the sum of one term each --
// regression: mean (e - o)^2 over the masked entries of the feature's channels (F.mse_loss);
// categorical (cardinality K, one output channel): torch's weighted cross-entropy over the masked (b, t) with the K
// estimate channels as logits and out.long() as the target (F.cross_entropy, weights or none, ignore_index -100) --
// and its gradients, without a host read.
//
// Operands: est [B, F_out, T] and out [B, F, T] with t-stride 1 and any (b, c) strides and element offset (the solver's
// time crops are read in place); mask bytes read through their (b, c, t) strides (c-stride 0 when the mask has one
// channel).  A device feature table holds, per feature, FD_TABLE ints: kind, estimate channel start, estimate width (K for
// a categorical feature), output channel start, weight offset (-1: unweighted) and lse slot (categorical only).
//
//   decoding_loss_partials_kernel  fixed grid (fd_blocks: shape and SM count); every CTA takes the same share of every
//                                  feature's work and stores fp64 partials per (CTA, feature) -- regression: (sum (e-o)^2,
//                                  count) over the rows of ml_load_chunk; categorical: (sum w_y (lse - z_y), sum w_y) with
//                                  threads along t and an online log-sum-exp over k (the K logits of one (b, t) lie one
//                                  channel stride apart: each warp reads 32 consecutive t of one channel per step), and the
//                                  lse of every (b, t) for the backward -- and a flag word (mask seen, bad targets)
//   decoding_loss_finalize_kernel  one CTA: the partials in a fixed order -> term_f = sum / count in fp32, loss = the terms
//                                  added in feature order (the reference's `loss += ...`), scale_f = 2 / N_f or 1 / W_f,
//                                  and the first error in the reference's order (904, then 905 / 906 per feature)
//   decoding_loss_bwd_kernel       one pass over every row of d_est (and of d_out): regression 2 (e - o) g / N,
//                                  categorical g w_y / W (softmax - onehot), 0 where the mask is False (a select);
//                                  contiguous outputs, float4 stores when T % 4 == 0 and both are 16-byte aligned
// No atomics on any result: loss and gradients are bitwise repeatable.  A target outside [0, K) is reported and never
// indexes anything.
#pragma once
#include "masked_loss.cuh"

namespace bm {

constexpr int FD_THREADS = 256;
constexpr int FD_TABLE = 6;            // ints per feature in the table
constexpr int FD_MAX_FEATURES = 15;    // flag word: bit 0 mask seen, bits 1 + 2f (target >= K) and 2 + 2f (bad negative)

enum DecodingFeatureKind { FD_REGRESSION = 0, FD_CATEGORICAL = 1 };
enum DecodingStatus { FD_NO_MASK = 904, FD_TARGET_TOO_LARGE = 905, FD_TARGET_NEGATIVE = 906 };

struct FdOperands {
    const float* est;
    long long e_sb, e_sc;
    const float* out;
    long long o_sb, o_sc;
    const unsigned char* mask;
    long long m_sb, m_sc, m_st;
    const int* table;
    const float* weights;
    int F, B, T;
};

// CTAs of the partials kernel: one per FD_THREADS (b, t) positions, at most four per SM
inline int fd_blocks(int B, int T) {
    long long n = ((long long)B * T + FD_THREADS - 1) / FD_THREADS;
    const long long cap = 4ll * num_sms();
    if (n > cap) n = cap;
    return n < 1 ? 1 : (int)n;
}

// The row loader's view of one feature's slice.  Regression: rows (b, c) of the estimate and output channels, the mask's
// channel c (or its one channel).  Categorical: rows (b, k) of the K logit channels, with the target channel as the
// "output" row of every k and the mask's one channel.
__device__ __forceinline__ MlOperands fd_slice(const FdOperands& p, int es, int width, int os, bool categorical) {
    return MlOperands{p.est + es * p.e_sc, p.e_sb, p.e_sc, p.out + os * p.o_sc, p.o_sb, categorical ? 0 : p.o_sc,
                      p.mask, p.m_sb, categorical ? 0 : p.m_sc, p.m_st, width, p.T};
}

// torch's out.long() of a target v with v < K: a class in [0, K), -100 (ignore_index), or -1 (any other negative
// class: out of bounds).  NaN never gets here (it fails v < K).
__device__ __forceinline__ int fd_target(float v) {
    if (v > -1.f) return (int)v;                            // truncation toward zero, as .long()
    if (v > -101.f && v <= -100.f) return -100;
    return -1;
}

__global__ void __launch_bounds__(FD_THREADS) decoding_loss_partials_kernel(FdOperands p, double* __restrict__ part,
                                                                            int* __restrict__ cta_flags,
                                                                            float* __restrict__ lse) {
    const int nb = gridDim.x, blk = blockIdx.x;
    const int nch = (p.T + 3) >> 2;
    unsigned bits = 0;
    for (int f = 0; f < p.F; ++f) {
        const int* row = p.table + FD_TABLE * f;
        const int kind = __ldg(row), es = __ldg(row + 1), w = __ldg(row + 2), os = __ldg(row + 3);
        double s = 0.0, n = 0.0;
        if (kind == FD_REGRESSION) {
            const MlOperands q = fd_slice(p, es, w, os, false);
            const long long items = (long long)p.B * w * nch;
            const long long j1 = items * (blk + 1) / nb;
            for (long long j = items * blk / nb + threadIdx.x; j < j1; j += FD_THREADS) {
                const long long r = j / nch;
                float e[4], o[4];
                bool m[4];
                ml_load_chunk(q, r, (int)(j - r * nch), e, o, m);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (!m[i]) continue;
                    const float d = e[i] - o[i];                // fp32, as torch forms the difference
                    s += (double)d * (double)d;
                    n += 1.0;
                    bits |= 1u;
                }
            }
        } else {
            const int woff = __ldg(row + 4), slot = __ldg(row + 5);
            const float kf = (float)w;
            const long long items = (long long)p.B * p.T;
            const long long j1 = items * (blk + 1) / nb;
            for (long long j = items * blk / nb + threadIdx.x; j < j1; j += FD_THREADS) {
                const int b = (int)(j / p.T), t = (int)(j - (long long)b * p.T);
                const float* z = p.est + b * p.e_sb + es * p.e_sc + t;
                const float v = __ldg(p.out + b * p.o_sb + os * p.o_sc + t);
                const bool m = __ldg(p.mask + b * p.m_sb + t * p.m_st) != 0;
                const int y = v < kf ? fd_target(v) : -2;
                float mx = -INFINITY, sum = 0.f, zy = 0.f;
#pragma unroll 4
                for (int k = 0; k < w; ++k) {
                    const float x = __ldg(z + k * p.e_sc);
                    zy = k == y ? x : zy;
                    if (x > mx) {
                        sum = sum * expf(mx - x) + 1.f;
                        mx = x;
                    } else if (!(x == -INFINITY)) {             // NaN goes in and propagates, as in torch
                        sum += expf(x - mx);
                    }
                }
                const float l = mx + logf(sum);
                lse[(long long)slot * items + j] = l;
                if (y == -2) bits |= 2u << (2 * f);             // assert K > output[:, start].max(): every position
                if (m) {
                    bits |= 1u;
                    if (y >= 0) {
                        const float wy = woff >= 0 ? __ldg(p.weights + woff + y) : 1.f;
                        s += (double)wy * (double)(l - zy);     // -log_softmax(z)[y] in fp32, weighted in fp64
                        n += (double)wy;
                    } else if (y == -1) {
                        bits |= 4u << (2 * f);
                    }
                }
            }
        }
        ml_block_sum(s, n);
        if (threadIdx.x == 0) {
            part[2 * ((long long)blk * p.F + f)] = s;
            part[2 * ((long long)blk * p.F + f) + 1] = n;
        }
        __syncthreads();                                        // ml_block_sum's shared words are reused
    }
    __shared__ unsigned sb[FD_THREADS / 32];
    bits = __reduce_or_sync(0xffffffffu, bits);
    if ((threadIdx.x & 31) == 0) sb[threadIdx.x >> 5] = bits;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned all = 0;
#pragma unroll
        for (int i = 0; i < FD_THREADS / 32; ++i) all |= sb[i];
        cta_flags[blk] = (int)all;
    }
}

// flag <- the reference's first error as code | (feature << 16), 0 when there is none; status (when given) <- the code if
// it is still 0, for a captured step
__global__ void __launch_bounds__(ML_FINAL_THREADS) decoding_loss_finalize_kernel(
    const double* __restrict__ part, const int* __restrict__ cta_flags, int nb, const int* __restrict__ table, int F,
    float* __restrict__ loss, float* __restrict__ scale, int* __restrict__ flag, int* __restrict__ status) {
    float total = 0.f;
    for (int f = 0; f < F; ++f) {
        double s = 0.0, n = 0.0;
        for (int i = threadIdx.x; i < nb; i += ML_FINAL_THREADS) {
            s += part[2 * ((long long)i * F + f)];
            n += part[2 * ((long long)i * F + f) + 1];
        }
        ml_block_sum(s, n);
        if (threadIdx.x == 0) {
            const float term = (float)s / (float)n;             // N_f = 0 or W_f = 0: NaN, as torch
            total = f == 0 ? term : total + term;
            scale[f] = table[FD_TABLE * f] == FD_REGRESSION ? (float)(2.0 / n) : (float)(1.0 / n);
        }
        __syncthreads();
    }
    __shared__ unsigned sb[ML_FINAL_THREADS / 32];
    unsigned bits = 0;
    for (int i = threadIdx.x; i < nb; i += ML_FINAL_THREADS) bits |= (unsigned)cta_flags[i];
    bits = __reduce_or_sync(0xffffffffu, bits);
    if ((threadIdx.x & 31) == 0) sb[threadIdx.x >> 5] = bits;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned all = 0;
#pragma unroll
        for (int i = 0; i < ML_FINAL_THREADS / 32; ++i) all |= sb[i];
        int code = (all & 1u) ? 0 : FD_NO_MASK, at = 0;
        for (int f = 0; f < F && code == 0; ++f) {
            if (all & (2u << (2 * f))) code = FD_TARGET_TOO_LARGE, at = f;
            else if (all & (4u << (2 * f))) code = FD_TARGET_NEGATIVE, at = f;
        }
        loss[0] = total;
        flag[0] = code == 0 ? 0 : code | (at << 16);
        if (code != 0 && status) atomicCAS(status, 0, code);
    }
}

__global__ void __launch_bounds__(FD_THREADS) decoding_loss_bwd_kernel(FdOperands p, int est_C, int out_C,
                                                                       const float* __restrict__ g,
                                                                       const float* __restrict__ scale,
                                                                       const float* __restrict__ lse,
                                                                       float* __restrict__ d_est,
                                                                       float* __restrict__ d_out, bool vec_out) {
    const float gv = __ldg(g);
    const int nch = (p.T + 3) >> 2;
    const long long est_items = d_est ? (long long)p.B * est_C * nch : 0;
    const long long items = est_items + (d_out ? (long long)p.B * out_C * nch : 0);
    for (long long j = blockIdx.x * (long long)FD_THREADS + threadIdx.x; j < items; j += (long long)gridDim.x * FD_THREADS) {
        const bool to_out = j >= est_items;
        const long long jj = to_out ? j - est_items : j;
        const int C = to_out ? out_C : est_C;
        const long long r = jj / nch;
        const int k = (int)(jj - r * nch);
        const int b = (int)(r / C), c = (int)(r - (long long)b * C);
        const int t0 = 4 * k, n = min(4, p.T - t0);
        float v[4] = {0.f, 0.f, 0.f, 0.f};                      // channels no feature holds, and d_out of a class channel
        for (int f = 0; f < p.F; ++f) {
            const int* row = p.table + FD_TABLE * f;
            const int kind = __ldg(row), es = __ldg(row + 1), w = __ldg(row + 2), os = __ldg(row + 3);
            const int start = to_out ? os : es, width = to_out && kind == FD_CATEGORICAL ? 1 : w;
            if (c < start || c >= start + width) continue;
            float e[4], o[4];
            bool m[4];
            const float sc = __ldg(scale + f);
            if (kind == FD_REGRESSION) {
                ml_load_chunk(fd_slice(p, es, w, os, false), (long long)b * w + (c - start), k, e, o, m);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float d = (e[i] - o[i]) * sc * gv;    // torch's mse_loss backward: (e - o) * (2 / N) * g
                    v[i] = m[i] ? (to_out ? -d : d) : 0.f;      // a select: a masked-out NaN or inf stays out
                }
            } else if (!to_out) {
                const int cls = c - es, woff = __ldg(row + 4), slot = __ldg(row + 5);
                ml_load_chunk(fd_slice(p, es, w, os, true), (long long)b * w + cls, k, e, o, m);
                const float* lrow = lse + ((long long)slot * p.B + b) * p.T + t0;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (i >= n || !m[i] || !(o[i] < (float)w)) continue;
                    const int y = fd_target(o[i]);
                    if (y < 0) continue;                        // ignore_index, or a reported bad target
                    const float wy = woff >= 0 ? __ldg(p.weights + woff + y) : 1.f;
                    const float pr = expf(e[i] - __ldg(lrow + i));
                    v[i] = gv * sc * wy * (pr - (cls == y ? 1.f : 0.f));
                }
            }
            break;
        }
        float* dst = (to_out ? d_out : d_est) + r * p.T + t0;
        if (vec_out && n == 4) {
            *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
            for (int i = 0; i < n; ++i) dst[i] = v[i];
        }
    }
}

}  // namespace bm
