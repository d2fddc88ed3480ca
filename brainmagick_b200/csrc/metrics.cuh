// Test metrics (bm/metrics.py: OnlineCorrelation, L1Reg, L2Reg, ClassificationAcc): per-column sums over dim 0 of
// [N, C, T] operands, accumulated on the device in fp64 across updates, and the finalize of each metric -- with no host
// read and no atomics.
//
// Operands: left and right are fp32 or fp64 read through their own (n, c, t) strides at any element offset (slices of dim 1
// and the solver's time crop are read in place); mask is one byte per entry read through its own strides (0 where it
// broadcasts).  A column is one (c, t); the accumulators are NP fp64 planes of C*T columns, the last one the count.
//
//   metric_update_kernel   threads along t (coalesced loads), one column per thread; grid (column blocks, splits): split s
//                          walks rows [N*s/splits, N*(s+1)/splits) in order with fp64 FMAs.  splits == 1: the sums go
//                          straight into the accumulators; else into fp64 partials per split
//   metric_combine_kernel  splits > 1: adds the partials in split order into the accumulators
//   metric_finalize_kernel one CTA: the metric per column in the output dtype and the flag bits (MetricFlag)
// The "seen a True mask entry" word is a ping-pong pair: an update reads seen[parity] (the accumulators are overwritten
// while it is 0, as the reference re-initialises while _count.sum() == 0) and only ever stores 1 into seen[parity ^ 1] (when
// seen[parity] is set or the update counted an entry).  The word it reads is never written in the same launch; the host
// flips the parity after each update without reading it.  A word left from two updates back is never larger than
// seen[parity], since the word only goes from 0 to 1.
#pragma once
#include "common.cuh"

namespace bm {

enum MetricKind { MT_CORRELATION = 0, MT_L1 = 1, MT_L2 = 2, MT_ACCURACY = 3 };
// bits of the finalize flag word; the reference's min() < -tol is False when a NaN is among the norms, hence the NaN bits
enum MetricFlag {
    MT_LEFT_UNSTABLE = 1, MT_LEFT_NAN = 2, MT_RIGHT_UNSTABLE = 4, MT_RIGHT_NAN = 8, MT_RESULT_NAN = 16, MT_COUNTED = 32
};

constexpr int MT_THREADS = 256;
constexpr int MT_FINAL_THREADS = 1024;
constexpr int MT_MAX_SPLITS = 64;
constexpr int MT_MAX_PLANES = 6;

// accumulator planes: (Σ l·r·m, Σ l·m, Σ r·m, Σ (l·m)², Σ (r·m)², count) for the correlation, (sum, count) otherwise
__host__ __device__ constexpr int mt_planes(int kind) { return kind == MT_CORRELATION ? 6 : 2; }

struct MtOperands {
    const void* l;
    long long l_sn, l_sc, l_st;
    const void* r;
    long long r_sn, r_sc, r_st;
    const unsigned char* m;
    long long m_sn, m_sc, m_st;
    int m_n;            // the mask's own first dimension, 1 or N: the count adds mask.sum(0) over it
    int N, C, T, K;     // C*T columns (C = 1 for the accuracy); K class channels of the accuracy's left operand
};

// row splits of an update: 1 when the column blocks alone give four CTAs per SM (enough loads in flight to approach HBM
// bandwidth) or there are no columns, else enough splits to make about four, at most MT_MAX_SPLITS and never more than
// there are rows.  Set by the shape and the SM count only.
inline int mt_splits(long long N, long long cols) {
    const long long blocks = (cols + MT_THREADS - 1) / MT_THREADS;
    if (N <= 1 || blocks == 0 || blocks >= 4ll * num_sms()) return 1;
    long long s = (4ll * num_sms() + blocks - 1) / blocks;
    if (s > MT_MAX_SPLITS) s = MT_MAX_SPLITS;
    if (s > N) s = N;
    return (int)s;
}

template <typename S>
__device__ __forceinline__ double mt_ld(const S* p) { return (double)__ldg(p); }

template <typename S, int KIND>
__global__ void __launch_bounds__(MT_THREADS) metric_update_kernel(MtOperands p, int splits, double* __restrict__ acc,
                                                                  int* __restrict__ seen, int parity,
                                                                  double* __restrict__ part) {
    constexpr int NP = mt_planes(KIND);
    const long long cols = (long long)p.C * p.T;
    const long long j = blockIdx.x * (long long)MT_THREADS + threadIdx.x;
    if (j >= cols) return;
    const int c = (int)(j / p.T), t = (int)(j - (long long)c * p.T);
    const int n0 = (int)((long long)p.N * blockIdx.y / splits), n1 = (int)((long long)p.N * (blockIdx.y + 1) / splits);
    const S* L = static_cast<const S*>(p.l) + c * p.l_sc + t * p.l_st;
    const S* R = static_cast<const S*>(p.r) + c * p.r_sc + t * p.r_st;
    const unsigned char* M = p.m + c * p.m_sc + t * p.m_st;
    double v[NP];
#pragma unroll
    for (int q = 0; q < NP; ++q) v[q] = 0.0;
#pragma unroll 4
    for (int n = n0; n < n1; ++n) {
        // the reference multiplies by the mask: a masked-out inf or NaN still gives NaN
        const double m = __ldg(M + n * p.m_sn) ? 1.0 : 0.0;
        if (KIND == MT_CORRELATION) {
            const double l = mt_ld(L + n * p.l_sn), r = mt_ld(R + n * p.r_sn);
            const double lm = l * m, rm = r * m;
            v[0] = fma(l * r, m, v[0]);                    // (l·r)·m is exact for m in {0, 1}: the fma rounds once
            v[1] += lm;
            v[2] += rm;
            v[3] = fma(lm, lm, v[3]);
            v[4] = fma(rm, rm, v[4]);
        } else if (KIND == MT_L1 || KIND == MT_L2) {
            const double d = (double)(S)(__ldg(L + n * p.l_sn) - __ldg(R + n * p.r_sn)) * m;   // l - r in the operands'
            v[0] = KIND == MT_L1 ? v[0] + fabs(d) : fma(d, d, v[0]);                          // dtype, as torch forms it
        } else {
            // torch's argmax: the first maximal index, a NaN counts as maximal
            const S* Ln = L + n * p.l_sn;
            S best = __ldg(Ln);
            int idx = 0;
            for (int k = 1; k < p.K; ++k) {
                const S x = __ldg(Ln + k * p.l_sc);
                if (!(best != best) && (x != x || x > best)) {
                    best = x;
                    idx = k;
                }
            }
            // the target equals the prediction only as equal values: -100, NaN and fractions never count
            v[0] += (m != 0.0 && (double)idx == mt_ld(R + n * p.r_sn)) ? 1.0 : 0.0;
        }
        v[NP - 1] += m;
    }
    if (p.m_n == 1) v[NP - 1] = blockIdx.y == 0 && __ldg(M) ? 1.0 : 0.0;   // a mask broadcast along N counts once
    if (splits == 1) {
        const bool was = __ldg(seen + parity) != 0;
#pragma unroll
        for (int q = 0; q < NP; ++q) acc[q * cols + j] = (was ? acc[q * cols + j] : 0.0) + v[q];
        if (was || v[NP - 1] != 0.0) seen[parity ^ 1] = 1;
    } else {
#pragma unroll
        for (int q = 0; q < NP; ++q) part[((long long)blockIdx.y * NP + q) * cols + j] = v[q];
    }
}

template <int NP>
__global__ void __launch_bounds__(MT_THREADS) metric_combine_kernel(const double* __restrict__ part, int splits,
                                                                   long long cols, double* __restrict__ acc,
                                                                   int* __restrict__ seen, int parity) {
    const long long j = blockIdx.x * (long long)MT_THREADS + threadIdx.x;
    if (j >= cols) return;
    const bool was = __ldg(seen + parity) != 0;
    double count = 0.0;
#pragma unroll
    for (int q = 0; q < NP; ++q) {
        double s = part[q * cols + j];
        for (int b = 1; b < splits; ++b) s += part[((long long)b * NP + q) * cols + j];
        acc[q * cols + j] = (was ? acc[q * cols + j] : 0.0) + s;
        count = s;
    }
    if (was || count != 0.0) seen[parity ^ 1] = 1;
}

// x.clamp(lo, inf) as torch: a NaN stays NaN (fmax would drop it)
__device__ __forceinline__ double mt_clamp_lo(double x, double lo) { return x < lo ? lo : x; }

// The reference's get() per column, in its order of operations (no contraction into FMAs):
//   correlation: n² = Σx² − |Σx|² / count for left and right (flags: n² < −tol, NaN), norm = sqrt(n².clamp(0)),
//                dot = Σlr − Σl·Σr / count, out = dot / (norm_l·norm_r).clamp(tol)
//   accumulative: out = sum / count
// Flags over every column: instability and NaN bits, and MT_COUNTED when any count is nonzero.
template <typename O, int KIND>
__global__ void __launch_bounds__(MT_FINAL_THREADS) metric_finalize_kernel(const double* __restrict__ acc, long long cols,
                                                                          double tol, O* __restrict__ out,
                                                                          int* __restrict__ flag) {
    int bits = 0;
    for (long long j = threadIdx.x; j < cols; j += MT_FINAL_THREADS) {
        double res;
        if (KIND == MT_CORRELATION) {
            const double sd = acc[j], sl = acc[cols + j], sr = acc[2 * cols + j];
            const double sll = acc[3 * cols + j], srr = acc[4 * cols + j], cnt = acc[5 * cols + j];
            const double nl2 = __dsub_rn(sll, __ddiv_rn(__dmul_rn(sl, sl), cnt));
            const double nr2 = __dsub_rn(srr, __ddiv_rn(__dmul_rn(sr, sr), cnt));
            bits |= (nl2 < -tol ? MT_LEFT_UNSTABLE : 0) | (isnan(nl2) ? MT_LEFT_NAN : 0) |
                    (nr2 < -tol ? MT_RIGHT_UNSTABLE : 0) | (isnan(nr2) ? MT_RIGHT_NAN : 0) |
                    (cnt != 0.0 ? MT_COUNTED : 0);
            const double den = mt_clamp_lo(__dmul_rn(__dsqrt_rn(mt_clamp_lo(nl2, 0.0)), __dsqrt_rn(mt_clamp_lo(nr2, 0.0))),
                                           tol);
            res = __ddiv_rn(__dsub_rn(sd, __ddiv_rn(__dmul_rn(sl, sr), cnt)), den);
        } else {
            const double cnt = acc[cols + j];
            res = __ddiv_rn(acc[j], cnt);
            bits |= cnt != 0.0 ? MT_COUNTED : 0;
        }
        bits |= isnan(res) ? MT_RESULT_NAN : 0;
        out[j] = (O)res;
    }
    int word = 0;
#pragma unroll
    for (int b = 1; b <= MT_COUNTED; b <<= 1) word |= __syncthreads_or(bits & b) ? b : 0;
    if (threadIdx.x == 0) flag[0] = word;
}

}  // namespace bm
