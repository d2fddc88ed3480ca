// Weight gradients on the tensor cores (3xTF32 wgmma engine of tc_common.cuh, or its single-pass TF32 / bf16 forms:
// passes = 1 / TC_BF16):
// for one tap shift s
//
//     P[ks][m][n] = sum_{b in split ks} sum_t  dY[b, t, m] * X[b, t + s, n]          (dY, X channels-last)
//
// i.e. a GEMM whose reduction runs over POSITIONS, so both operands are M/N-contiguous in memory; the engine transposes
// them on their way into its K-major shared-memory tiles.  Per CTA: one 128(m) x 128(n) tile for one tap and one slice of
// the batch (X rows shifted outside [0,T) are zeros = the conv padding).  The partial tiles go to the workspace and
// `wgrad_reduce_kernel` sums the batch slices in a fixed order (deterministic) into the nn.Conv1d layout [m][n][tap];
// "direct" calls (one tap, one slice) write the output itself, and the grouped form writes one plane per group.
#pragma once
#include "../../include/bm_b200.h"
#include "tc_common.cuh"

namespace bm {
namespace tc {

constexpr int WG_BM = HG_BM;

// dW[m][n][tap] = sum_ks P[tap][ks][m][n]   (fixed summation order => deterministic), n < Ntrue only
__global__ void wgrad_reduce_kernel(const float* __restrict__ P, float* __restrict__ dW, int taps, int ksplit, int Mpad,
                                    int M, int N, int Ntrue) {
    long long total = (long long)M * Ntrue * taps;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        int j = (int)(idx % taps);
        long long mn = idx / taps;
        int n = (int)(mn % Ntrue), m = (int)(mn / Ntrue);
        const float* src = P + ((long long)j * ksplit * Mpad + m) * N + n;
        float s = 0.f;
        for (int k = 0; k < ksplit; ++k) s += src[(long long)k * Mpad * N];
        dW[idx] = s;
    }
}

// N tile (= 2*nh) selection: nh in {160,128,96,64} with N % (2*nh) == 0
inline int wgrad_pick_nh(int N) {
    for (int nh = 160; nh >= 64; nh -= 32)
        if (N % (2 * nh) == 0) return nh;
    return 0;
}
bool wgrad_tc_supported(int M, int N) { return wgrad_pick_nh(N) != 0 && M >= 32 && (M % 4) == 0; }
inline void wgrad_geometry(int B, int M, int N, int taps, int* nh, int* mblocks, int* ksplit, int* bchunk) {
    *nh = wgrad_pick_nh(N);
    *mblocks = (M + WG_BM - 1) / WG_BM;
    const int bn = hg_pick_bn(N);
    int tiles = (*mblocks) * ((N + bn - 1) / bn) * taps;
    int want = num_sms() / tiles;                 // floor: the whole grid must fit in ONE wave (1 CTA per SM)
    if (want < 1) want = 1;
    if (want > B) want = B;
    *bchunk = (B + want - 1) / want;
    *ksplit = (B + *bchunk - 1) / *bchunk;
}
inline size_t wgrad_workspace_floats(int B, int M, int N, int taps) {
    int nh, mb, ks, bc;
    wgrad_geometry(B, M, N, taps, &nh, &mb, &ks, &bc);
    return (size_t)taps * ks * mb * WG_BM * N;
}

struct WgradOp {
    static constexpr bool A_KCONTIG = false, B_KCONTIG = false;
    int B, T, M, N, taps, dilation, ntiles;
    int bchunk;                 // batch slices: slice ks covers samples [ks*bchunk, min(B, (ks+1)*bchunk))
    const int* zlist;           // grouped mode: slice ks = samples zlist[seg_off[ks] .. seg_off[ks+1])
    const int* seg_off;
    const float* dY;            // [B,T,M]
    const float* X;             // [B,T,N]
    float* P;                   // output planes
    long long plane;            // floats per (tap, slice) plane of P
    int rows;                   // rows of a plane that are written
    int ksplit;

    struct Cta { int tap, shift, m0, n0, ks, b_begin, b_end, tchunks; };
    template <int BN> __device__ Cta cta() const {
        Cta c;
        c.tap = blockIdx.x / ntiles;
        c.shift = (c.tap - taps / 2) * dilation;
        c.n0 = (blockIdx.x - c.tap * ntiles) * BN;
        c.m0 = blockIdx.y * HG_BM;
        c.ks = blockIdx.z;
        c.b_begin = seg_off ? seg_off[c.ks] : c.ks * bchunk;
        c.b_end = seg_off ? seg_off[c.ks + 1] : min(B, c.b_begin + bchunk);
        c.tchunks = (T + HG_BK - 1) / HG_BK;
        return c;
    }
    __device__ int kblocks(const Cta& c) const { return max(0, c.b_end - c.b_begin) * c.tchunks; }
    __device__ int sample(const Cta& c, int kb) const {
        const int b = c.b_begin + kb / c.tchunks;
        return zlist ? zlist[b] : b;
    }
    __device__ float4 a4(const Cta& c, int kb, int k, int q) const {         // dY^T: rows m, reduction over positions
        const int t = (kb % c.tchunks) * HG_BK + k, m = c.m0 + 4 * q;
        if (t >= T || m >= M) return make_float4(0.f, 0.f, 0.f, 0.f);
        return __ldg(reinterpret_cast<const float4*>(dY + ((long long)sample(c, kb) * T + t) * M + m));
    }
    __device__ float4 b4(const Cta& c, int kb, int k, int q) const {         // X^T shifted by the tap, zeros across the edges
        const int t = (kb % c.tchunks) * HG_BK + k, ts = t + c.shift, n = c.n0 + 4 * q;
        if (t >= T || ts < 0 || ts >= T || n >= N) return make_float4(0.f, 0.f, 0.f, 0.f);
        return __ldg(reinterpret_cast<const float4*>(X + ((long long)sample(c, kb) * T + ts) * N + n));
    }
    template <int BN> __device__ void epilogue(const Cta& c, const float* acc, int m0) const {
        HgStore s{P + ((long long)c.tap * ksplit + c.ks) * plane, N, rows, N};
        s.store<BN>(acc, c.m0 + m0, c.n0);
    }
};

// dY [B,T,M], X [B,T,N] -> dW [M][Ntrue][taps]; ws: wgrad_workspace_floats() floats
int launch_wgrad_tc(const float* dY, const float* X, int B, int T, int M, int N, int Ntrue, int taps, int dilation,
                    float* ws, float* dW, int passes, cudaStream_t st, float* dbias) {
    int nh, mblocks, ksplit, bchunk;
    wgrad_geometry(B, M, N, taps, &nh, &mblocks, &ksplit, &bchunk);
    if (nh == 0) return set_error(2, "%s: unsupported N%s", __func__);
    const int Mpad = mblocks * WG_BM;
    const bool direct = taps == 1 && ksplit == 1 && Ntrue == N;
    WgradOp o;
    const int bn = hg_pick_bn(N);
    o.B = B; o.T = T; o.M = M; o.N = N; o.taps = taps; o.dilation = dilation; o.ntiles = (N + bn - 1) / bn;
    o.bchunk = bchunk; o.zlist = nullptr; o.seg_off = nullptr; o.dY = dY; o.X = X; o.ksplit = ksplit;
    o.P = direct ? dW : ws;
    o.plane = (long long)(direct ? M : Mpad) * N;
    o.rows = direct ? M : Mpad;
    if (int rc = hg_launch_bn(bn, o, dim3(o.ntiles * taps, mblocks, ksplit), passes, st, __func__)) return rc;
    if (dbias)                 // bias gradient sum_{b,t} dY[b,t,m]
        if (int rc = bm_col_sum(dY, (long long)B * T, M, dbias, st)) return rc;
    if (direct) return 0;
    wgrad_reduce_kernel<<<ew_grid((long long)M * Ntrue * taps), 256, 0, st>>>(ws, dW, taps, ksplit, Mpad, M, N, Ntrue);
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: reduce launch failed: %s", __func__, cudaGetErrorString(e));
    return 0;
}

// grouped pointwise weight gradient: out[g][m][n] = sum_{b in group g} sum_t dY[b,t,m] X[b,t,n]; out is [G][Mpad][N] with
// Mpad = ceil(M/128)*128 (rows >= M are zero); groups given as CSR (zlist, seg_off[G+1]) over the samples.
inline int launch_wgrad_tc_grouped(const float* dY, const float* X, const int* zlist, const int* seg_off, int G, int B,
                                   int T, int M, int N, float* out, int passes, cudaStream_t st) {
    if (wgrad_pick_nh(N) == 0) return set_error(2, "%s: unsupported N%s", __func__);
    if (G > 65535) return set_error(2, "%s: too many groups%s", __func__);
    const int mblocks = (M + WG_BM - 1) / WG_BM;
    WgradOp o;
    o.B = B; o.T = T; o.M = M; o.N = N; o.taps = 1; o.dilation = 1; o.ntiles = (N + HG_BN - 1) / HG_BN;
    o.bchunk = 0; o.zlist = zlist; o.seg_off = seg_off; o.dY = dY; o.X = X; o.ksplit = G;
    o.P = out; o.plane = (long long)mblocks * WG_BM * N; o.rows = mblocks * WG_BM;
    // 128 columns: one CTA per (tile, group) and no K-slice count to raise, so fewer, wider tiles fill the waves worse
    // (27 groups of 320 x 320: 162 CTAs at 160, a second wave of 30 on 132 SMs, ran slower than 243 at 128)
    return hg_launch<HG_BN>(o, dim3(o.ntiles, mblocks, G), passes, st, __func__);
}

}  // namespace tc
}  // namespace bm
