// Weight gradient of a (dilated) k-tap conv (3xTF32 wgmma engine of tc_common.cuh, or its single-pass TF32 form):
//
//     dW[m][n][tap] = sum_p dY[p, m] * X[p + shift(tap), n]          p = b*T + t flattened rows, channels-last operands
//
// as ONE GEMM whose OUTPUT ROWS are the (tap, n) pairs and whose columns are the dY channels:
//
//     G[(tap, n)][m] = sum_p Xs[p, (tap, n)] * dY[p, m],     Xs[p, (tap, n)] = X[p + shift(tap), n] (0 across a sample edge)
//
// so the taps share one tile grid (3 x 320 rows = 7.5 tiles of 128 instead of 3 x 3) and the reduction runs over the
// flattened rows in exact blocks of 32.  One CTA = one (128-row tile, 128- or 160-column tile, K slice) of hw_wgrad_kernel
// (tc_common.cuh: X and dY by TMA, X transposed in registers, dY in shared memory); partial tiles go to the workspace and
// `wgradp_reduce_kernel` sums the K slices in a fixed order (deterministic) while scattering into the nn.Conv1d layout
// [m][n][tap].
#pragma once
#include "tc_wgrad.cuh"

namespace bm {
namespace tc {

struct WgradPOp {
    int R, T, Mdy, Nx, taps, dilation, rows, per_split, chunks;
    const float* dY; const float* X;
    float* P;                   // [ks][rows_pad][Mdy]
    int rows_pad;
    int* err;                   // pipeline status (HC_ERR_FULL / HC_ERR_EMPTY), or null

    struct Cta { int m0, n0, c0, c1; };
    template <int BN> __device__ Cta cta() const {
        Cta c;
        c.n0 = blockIdx.x * BN;
        c.m0 = blockIdx.y * HG_BM;
        c.c0 = blockIdx.z * per_split;
        c.c1 = min(chunks, c.c0 + per_split);
        return c;
    }
    __device__ int kblocks(const Cta& c) const { return max(0, c.c1 - c.c0); }
    __device__ int row0(const Cta& c) const { return c.c0 * HG_BK; }
    // box j of the A tile (tile rows 32 j .. 32 j + 31 = Xs rows (tap, n .. n + 31)): {n, shift(tap)}; rows past the last
    // tap are padding: shift T (every element is zeroed)
    __device__ int2 a_box(const Cta& c, int j) const {
        const int r = c.m0 + 32 * j;
        if (r >= rows) return make_int2(0, T);
        const int tap = r / Nx;
        return make_int2(r - tap * Nx, (tap - taps / 2) * dilation);
    }
    // box j of block kb's dY tile (tile columns 32 j .. 32 j + 31): {first channel m, first row p} in the dY map; channels
    // m >= Mdy and rows p >= R arrive as zeros
    __device__ int2 b_box(const Cta& c, int kb, int j) const {
        return make_int2(c.n0 + 32 * j, (c.c0 + kb) * HG_BK);
    }
    template <int BN> __device__ void epilogue(const Cta& c, const float* acc, int m0) const {
        HgStore s{P + (long long)blockIdx.z * rows_pad * Mdy, Mdy, rows_pad, Mdy};
        s.store<BN>(acc, c.m0 + m0, c.n0);
    }
};

// dW[m][n][tap] = sum_ks P[ks][tap*Nx + n][m]   (fixed order => deterministic), n < Ntrue only
__global__ void wgradp_reduce_kernel(const float* __restrict__ P, float* __restrict__ dW, int taps, int ks, int rows_pad,
                                     int Mdy, int Nx, int Ntrue) {
    // thread per (n, tap, m) with m fastest on the READ side (coalesced over the K-slice planes)
    const long long total = (long long)Mdy * Ntrue * taps;
    const long long plane = (long long)rows_pad * Mdy;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(idx % Mdy);
        const long long r = idx / Mdy;
        const int n = (int)(r % Ntrue), tap = (int)(r / Ntrue);
        const float* src = P + ((long long)tap * Nx + n) * Mdy + m;
        float s = 0.f;
        for (int k = 0; k < ks; ++k) s += src[(long long)k * plane];
        dW[((long long)m * Ntrue + n) * taps + tap] = s;
    }
}

struct WgradPPGeom { int mtiles, ks, chunks, per_split, rows, bn; };

inline bool wgradp_supported(int T, int Mdy, int Nx, int taps) {
    return T >= HG_BK && Nx % 32 == 0 && Nx >= 32 && taps >= 1 && taps <= 3 && Mdy % 64 == 0;
}
inline WgradPPGeom wgradp_geometry(int B, int T, int Mdy, int Nx, int taps) {
    WgradPPGeom g;
    g.rows = taps * Nx;
    g.mtiles = (g.rows + 255) / 256;
    const long long R = (long long)B * T;
    g.chunks = (int)((R + HG_BK - 1) / HG_BK);
    g.bn = hg_pick_bn(Mdy);
    const int tiles = 2 * g.mtiles * ((Mdy + g.bn - 1) / g.bn);
    int ks = num_sms() / tiles;                              // one wave of 128 x bn tiles
    if (ks < 1) ks = 1;
    if (ks > g.chunks) ks = g.chunks;
    g.per_split = (g.chunks + ks - 1) / ks;
    g.ks = (g.chunks + g.per_split - 1) / g.per_split;
    return g;
}
inline size_t wgradp_workspace_floats(int B, int T, int Mdy, int Nx, int taps) {
    const WgradPPGeom g = wgradp_geometry(B, T, Mdy, Nx, taps);
    return (size_t)g.ks * g.mtiles * 256 * Mdy;
}

// dY [B,T,Mdy], X [B,T,Nx] channels-last -> dW [Mdy][Ntrue][taps]; ws: wgradp_workspace_floats() floats
inline int launch_wgrad_pp(const float* dY, const float* X, int B, int T, int Mdy, int Nx, int Ntrue, int taps,
                           int dilation, float* ws, float* dW, int passes, int* err, cudaStream_t st) {
    const WgradPPGeom g = wgradp_geometry(B, T, Mdy, Nx, taps);
    const long long R = (long long)B * T;
    if (R >= (1ll << 31)) return set_error(2, "%s: too many rows%s", __func__);
    if (reinterpret_cast<uintptr_t>(dY) & 15) return set_error(2, "%s: dy must be 16-byte aligned%s", __func__);
    WgradPOp o;
    o.R = (int)R; o.T = T; o.Mdy = Mdy; o.Nx = Nx; o.taps = taps; o.dilation = dilation; o.rows = g.rows;
    o.per_split = g.per_split; o.chunks = g.chunks; o.dY = dY; o.X = X; o.P = ws; o.rows_pad = g.mtiles * 256;
    o.err = err;
    const dim3 grid((Mdy + g.bn - 1) / g.bn, o.rows_pad / HG_BM, g.ks);
    if (int rc = hw_launch_bn(g.bn, o, grid, passes, st, __func__)) return rc;
    wgradp_reduce_kernel<<<ew_grid((long long)Mdy * Ntrue * taps), 256, 0, st>>>(ws, dW, taps, g.ks, o.rows_pad, Mdy, Nx,
                                                                                Ntrue);
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: reduce launch failed: %s", __func__, cudaGetErrorString(e));
    return 0;
}

}  // namespace tc
}  // namespace bm
