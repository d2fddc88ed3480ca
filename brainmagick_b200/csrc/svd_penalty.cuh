// Spectral-norm penalty (bm/svd.py: svd_penalty): for every selected weight, the estimate of its largest squared singular
// value that torch.svd_lowrank(p, q, niter)[1][0] ** 2 gives, and its gradient -- grouped over all weights, so the launch
// count does not depend on how many there are.
//
// Each weight P (row-major [rows_p, cols_p], the stored layout viewed as [shape[0], -1]) is read in its tall orientation
// A [m, n], m >= n: A = P, or A = Pᵀ read through a transpose flag (never copied).  With the draw R [n, q] and S = 2 niter + 1
// orthonormalisation steps (step k: X_k = A·Qin_k for even k, X_k = Aᵀ·Qin_k for odd k; Qin_0 = R, Qin_k = Y_{k-1}):
//   Y_k Rx_k = X_k                    Cholesky QR with the Gram matrix accumulated in fp64 (only the span matters)
//   Yt = Aᵀ Y_{S-1};  λ, w = top eigenpair of Ytᵀ Yt  (= S[0]² of svd(Qᵀ A) in the reference)
// When n <= q the span already holds A's whole range: λ, w is then the top eigenpair of Aᵀ A and u = A w ("exact" weights).
// A panel of rank below q (a weight of rank < q, e.g. with fewer than q nonzero rows) keeps only the columns with a pivot
// above SV_PIVOT_REL: Y_k holds an orthonormal basis of the panel's span plus zero columns, Rx_k⁻¹ is the inverse on the
// kept columns and zero elsewhere, and the value and gradient stay finite (then σ₁² and 2 σ₁ u₁ v₁ᵀ when the span holds
// A's range).  The gradient is then the one along perturbations that keep the span's dimension.
// Backward, with z = Y_{S-1} w and the upstream scale s = gout / proba:
//   dA = s · (2 z (Yt w)ᵀ + Σ_k pair_k),  gQ_{S-1} = 2 (A Yt w) wᵀ,  gX_k = (I - Y_k Y_kᵀ) gQ_k Rx_k⁻ᵀ,
//   even k: pair_k = gX_k Qin_kᵀ, gQ_{k-1} = Aᵀ gX_k;  odd k: pair_k = Y_{k-1} gX_kᵀ, gQ_{k-1} = A gX_k
//   exact weights: dA = s · 2 u wᵀ.
//
// Kernels (one launch per stage for every weight; a weight's blocks found by binary search in the table's tile starts):
//   sv_product_kernel  op(A)·Y for [rows, nc] panels (nc <= SV_QMAX), SV_TR output rows per block, fp32 FMA, fixed k order
//   sv_orth_kernel     one block per weight: fp64 Gram, Cholesky, Rx⁻¹ kept in fp64, Y = X Rx⁻¹ in place
//   sv_eig_kernel      one block per weight: fp64 Gram of Yt (or of A), top eigenpair by repeated squaring, λ and w
//   sv_sum_kernel      one thread: Σ λ in weight order, / proba
//   sv_bwd_start_kernel, sv_project_kernel: z, Yt w; gX_k in place of gQ_k (one block per weight)
//   sv_write_kernel    every gradient element once: 64x64 tiles of dP over the rank-(1 + S q) factor pairs
// No atomics and no data-dependent order anywhere, so repeated calls are bitwise identical.  Everything is FP32 FMA or fp64:
// neither the TF32 flag nor autocast changes it.
#pragma once
#include "common.cuh"

namespace bm {

constexpr int SV_QMAX = 32;          // largest q (the drop-in's `dim`)
constexpr int SV_THREADS = 256;
constexpr int SV_TR = 32;            // output rows per product block
constexpr int SV_TK = 64;            // reduction rows staged per product iteration
constexpr int SV_WT = 64;            // gradient tile edge
constexpr int SV_GRAM_ROWS = 32;     // rows staged per Gram iteration
constexpr int SV_SQUARINGS = 48;     // eigenvector: the top direction of M^(2^48)
// Cholesky pivots at or below this fraction of the Gram matrix's largest diagonal drop their column: its residual norm is
// below 1e-4 of the largest column's.  The fp32 products leave residuals up to about 1e-6 in a panel whose true rank is
// below q, and normalising such rounding into a column of Y would amplify it through Rx⁻¹ in the backward
constexpr double SV_PIVOT_REL = 1e-8;

// the int64 table, one row of SV_FIELDS per weight
enum SvField { SV_P = 0, SV_M, SV_N, SV_TRANS, SV_EXACT, SV_WS, SV_WS64, SV_R, SV_G, SV_TILE_M, SV_TILE_N, SV_TILE_W, SV_FIELDS };

// buffers of a weight's float workspace: Y_k and G_k (gQ_k, then gX_k) are [rows_k, q], rows_k = m for even k, n for odd
__host__ __device__ inline long long sv_yoff(long long m, long long n, int q, int k) {
    return (long long)q * (((k + 1) / 2) * m + (k / 2) * n);
}
__host__ __device__ inline long long sv_ws_floats(long long m, long long n, int q, int S) {
    return 2 * sv_yoff(m, n, q, S) + n * q + 2 * m + n;          // Y_k, G_k, Yt, z [m], v [n], a [m]
}
__host__ __device__ inline long long sv_ws64_doubles(int q, int S) { return (long long)S * q * q + q + 1; }   // Rx⁻¹_k, w, λ

struct SvW {
    const float* p;
    int m, n, trans, exact;
    long long ws, ws64, r, g;
    __device__ explicit SvW(const long long* t)
        : p(reinterpret_cast<const float*>(t[SV_P])), m((int)t[SV_M]), n((int)t[SV_N]), trans((int)t[SV_TRANS]),
          exact((int)t[SV_EXACT]), ws(t[SV_WS]), ws64(t[SV_WS64]), r(t[SV_R]), g(t[SV_G]) {}
    __device__ float a(int i, int j) const { return trans ? __ldg(p + (long long)j * m + i) : __ldg(p + (long long)i * n + j); }
    __device__ int rows(int k) const { return (k & 1) ? n : m; }
};

// buffer selectors of sv_product_kernel
enum SvBuf { SVB_R = 0, SVB_Y = 1, SVB_G = 2, SVB_YT = 3, SVB_V = 4, SVB_A = 5 };
__device__ inline float* sv_buf(const SvW& w, float* ws, const float* R, int q, int S, int sel, int k) {
    float* base = ws + w.ws;
    const long long SY = sv_yoff(w.m, w.n, q, S);
    switch (sel) {
        case SVB_R: return const_cast<float*>(R) + w.r;
        case SVB_Y: return base + sv_yoff(w.m, w.n, q, k);
        case SVB_G: return base + SY + sv_yoff(w.m, w.n, q, k);
        case SVB_YT: return base + 2 * SY;
        case SVB_V: return base + 2 * SY + (long long)w.n * q + w.m;
        default: return base + 2 * SY + (long long)w.n * q + w.m + w.n;
    }
}
__device__ inline float* sv_z(const SvW& w, float* ws, int q, int S) { return ws + w.ws + 2 * sv_yoff(w.m, w.n, q, S) + (long long)w.n * q; }

// the weight owning grouped block b: the last row whose tile start is <= b (rows with no tiles are passed over)
__device__ inline int sv_owner(const long long* tab, int W, int field, long long b) {
    int lo = 0, hi = W - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) / 2;
        if (tab[(long long)mid * SV_FIELDS + field] <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// out [rows, nc] = op(A) · in [K, nc]: op 0 A (rows m, K n), op 1 Aᵀ (rows n, K m).  Exact weights have no tiles; in the
// backward (bwd != 0) weights without a gradient return at once.
__global__ void __launch_bounds__(SV_THREADS) sv_product_kernel(const long long* tab, int W, int q, int S, int op, int nc,
                                                                int in_sel, int in_k, int out_sel, int out_k, int bwd,
                                                                const float* R, float* ws) {
    const int field = op ? SV_TILE_N : SV_TILE_M;
    const int i = sv_owner(tab, W, field, blockIdx.x);
    const long long* t = tab + (long long)i * SV_FIELDS;
    const SvW w(t);
    if (bwd && w.g < 0) return;
    const int rows = op ? w.n : w.m, K = op ? w.m : w.n;
    const int r0 = (int)(blockIdx.x - t[field]) * SV_TR;
    const float* in = sv_buf(w, ws, R, q, S, in_sel, in_k);
    float* out = sv_buf(w, ws, R, q, S, out_sel, out_k);
    // op(A)(r, k) = p[r*ld + k] when it runs along P's rows (op == trans), else p[k*ld + r]
    const bool along_k = (op == w.trans);
    const long long ld = w.trans ? w.m : w.n;
    __shared__ float sA[SV_TR][SV_TK + 1];
    __shared__ float sY[SV_TK][SV_QMAX];
    const int tr = threadIdx.x / 8, tc = threadIdx.x % 8;
    float acc[SV_QMAX / 8] = {};
    for (int k0 = 0; k0 < K; k0 += SV_TK) {
        for (int e = threadIdx.x; e < SV_TR * SV_TK; e += SV_THREADS) {
            const int r = along_k ? e / SV_TK : e % SV_TR, k = along_k ? e % SV_TK : e / SV_TR;
            const int gr = r0 + r, gk = k0 + k;
            sA[r][k] = (gr < rows && gk < K) ? __ldg(w.p + (along_k ? gr * ld + gk : gk * ld + gr)) : 0.f;
        }
        for (int e = threadIdx.x; e < SV_TK * nc; e += SV_THREADS) {
            const int k = e / nc, c = e % nc;
            sY[k][c] = (k0 + k < K) ? in[(long long)(k0 + k) * nc + c] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < SV_TK; ++kk) {
            const float av = sA[tr][kk];
#pragma unroll
            for (int j = 0; j < SV_QMAX / 8; ++j)
                if (tc + 8 * j < nc) acc[j] = fmaf(av, sY[kk][tc + 8 * j], acc[j]);
        }
        __syncthreads();
    }
    if (r0 + tr < rows) {
#pragma unroll
        for (int j = 0; j < SV_QMAX / 8; ++j)
            if (tc + 8 * j < nc) out[(long long)(r0 + tr) * nc + tc + 8 * j] = acc[j];
    }
}

// G[a*q + b] = Σ_r x(r, a) y(r, b) over r < rows in fp64, a, b < d, in row order (block-wide; ends synchronised)
template <typename LX, typename LY>
__device__ void sv_gram(LX x, LY y, int rows, int d, double* G) {
    __shared__ float sx[SV_GRAM_ROWS][SV_QMAX], sy[SV_GRAM_ROWS][SV_QMAX];
    double acc[SV_QMAX * SV_QMAX / SV_THREADS] = {};
    for (int r0 = 0; r0 < rows; r0 += SV_GRAM_ROWS) {
        for (int e = threadIdx.x; e < SV_GRAM_ROWS * d; e += SV_THREADS) {
            const int r = e / d, c = e % d;
            sx[r][c] = r0 + r < rows ? x(r0 + r, c) : 0.f;
            sy[r][c] = r0 + r < rows ? y(r0 + r, c) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SV_QMAX * SV_QMAX / SV_THREADS; ++j) {
            const int e = threadIdx.x + j * SV_THREADS;
            if (e < d * d) {
                const int a = e / d, b = e % d;
                for (int r = 0; r < SV_GRAM_ROWS; ++r) acc[j] = fma((double)sx[r][a], (double)sy[r][b], acc[j]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < SV_QMAX * SV_QMAX / SV_THREADS; ++j) {
        const int e = threadIdx.x + j * SV_THREADS;
        if (e < d * d) G[(e / d) * d + e % d] = acc[j];
    }
    __syncthreads();
}

// Cholesky QR of X [rows, q] at step k, in place: Y = X Rx⁻¹ with Rx upper triangular, XᵀX = RxᵀRx; Rx⁻¹ to ws64
__global__ void __launch_bounds__(SV_THREADS) sv_orth_kernel(const long long* tab, int q, int S, int k, float* ws, double* ws64) {
    const SvW w(tab + (long long)blockIdx.x * SV_FIELDS);
    if (w.exact) return;
    const int rows = w.rows(k);
    float* X = ws + w.ws + sv_yoff(w.m, w.n, q, k);
    __shared__ double G[SV_QMAX * SV_QMAX], Ri[SV_QMAX * SV_QMAX];
    auto ld = [&](int r, int c) { return X[(long long)r * q + c]; };
    sv_gram(ld, ld, rows, q, G);
    // right-looking Cholesky on the upper triangle: row c of Rx, then the trailing update.  A pivot at or below
    // SV_PIVOT_REL of the largest diagonal is a column the earlier ones already span (to the panel's fp32 rounding): its
    // row of Rx is zero, and so are its column of Y and its row and column of Rx⁻¹ (see the header comment)
    __shared__ double tol;
    if (threadIdx.x == 0) {
        double mx = 0.0;
        for (int a = 0; a < q; ++a) mx = fmax(mx, G[a * q + a]);
        tol = SV_PIVOT_REL * mx;
    }
    __syncthreads();
    for (int c = 0; c < q; ++c) {
        if (threadIdx.x == 0) {
            const double d = G[c * q + c];
            G[c * q + c] = d > tol ? sqrt(d) : 0.0;
        }
        __syncthreads();
        const double rc = G[c * q + c];
        for (int j = c + 1 + threadIdx.x; j < q; j += SV_THREADS) G[c * q + j] = rc > 0.0 ? G[c * q + j] / rc : 0.0;
        __syncthreads();
        for (int e = threadIdx.x; e < q * q; e += SV_THREADS) {
            const int a = e / q, b = e % q;
            if (a > c && b >= a) G[a * q + b] -= G[c * q + a] * G[c * q + b];
        }
        __syncthreads();
    }
    // Rx⁻¹ by columns (upper triangular): the inverse of Rx restricted to the kept columns, zero elsewhere
    if (threadIdx.x < q) {
        const int c = threadIdx.x;
        for (int a = 0; a < q; ++a) Ri[a * q + c] = 0.0;
        if (G[c * q + c] > 0.0) {
            Ri[c * q + c] = 1.0 / G[c * q + c];
            for (int a = c - 1; a >= 0; --a) {
                if (G[a * q + a] == 0.0) continue;
                double s = 0.0;
                for (int l = a + 1; l <= c; ++l) s = fma(G[a * q + l], Ri[l * q + c], s);
                Ri[a * q + c] = -s / G[a * q + a];
            }
        }
    }
    __syncthreads();
    double* Rk = ws64 + w.ws64 + (long long)k * q * q;
    for (int e = threadIdx.x; e < q * q; e += SV_THREADS) Rk[e] = Ri[e];
    for (int r = threadIdx.x; r < rows; r += SV_THREADS) {
        float x[SV_QMAX];
#pragma unroll
        for (int c = 0; c < SV_QMAX; ++c) x[c] = c < q ? X[(long long)r * q + c] : 0.f;
#pragma unroll
        for (int c = 0; c < SV_QMAX; ++c) {
            if (c < q) {
                double s = 0.0;
#pragma unroll
                for (int l = 0; l < SV_QMAX; ++l)
                    if (l <= c) s = fma((double)x[l], Ri[l * q + c], s);
                X[(long long)r * q + c] = (float)s;
            }
        }
    }
}

// the top eigenpair of M [d, d] (symmetric positive semi-definite, in shared memory): v from the trace-normalised powers
// M^(2^j), λ the Rayleigh quotient of v.  Block-wide; writes w[0..q) (zero past d) and lam.
__device__ void sv_top_eig(const double* M, int d, int q, double* w_out, double* lam_out) {
    __shared__ double P[SV_QMAX * SV_QMAX], T[SV_QMAX * SV_QMAX], v[SV_QMAX];
    __shared__ double tr;
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int a = 0; a < d; ++a) s += M[a * d + a];
        tr = s;
    }
    __syncthreads();
    const double t0 = tr;
    for (int e = threadIdx.x; e < d * d; e += SV_THREADS) P[e] = t0 > 0.0 ? M[e] / t0 : 0.0;
    __syncthreads();
    for (int it = 0; it < SV_SQUARINGS && t0 > 0.0; ++it) {
        for (int e = threadIdx.x; e < d * d; e += SV_THREADS) {
            const int a = e / d, b = e % d;
            double s = 0.0;
            for (int l = 0; l < d; ++l) s = fma(P[a * d + l], P[l * d + b], s);
            T[e] = s;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double s = 0.0;
            for (int a = 0; a < d; ++a) s += T[a * d + a];
            tr = s;
        }
        __syncthreads();
        const double ts = tr;
        for (int e = threadIdx.x; e < d * d; e += SV_THREADS) P[e] = T[e] / ts;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int best = 0;
        for (int a = 1; a < d; ++a)
            if (P[a * d + a] > P[best * d + best]) best = a;
        double nn = 0.0;
        for (int a = 0; a < d; ++a) {
            v[a] = t0 > 0.0 ? P[a * d + best] : (a == 0 ? 1.0 : 0.0);
            nn += v[a] * v[a];
        }
        const double inv = 1.0 / sqrt(nn);
        double lam = 0.0;
        for (int a = 0; a < d; ++a) v[a] *= inv;
        for (int a = 0; a < d; ++a) {
            double s = 0.0;
            for (int b = 0; b < d; ++b) s = fma(M[a * d + b], v[b], s);
            lam = fma(v[a], s, lam);
        }
        for (int a = 0; a < q; ++a) w_out[a] = a < d ? v[a] : 0.0;
        *lam_out = lam;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(SV_THREADS) sv_eig_kernel(const long long* tab, int q, int S, float* ws, double* ws64) {
    const SvW w(tab + (long long)blockIdx.x * SV_FIELDS);
    __shared__ double M[SV_QMAX * SV_QMAX];
    double* wv = ws64 + w.ws64 + (long long)S * q * q;
    if (w.exact) {
        auto la = [&](int r, int c) { return w.a(r, c); };
        sv_gram(la, la, w.m, w.n, M);
        sv_top_eig(M, w.n, q, wv, wv + q);
        if (w.g >= 0) {                                          // u = A w for the gradient 2 u wᵀ
            float* u = sv_z(w, ws, q, S);
            for (int r = threadIdx.x; r < w.m; r += SV_THREADS) {
                double s = 0.0;
                for (int c = 0; c < w.n; ++c) s = fma((double)w.a(r, c), wv[c], s);
                u[r] = (float)s;
            }
        }
    } else {
        const float* Yt = ws + w.ws + 2 * sv_yoff(w.m, w.n, q, S);
        auto ly = [&](int r, int c) { return Yt[(long long)r * q + c]; };
        sv_gram(ly, ly, w.n, q, M);
        sv_top_eig(M, q, q, wv, wv + q);
    }
}

__global__ void sv_sum_kernel(const long long* tab, int W, int q, int S, const double* ws64, double proba, float* out) {
    double s = 0.0;
    for (int i = 0; i < W; ++i) s += ws64[tab[(long long)i * SV_FIELDS + SV_WS64] + (long long)S * q * q + q];
    out[0] = (float)(s / proba);
}

// z = Y_{S-1} w [m] and v = Yt w [n] of every weight with a gradient
__global__ void __launch_bounds__(SV_THREADS) sv_bwd_start_kernel(const long long* tab, int q, int S, float* ws, const double* ws64) {
    const SvW w(tab + (long long)blockIdx.x * SV_FIELDS);
    if (w.exact || w.g < 0) return;
    const double* wv = ws64 + w.ws64 + (long long)S * q * q;
    const float* Y = sv_buf(w, ws, nullptr, q, S, SVB_Y, S - 1);
    const float* Yt = sv_buf(w, ws, nullptr, q, S, SVB_YT, 0);
    float* z = sv_z(w, ws, q, S);
    float* v = sv_buf(w, ws, nullptr, q, S, SVB_V, 0);
    for (int r = threadIdx.x; r < w.m + w.n; r += SV_THREADS) {
        const float* row = r < w.m ? Y + (long long)r * q : Yt + (long long)(r - w.m) * q;
        double s = 0.0;
        for (int c = 0; c < q; ++c) s = fma((double)row[c], wv[c], s);
        (r < w.m ? z[r] : v[r - w.m]) = (float)s;
    }
}

// gX_k = (I - Y_k Y_kᵀ) gQ_k Rx_k⁻ᵀ in place of gQ_k; at the last step gQ = 2 a wᵀ (a = A Yt w) is formed first
__global__ void __launch_bounds__(SV_THREADS) sv_project_kernel(const long long* tab, int q, int S, int k, float* ws, const double* ws64) {
    const SvW w(tab + (long long)blockIdx.x * SV_FIELDS);
    if (w.exact || w.g < 0) return;
    const int rows = w.rows(k);
    const float* Y = sv_buf(w, ws, nullptr, q, S, SVB_Y, k);
    float* Gk = sv_buf(w, ws, nullptr, q, S, SVB_G, k);
    const double* Ri = ws64 + w.ws64 + (long long)k * q * q;
    if (k == S - 1) {
        const double* wv = ws64 + w.ws64 + (long long)S * q * q;
        const float* a = sv_buf(w, ws, nullptr, q, S, SVB_A, 0);
        for (int e = threadIdx.x; e < rows * q; e += SV_THREADS) Gk[e] = (float)(2.0 * a[e / q] * wv[e % q]);
        __syncthreads();
    }
    __shared__ double C[SV_QMAX * SV_QMAX];
    auto ly = [&](int r, int c) { return Y[(long long)r * q + c]; };
    auto lg = [&](int r, int c) { return Gk[(long long)r * q + c]; };
    sv_gram(ly, lg, rows, q, C);                                   // C = Yᵀ gQ
    for (int r = threadIdx.x; r < rows; r += SV_THREADS) {
        double h[SV_QMAX];
        float y[SV_QMAX];
#pragma unroll
        for (int c = 0; c < SV_QMAX; ++c) {
            y[c] = c < q ? Y[(long long)r * q + c] : 0.f;
            h[c] = c < q ? (double)Gk[(long long)r * q + c] : 0.0;
        }
#pragma unroll
        for (int a = 0; a < SV_QMAX; ++a) {
            if (a < q) {
                double s = h[a];
#pragma unroll
                for (int c = 0; c < SV_QMAX; ++c)
                    if (c < q) s = fma(-(double)y[c], C[c * q + a], s);
                h[a] = s;
            }
        }
#pragma unroll
        for (int b = 0; b < SV_QMAX; ++b) {
            if (b < q) {
                double s = 0.0;
#pragma unroll
                for (int a = 0; a < SV_QMAX; ++a)
                    if (a >= b && a < q) s = fma(h[a], Ri[b * q + a], s);
                Gk[(long long)r * q + b] = (float)s;
            }
        }
    }
}

// dP = (gout / proba) · Σ pairs, one SV_WT x SV_WT tile per block, every element written once
__global__ void __launch_bounds__(SV_THREADS) sv_write_kernel(const long long* tab, int W, int q, int S, const float* R,
                                                              float* ws, const double* ws64, const float* gout,
                                                              double proba, float* grad) {
    const int i = sv_owner(tab, W, SV_TILE_W, blockIdx.x);
    const long long* t = tab + (long long)i * SV_FIELDS;
    const SvW w(t);
    const int rows_p = w.trans ? w.n : w.m, cols_p = w.trans ? w.m : w.n;
    const int tiles_c = (cols_p + SV_WT - 1) / SV_WT;
    const int tile = (int)(blockIdx.x - t[SV_TILE_W]);
    const int r0 = (tile / tiles_c) * SV_WT, c0 = (tile % tiles_c) * SV_WT;
    // rows padded to 66 floats: a warp's (row, l) stores at q = 16 (l fastest, two rows) land in 32 distinct banks
    __shared__ float sR[SV_QMAX][SV_WT + 2], sC[SV_QMAX][SV_WT + 2];
    const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
    float acc[4][4] = {};
    const double* wv = ws64 + w.ws64 + (long long)S * q * q;
    const int npairs = w.exact ? 1 : S + 1;
    for (int pi = 0; pi < npairs; ++pi) {
        // the pair's m-side factor U [m, L] and n-side factor V [n, L]; a null V is the weight's w (exact rank-1 pair)
        const float *U, *V = nullptr;
        int L = q;
        float uscale = 1.f;
        if (pi == 0) {
            L = 1;
            uscale = 2.f;
            U = sv_z(w, ws, q, S);
            if (!w.exact) V = sv_buf(w, ws, R, q, S, SVB_V, 0);
        } else {
            const int k = pi - 1;
            if (k % 2 == 0) {
                U = sv_buf(w, ws, R, q, S, SVB_G, k);
                V = k == 0 ? sv_buf(w, ws, R, q, S, SVB_R, 0) : sv_buf(w, ws, R, q, S, SVB_Y, k - 1);
            } else {
                U = sv_buf(w, ws, R, q, S, SVB_Y, k - 1);
                V = sv_buf(w, ws, R, q, S, SVB_G, k);
            }
        }
        // P rows are A rows (U) unless transposed
        for (int e = threadIdx.x; e < SV_WT * L; e += SV_THREADS) {
            const int rr = e / L, l = e % L;
            const int gr = r0 + rr, gc = c0 + rr;
            auto fu = [&](int x) { return x < w.m ? uscale * U[(long long)x * L + l] : 0.f; };
            auto fv = [&](int x) { return x < w.n ? (V ? V[(long long)x * L + l] : (float)wv[x]) : 0.f; };
            sR[l][rr] = w.trans ? fv(gr) : fu(gr);
            sC[l][rr] = w.trans ? fu(gc) : fv(gc);
        }
        __syncthreads();
        for (int l = 0; l < L; ++l) {
            float a[4], b[4];
#pragma unroll
            for (int x = 0; x < 4; ++x) { a[x] = sR[l][ty + 16 * x]; b[x] = sC[l][tx + 16 * x]; }
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
                for (int y = 0; y < 4; ++y) acc[x][y] = fmaf(a[x], b[y], acc[x][y]);
        }
        __syncthreads();
    }
    const float s = (float)((double)gout[0] / proba);
    float* dP = grad + w.g;
#pragma unroll
    for (int x = 0; x < 4; ++x) {
        const int r = r0 + ty + 16 * x;
        if (r >= rows_p) continue;
#pragma unroll
        for (int y = 0; y < 4; ++y) {
            const int c = c0 + tx + 16 * y;
            if (c < cols_p) dP[(long long)r * cols_p + c] = s * acc[x][y];
        }
    }
}

}  // namespace bm
