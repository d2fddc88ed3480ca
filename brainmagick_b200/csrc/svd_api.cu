// C-ABI entry points of the spectral-norm penalty (see include/bm_b200.h for the contract).
#include "api.cuh"
#include "svd_penalty.cuh"

using namespace bm;

// Spectral-norm penalty (bm/svd.py): grouped randomized subspace iteration over every selected weight (svd_penalty.cuh)
extern "C" int bm_svd_table(int W, const long long* ptrs, const long long* rows_p, const long long* cols_p, const int* grad,
                            int q, int niter, long long* table, long long* sizes) {
    BM_CHECK_ARG(W >= 1 && q >= 1 && q <= SV_QMAX && niter >= 0 && ptrs && rows_p && cols_p && grad && table && sizes);
    const int S = 2 * niter + 1;
    long long ws = 0, ws64 = 0, r = 0, g = 0, tm = 0, tn = 0, tw = 0;
    for (int i = 0; i < W; ++i) {
        BM_CHECK_ARG(ptrs[i] && rows_p[i] >= 1 && cols_p[i] >= 1 && rows_p[i] * cols_p[i] < (1ll << 31));
        const int trans = rows_p[i] < cols_p[i];
        const long long m = trans ? cols_p[i] : rows_p[i], n = trans ? rows_p[i] : cols_p[i];
        const int exact = n <= q;
        long long* t = table + (long long)i * SV_FIELDS;
        t[SV_P] = ptrs[i];
        t[SV_M] = m;
        t[SV_N] = n;
        t[SV_TRANS] = trans;
        t[SV_EXACT] = exact;
        t[SV_WS] = ws;
        t[SV_WS64] = ws64;
        t[SV_R] = r;
        t[SV_G] = grad[i] ? g : -1;
        t[SV_TILE_M] = tm;
        t[SV_TILE_N] = tn;
        t[SV_TILE_W] = tw;
        ws += sv_ws_floats(m, n, q, S);
        ws64 += sv_ws64_doubles(q, S);
        r += n * q;
        if (grad[i]) {
            g += m * n;
            tw += ((rows_p[i] + SV_WT - 1) / SV_WT) * ((cols_p[i] + SV_WT - 1) / SV_WT);
        }
        if (!exact) {
            tm += (m + SV_TR - 1) / SV_TR;
            tn += (n + SV_TR - 1) / SV_TR;
        }
    }
    const long long out[7] = {ws, ws64, r, g, tm, tn, tw};
    for (int k = 0; k < 7; ++k) sizes[k] = out[k];
    return 0;
}
extern "C" int bm_svd_penalty_fwd(const long long* table, int W, int q, int niter, long long tiles_m, long long tiles_n,
                                  const float* R, float* ws, double* ws64, double proba, float* out, bm_stream_t stream) {
    BM_CHECK_ARG(table && W >= 1 && q >= 1 && q <= SV_QMAX && niter >= 0 && tiles_m >= 0 && tiles_n >= 0);
    BM_CHECK_ARG(R && ws && ws64 && out && proba > 0.0);
    const int S = 2 * niter + 1;
    const cudaStream_t st = ST(stream);
    for (int k = 0; k < S; ++k) {
        const int op = k & 1;
        const long long tiles = op ? tiles_n : tiles_m;
        if (tiles) {
            sv_product_kernel<<<(unsigned)tiles, SV_THREADS, 0, st>>>(table, W, q, S, op, q, k ? SVB_Y : SVB_R, k - 1, SVB_Y,
                                                                      k, 0, R, ws);
            BM_CHECK_LAUNCH();
        }
        sv_orth_kernel<<<W, SV_THREADS, 0, st>>>(table, q, S, k, ws, ws64);
        BM_CHECK_LAUNCH();
    }
    if (tiles_n) {
        sv_product_kernel<<<(unsigned)tiles_n, SV_THREADS, 0, st>>>(table, W, q, S, 1, q, SVB_Y, S - 1, SVB_YT, 0, 0, R, ws);
        BM_CHECK_LAUNCH();
    }
    sv_eig_kernel<<<W, SV_THREADS, 0, st>>>(table, q, S, ws, ws64);
    BM_CHECK_LAUNCH();
    sv_sum_kernel<<<1, 1, 0, st>>>(table, W, q, S, ws64, proba, out);
    BM_CHECK_LAUNCH();
    return 0;
}
extern "C" int bm_svd_penalty_bwd(const long long* table, int W, int q, int niter, long long tiles_m, long long tiles_n,
                                  long long tiles_w, const float* R, float* ws, const double* ws64, const float* gout,
                                  double proba, float* grad, bm_stream_t stream) {
    BM_CHECK_ARG(table && W >= 1 && q >= 1 && q <= SV_QMAX && niter >= 0 && tiles_m >= 0 && tiles_n >= 0 && tiles_w >= 0);
    BM_CHECK_ARG(R && ws && ws64 && gout && proba > 0.0 && (grad || tiles_w == 0));
    const int S = 2 * niter + 1;
    const cudaStream_t st = ST(stream);
    sv_bwd_start_kernel<<<W, SV_THREADS, 0, st>>>(table, q, S, ws, ws64);
    BM_CHECK_LAUNCH();
    if (tiles_m) {
        sv_product_kernel<<<(unsigned)tiles_m, SV_THREADS, 0, st>>>(table, W, q, S, 0, 1, SVB_V, 0, SVB_A, 0, 1, R, ws);
        BM_CHECK_LAUNCH();
    }
    for (int k = S - 1; k >= 0; --k) {
        sv_project_kernel<<<W, SV_THREADS, 0, st>>>(table, q, S, k, ws, ws64);
        BM_CHECK_LAUNCH();
        const int op = (k % 2 == 0) ? 1 : 0;                 // X_k = A Qin: gQin = Aᵀ gX; X_k = Aᵀ Qin: gQin = A gX
        const long long tiles = op ? tiles_n : tiles_m;
        if (k > 0 && tiles) {
            sv_product_kernel<<<(unsigned)tiles, SV_THREADS, 0, st>>>(table, W, q, S, op, q, SVB_G, k, SVB_G, k - 1, 1, R, ws);
            BM_CHECK_LAUNCH();
        }
    }
    if (tiles_w) {
        sv_write_kernel<<<(unsigned)tiles_w, SV_THREADS, 0, st>>>(table, W, q, S, R, ws, ws64, gout, proba, grad);
        BM_CHECK_LAUNCH();
    }
    return 0;
}
