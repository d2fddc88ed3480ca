// C-ABI entry points of the masked regression losses, FeatureDecodingLoss and the test metrics (see include/bm_b200.h
// for the contract).
#include "api.cuh"
#include "masked_loss.cuh"
#include "decoding_loss.cuh"
#include "metrics.cuh"

using namespace bm;

// masked L1 / L2 loss (bm/losses.py:11-26): fixed-grid fp64 partials, a one-CTA finalize, an elementwise backward
extern "C" long long bm_masked_loss_workspace(int B, int C, int T) {
    return (B < 0 || C < 0 || T < 0) ? 0 : 4ll * ml_blocks((long long)B * C);      // (sum, count) fp64 per CTA
}
extern "C" int bm_masked_loss_fwd(int kind, const float* est, long long est_sb, long long est_sc, const float* out,
                                  long long out_sb, long long out_sc, const unsigned char* mask, long long mask_sb,
                                  long long mask_sc, long long mask_st, int B, int C, int T, float* workspace,
                                  long long workspace_floats, float* loss, float* inv_n, bm_stream_t stream) {
    BM_CHECK_ARG((kind == ML_L1 || kind == ML_L2) && B >= 0 && C >= 0 && T >= 0 && loss && inv_n);
    BM_CHECK_ARG(((long long)B * C * T == 0) || (est && out && mask));
    BM_CHECK_WS(bm_masked_loss_workspace(B, C, T));
    const long long rows = (long long)B * C * (T > 0);
    const MlOperands p{est, est_sb, est_sc, out, out_sb, out_sc, mask, mask_sb, mask_sc, mask_st, C, T};
    const int nb = ml_blocks(rows);
    double* part = reinterpret_cast<double*>(workspace);
    if (kind == ML_L1) masked_loss_partials_kernel<ML_L1><<<nb, ML_THREADS, 0, ST(stream)>>>(p, rows, part);
    else masked_loss_partials_kernel<ML_L2><<<nb, ML_THREADS, 0, ST(stream)>>>(p, rows, part);
    BM_CHECK_LAUNCH();
    masked_loss_finalize_kernel<<<1, ML_FINAL_THREADS, 0, ST(stream)>>>(part, nb, loss, inv_n);
    BM_CHECK_LAUNCH();
    return 0;
}
extern "C" int bm_masked_loss_bwd(int kind, const float* gout, const float* inv_n, const float* est, long long est_sb,
                                  long long est_sc, const float* out, long long out_sb, long long out_sc,
                                  const unsigned char* mask, long long mask_sb, long long mask_sc, long long mask_st, int B,
                                  int C, int T, float* d_est, float* d_out, bm_stream_t stream) {
    BM_CHECK_ARG((kind == ML_L1 || kind == ML_L2) && B >= 0 && C >= 0 && T >= 0 && gout && inv_n);
    const long long rows = (long long)B * C;
    if (rows * T == 0 || (!d_est && !d_out)) return 0;
    BM_CHECK_ARG(est && out && mask);
    const MlOperands p{est, est_sb, est_sc, out, out_sb, out_sc, mask, mask_sb, mask_sc, mask_st, C, T};
    const bool vec_out = T % 4 == 0 && aligned16(d_est, d_out);
    const int grid = ew_grid(rows * ((T + 3) / 4), ML_THREADS);
    if (kind == ML_L1)
        masked_loss_bwd_kernel<ML_L1><<<grid, ML_THREADS, 0, ST(stream)>>>(p, rows, gout, inv_n, d_est, d_out, vec_out);
    else
        masked_loss_bwd_kernel<ML_L2><<<grid, ML_THREADS, 0, ST(stream)>>>(p, rows, gout, inv_n, d_est, d_out, vec_out);
    BM_CHECK_LAUNCH();
    return 0;
}

// FeatureDecodingLoss (bm/losses.py:117-173): fixed-grid fp64 partials per (CTA, feature), a one-CTA finalize, one
// backward pass over every gradient row
extern "C" long long bm_decoding_loss_workspace(int B, int T, int F) {
    if (B < 0 || T < 0 || F < 1 || F > FD_MAX_FEATURES) return 0;
    const long long nb = fd_blocks(B, T);
    return 4 * nb * F + nb + (nb & 1);              // (sum, count) fp64 per (CTA, feature), then one flag word per CTA
}
extern "C" int bm_decoding_loss_fwd(const float* est, long long est_sb, long long est_sc, const float* out, long long out_sb,
                                    long long out_sc, const unsigned char* mask, long long mask_sb, long long mask_sc,
                                    long long mask_st, int B, int T, const int* table, int F, const float* weights,
                                    float* lse, float* workspace, long long workspace_floats, float* loss, float* scale,
                                    int* flag, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(B >= 0 && T >= 0 && F >= 1 && F <= FD_MAX_FEATURES && table && loss && scale && flag);
    BM_CHECK_ARG(((long long)B * T == 0) || (est && out && mask && lse));
    BM_CHECK_WS(bm_decoding_loss_workspace(B, T, F));
    const int nb = fd_blocks(B, T);
    const FdOperands p{est, est_sb, est_sc, out, out_sb, out_sc, mask, mask_sb, mask_sc, mask_st, table, weights, F, B, T};
    double* part = reinterpret_cast<double*>(workspace);
    int* cta_flags = reinterpret_cast<int*>(workspace + 4ll * nb * F);
    decoding_loss_partials_kernel<<<nb, FD_THREADS, 0, ST(stream)>>>(p, part, cta_flags, lse);
    BM_CHECK_LAUNCH();
    decoding_loss_finalize_kernel<<<1, ML_FINAL_THREADS, 0, ST(stream)>>>(part, cta_flags, nb, table, F, loss, scale, flag,
                                                                           status);
    BM_CHECK_LAUNCH();
    return 0;
}
extern "C" int bm_decoding_loss_bwd(const float* gout, const float* scale, const float* lse, const float* est,
                                    long long est_sb, long long est_sc, const float* out, long long out_sb, long long out_sc,
                                    const unsigned char* mask, long long mask_sb, long long mask_sc, long long mask_st, int B,
                                    int T, int est_C, int out_C, const int* table, int F, const float* weights, float* d_est,
                                    float* d_out, bm_stream_t stream) {
    BM_CHECK_ARG(B >= 0 && T >= 0 && est_C >= 0 && out_C >= 0 && F >= 1 && F <= FD_MAX_FEATURES && gout && scale && table);
    if ((long long)B * T == 0 || (!d_est && !d_out)) return 0;
    BM_CHECK_ARG(est && out && mask && lse);
    const FdOperands p{est, est_sb, est_sc, out, out_sb, out_sc, mask, mask_sb, mask_sc, mask_st, table, weights, F, B, T};
    const bool vec_out = T % 4 == 0 && aligned16(d_est, d_out);
    const long long rows = (long long)B * ((d_est ? est_C : 0) + (d_out ? out_C : 0));
    decoding_loss_bwd_kernel<<<ew_grid(rows * ((T + 3) / 4), FD_THREADS), FD_THREADS, 0, ST(stream)>>>(
        p, est_C, out_C, gout, scale, lse, d_est, d_out, vec_out);
    BM_CHECK_LAUNCH();
    return 0;
}

// Test metrics (bm/metrics.py): per-column fp64 sums over dim 0 into device accumulators, and one finalize per get()
namespace {
template <typename S>
int metric_update_launch(int kind, const MtOperands& p, int splits, double* acc, int* seen, int parity, double* part,
                         cudaStream_t st) {
    const long long cols = (long long)p.C * p.T;
    const dim3 grid((unsigned)((cols + MT_THREADS - 1) / MT_THREADS), (unsigned)splits);
    switch (kind) {
        case MT_CORRELATION: metric_update_kernel<S, MT_CORRELATION><<<grid, MT_THREADS, 0, st>>>(p, splits, acc, seen, parity, part); break;
        case MT_L1: metric_update_kernel<S, MT_L1><<<grid, MT_THREADS, 0, st>>>(p, splits, acc, seen, parity, part); break;
        case MT_L2: metric_update_kernel<S, MT_L2><<<grid, MT_THREADS, 0, st>>>(p, splits, acc, seen, parity, part); break;
        default: metric_update_kernel<S, MT_ACCURACY><<<grid, MT_THREADS, 0, st>>>(p, splits, acc, seen, parity, part); break;
    }
    BM_CHECK_LAUNCH();
    if (splits > 1) {
        if (kind == MT_CORRELATION)
            metric_combine_kernel<6><<<grid.x, MT_THREADS, 0, st>>>(part, splits, cols, acc, seen, parity);
        else
            metric_combine_kernel<2><<<grid.x, MT_THREADS, 0, st>>>(part, splits, cols, acc, seen, parity);
        BM_CHECK_LAUNCH();
    }
    return 0;
}
template <typename O>
int metric_finalize_launch(int kind, const double* acc, long long cols, double tol, void* out, int* flag, cudaStream_t st) {
    if (kind == MT_CORRELATION)
        metric_finalize_kernel<O, MT_CORRELATION><<<1, MT_FINAL_THREADS, 0, st>>>(acc, cols, tol, static_cast<O*>(out), flag);
    else
        metric_finalize_kernel<O, MT_L1><<<1, MT_FINAL_THREADS, 0, st>>>(acc, cols, tol, static_cast<O*>(out), flag);
    BM_CHECK_LAUNCH();
    return 0;
}
}  // namespace

extern "C" long long bm_metric_workspace(int N, int C, int T) {
    if (N < 0 || C < 0 || T < 0) return 0;
    const long long cols = (long long)C * T;
    const int s = mt_splits(N, cols);
    return s > 1 ? 2ll * MT_MAX_PLANES * s * cols : 0;      // fp64 partials: NP planes per split
}
extern "C" int bm_metric_update(int kind, int dtype, const void* left, long long left_sn, long long left_sc,
                                long long left_st, const void* right, long long right_sn, long long right_sc,
                                long long right_st, const unsigned char* mask, long long mask_sn, long long mask_sc,
                                long long mask_st, int mask_n, int N, int C, int T, int K, double* acc, int* seen,
                                int parity, float* workspace, long long workspace_floats, bm_stream_t stream) {
    BM_CHECK_ARG(kind >= MT_CORRELATION && kind <= MT_ACCURACY && (dtype == 0 || dtype == 1));
    BM_CHECK_ARG(N >= 0 && C >= 0 && T >= 0 && (mask_n == 1 || mask_n == N) && (parity == 0 || parity == 1));
    BM_CHECK_ARG(kind != MT_ACCURACY || (C == 1 && K >= 1));
    const long long cols = (long long)C * T;
    if (cols == 0) return 0;                                // an empty slice or time crop: nothing to add
    BM_CHECK_ARG(acc && seen && left && right && mask);
    const int splits = mt_splits(N, cols);
    if (splits > 1) BM_CHECK_WS(bm_metric_workspace(N, C, T));
    const MtOperands p{left, left_sn, left_sc, left_st, right, right_sn, right_sc, right_st, mask, mask_sn, mask_sc, mask_st,
                       mask_n, N, C, T, K};
    double* part = reinterpret_cast<double*>(workspace);
    return dtype == 0 ? metric_update_launch<float>(kind, p, splits, acc, seen, parity, part, ST(stream))
                      : metric_update_launch<double>(kind, p, splits, acc, seen, parity, part, ST(stream));
}
extern "C" int bm_metric_finalize(int kind, const double* acc, int C, int T, double tol, void* out, int out_dtype, int* flag,
                                  bm_stream_t stream) {
    BM_CHECK_ARG(kind >= MT_CORRELATION && kind <= MT_ACCURACY && (out_dtype == 0 || out_dtype == 1));
    const long long cols = (long long)C * T;
    BM_CHECK_ARG(C >= 0 && T >= 0 && flag && (cols == 0 || (acc && out)));
    return out_dtype == 0 ? metric_finalize_launch<float>(kind, acc, cols, tol, out, flag, ST(stream))
                          : metric_finalize_launch<double>(kind, acc, cols, tol, out, flag, ST(stream));
}
