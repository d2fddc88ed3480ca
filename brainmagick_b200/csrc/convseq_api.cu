// C-ABI entry points of the ConvSequence layers and the head on the FP32-FMA path: conv, BatchNorm statistics, the layer
// epilogue family, GLU and GELU backward, column sums (see include/bm_b200.h for the contract).
#include "api.cuh"
#include "elementwise.cuh"
#include "convseq.cuh"

using namespace bm;

namespace bm {
template <class T>
int reduce_rows(const T* part, long long n, int W, T* out, cudaStream_t st) {
    reduce_rows_kernel<T><<<(W + 127) / 128, 128, 0, st>>>(part, n, W, out);
    BM_CHECK_LAUNCH();
    return 0;
}
template int reduce_rows<float>(const float*, long long, int, float*, cudaStream_t);
template int reduce_rows<double>(const double*, long long, int, double*, cudaStream_t);

int colsum(const float* X, long long rows, int C, int ld, float* part, float* out, cudaStream_t st) {
    dim3 grid((unsigned)blocks_of(rows, COLSUM_RPB), (C + 127) / 128);
    if (ld == C) colsum_cl_kernel<true><<<grid, 128, 0, st>>>(X, part, rows, C, COLSUM_RPB);
    else colsum_strided_kernel<true><<<grid, 128, 0, st>>>(X, part, rows, C, ld, COLSUM_RPB);
    BM_CHECK_LAUNCH();
    return reduce_rows(part, (long long)grid.x, C, out, st);
}
}  // namespace bm

namespace {
// workspaces of the deterministic forms (api.cuh)
constexpr int COLSTATS_RPB = 128;
inline long long colstats_ws_floats(long long rows, int C) { return blocks_of(rows, COLSTATS_RPB) * 4ll * C; }  // fp64 [nb][2C]
inline long long glu_bwd_ws_floats(long long rows, int H) { return blocks_of(rows, CS_ROWS_PER_BLOCK) * 2ll * H; }
inline long long head_ws_floats(int B, int T, int H, int F) {
    return std::max({(long long)B * F, colsum_ws_floats((long long)B * T, 2 * H), planes_floats(B, 2 * H, F),
                     planes_floats(B, 2 * H, H)});
}
}  // namespace

// =================================================================================================
// K3 / K4
// =================================================================================================
extern "C" int bm_conv_weight_prep(const float* w, int Cout, int Cin, int Kw, float* wf, float* wb,
                                   bm_stream_t stream) {
    BM_CHECK_ARG(w && (wf || wb) && Cout > 0 && Cin > 0 && Kw > 0);
    weight_prep_kernel<<<ew_grid((long long)Cout * Cin * Kw), 256, 0, ST(stream)>>>(w, wf, wb, Cout, Cin, Kw);
    BM_CHECK_LAUNCH();
    return 0;
}

static int conv_gemm(const float* x, const float* wmat, const float* bias, const float* addend, int B, int T,
                     int K, int N, int Kw, int dilation, int sign, float* y, double* stats, int glu, float* glu_out,
                     cudaStream_t st) {
    BM_CHECK_ARG(Kw >= 1 && Kw <= 3 && (Kw % 2) == 1);
    GemmP g = gemm_defaults();
    g.M = T; g.N = N; g.K = K; g.kchunk = K; g.taps = Kw;
    g.Z = B; g.nseg = B; g.zchunk = 1;
    g.A = x; g.lda_z = (long long)T * K; g.lda_m = K; g.lda_k = 1;
    for (int j = 0; j < Kw; ++j) g.a_shift_m[j] = sign * (j - Kw / 2) * dilation;
    g.B = wmat; g.ldb_z = 0; g.ldb_tap = (long long)K * N; g.ldb_k = N; g.ldb_n = 1; g.b_ncontig = 1;
    g.D = y; g.ldd_z = (long long)T * N; g.ldd_m = N; g.ldd_n = 1;
    g.bias = bias; g.addend = addend; g.stats = stats;
    if (glu) {
        g.glu = 1; g.glu_out = glu_out;
        g.ldg_z = (long long)T * (N / 2); g.ldg_m = N / 2; g.ldg_n = 1;
    }
    BM_CUDA(launch_gemm(g, st));
    return 0;
}

extern "C" int bm_conv1d_fwd(const float* x, const float* wf, const float* bias, int B, int T, int Cin, int Cout,
                             int Kw, int dilation, float* y, double* stats, bm_stream_t stream) {
    BM_CHECK_ARG(x && wf && y && B > 0 && T > 0 && Cin > 0 && Cout > 0 && dilation >= 1);
    cudaStream_t st = ST(stream);
    if (stats) BM_CUDA(cudaMemsetAsync(stats, 0, sizeof(double) * 2 * Cout, st));
    return conv_gemm(x, wf, bias, nullptr, B, T, Cin, Cout, Kw, dilation, +1, y, stats, 0, nullptr, st);
}

extern "C" int bm_bn_stats_finalize(const double* stats, long long n, float eps, float momentum,
                                    float* running_mean, float* running_var, float* mean, float* invstd, int C,
                                    bm_stream_t stream) {
    BM_CHECK_ARG(stats && mean && invstd && C > 0 && n > 0);
    BM_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr));
    bn_finalize_kernel<<<(C + 127) / 128, 128, 0, ST(stream)>>>(stats, (double)n, eps, momentum, nullptr, running_mean,
                                                               running_var, mean, invstd, C);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_bn_stats_finalize_cumulative(const double* stats, long long n, float eps,
                                               const long long* num_batches_tracked, float* running_mean,
                                               float* running_var, float* mean, float* invstd, int C, bm_stream_t stream) {
    BM_CHECK_ARG(stats && num_batches_tracked && running_mean && running_var && mean && invstd && C > 0 && n > 0);
    bn_finalize_kernel<<<(C + 127) / 128, 128, 0, ST(stream)>>>(stats, (double)n, eps, 0.f, num_batches_tracked,
                                                               running_mean, running_var, mean, invstd, C);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_bn_stats_finalize_counted(const double* stats, float eps, float momentum, float* running_mean,
                                            float* running_var, float* mean, float* invstd, int C, bm_stream_t stream) {
    BM_CHECK_ARG(stats && mean && invstd && C > 0);
    BM_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr));
    bn_finalize_kernel<true><<<(C + 127) / 128, 128, 0, ST(stream)>>>(stats, 0.0, eps, momentum, nullptr, running_mean,
                                                                     running_var, mean, invstd, C);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_bn_stats_finalize_counted_cumulative(const double* stats, float eps, const long long* num_batches_tracked,
                                                       float* running_mean, float* running_var, float* mean, float* invstd,
                                                       int C, bm_stream_t stream) {
    BM_CHECK_ARG(stats && num_batches_tracked && running_mean && running_var && mean && invstd && C > 0);
    bn_finalize_kernel<true><<<(C + 127) / 128, 128, 0, ST(stream)>>>(stats, 0.0, eps, 0.f, num_batches_tracked,
                                                                     running_mean, running_var, mean, invstd, C);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_bn_eval_stats(const float* running_mean, const float* running_var, float eps, float* mean,
                                float* invstd, int C, bm_stream_t stream) {
    BM_CHECK_ARG(running_mean && running_var && mean && invstd && C > 0);
    bn_eval_stats_kernel<<<(C + 127) / 128, 128, 0, ST(stream)>>>(running_mean, running_var, eps, mean, invstd, C);
    BM_CHECK_LAUNCH();
    return 0;
}

// ---- ConvSequence layer epilogue (convseq.cuh): one implementation behind every bm_bn_gelu_skip_*, bm_bn_act_skip_* and
// bm_bn_act_gain_skip_* entry point; the column-stationary or the generic kernels by shape and alignment alone ----------------
struct Epi {
    const float *mean, *invstd, *gamma, *beta;      // mean == NULL: no BatchNorm
    int act;
    float slope;
    const float *scale = nullptr, *post = nullptr;  // residual gains, NULL = 1
    float boost = 0.f;
    bool gain_grads = false;                        // dscale / dpost asked for: S is summed even when both gains are NULL
    bool bn() const { return mean != nullptr; }
    bool gain() const { return scale || post || gain_grads; }
    int width(int C) const { return (gain() ? 3 : 2) * C; }   // fp64 sums: (sum dz, sum dz*yhat[, S = sum g*branch])
};

// C % 4 == 0 and every operand the call touches 16-byte aligned: the column-stationary kernels up to C / 4 <= 256, above it
// the float4 form (VEC = 4) of the generic ones
static bool epi_vec(const Epi& e, int C, std::initializer_list<const void*> ops) {
    uintptr_t bits = reinterpret_cast<uintptr_t>(e.mean) | reinterpret_cast<uintptr_t>(e.invstd) |
                     reinterpret_cast<uintptr_t>(e.gamma) | reinterpret_cast<uintptr_t>(e.beta) |
                     reinterpret_cast<uintptr_t>(e.scale) | reinterpret_cast<uintptr_t>(e.post);
    for (const void* p : ops) bits |= reinterpret_cast<uintptr_t>(p);
    return C % 4 == 0 && (bits & 15) == 0;
}
static bool epi_cs(const Epi& e, int C, std::initializer_list<const void*> ops) { return epi_vec(e, C, ops) && C / 4 <= 256; }
static dim3 epi_cs_block(int C) { return dim3(C / 4, std::max(1, 320 / (C / 4))); }

// f(ACT, BN, GAIN) with the epilogue's form as std::integral_constant arguments: the kernels' instantiation
template <class F>
static void epi_form(const Epi& e, F&& f) {
    auto with = [&](auto act) {
        using T = std::true_type;
        using N = std::false_type;
        if (e.bn()) e.gain() ? f(act, T{}, T{}) : f(act, T{}, N{});
        else e.gain() ? f(act, N{}, T{}) : f(act, N{}, N{});
    };
    if (e.act == ACT_GELU) with(std::integral_constant<int, ACT_GELU>{});
    else if (e.act == ACT_LRELU) with(std::integral_constant<int, ACT_LRELU>{});
    else with(std::integral_constant<int, ACT_NONE>{});
}
#define EPI_T(A, B, G) decltype(A)::value, decltype(B)::value, decltype(G)::value

static int epi_fwd(const float* y, const Epi& e, const float* x_old, float* x_new, long long rows, int C, float* amax_out,
                   cudaStream_t st) {
    BM_CHECK_ARG(y && x_new && rows > 0 && C > 0 && e.act >= 0 && e.act <= 2);
    BM_CHECK_ARG(!e.mean || (e.invstd && e.gamma && e.beta));
    if (int rc = amax_begin(amax_out, st)) return rc;
    const bool vec = epi_vec(e, C, {y, x_old, x_new}), cs = vec && C / 4 <= 256;
    epi_form(e, [&](auto A, auto B, auto G) {
        if (cs)
            epi_fwd_cs_kernel<EPI_T(A, B, G)><<<(unsigned)blocks_of(rows, CS_ROWS_PER_BLOCK), epi_cs_block(C), 0, st>>>(
                y, e.mean, e.invstd, e.gamma, e.beta, x_old, x_new, rows, C, reinterpret_cast<unsigned int*>(amax_out), e.slope,
                e.scale, e.boost, e.post);
        else if (vec)
            epi_fwd_kernel<EPI_T(A, B, G), 4><<<ew_grid(rows * C, 256, 4), 256, 0, st>>>(
                y, e.mean, e.invstd, e.gamma, e.beta, x_old, x_new, rows * C, C, e.slope, e.scale, e.boost, e.post);
        else
            epi_fwd_kernel<EPI_T(A, B, G), 1><<<ew_grid(rows * C), 256, 0, st>>>(
                y, e.mean, e.invstd, e.gamma, e.beta, x_old, x_new, rows * C, C, e.slope, e.scale, e.boost, e.post);
    });
    BM_CHECK_LAUNCH();
    if (amax_out && !cs) return tc::launch_amax(x_new, rows * C, amax_out, st);
    return 0;
}

// The backward in its two halves, which a SyncBatchNorm caller runs as two calls with the all-reduce of the sums between them
// (the _reduce / _apply entry points); epi_bwd runs them back to back.
// reduce half: sums [e.width(C)] over the call's rows, then the parameter gradients (each nullable) from them.
// part: NULL (fp64 atomics into sums, zeroed here) or the epi_ws_floats partials of the deterministic form: fp64 [nb][W], nb
// the block count of the column-stationary kernel (CS_ROWS_PER_BLOCK = 96 rows per block; the generic one takes 128)
inline long long epi_ws_floats(long long rows, int W) { return blocks_of(rows, CS_ROWS_PER_BLOCK) * 2ll * W; }
static int epi_bwd_reduce(const float* g, const float* y, const Epi& e, long long rows, int C, bool cs, double* sums,
                          float* dgamma, float* dbeta, float* dscale, float* dpost, double* part, cudaStream_t st) {
    const int W = e.width(C);
    if (!part) BM_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * W, st));
    double* out = part ? part : sums;
    const int rpb = cs ? CS_ROWS_PER_BLOCK : 128;   // the generic kernel: one thread per column, 128 rows per block
    const long long nblk = blocks_of(rows, rpb);
    epi_form(e, [&](auto A, auto B, auto G) {
        if constexpr (decltype(B)::value || decltype(G)::value) {   // without either there is nothing to reduce
            if (cs) {
                const dim3 block = epi_cs_block(C);
                auto* kernel = part ? epi_bwd_reduce_cs_kernel<EPI_T(A, B, G), true> : epi_bwd_reduce_cs_kernel<EPI_T(A, B, G)>;
                kernel<<<(unsigned)nblk, block, sizeof(float) * W * block.y, st>>>(g, y, e.mean, e.invstd, e.gamma, e.beta, out,
                                                                                 rows, C, e.slope, e.scale, e.boost, e.post);
            } else {
                auto* kernel = part ? epi_bwd_reduce_kernel<EPI_T(A, B, G), true> : epi_bwd_reduce_kernel<EPI_T(A, B, G)>;
                kernel<<<dim3((unsigned)nblk, (C + 127) / 128), 128, 0, st>>>(g, y, e.mean, e.invstd, e.gamma, e.beta, out,
                                                                             rows, C, rpb, e.slope, e.scale, e.boost, e.post);
            }
        }
    });
    BM_CHECK_LAUNCH();
    if (part)
        if (int rc = reduce_rows(part, nblk, W, sums, st)) return rc;
    epi_param_grad_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums, C, e.scale, e.boost, e.post, dgamma, dbeta, dscale, dpost);
    BM_CHECK_LAUNCH();
    return 0;
}

// apply half: dy.  counted: the sums and the row count n come from `sums` [2C + 1] (n in sums[2C], read on the device);
// else n = rows and the column-stationary kernel takes the sums as dgamma / dbeta.  Both give the same bits for the same n.
static int epi_bwd_apply(const float* g, const float* y, const Epi& e, int batch_stats, long long rows, int C, bool cs,
                         bool vec, const double* sums, const float* dgamma, const float* dbeta, bool counted, float* dy, float* amax_out,
                         cudaStream_t st) {
    const long long total = rows * C;
    const float rn = (float)(1.0 / (double)rows);
    unsigned int* amax = reinterpret_cast<unsigned int*>(amax_out);
    epi_form(e, [&](auto A, auto B, auto G) {
        const unsigned nblk = (unsigned)blocks_of(rows, CS_ROWS_PER_BLOCK);
        if (counted) {   // the SyncBatchNorm apply half: a BatchNorm and no gain (epi_bwd_apply_half)
            if constexpr (decltype(B)::value && !decltype(G)::value) {
                if (cs)
                    epi_bwd_apply_cs_kernel<EPI_T(A, B, G), true><<<nblk, epi_cs_block(C), 0, st>>>(
                        g, y, e.mean, e.invstd, e.gamma, e.beta, nullptr, nullptr, sums, 0.f, 1, dy, rows, C, amax, e.slope,
                        e.scale, e.boost, e.post);
                else if (vec)
                    epi_bwd_apply_kernel<EPI_T(A, B, G), 4, true><<<ew_grid(total, 256, 4), 256, 0, st>>>(
                        g, y, e.mean, e.invstd, e.gamma, e.beta, sums, 0.0, 1, dy, total, C, e.slope, e.scale, e.boost, e.post);
                else
                    epi_bwd_apply_kernel<EPI_T(A, B, G), 1, true><<<ew_grid(total), 256, 0, st>>>(
                        g, y, e.mean, e.invstd, e.gamma, e.beta, sums, 0.0, 1, dy, total, C, e.slope, e.scale, e.boost, e.post);
            }
        } else if (cs) {
            epi_bwd_apply_cs_kernel<EPI_T(A, B, G)><<<nblk, epi_cs_block(C), 0, st>>>(
                g, y, e.mean, e.invstd, e.gamma, e.beta, dgamma, dbeta, nullptr, rn, batch_stats, dy, rows, C, amax, e.slope,
                e.scale, e.boost, e.post);
        } else if (vec) {
            epi_bwd_apply_kernel<EPI_T(A, B, G), 4><<<ew_grid(total, 256, 4), 256, 0, st>>>(
                g, y, e.mean, e.invstd, e.gamma, e.beta, sums, (double)rows, batch_stats, dy, total, C, e.slope, e.scale, e.boost,
                e.post);
        } else {
            epi_bwd_apply_kernel<EPI_T(A, B, G), 1><<<ew_grid(total), 256, 0, st>>>(
                g, y, e.mean, e.invstd, e.gamma, e.beta, sums, (double)rows, batch_stats, dy, total, C, e.slope, e.scale, e.boost,
                e.post);
        }
    });
    BM_CHECK_LAUNCH();
    if (amax_out && !cs) return tc::launch_amax(dy, total, amax_out, st);
    return 0;
}

// The BatchNorm sums are reduced unless batch_stats == 0 and dgamma == dbeta == NULL: the data gradient of an eval-mode
// BatchNorm whose affine parameters are frozen is then one elementwise pass (the apply kernels read the sums / dgamma / dbeta
// only when use_batch_stats is set, so its dy is bitwise the reducing form's).  The gains' S is reduced for dscale / dpost.
static bool epi_bn_reduces(const Epi& e, int batch_stats, const float* dgamma, const float* dbeta) {
    return e.bn() && (batch_stats || dgamma || dbeta);
}

// part: NULL (fp64 atomics into sums) or the epi_ws_floats partials of the deterministic form
static int epi_bwd(const float* g, const float* y, const Epi& e, int batch_stats, long long rows, int C, double* sums,
                   float* dy, float* dgamma, float* dbeta, float* dscale, float* dpost, float* amax_out, double* part,
                   cudaStream_t st) {
    BM_CHECK_ARG(g && y && dy && rows > 0 && C > 0 && e.act >= 0 && e.act <= 2);
    BM_CHECK_ARG(!e.mean || (e.invstd && e.gamma && e.beta));
    const bool bn_reduce = epi_bn_reduces(e, batch_stats, dgamma, dbeta);
    BM_CHECK_ARG(!bn_reduce || (dgamma && dbeta));
    const bool reduce = bn_reduce || dscale || dpost;
    BM_CHECK_ARG(!reduce || sums);
    if (int rc = amax_begin(amax_out, st)) return rc;
    const bool vec = epi_vec(e, C, {g, y, dy, dgamma, dbeta}), cs = vec && C / 4 <= 256;
    if (reduce)
        if (int rc = epi_bwd_reduce(g, y, e, rows, C, cs, sums, bn_reduce ? dgamma : nullptr, bn_reduce ? dbeta : nullptr,
                                    dscale, dpost, part, st))
            return rc;
    return epi_bwd_apply(g, y, e, bn_reduce && batch_stats, rows, C, cs, vec, sums, dgamma, dbeta, false, dy, amax_out, st);
}

// the deterministic form: the workspace is used (and checked) only when something is reduced
static int epi_bwd_det(const float* g, const float* y, const Epi& e, int batch_stats, long long rows, int C, double* sums,
                       float* dy, float* dgamma, float* dbeta, float* dscale, float* dpost, float* amax_out, float* workspace,
                       long long workspace_floats, cudaStream_t st) {
    BM_CHECK_ARG(rows > 0 && C > 0);
    double* part = nullptr;
    if (epi_bn_reduces(e, batch_stats, dgamma, dbeta) || dscale || dpost) {
        BM_CHECK_WS(epi_ws_floats(rows, e.width(C)));
        part = reinterpret_cast<double*>(workspace);
    }
    return epi_bwd(g, y, e, batch_stats, rows, C, sums, dy, dgamma, dbeta, dscale, dpost, amax_out, part, st);
}

// SyncBatchNorm halves of epi_bwd with a training-mode BatchNorm and no gain (the kernel choice is epi_bwd's, so the pair
// gives its bits for the same sums and n)
static int epi_bwd_reduce_half(const float* g, const float* y, const Epi& e, long long rows, int C, double* sums, float* dgamma,
                               float* dbeta, double* part, cudaStream_t st) {
    BM_CHECK_ARG(g && y && e.mean && e.invstd && e.gamma && e.beta && sums && dgamma && dbeta && rows > 0 && C > 0 &&
                 e.act >= 0 && e.act <= 2);
    return epi_bwd_reduce(g, y, e, rows, C, epi_cs(e, C, {g, y, dgamma, dbeta}), sums, dgamma, dbeta, nullptr, nullptr, part,
                          st);
}
static int epi_bwd_reduce_half_det(const float* g, const float* y, const Epi& e, long long rows, int C, double* sums,
                                   float* dgamma, float* dbeta, float* workspace, long long workspace_floats, cudaStream_t st) {
    BM_CHECK_ARG(rows > 0 && C > 0);
    BM_CHECK_WS(epi_ws_floats(rows, 2 * C));
    return epi_bwd_reduce_half(g, y, e, rows, C, sums, dgamma, dbeta, reinterpret_cast<double*>(workspace), st);
}
static int epi_bwd_apply_half(const float* g, const float* y, const Epi& e, long long rows, int C, const double* sums,
                              float* dy, cudaStream_t st) {
    BM_CHECK_ARG(g && y && e.mean && e.invstd && e.gamma && e.beta && sums && dy && rows > 0 && C > 0 && e.act >= 0 &&
                 e.act <= 2);
    const bool vec = epi_vec(e, C, {g, y, dy});
    return epi_bwd_apply(g, y, e, 1, rows, C, vec && C / 4 <= 256, vec, sums, nullptr, nullptr, true, dy, nullptr, st);
}

// BatchNorm + GELU (SimpleConv's layers): the BatchNorm is required
extern "C" int bm_bn_gelu_skip_fwd(const float* y, const float* mean, const float* invstd, const float* gamma,
                                   const float* beta, const float* x_old, float* x_new, long long rows, int C,
                                   float* amax_out, bm_stream_t stream) {
    BM_CHECK_ARG(mean);
    const Epi e{mean, invstd, gamma, beta, ACT_GELU, 0.f};
    return epi_fwd(y, e, x_old, x_new, rows, C, amax_out, ST(stream));
}
extern "C" int bm_bn_gelu_skip_bwd(const float* g, const float* y, const float* mean, const float* invstd,
                                   const float* gamma, const float* beta, int batch_stats, long long rows, int C,
                                   double* sums, float* dy, float* dgamma, float* dbeta, float* amax_out,
                                   bm_stream_t stream) {
    BM_CHECK_ARG(mean);
    const Epi e{mean, invstd, gamma, beta, ACT_GELU, 0.f};
    return epi_bwd(g, y, e, batch_stats, rows, C, sums, dy, dgamma, dbeta, nullptr, nullptr, amax_out, nullptr, ST(stream));
}
extern "C" long long bm_bn_gelu_skip_bwd_det_workspace(long long rows, int C) {
    return rows > 0 && C > 0 ? epi_ws_floats(rows, 2 * C) : 0;
}
extern "C" int bm_bn_gelu_skip_bwd_det(const float* g, const float* y, const float* mean, const float* invstd,
                                       const float* gamma, const float* beta, int batch_stats, long long rows, int C,
                                       double* sums, float* dy, float* dgamma, float* dbeta, float* amax_out,
                                       float* workspace, long long workspace_floats, bm_stream_t stream) {
    BM_CHECK_ARG(mean);
    const Epi e{mean, invstd, gamma, beta, ACT_GELU, 0.f};
    return epi_bwd_det(g, y, e, batch_stats, rows, C, sums, dy, dgamma, dbeta, nullptr, nullptr, amax_out, workspace,
                       workspace_floats, ST(stream));
}
extern "C" int bm_bn_gelu_skip_bwd_reduce(const float* g, const float* y, const float* mean, const float* invstd,
                                          const float* gamma, const float* beta, long long rows, int C, double* sums,
                                          float* dgamma, float* dbeta, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, ACT_GELU, 0.f};
    return epi_bwd_reduce_half(g, y, e, rows, C, sums, dgamma, dbeta, nullptr, ST(stream));
}
extern "C" long long bm_bn_gelu_skip_bwd_reduce_det_workspace(long long rows, int C) {
    return rows > 0 && C > 0 ? epi_ws_floats(rows, 2 * C) : 0;
}
extern "C" int bm_bn_gelu_skip_bwd_reduce_det(const float* g, const float* y, const float* mean, const float* invstd,
                                              const float* gamma, const float* beta, long long rows, int C, double* sums,
                                              float* dgamma, float* dbeta, float* workspace, long long workspace_floats,
                                              bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, ACT_GELU, 0.f};
    return epi_bwd_reduce_half_det(g, y, e, rows, C, sums, dgamma, dbeta, workspace, workspace_floats, ST(stream));
}
extern "C" int bm_bn_gelu_skip_bwd_apply(const float* g, const float* y, const float* mean, const float* invstd,
                                         const float* gamma, const float* beta, long long rows, int C, const double* sums,
                                         float* dy, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, ACT_GELU, 0.f};
    return epi_bwd_apply_half(g, y, e, rows, C, sums, dy, ST(stream));
}

extern "C" int bm_conv1d_bwd_data(const float* dy, const float* wb, const float* addend, int B, int T, int Cin,
                                  int Cout, int Kw, int dilation, float* dx, bm_stream_t stream) {
    BM_CHECK_ARG(dy && wb && dx && B > 0 && T > 0 && Cin > 0 && Cout > 0 && dilation >= 1);
    return conv_gemm(dy, wb, nullptr, addend, B, T, Cout, Cin, Kw, dilation, -1, dx, nullptr, 0, nullptr,
                     ST(stream));
}

// part: NULL (atomic reductions) or the colsum_ws_floats(B*T, Cout) partials of the deterministic form
static int conv1d_bwd_weight(const float* dy, const float* x, int B, int T, int Cin, int Cout, int Kw, int dilation, float* dw,
                             float* dbias, float* part, cudaStream_t st) {
    BM_CHECK_ARG(dy && x && dw && B > 0 && T > 0 && Cin > 0 && Cout > 0 && Kw >= 1 && Kw <= 3);
    if (!part) BM_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)Cout * Cin * Kw, st));
    int nseg = pick_chunks(B, tiles_of(Cout, Cin) * Kw);
    int zchunk = (B + nseg - 1) / nseg;
    nseg = (B + zchunk - 1) / zchunk;
    for (int j = 0; j < Kw; ++j) {
        GemmP g = gemm_defaults();
        g.M = Cout; g.N = Cin; g.K = T; g.kchunk = T;
        g.Z = B; g.nseg = nseg; g.zchunk = zchunk;
        g.A = dy; g.lda_z = (long long)T * Cout; g.lda_m = 1; g.lda_k = Cout; g.a_mcontig = 1;
        g.B = x; g.ldb_z = (long long)T * Cin; g.ldb_n = 1; g.ldb_k = Cin; g.b_ncontig = 1;
        g.b_shift_k[0] = (j - Kw / 2) * dilation;
        g.D = dw + j; g.ldd_z = 0; g.ldd_m = (long long)Cin * Kw; g.ldd_n = Kw; g.atomic = 1;
        if (part) BM_CUDA(launch_gemm_planes(g, dw, (long long)Cout * Cin * Kw, part, st));
        else BM_CUDA(launch_gemm(g, st));
    }
    if (part) {                                     // every tap's planes are written: sum them, then the bias (reusing part)
        if (int rc = sum_planes(part, nseg, (long long)Cout * Cin * Kw, dw, st)) return rc;
        return dbias ? colsum(dy, (long long)B * T, Cout, Cout, part, dbias, st) : 0;
    }
    if (dbias) {
        BM_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float) * Cout, st));
        long long rows = (long long)B * T;
        dim3 grid((unsigned)((rows + 255) / 256), (Cout + 127) / 128);
        colsum_cl_kernel<<<grid, 128, 0, st>>>(dy, dbias, rows, Cout, 256);
        BM_CHECK_LAUNCH();
    }
    return 0;
}

extern "C" int bm_conv1d_bwd_weight(const float* dy, const float* x, int B, int T, int Cin, int Cout, int Kw,
                                    int dilation, float* dw, float* dbias, bm_stream_t stream) {
    return conv1d_bwd_weight(dy, x, B, T, Cin, Cout, Kw, dilation, dw, dbias, nullptr, ST(stream));
}
extern "C" long long bm_conv1d_bwd_weight_det_workspace(int B, int T, int Cin, int Cout, int Kw) {
    if (B <= 0 || T <= 0 || Cin <= 0 || Cout <= 0 || Kw <= 0) return 0;
    return std::max(colsum_ws_floats((long long)B * T, Cout), planes_floats(B, Cout, Cin, Kw));
}
extern "C" int bm_conv1d_bwd_weight_det(const float* dy, const float* x, int B, int T, int Cin, int Cout, int Kw,
                                        int dilation, float* dw, float* dbias, float* workspace, long long workspace_floats,
                                        bm_stream_t stream) {
    BM_CHECK_ARG(B > 0 && T > 0 && Cin > 0 && Cout > 0 && Kw >= 1 && Kw <= 3);
    BM_CHECK_WS(bm_conv1d_bwd_weight_det_workspace(B, T, Cin, Cout, Kw));
    return conv1d_bwd_weight(dy, x, B, T, Cin, Cout, Kw, dilation, dw, dbias, workspace, ST(stream));
}

extern "C" int bm_conv1d_glu_fwd(const float* x, const float* wf, const float* bias, int B, int T, int Cin, int H,
                                 int Kw, float* h, float* out, bm_stream_t stream) {
    BM_CHECK_ARG(x && wf && out && B > 0 && T > 0 && Cin > 0 && H > 0);
    return conv_gemm(x, wf, bias, nullptr, B, T, Cin, 2 * H, Kw, 1, +1, h, nullptr, 1, out, ST(stream));
}

// part: NULL (atomic reductions) or the glu_bwd_ws_floats(rows, H) partials of the deterministic form
static int glu_bwd(const float* g, const float* h, long long rows, int H, float* dh, float* dbias, float* amax_out, float* part,
                   cudaStream_t st) {
    BM_CHECK_ARG(g && h && dh && rows > 0 && H > 0);
    if (dbias && !part) BM_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float) * 2 * H, st));
    if (int rc = amax_begin(amax_out, st)) return rc;
    if (H % 4 == 0 && H / 4 <= 256 && aligned16(g, h, dh)) {
        const int cx = H / 4, ry = std::max(1, 320 / cx);
        const unsigned nblk = (unsigned)((rows + CS_ROWS_PER_BLOCK - 1) / CS_ROWS_PER_BLOCK);
        if (dbias && part) {
            glu_bwd_cs_kernel<true><<<nblk, dim3(cx, ry), sizeof(float) * 2 * H * ry, st>>>(
                g, h, dh, part, rows, H, reinterpret_cast<unsigned int*>(amax_out));
            BM_CHECK_LAUNCH();
            return reduce_rows(part, (long long)nblk, 2 * H, dbias, st);
        }
        glu_bwd_cs_kernel<<<nblk, dim3(cx, ry), dbias ? sizeof(float) * 2 * H * ry : 0, st>>>(
            g, h, dh, dbias, rows, H, reinterpret_cast<unsigned int*>(amax_out));
        BM_CHECK_LAUNCH();
        return 0;
    }
    if (H % 4 == 0 && aligned16(g, h, dh))
        glu_bwd_v4_kernel<<<ew_grid(rows * H / 4), 256, 0, st>>>(
            reinterpret_cast<const float4*>(g), reinterpret_cast<const float4*>(h), reinterpret_cast<float4*>(dh), rows, H);
    else
        glu_bwd_kernel<<<ew_grid(rows * H), 256, 0, st>>>(g, h, dh, rows, H);
    BM_CHECK_LAUNCH();
    if (dbias && part) {
        if (int rc = colsum(dh, rows, 2 * H, 2 * H, part, dbias, st)) return rc;
    } else if (dbias) {
        dim3 grid((unsigned)((rows + 255) / 256), (2 * H + 127) / 128);
        colsum_cl_kernel<<<grid, 128, 0, st>>>(dh, dbias, rows, 2 * H, 256);
        BM_CHECK_LAUNCH();
    }
    if (amax_out) return tc::launch_amax(dh, rows * 2 * H, amax_out, st);
    return 0;
}

extern "C" int bm_glu_bwd(const float* g, const float* h, long long rows, int H, float* dh, float* dbias,
                          float* amax_out, bm_stream_t stream) {
    return glu_bwd(g, h, rows, H, dh, dbias, amax_out, nullptr, ST(stream));
}
extern "C" long long bm_glu_bwd_det_workspace(long long rows, int H) {
    // the column-stationary kernel's partial rows, or the colsum's for the generic kernels (fewer rows of 2H)
    return rows > 0 && H > 0 ? glu_bwd_ws_floats(rows, H) : 0;
}
extern "C" int bm_glu_bwd_det(const float* g, const float* h, long long rows, int H, float* dh, float* dbias,
                              float* amax_out, float* workspace, long long workspace_floats, bm_stream_t stream) {
    BM_CHECK_ARG(rows > 0 && H > 0);
    if (!dbias)                                  // no bias gradient: nothing is reduced, the workspace is not used
        return glu_bwd(g, h, rows, H, dh, nullptr, amax_out, nullptr, ST(stream));
    BM_CHECK_WS(glu_bwd_ws_floats(rows, H));
    return glu_bwd(g, h, rows, H, dh, dbias, amax_out, workspace, ST(stream));
}

// =================================================================================================
// K5
// =================================================================================================
extern "C" int bm_head_fwd(const float* x, const float* w0, const float* b0, const float* w2, const float* b2,
                           int B, int T, int H, int F, float* h1, float* q, float* est, bm_stream_t stream) {
    BM_CHECK_ARG(x && w0 && b0 && w2 && b2 && q && est && B > 0 && T > 0 && H > 0 && F > 0);
    cudaStream_t st = ST(stream);
    const int H2 = 2 * H;
    {   // h1 = x w0^T + b0 ; q = GELU(h1)
        GemmP g = gemm_defaults();
        g.M = B * T; g.N = H2; g.K = H; g.kchunk = H;
        g.A = x; g.lda_m = H; g.lda_k = 1;
        g.B = w0; g.ldb_n = H; g.ldb_k = 1;
        g.D = q; g.ldd_m = H2; g.ldd_n = 1;
        g.bias = b0; g.aux = h1; g.act = 1;
        BM_CUDA(launch_gemm(g, st));
    }
    {   // est[b][f][t] = b2[f] + sum_i q[b][t][i] w2[i][f]
        GemmP g = gemm_defaults();
        g.M = T; g.N = F; g.K = H2; g.kchunk = H2;
        g.Z = B; g.nseg = B; g.zchunk = 1;
        g.A = q; g.lda_z = (long long)T * H2; g.lda_m = H2; g.lda_k = 1;
        g.B = w2; g.ldb_n = 1; g.ldb_k = F; g.b_ncontig = 1;
        g.D = est; g.ldd_z = (long long)F * T; g.ldd_m = 1; g.ldd_n = T;
        g.bias = b2;
        BM_CUDA(launch_gemm(g, st));
    }
    return 0;
}

// dW2, db2, dh1 = dq*GELU'(h1) (in place in dq), dW0, db0 -- the parameter-gradient half of the head backward
// part: NULL (atomic reductions) or the head_ws_floats(B, T, H, F) partials of the deterministic form.  Each of dw0, db0, dw2,
// db2 may be NULL (a frozen parameter): its GEMM / reduction is skipped.  want_dh1 = 0: dq is not turned into dh1 (nothing
// reads it: the caller wants neither dx nor dw0 / db0).
static int head_bwd_params(const float* dest, const float* x, const float* h1, const float* q, int B, int T, int H, int F,
                           float* dq, float* dw0, float* db0, float* dw2, float* db2, float* part, cudaStream_t st,
                           bool want_dh1 = true) {
    BM_CHECK_ARG(dest && (!want_dh1 || (h1 && dq)) && (!dw0 || x) && (!dw2 || q));
    BM_CHECK_ARG(want_dh1 || (!dw0 && !db0));
    const int H2 = 2 * H;
    const long long rows = (long long)B * T;
    if (dw2) {   // dw2[i][f] = sum_{b,t} q[b][t][i] dest[b][f][t]
        GemmP g = gemm_defaults();
        g.M = H2; g.N = F; g.K = T; g.kchunk = T;
        g.Z = B; g.nseg = pick_chunks(B, tiles_of(H2, F)); g.zchunk = (B + g.nseg - 1) / g.nseg;
        g.nseg = (B + g.zchunk - 1) / g.zchunk;
        g.A = q; g.lda_z = (long long)T * H2; g.lda_m = 1; g.lda_k = H2; g.a_mcontig = 1;
        g.B = dest; g.ldb_z = (long long)F * T; g.ldb_n = T; g.ldb_k = 1; g.b_ncontig = 0;
        g.D = dw2; g.ldd_m = F; g.ldd_n = 1; g.atomic = 1;
        if (part) {
            BM_CUDA(launch_gemm_planes(g, dw2, (long long)H2 * F, part, st));
            if (int rc = sum_planes(part, g.nseg, (long long)H2 * F, dw2, st)) return rc;
        } else {
            BM_CUDA(cudaMemsetAsync(dw2, 0, sizeof(float) * (size_t)H2 * F, st));
            BM_CUDA(launch_gemm(g, st));
        }
    }
    if (db2) {   // db2[f] = sum_{b,t} dest[b][f][t]
        long long nrows = (long long)B * F;
        if (part) {
            rowsum_cm_kernel<true><<<(unsigned)((nrows + 7) / 8), 256, 0, st>>>(dest, part, B, F, T);
            BM_CHECK_LAUNCH();
            if (int rc = reduce_rows(part, (long long)B, F, db2, st)) return rc;
        } else {
            BM_CUDA(cudaMemsetAsync(db2, 0, sizeof(float) * F, st));
            rowsum_cm_kernel<<<(unsigned)((nrows + 7) / 8), 256, 0, st>>>(dest, db2, B, F, T);
            BM_CHECK_LAUNCH();
        }
    }
    if (!want_dh1) return 0;
    gelu_bwd_kernel<<<ew_grid(rows * H2), 256, 0, st>>>(dq, h1, dq, rows * H2);   // dq <- dh1
    BM_CHECK_LAUNCH();
    if (dw0) {   // dw0[n][k] = sum_rows dh1[row][n] x[row][k]
        GemmP g = gemm_defaults();
        g.M = H2; g.N = H; g.K = T; g.kchunk = T;
        g.Z = B; g.nseg = pick_chunks(B, tiles_of(H2, H)); g.zchunk = (B + g.nseg - 1) / g.nseg;
        g.nseg = (B + g.zchunk - 1) / g.zchunk;
        g.A = dq; g.lda_z = (long long)T * H2; g.lda_m = 1; g.lda_k = H2; g.a_mcontig = 1;
        g.B = x; g.ldb_z = (long long)T * H; g.ldb_n = 1; g.ldb_k = H; g.b_ncontig = 1;
        g.D = dw0; g.ldd_m = H; g.ldd_n = 1; g.atomic = 1;
        if (part) {
            BM_CUDA(launch_gemm_planes(g, dw0, (long long)H2 * H, part, st));
            if (int rc = sum_planes(part, g.nseg, (long long)H2 * H, dw0, st)) return rc;
        } else {
            BM_CUDA(cudaMemsetAsync(dw0, 0, sizeof(float) * (size_t)H2 * H, st));
            BM_CUDA(launch_gemm(g, st));
        }
    }
    if (!db0) return 0;
    if (part) return colsum(dq, rows, H2, H2, part, db0, st);   // db0; the partials buffer is reused stage after stage
    {   // db0
        BM_CUDA(cudaMemsetAsync(db0, 0, sizeof(float) * H2, st));
        dim3 grid((unsigned)((rows + 255) / 256), (H2 + 127) / 128);
        colsum_cl_kernel<<<grid, 128, 0, st>>>(dq, db0, rows, H2, 256);
        BM_CHECK_LAUNCH();
    }
    return 0;
}

extern "C" int bm_head_bwd_params(const float* dest, const float* x, const float* h1, const float* q, int B, int T,
                                  int H, int F, float* dq, float* dw0, float* db0, float* dw2, float* db2,
                                  bm_stream_t stream) {
    return head_bwd_params(dest, x, h1, q, B, T, H, F, dq, dw0, db0, dw2, db2, nullptr, ST(stream));
}
extern "C" long long bm_head_bwd_params_det_workspace(int B, int T, int H, int F) {
    return B > 0 && T > 0 && H > 0 && F > 0 ? head_ws_floats(B, T, H, F) : 0;
}
extern "C" int bm_head_bwd_params_det(const float* dest, const float* x, const float* h1, const float* q, int B, int T,
                                      int H, int F, float* dq, float* dw0, float* db0, float* dw2, float* db2,
                                      float* workspace, long long workspace_floats, bm_stream_t stream) {
    BM_CHECK_ARG(B > 0 && T > 0 && H > 0 && F > 0);
    if (dw0 || db0 || dw2 || db2) BM_CHECK_WS(head_ws_floats(B, T, H, F));
    return head_bwd_params(dest, x, h1, q, B, T, H, F, dq, dw0, db0, dw2, db2, workspace, ST(stream));
}

static int head_bwd(const float* dest, const float* x, const float* w0, const float* w2, const float* h1, const float* q, int B,
                    int T, int H, int F, float* dq, float* dx, float* dw0, float* db0, float* dw2, float* db2, float* part,
                    cudaStream_t st) {
    const bool want_dh1 = dx || dw0 || db0;       // else only dw2 / db2 (or nothing) is asked for: no dq, no GELU'
    BM_CHECK_ARG(dest && (!want_dh1 || (w2 && h1 && dq)) && (!dx || w0));
    const int H2 = 2 * H;
    const long long rows = (long long)B * T;
    if (want_dh1) {   // dq[b][t][i] = sum_f dest[b][f][t] w2[i][f]
        GemmP g = gemm_defaults();
        g.M = T; g.N = H2; g.K = F; g.kchunk = F;
        g.Z = B; g.nseg = B; g.zchunk = 1;
        g.A = dest; g.lda_z = (long long)F * T; g.lda_m = 1; g.lda_k = T; g.a_mcontig = 1;
        g.B = w2; g.ldb_n = F; g.ldb_k = 1;
        g.D = dq; g.ldd_z = (long long)T * H2; g.ldd_m = H2; g.ldd_n = 1;
        BM_CUDA(launch_gemm(g, st));
    }
    int rc = head_bwd_params(dest, x, h1, q, B, T, H, F, dq, dw0, db0, dw2, db2, part, st, want_dh1);
    if (rc) return rc;
    if (dx) {   // dx[row][k] = sum_n dh1[row][n] w0[n][k]
        GemmP g = gemm_defaults();
        g.M = (int)rows; g.N = H; g.K = H2; g.kchunk = H2;
        g.A = dq; g.lda_m = H2; g.lda_k = 1;
        g.B = w0; g.ldb_n = 1; g.ldb_k = H; g.b_ncontig = 1;
        g.D = dx; g.ldd_m = H; g.ldd_n = 1;
        BM_CUDA(launch_gemm(g, st));
    }
    return 0;
}

extern "C" int bm_head_bwd(const float* dest, const float* x, const float* w0, const float* w2, const float* h1,
                           const float* q, int B, int T, int H, int F, float* dq, float* dx, float* dw0,
                           float* db0, float* dw2, float* db2, bm_stream_t stream) {
    return head_bwd(dest, x, w0, w2, h1, q, B, T, H, F, dq, dx, dw0, db0, dw2, db2, nullptr, ST(stream));
}
extern "C" long long bm_head_bwd_det_workspace(int B, int T, int H, int F) {
    return bm_head_bwd_params_det_workspace(B, T, H, F);
}
extern "C" int bm_head_bwd_det(const float* dest, const float* x, const float* w0, const float* w2, const float* h1,
                               const float* q, int B, int T, int H, int F, float* dq, float* dx, float* dw0,
                               float* db0, float* dw2, float* db2, float* workspace, long long workspace_floats,
                               bm_stream_t stream) {
    BM_CHECK_ARG(B > 0 && T > 0 && H > 0 && F > 0);
    if (dw0 || db0 || dw2 || db2) BM_CHECK_WS(head_ws_floats(B, T, H, F));
    return head_bwd(dest, x, w0, w2, h1, q, B, T, H, F, dq, dx, dw0, db0, dw2, db2, workspace, ST(stream));
}

// =================================================================================================
// Stand-alone ConvSequence epilogues (the forms of epi_fwd / epi_bwd above)
// =================================================================================================
// any activation, BatchNorm optional (mean == NULL), with or without the residual gains
extern "C" int bm_bn_act_skip_fwd(const float* y, const float* mean, const float* invstd, const float* gamma,
                                  const float* beta, const float* x_old, float* x_new, long long rows, int C, int act,
                                  float slope, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope};
    return epi_fwd(y, e, x_old, x_new, rows, C, nullptr, ST(stream));
}
extern "C" int bm_bn_act_skip_bwd(const float* g, const float* y, const float* mean, const float* invstd,
                                  const float* gamma, const float* beta, int batch_stats, long long rows, int C,
                                  int act, float slope, double* sums, float* dy, float* dgamma, float* dbeta,
                                  bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope};
    return epi_bwd(g, y, e, batch_stats, rows, C, sums, dy, dgamma, dbeta, nullptr, nullptr, nullptr, nullptr, ST(stream));
}
extern "C" long long bm_bn_act_skip_bwd_det_workspace(long long rows, int C) {
    return rows > 0 && C > 0 ? epi_ws_floats(rows, 2 * C) : 0;
}
extern "C" int bm_bn_act_skip_bwd_det(const float* g, const float* y, const float* mean, const float* invstd,
                                      const float* gamma, const float* beta, int batch_stats, long long rows, int C,
                                      int act, float slope, double* sums, float* dy, float* dgamma, float* dbeta,
                                      float* workspace, long long workspace_floats, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope};
    return epi_bwd_det(g, y, e, batch_stats, rows, C, sums, dy, dgamma, dbeta, nullptr, nullptr, nullptr, workspace,
                       workspace_floats, ST(stream));
}
extern "C" int bm_bn_act_skip_bwd_reduce(const float* g, const float* y, const float* mean, const float* invstd,
                                         const float* gamma, const float* beta, long long rows, int C, int act, float slope,
                                         double* sums, float* dgamma, float* dbeta, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope};
    return epi_bwd_reduce_half(g, y, e, rows, C, sums, dgamma, dbeta, nullptr, ST(stream));
}
extern "C" long long bm_bn_act_skip_bwd_reduce_det_workspace(long long rows, int C) {
    return rows > 0 && C > 0 ? epi_ws_floats(rows, 2 * C) : 0;
}
extern "C" int bm_bn_act_skip_bwd_reduce_det(const float* g, const float* y, const float* mean, const float* invstd,
                                             const float* gamma, const float* beta, long long rows, int C, int act,
                                             float slope, double* sums, float* dgamma, float* dbeta, float* workspace,
                                             long long workspace_floats, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope};
    return epi_bwd_reduce_half_det(g, y, e, rows, C, sums, dgamma, dbeta, workspace, workspace_floats, ST(stream));
}
extern "C" int bm_bn_act_skip_bwd_apply(const float* g, const float* y, const float* mean, const float* invstd,
                                        const float* gamma, const float* beta, long long rows, int C, int act, float slope,
                                        const double* sums, float* dy, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope};
    return epi_bwd_apply_half(g, y, e, rows, C, sums, dy, ST(stream));
}
extern "C" int bm_bn_act_gain_skip_fwd(const float* y, const float* mean, const float* invstd, const float* gamma,
                                       const float* beta, const float* x_old, float* x_new, long long rows, int C, int act,
                                       float slope, const float* scale, float boost, const float* post, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope, scale, post, boost};
    return epi_fwd(y, e, x_old, x_new, rows, C, nullptr, ST(stream));
}
extern "C" int bm_bn_act_gain_skip_bwd(const float* g, const float* y, const float* mean, const float* invstd,
                                       const float* gamma, const float* beta, int batch_stats, long long rows, int C, int act,
                                       float slope, const float* scale, float boost, const float* post, double* sums,
                                       float* dy, float* dgamma, float* dbeta, float* dscale, float* dpost,
                                       bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope, scale, post, boost, dscale || dpost};
    return epi_bwd(g, y, e, batch_stats, rows, C, sums, dy, dgamma, dbeta, dscale, dpost, nullptr, nullptr, ST(stream));
}
extern "C" long long bm_bn_act_gain_skip_bwd_det_workspace(long long rows, int C) {
    return rows > 0 && C > 0 ? epi_ws_floats(rows, 3 * C) : 0;
}
extern "C" int bm_bn_act_gain_skip_bwd_det(const float* g, const float* y, const float* mean, const float* invstd,
                                           const float* gamma, const float* beta, int batch_stats, long long rows, int C,
                                           int act, float slope, const float* scale, float boost, const float* post,
                                           double* sums, float* dy, float* dgamma, float* dbeta, float* dscale, float* dpost,
                                           float* workspace, long long workspace_floats, bm_stream_t stream) {
    const Epi e{mean, invstd, gamma, beta, act, slope, scale, post, boost, dscale || dpost};
    return epi_bwd_det(g, y, e, batch_stats, rows, C, sums, dy, dgamma, dbeta, dscale, dpost, nullptr, workspace,
                       workspace_floats, ST(stream));
}

// per-column sum / sum of squares of a channels-last matrix (BatchNorm batch statistics after bm_tc_conv1d)
extern "C" int bm_col_stats(const float* y, long long rows, int C, double* stats, bm_stream_t stream) {
    BM_CHECK_ARG(y && stats && rows > 0 && C > 0);
    cudaStream_t st = ST(stream);
    BM_CUDA(cudaMemsetAsync(stats, 0, sizeof(double) * 2 * C, st));
    {
        const int rpb = 128;
        dim3 grid((unsigned)((rows + rpb - 1) / rpb), (C + 127) / 128);
        col_stats_kernel<<<grid, 128, 0, st>>>(y, stats, rows, C, rpb);
    }
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" long long bm_col_stats_det_workspace(long long rows, int C) {
    return rows > 0 && C > 0 ? colstats_ws_floats(rows, C) : 0;
}
extern "C" int bm_col_stats_det(const float* y, long long rows, int C, float* workspace, long long workspace_floats,
                                double* stats, bm_stream_t stream) {
    BM_CHECK_ARG(y && stats && rows > 0 && C > 0);
    BM_CHECK_WS(colstats_ws_floats(rows, C));
    cudaStream_t st = ST(stream);
    double* part = reinterpret_cast<double*>(workspace);
    dim3 grid((unsigned)blocks_of(rows, COLSTATS_RPB), (C + 127) / 128);
    col_stats_kernel<true><<<grid, 128, 0, st>>>(y, part, rows, C, COLSTATS_RPB);
    BM_CHECK_LAUNCH();
    return reduce_rows(part, (long long)grid.x, 2 * C, stats, st);
}

extern "C" int bm_col_sum(const float* x, long long rows, int C, float* out, bm_stream_t stream) {
    BM_CHECK_ARG(x && out && rows > 0 && C > 0);
    cudaStream_t st = ST(stream);
    BM_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * C, st));
    {
        dim3 grid((unsigned)((rows + 255) / 256), (C + 127) / 128);
        colsum_cl_kernel<<<grid, 128, 0, st>>>(x, out, rows, C, 256);
    }
    BM_CHECK_LAUNCH();
    return 0;
}
extern "C" long long bm_col_sum_det_workspace(long long rows, int C) {
    return rows > 0 && C > 0 ? colsum_ws_floats(rows, C) : 0;
}
extern "C" int bm_col_sum_det(const float* x, long long rows, int C, float* workspace, long long workspace_floats, float* out,
                              bm_stream_t stream) {
    BM_CHECK_ARG(x && out && rows > 0 && C > 0);
    BM_CHECK_WS(colsum_ws_floats(rows, C));
    return colsum(x, rows, C, C, workspace, out, ST(stream));
}

// dh = dq * GELU'(h)  (elementwise; dh may alias dq)
extern "C" int bm_gelu_bwd(const float* dq, const float* h, long long n, float* dh, bm_stream_t stream) {
    BM_CHECK_ARG(dq && h && dh && n > 0);
    if (n % 4 == 0 && aligned16(dq, h, dh))
        gelu_bwd_v4_kernel<<<ew_grid(n / 4), 256, 0, ST(stream)>>>(
            reinterpret_cast<const float4*>(dq), reinterpret_cast<const float4*>(h), reinterpret_cast<float4*>(dh), n / 4);
    else
        gelu_bwd_kernel<<<ew_grid(n), 256, 0, ST(stream)>>>(dq, h, dh, n);
    BM_CHECK_LAUNCH();
    return 0;
}
