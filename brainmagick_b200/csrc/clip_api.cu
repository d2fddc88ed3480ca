// C-ABI entry points of ClipLoss: scores, losses and their gradients, over contiguous or pooled candidates (see
// include/bm_b200.h for the contract).
#include "api.cuh"
#include "tc_clip.cuh"
#include "tc_gemm_nt.cuh"

using namespace bm;

// =================================================================================================
// K6
// =================================================================================================
// Scratch (caller-owned, passed to every call): bm_clip_workspace() floats.  Tensor-core path: split-K partial score
// tiles + fp64 partial sums of squares + the finalize ticket (csrc/tc_clip.cuh); FP32-FMA path: fp64 sums of squares.
extern "C" long long bm_clip_workspace(int Bn, int Bc, long long KT) {
    if (Bn <= 0 || Bc <= 0 || KT <= 0) return 0;
    if (tc::clip_tc_supported(Bn, Bc, KT)) return tc::clip_ws_floats(Bn, Bc, KT);
    return 2ll * Bc + 2;
}

// det: one block per candidate (one add per slot), else up to 32 K splits per candidate
static int candidate_inv_norms(const float* cand, int Bc, long long KT, double* ss, float* inv_norm, bool det, cudaStream_t st) {
    BM_CHECK_ARG(cand && ss && inv_norm && Bc > 0 && KT > 0);
    BM_CUDA(cudaMemsetAsync(ss, 0, sizeof(double) * Bc, st));
    int splits = (int)((KT + 65535) / 65536);
    if (splits > 32) splits = 32;
    if (det) splits = 1;
    row_sumsq_kernel<<<dim3(Bc, splits), 256, 0, st>>>(cand, ss, KT);
    BM_CHECK_LAUNCH();
    inv_norm_kernel<<<(Bc + 127) / 128, 128, 0, st>>>(ss, inv_norm, Bc);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_candidate_inv_norms(const float* cand, int Bc, long long KT, double* ss, float* inv_norm,
                                      bm_stream_t stream) {
    return candidate_inv_norms(cand, Bc, KT, ss, inv_norm, false, ST(stream));
}
extern "C" int bm_candidate_inv_norms_det(const float* cand, int Bc, long long KT, double* ss, float* inv_norm,
                                          bm_stream_t stream) {
    return candidate_inv_norms(cand, Bc, KT, ss, inv_norm, true, ST(stream));
}

namespace {
// scores (+ probs / row_loss / loss) on whichever kernel the shape allows
// det: the candidate sums of squares one block per candidate, the FP32-FMA score GEMM without a K split
int clip_forward(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given, int target_offset,
                 float* inv_norm, float* scores, float* probs, float* row_loss, float* loss, float* ws,
                 long long ws_floats, int* status, bool det, int passes, cudaStream_t st) {
    BM_CHECK_ARG(est && cand && inv_norm && scores && ws && Bn > 0 && Bc > 0 && KT > 0);
    BM_CHECK_ARG(KT < (1ll << 31));
    BM_CHECK_ARG(ws_floats >= bm_clip_workspace(Bn, Bc, KT));
    BM_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 7) == 0);
    if (tc::clip_tc_supported(Bn, Bc, KT))
        return tc::launch_clip_scores(est, cand, Bn, Bc, KT, norms_given, target_offset, inv_norm, scores, probs, row_loss,
                                      loss, ws, passes, status, st, det);
    // FP32-FMA GEMM (feature sizes not a multiple of 4 floats: no TMA row pitch)
    if (!norms_given) {
        int rc = candidate_inv_norms(cand, Bc, KT, reinterpret_cast<double*>(ws), inv_norm, det, st);
        if (rc) return rc;
    }
    BM_CUDA(cudaMemsetAsync(scores, 0, sizeof(float) * (size_t)Bn * Bc, st));
    GemmP g = gemm_defaults();
    g.M = Bn; g.N = Bc; g.K = (int)KT;
    int tiles = tiles_of(Bn, Bc);
    int ks = det ? 1 : (2 * num_sms() + tiles - 1) / tiles;
    long long kchunk = (KT + ks - 1) / ks;
    kchunk = ((kchunk + GBK - 1) / GBK) * GBK;
    ks = (int)((KT + kchunk - 1) / kchunk);
    g.ksplit = ks; g.kchunk = (int)kchunk;
    g.A = est; g.lda_m = KT; g.lda_k = 1;
    g.B = cand; g.ldb_n = KT; g.ldb_k = 1;
    g.D = scores; g.ldd_m = Bc; g.ldd_n = 1; g.atomic = 1;
    g.colscale = inv_norm;
    BM_CUDA(launch_gemm(g, st));
    if (probs || row_loss) {
        clip_ce_rows_kernel<<<Bn, 256, 0, st>>>(scores, Bn, Bc, target_offset, row_loss, probs);
        BM_CHECK_LAUNCH();
    }
    if (loss) {
        mean_kernel<<<1, 256, 0, st>>>(row_loss, Bn, loss);
        BM_CHECK_LAUNCH();
    }
    return 0;
}
int clip_scores(int passes, bool det, const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given,
                float* inv_norm, float* scores, float* probs, float* workspace, long long workspace_floats, int* status,
                bm_stream_t stream) {
    return clip_forward(est, cand, Bn, Bc, KT, norms_given, 0, inv_norm, scores, probs, nullptr, nullptr, workspace,
                        workspace_floats, status, det, passes, ST(stream));
}
int clip_loss_fwd(int passes, bool det, const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset,
                  float* inv_norm, float* scores, float* probs, float* row_loss, float* loss, float* workspace,
                  long long workspace_floats, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(probs && row_loss && loss);
    BM_CHECK_ARG(target_offset >= 0 && target_offset + Bn <= Bc);
    return clip_forward(est, cand, Bn, Bc, KT, 0, target_offset, inv_norm, scores, probs, row_loss, loss, workspace,
                        workspace_floats, status, det, passes, ST(stream));
}
}  // namespace

#define BM_CLIP_SCORES_PARAMS                                                                                            \
    (const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given, float* inv_norm, float* scores, \
     float* probs, float* workspace, long long workspace_floats, int* status, bm_stream_t stream)
#define BM_CLIP_SCORES_ARGS(det) \
    (det, est, cand, Bn, Bc, KT, norms_given, inv_norm, scores, probs, workspace, workspace_floats, status, stream)
BM_TC_FORMS(bm_clip_scores, clip_scores, BM_CLIP_SCORES_PARAMS, BM_CLIP_SCORES_ARGS(false))
BM_TC_FORMS(bm_clip_scores_det, clip_scores, BM_CLIP_SCORES_PARAMS, BM_CLIP_SCORES_ARGS(true))

#define BM_CLIP_LOSS_FWD_PARAMS                                                                                          \
    (const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset, float* inv_norm,              \
     float* scores, float* probs, float* row_loss, float* loss, float* workspace, long long workspace_floats,            \
     int* status, bm_stream_t stream)
#define BM_CLIP_LOSS_FWD_ARGS(det)                                                                                       \
    (det, est, cand, Bn, Bc, KT, target_offset, inv_norm, scores, probs, row_loss, loss, workspace, workspace_floats,    \
     status, stream)
BM_TC_FORMS(bm_clip_loss_fwd, clip_loss_fwd, BM_CLIP_LOSS_FWD_PARAMS, BM_CLIP_LOSS_FWD_ARGS(false))
BM_TC_FORMS(bm_clip_loss_fwd_det, clip_loss_fwd, BM_CLIP_LOSS_FWD_PARAMS, BM_CLIP_LOSS_FWD_ARGS(true))

namespace {
// dest = G @ cand, the GEMM of the CLIP backward.  fill(transposed) writes G [Bn][Bc] (transposed: [Bc][Bn]) in the layout
// the chosen GEMM reads.
template <class Fill>
int clip_dest_gemm(Fill fill, const float* cand, int Bn, int Bc, long long KT, float* G, float* dest, int passes,
                   int* status, cudaStream_t st) {
    if (tc::gemm_nt_pp_supported(Bn, (int)KT, Bc) && Bn >= 192) {
        // csrc/tc_gemm_nt.cuh: dE = G C with G [Bn][Bc], C [Bc][KT]; smaller batches take the weight-gradient form below
        if (int rc = fill(0)) return rc;
        return tc::launch_gemm_nt_pp(G, cand, dest, Bn, (int)KT, Bc, passes, status, st);
    }
    if (tc::wgrad_tc_supported(Bn, (int)KT)) {
        // tensor cores: dE[b][k] = sum_o G^T[o][b] C[o][k]  == weight-gradient GEMM with "positions" = candidates
        if (int rc = fill(1)) return rc;
        return tc::launch_wgrad_tc(G, cand, 1, Bc, Bn, (int)KT, (int)KT, 1, 1, dest, dest, passes, st, nullptr);   // direct
    }
    if (int rc = fill(0)) return rc;
    GemmP g = gemm_defaults();
    g.M = Bn; g.N = (int)KT; g.K = Bc; g.kchunk = Bc;
    g.A = G; g.lda_m = Bc; g.lda_k = 1;
    g.B = cand; g.ldb_n = 1; g.ldb_k = KT; g.b_ncontig = 1;
    g.D = dest; g.ldd_m = KT; g.ldd_n = 1;
    BM_CUDA(launch_gemm(g, st));
    return 0;
}

// dcand[o] = sum_b G[b][o] est[b] - coef[o] cand[o] (see clip_cand_coef_kernel); fill as in clip_dest_gemm
template <class Fill>
int clip_dcand_gemm(Fill fill, const float* scores, const float* inv_norm, const float* est, const float* cand, int Bn, int Bc,
                    long long KT, float* G, float* coef, float* dcand, int passes, int* status, cudaStream_t st) {
    if (int rc = fill(0)) return rc;
    clip_cand_coef_kernel<<<(Bc + 127) / 128, 128, 0, st>>>(G, scores, inv_norm, Bn, Bc, coef);     // needs G as [Bn][Bc]
    BM_CHECK_LAUNCH();
    // dcand[o][k] = sum_b G[b][o] est[b][k]
    if (tc::gemm_nt_pp_supported(Bc, (int)KT, Bn)) {
        // csrc/tc_gemm_nt.cuh: A = G^T [Bc][Bn] (rewritten into the same scratch), B = est [Bn][KT]
        if (int rc = fill(1)) return rc;
        int rc = tc::launch_gemm_nt_pp(G, est, dcand, Bc, (int)KT, Bn, passes, status, st);
        if (rc) return rc;
    } else if (tc::wgrad_tc_supported(Bc, (int)KT)) {
        int rc = tc::launch_wgrad_tc(G, est, 1, Bn, Bc, (int)KT, (int)KT, 1, 1, dcand, dcand, passes, st, nullptr);   // direct
        if (rc) return rc;
    } else {
        GemmP g = gemm_defaults();
        g.M = Bc; g.N = (int)KT; g.K = Bn; g.kchunk = Bn;
        g.A = G; g.lda_m = 1; g.lda_k = Bc; g.a_mcontig = 1;
        g.B = est; g.ldb_n = 1; g.ldb_k = KT; g.b_ncontig = 1;
        g.D = dcand; g.ldd_m = KT; g.ldd_n = 1;
        BM_CUDA(launch_gemm(g, st));
    }
    clip_cand_correct_kernel<<<ew_grid((long long)Bc * KT), 256, 0, st>>>(cand, coef, KT, (long long)Bc * KT, dcand);
    BM_CHECK_LAUNCH();
    return 0;
}

int clip_loss_bwd(int passes, const float* probs, const float* inv_norm, const float* cand, const float* gout, int Bn, int Bc,
                  long long KT, int target_offset, float* G, float* dest, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(probs && inv_norm && cand && gout && G && dest && Bn > 0 && Bc > 0 && KT > 0);
    BM_CHECK_ARG(KT < (1ll << 31));
    cudaStream_t st = ST(stream);
    auto fill = [&](int transposed) {
        clip_ce_bwd_kernel<<<ew_grid((long long)Bn * Bc), 256, 0, st>>>(probs, inv_norm, gout, Bn, Bc, target_offset, G,
                                                                        transposed);
        BM_CHECK_LAUNCH();
        return 0;
    };
    return clip_dest_gemm(fill, cand, Bn, Bc, KT, G, dest, passes, status, st);
}
}  // namespace

BM_TC_FORMS(bm_clip_loss_bwd, clip_loss_bwd,
            (const float* probs, const float* inv_norm, const float* cand, const float* gout, int Bn, int Bc, long long KT,
             int target_offset, float* G, float* dest, int* status, bm_stream_t stream),
            (probs, inv_norm, cand, gout, Bn, Bc, KT, target_offset, G, dest, status, stream))

// ---- pooled candidates (negatives.py): candidate o is cand[o] for o < Bb, else arena[slots[o - Bb]] ----------------------
namespace {
int check_pooled(const float* cand, int Bb, const float* arena, const int* slots, int Bn, int Bc, long long KT) {
    BM_CHECK_ARG(cand && Bn > 0 && Bb >= 0 && Bb <= Bc && (Bb == Bc || (arena && slots)));
    BM_CHECK_ARG(tc::clip_tc_supported(Bn, Bc, KT));
    return 0;
}

int clip_loss_fwd_pooled(int passes, bool det, const float* est, const float* cand, int Bb, const float* arena,
                         const int* slots, int Bn, int Bc, long long KT, int target_offset, float* inv_norm, float* scores,
                         float* probs, float* row_loss, float* loss, float* workspace, long long workspace_floats, int* status,
                         bm_stream_t stream) {
    if (int rc = check_pooled(cand, Bb, arena, slots, Bn, Bc, KT)) return rc;
    BM_CHECK_ARG(est && inv_norm && scores && probs && row_loss && loss && workspace);
    BM_CHECK_ARG(target_offset >= 0 && target_offset + Bn <= Bc);
    BM_CHECK_ARG(workspace_floats >= bm_clip_workspace(Bn, Bc, KT));
    BM_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0);
    return tc::launch_clip_scores(est, cand, Bn, Bc, KT, 0, target_offset, inv_norm, scores, probs, row_loss, loss,
                                  workspace, passes, status, ST(stream), det, Bb, arena, Bb < Bc ? slots : nullptr);
}

int clip_loss_bwd_pooled(int passes, const float* probs, const float* inv_norm, const float* cand, int Bb, const float* arena,
                         const int* slots, const float* gout, int Bn, int Bc, long long KT, int target_offset, float* G,
                         float* dest, int* status, bm_stream_t stream) {
    (void)status;
    if (int rc = check_pooled(cand, Bb, arena, slots, Bn, Bc, KT)) return rc;
    BM_CHECK_ARG(probs && inv_norm && gout && G && dest);
    cudaStream_t st = ST(stream);
    const int ldg = (Bc + 3) / 4 * 4;
    clip_ce_bwd_padded_kernel<<<ew_grid((long long)Bn * ldg), 256, 0, st>>>(probs, inv_norm, gout, Bn, Bc, ldg,
                                                                            target_offset, G);
    BM_CHECK_LAUNCH();
    return tc::launch_gemm_nt_pooled(G, ldg, cand, Bb, arena, slots, Bc, dest, Bn, (int)KT, passes, st);
}
}  // namespace

#define BM_CLIP_LOSS_FWD_POOLED_PARAMS                                                                                   \
    (const float* est, const float* cand, int Bb, const float* arena, const int* slots, int Bn, int Bc, long long KT,   \
     int target_offset, float* inv_norm, float* scores, float* probs, float* row_loss, float* loss, float* workspace,   \
     long long workspace_floats, int* status, bm_stream_t stream)
#define BM_CLIP_LOSS_FWD_POOLED_ARGS(det)                                                                                \
    (det, est, cand, Bb, arena, slots, Bn, Bc, KT, target_offset, inv_norm, scores, probs, row_loss, loss, workspace,   \
     workspace_floats, status, stream)
BM_TC_FORMS(bm_clip_loss_fwd_pooled, clip_loss_fwd_pooled, BM_CLIP_LOSS_FWD_POOLED_PARAMS,
            BM_CLIP_LOSS_FWD_POOLED_ARGS(false))
BM_TC_FORMS(bm_clip_loss_fwd_pooled_det, clip_loss_fwd_pooled, BM_CLIP_LOSS_FWD_POOLED_PARAMS,
            BM_CLIP_LOSS_FWD_POOLED_ARGS(true))
BM_TC_FORMS(bm_clip_loss_bwd_pooled, clip_loss_bwd_pooled,
            (const float* probs, const float* inv_norm, const float* cand, int Bb, const float* arena, const int* slots,
             const float* gout, int Bn, int Bc, long long KT, int target_offset, float* G, float* dest, int* status,
             bm_stream_t stream),
            (probs, inv_norm, cand, Bb, arena, slots, gout, Bn, Bc, KT, target_offset, G, dest, status, stream))

static int clip_loss_bwd_cand(int passes, const float* probs, const float* scores, const float* inv_norm, const float* est,
                              const float* cand, const float* gout, int Bn, int Bc, long long KT, int target_offset, float* G,
                              float* coef, float* dcand, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(probs && scores && inv_norm && est && cand && gout && G && coef && dcand);
    BM_CHECK_ARG(Bn > 0 && Bc > 0 && KT > 0 && KT < (1ll << 31));
    cudaStream_t st = ST(stream);
    auto fill = [&](int transposed) {
        clip_ce_bwd_kernel<<<ew_grid((long long)Bn * Bc), 256, 0, st>>>(probs, inv_norm, gout, Bn, Bc, target_offset, G,
                                                                        transposed);
        BM_CHECK_LAUNCH();
        return 0;
    };
    return clip_dcand_gemm(fill, scores, inv_norm, est, cand, Bn, Bc, KT, G, coef, dcand, passes, status, st);
}
BM_TC_FORMS(bm_clip_loss_bwd_cand, clip_loss_bwd_cand,
            (const float* probs, const float* scores, const float* inv_norm, const float* est, const float* cand,
             const float* gout, int Bn, int Bc, long long KT, int target_offset, float* G, float* coef, float* dcand,
             int* status, bm_stream_t stream),
            (probs, scores, inv_norm, est, cand, gout, Bn, Bc, KT, target_offset, G, coef, dcand, status, stream))

static int clip_scores_bwd(int passes, const float* dscores, const float* scores, const float* inv_norm, const float* est,
                           const float* cand, int Bn, int Bc, long long KT, float* G, float* coef, float* dest, float* dcand,
                           int* status, bm_stream_t stream) {
    BM_CHECK_ARG(dscores && inv_norm && cand && G && Bn > 0 && Bc > 0 && KT > 0 && KT < (1ll << 31));
    BM_CHECK_ARG(!dcand || (scores && est && coef));
    cudaStream_t st = ST(stream);
    auto fill = [&](int transposed) {
        clip_scores_grad_kernel<<<ew_grid((long long)Bn * Bc), 256, 0, st>>>(dscores, inv_norm, Bn, Bc, G, transposed);
        BM_CHECK_LAUNCH();
        return 0;
    };
    if (dest)
        if (int rc = clip_dest_gemm(fill, cand, Bn, Bc, KT, G, dest, passes, status, st)) return rc;
    if (dcand)
        if (int rc = clip_dcand_gemm(fill, scores, inv_norm, est, cand, Bn, Bc, KT, G, coef, dcand, passes, status, st))
            return rc;
    return 0;
}
BM_TC_FORMS(bm_clip_scores_bwd, clip_scores_bwd,
            (const float* dscores, const float* scores, const float* inv_norm, const float* est, const float* cand, int Bn,
             int Bc, long long KT, float* G, float* coef, float* dest, float* dcand, int* status, bm_stream_t stream),
            (dscores, scores, inv_norm, est, cand, Bn, Bc, KT, G, coef, dest, dcand, status, stream))
