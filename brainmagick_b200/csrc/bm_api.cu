// C-ABI entry points of libbm_b200.so (see include/bm_b200.h for the contract and the reference citations).
#include <algorithm>
#include "../../include/bm_b200.h"
#include "common.cuh"
#include "elementwise.cuh"
#include "gemm_simt.cuh"
#include "tc_conv.cuh"
#include "tc_wgrad.cuh"
#include "tc_clip.cuh"
#include "tc_wgradp.cuh"
#include "tc_gemm_nt.cuh"
#include "retrieval.cuh"
#include "prep.cuh"
#include "convseq.cuh"
#include "channel_join.cuh"
#include "masked_loss.cuh"
#include "decoding_loss.cuh"
#include "metrics.cuh"
#include "svd_penalty.cuh"

namespace bm {
thread_local char g_last_error[512] = "";
unsigned long long g_launches = 0;
int g_debug_flags = 0;
long long* g_debug_buf = nullptr;
}
using namespace bm;

#define ST(s) reinterpret_cast<cudaStream_t>(s)

// ---- TF32 and bf16 forms (the `_tf32` and `_bf16` entry points) ---------------------------------------------------------
// Every entry point that runs a tensor-core contraction is a static implementation whose first argument is the engine's
// operand mode (tc_common.cuh).  BM_TC_FORMS defines over it the default entry point (3xTF32), its `_tf32` twin
// (single-pass TF32: each fp32 operand element rounded once to tf32) and its `_bf16` twin (each fp32 operand element
// rounded once to bf16), with identical arguments.
#define BM_ARGS(...) __VA_ARGS__
#define BM_TC_FORMS(name, impl, params, args)                                                                            \
    extern "C" int name params { return impl(tc::TC_3XTF32, BM_ARGS args); }                                              \
    extern "C" int name##_tf32 params { return impl(tc::TC_TF32, BM_ARGS args); }                                         \
    extern "C" int name##_bf16 params { return impl(tc::TC_BF16, BM_ARGS args); }

extern "C" const char* bm_last_error(void) { return bm::g_last_error; }
extern "C" int bm_abi_version(void) { return 1; }
extern "C" unsigned long long bm_launch_count(void) { return bm::g_launches; }
extern "C" int bm_set_debug_buffer(long long* buf) { bm::g_debug_buf = buf; return 0; }
extern "C" int bm_set_debug_flags(int flags) { int old = bm::g_debug_flags; bm::g_debug_flags = flags; return old; }
#ifdef BM_HC_PHASES
// the per-phase probe's counters (tc_common.cuh HcPhase): out[kernel * HP_N + phase] after the device is idle; reset: zero
// them.  Only in the probe build of profiles/conv_phase_probe.py, not part of the ABI.
extern "C" int bm_hc_phases(unsigned long long* out, int reset) {
    BM_CUDA(cudaDeviceSynchronize());
    BM_CUDA(cudaMemcpyFromSymbol(out, tc::g_hc_phases, sizeof(tc::g_hc_phases)));
    if (reset) {
        static const unsigned long long zeros[2 * tc::HP_N] = {};
        BM_CUDA(cudaMemcpyToSymbol(tc::g_hc_phases, zeros, sizeof(zeros)));
    }
    return 0;
}
#endif

namespace {

// number of z-chunks so that a reduction GEMM with `tiles` output tiles fills the machine ~2x
inline int pick_chunks(int Z, int tiles) {
    int want = (2 * num_sms() + tiles - 1) / tiles;
    if (want < 1) want = 1;
    if (want > Z) want = Z;
    return want;
}
inline int tiles_of(int M, int N) { return ((M + GBM - 1) / GBM) * ((N + GBN - 1) / GBN); }

// ---- deterministic forms (the `_det` entry points) -------------------------------------------------------------------
// Every floating-point reduction that the default entry points finish with atomics is split in two: each block stores its
// partial row into a caller-owned [n_blocks][width] buffer, and reduce_rows_kernel sums the rows in index order.  The
// split-batch FP32-FMA weight-gradient GEMMs store one partial plane per batch segment ([nseg][output], the segment count of
// the atomic form, which follows the SM count) and sum the planes in segment order; the remaining split GEMMs (dheads over
// the recordings, the FP32-FMA CLIP scores) run unsplit: one CTA per output tile adds onto the zeroed output exactly once.
constexpr int COLSUM_RPB = 256, COLSTATS_RPB = 128;
inline long long blocks_of(long long rows, int rpb) { return (rows + rpb - 1) / rpb; }
inline long long colsum_ws_floats(long long rows, int C) { return blocks_of(rows, COLSUM_RPB) * C; }
inline long long colstats_ws_floats(long long rows, int C) { return blocks_of(rows, COLSTATS_RPB) * 4ll * C; }  // fp64 [nb][2C]
inline long long glu_bwd_ws_floats(long long rows, int H) { return blocks_of(rows, CS_ROWS_PER_BLOCK) * 2ll * H; }
// batch segments of the split weight-gradient GEMMs (the atomic form's count); planes = segments x output elements
inline int wgrad_segments(int B, int tiles) {
    const int zchunk = (B + pick_chunks(B, tiles) - 1) / pick_chunks(B, tiles);
    return (B + zchunk - 1) / zchunk;
}
inline long long planes_floats(int B, int M, int N, int taps = 1) {
    return (long long)wgrad_segments(B, tiles_of(M, N) * taps) * M * N * taps;
}
inline long long head_ws_floats(int B, int T, int H, int F) {
    return std::max({(long long)B * F, colsum_ws_floats((long long)B * T, 2 * H), planes_floats(B, 2 * H, F),
                     planes_floats(B, 2 * H, H)});
}

template <class T>
int reduce_rows(const T* part, long long n, int W, T* out, cudaStream_t st) {
    reduce_rows_kernel<T><<<(W + 127) / 128, 128, 0, st>>>(part, n, W, out);
    BM_CHECK_LAUNCH();
    return 0;
}

// out[c] = sum_r X[r*ld + c] over `rows` rows: atomically (part == NULL, out zeroed here) or through the partials `part`
int colsum(const float* X, long long rows, int C, int ld, float* part, float* out, cudaStream_t st) {
    dim3 grid((unsigned)blocks_of(rows, COLSUM_RPB), (C + 127) / 128);
    if (!part) BM_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * C, st));
    if (ld == C) {
        if (part) colsum_cl_kernel<true><<<grid, 128, 0, st>>>(X, part, rows, C, COLSUM_RPB);
        else colsum_cl_kernel<<<grid, 128, 0, st>>>(X, out, rows, C, COLSUM_RPB);
    } else {
        if (part) colsum_strided_kernel<true><<<grid, 128, 0, st>>>(X, part, rows, C, ld, COLSUM_RPB);
        else colsum_strided_kernel<<<grid, 128, 0, st>>>(X, out, rows, C, ld, COLSUM_RPB);
    }
    BM_CHECK_LAUNCH();
    return part ? reduce_rows(part, (long long)grid.x, C, out, st) : 0;
}

// the split GEMM g (atomic form: g.D inside the output `out` of `elems` elements, g.atomic = 1) with one partial plane per
// segment: segment s writes part[s * elems + (g.D - out) + ...]; sum_planes adds the planes in segment order
cudaError_t launch_gemm_planes(GemmP g, const float* out, long long elems, float* part, cudaStream_t st) {
    g.D = part + (g.D - out);
    g.ldd_z = elems;
    g.atomic = 0;
    return launch_gemm(g, st);
}
int sum_planes(const float* part, int nseg, long long elems, float* out, cudaStream_t st) {
    return reduce_rows(part, (long long)nseg, (int)elems, out, st);
}

#define BM_CHECK_WS(need)                                                                              \
    BM_CHECK_ARG(workspace && workspace_floats >= (need) && (reinterpret_cast<uintptr_t>(workspace) & 7) == 0)

}  // namespace

// =================================================================================================
// K1
// =================================================================================================
extern "C" int bm_attention_weights_fwd(const float* positions, const float* freq, const float* heads,
                                        const float* ban_centre, float radius, int R, int C, int O, int P,
                                        float* emb, float* weights, bm_stream_t stream) {
    BM_CHECK_ARG(positions && freq && heads && emb && weights);
    BM_CHECK_ARG(R > 0 && C > 0 && O > 0 && P > 0 && P % 2 == 0);
    int n = 0;
    while ((n + 1) * (n + 1) * 2 <= P) ++n;
    BM_CHECK_ARG(n * n * 2 == P);
    cudaStream_t st = ST(stream);
    fourier_emb_kernel<<<ew_grid((long long)R * C * n * n), 256, 0, st>>>(positions, freq, 0.2f, R * C, n, emb);
    BM_CHECK_LAUNCH();
    // scores[r][o][c] = <emb[r][c][:], heads[o][:]>
    GemmP g = gemm_defaults();
    g.M = C; g.N = O; g.K = P;
    g.Z = R; g.nseg = R; g.zchunk = 1; g.kchunk = P;
    g.A = emb; g.lda_z = (long long)C * P; g.lda_m = P; g.lda_k = 1; g.a_mcontig = 0;
    g.B = heads; g.ldb_z = 0; g.ldb_n = P; g.ldb_k = 1; g.b_ncontig = 0;
    g.D = weights; g.ldd_z = (long long)O * C; g.ldd_m = 1; g.ldd_n = C;
    BM_CUDA(launch_gemm(g, st));
    int rows = R * O;
    masked_softmax_kernel<<<(rows + 7) / 8, 256, 0, st>>>(weights, positions, ban_centre, radius, -0.1f, R, O, C);
    BM_CHECK_LAUNCH();
    return 0;
}

static int attention_weights_bwd(const float* dweights, const float* weights, const float* emb, int R, int C, int O, int P,
                                 float* dscores, float* dheads, bool det, cudaStream_t st) {
    BM_CHECK_ARG(dweights && weights && emb && dscores && dheads);
    int rows = R * O;
    softmax_bwd_kernel<<<(rows + 7) / 8, 256, 0, st>>>(weights, dweights, dscores, rows, C);
    BM_CHECK_LAUNCH();
    // dheads[o][p] = sum_{r,c} ds[r][o][c] emb[r][c][p]
    BM_CUDA(cudaMemsetAsync(dheads, 0, sizeof(float) * O * P, st));
    GemmP g = gemm_defaults();
    g.M = O; g.N = P; g.K = C; g.kchunk = C;
    g.Z = R; g.zchunk = det ? R : 1; g.nseg = det ? 1 : R;
    g.A = dscores; g.lda_z = (long long)O * C; g.lda_m = C; g.lda_k = 1; g.a_mcontig = 0;
    g.B = emb; g.ldb_z = (long long)C * P; g.ldb_n = 1; g.ldb_k = P; g.b_ncontig = 1;
    g.D = dheads; g.ldd_z = 0; g.ldd_m = P; g.ldd_n = 1; g.atomic = 1;
    BM_CUDA(launch_gemm(g, st));
    return 0;
}

extern "C" int bm_attention_weights_bwd(const float* dweights, const float* weights, const float* emb, int R,
                                        int C, int O, int P, float* dscores, float* dheads, bm_stream_t stream) {
    return attention_weights_bwd(dweights, weights, emb, R, C, O, P, dscores, dheads, false, ST(stream));
}
extern "C" int bm_attention_weights_bwd_det(const float* dweights, const float* weights, const float* emb, int R,
                                            int C, int O, int P, float* dscores, float* dheads, bm_stream_t stream) {
    return attention_weights_bwd(dweights, weights, emb, R, C, O, P, dscores, dheads, true, ST(stream));
}

// =================================================================================================
// K2
// =================================================================================================
// ---- pieces (leading dimensions explicit so that u / v / x0 may be kept channel-padded for the tensor-core layers) ----
extern "C" int bm_sensor_mix_fwd(const float* meg, const float* weights, const int* rec_of_sample, int B, int C, int T,
                                 int O, int ld_u, float* u, bm_stream_t stream) {
    BM_CHECK_ARG(meg && weights && rec_of_sample && u && ld_u >= O);
    // u[b][t][o] = sum_c meg[b][c][t] w[rec_b][o][c]
    GemmP g = gemm_defaults();
    g.M = T; g.N = O; g.K = C; g.kchunk = C;
    g.Z = B; g.nseg = B; g.zchunk = 1;
    g.A = meg; g.lda_z = (long long)C * T; g.lda_m = 1; g.lda_k = T; g.a_mcontig = 1;
    g.B = weights; g.bsel = rec_of_sample; g.ldb_z = (long long)O * C; g.ldb_n = C; g.ldb_k = 1; g.b_ncontig = 0;
    g.D = u; g.ldd_z = (long long)T * ld_u; g.ldd_m = ld_u; g.ldd_n = 1;
    BM_CUDA(launch_gemm(g, ST(stream)));
    return 0;
}

extern "C" int bm_initial_linear_fwd(const float* u, int ld_u, const float* il_w, const float* il_b, int B, int T, int O,
                                     int IL, int ld_v, float* v, bm_stream_t stream) {
    BM_CHECK_ARG(u && il_w && il_b && v && ld_u >= O && ld_v >= IL);
    // v[row][p] = il_b[p] + sum_o u[row][o] il_w[p][o]
    GemmP g = gemm_defaults();
    g.M = B * T; g.N = IL; g.K = O; g.kchunk = O;
    g.A = u; g.lda_m = ld_u; g.lda_k = 1;
    g.B = il_w; g.ldb_n = O; g.ldb_k = 1;
    g.D = v; g.ldd_m = ld_v; g.ldd_n = 1;
    g.bias = il_b;
    BM_CUDA(launch_gemm(g, ST(stream)));
    return 0;
}

extern "C" int bm_subject_layers_fwd(const float* v, int ld_v, const float* subj_w, const int* subject, int B, int T,
                                     int IL, int D, int ld_x0, float* x0, bm_stream_t stream) {
    BM_CHECK_ARG(v && subj_w && subject && x0 && ld_v >= IL && ld_x0 >= D);
    // x0[b][t][d] = sum_p v[b][t][p] M[s_b][p][d]
    GemmP g = gemm_defaults();
    g.M = T; g.N = D; g.K = IL; g.kchunk = IL;
    g.Z = B; g.nseg = B; g.zchunk = 1;
    g.A = v; g.lda_z = (long long)T * ld_v; g.lda_m = ld_v; g.lda_k = 1;
    g.B = subj_w; g.bsel = subject; g.ldb_z = (long long)IL * D; g.ldb_n = 1; g.ldb_k = D; g.b_ncontig = 1;
    g.D = x0; g.ldd_z = (long long)T * ld_x0; g.ldd_m = ld_x0; g.ldd_n = 1;
    BM_CUDA(launch_gemm(g, ST(stream)));
    return 0;
}

extern "C" int bm_sensor_chain_fwd(const float* meg, const float* weights, const int* rec_of_sample,
                                   const float* il_w, const float* il_b, const float* subj_w, const int* subject,
                                   int B, int C, int T, int O, int IL, int D, int ld_x0, float* u, float* v,
                                   float* x0, bm_stream_t stream) {
    BM_CHECK_ARG(meg && weights && rec_of_sample && il_w && il_b && subj_w && subject && u && v && x0);
    BM_CHECK_ARG(ld_x0 >= D);
    int rc = bm_sensor_mix_fwd(meg, weights, rec_of_sample, B, C, T, O, O, u, stream);
    if (!rc) rc = bm_initial_linear_fwd(u, O, il_w, il_b, B, T, O, IL, IL, v, stream);
    if (!rc) rc = bm_subject_layers_fwd(v, IL, subj_w, subject, B, T, IL, D, ld_x0, x0, stream);
    return rc;
}

extern "C" int bm_subject_layers_bwd(const float* dx0, int ld_x0, const float* v, int ld_v, const float* subj_w,
                                     const int* subject, const int* subj_order, const int* subj_off, int B, int T, int IL,
                                     int D, int S, int ld_dv, float* dv, float* d_subj_w, bm_stream_t stream) {
    // dv NULL: no data gradient (nothing below needs it); d_subj_w NULL: frozen weights
    BM_CHECK_ARG(dx0 && (!dv || (subj_w && subject)) && (!d_subj_w || (v && subj_order && subj_off)));
    BM_CHECK_ARG(ld_x0 >= D && ld_v >= IL && ld_dv >= IL);
    cudaStream_t st = ST(stream);
    if (dv) {   // dv[b][t][p] = sum_d g[b][t][d] M[s_b][p][d]
        GemmP g = gemm_defaults();
        g.M = T; g.N = IL; g.K = D; g.kchunk = D;
        g.Z = B; g.nseg = B; g.zchunk = 1;
        g.A = dx0; g.lda_z = (long long)T * ld_x0; g.lda_m = ld_x0; g.lda_k = 1;
        g.B = subj_w; g.bsel = subject; g.ldb_z = (long long)IL * D; g.ldb_n = D; g.ldb_k = 1;
        g.D = dv; g.ldd_z = (long long)T * ld_dv; g.ldd_m = ld_dv; g.ldd_n = 1;
        BM_CUDA(launch_gemm(g, st));
    }
    if (d_subj_w) {   // dM[s][p][d] = sum_{b in s} sum_t v[b][t][p] g[b][t][d]
        GemmP g = gemm_defaults();
        g.M = IL; g.N = D; g.K = T; g.kchunk = T;
        g.Z = B; g.nseg = S; g.seg_off = subj_off; g.zlist = subj_order;
        g.A = v; g.lda_z = (long long)T * ld_v; g.lda_m = 1; g.lda_k = ld_v; g.a_mcontig = 1;
        g.B = dx0; g.ldb_z = (long long)T * ld_x0; g.ldb_n = 1; g.ldb_k = ld_x0; g.b_ncontig = 1;
        g.D = d_subj_w; g.ldd_z = (long long)IL * D; g.ldd_m = D; g.ldd_n = 1;
        BM_CUDA(launch_gemm(g, st));
    }
    return 0;
}

// part: NULL (atomic reductions) or the colsum_ws_floats(B*T, IL) partials of the deterministic form.
// du, d_il_w, d_il_b may each be NULL (no data gradient below / frozen parameter): its GEMM or reduction is skipped.
static int initial_linear_bwd(const float* dv, int ld_dv, const float* u, int ld_u, const float* il_w, int B, int T, int O,
                              int IL, int ld_du, float* du, float* d_il_w, float* d_il_b, float* part, cudaStream_t st) {
    BM_CHECK_ARG(dv && (!du || il_w) && (!d_il_w || u) && ld_dv >= IL && ld_u >= O && ld_du >= O);
    if (d_il_w) {   // d_il_w[p][o] = sum_{b,t} dv[b][t][p] u[b][t][o]
        BM_CUDA(cudaMemsetAsync(d_il_w, 0, sizeof(float) * IL * O, st));
        GemmP g = gemm_defaults();
        g.M = IL; g.N = O; g.K = T; g.kchunk = T;
        g.Z = B; g.nseg = pick_chunks(B, tiles_of(IL, O)); g.zchunk = (B + g.nseg - 1) / g.nseg;
        g.nseg = (B + g.zchunk - 1) / g.zchunk;
        g.A = dv; g.lda_z = (long long)T * ld_dv; g.lda_m = 1; g.lda_k = ld_dv; g.a_mcontig = 1;
        g.B = u; g.ldb_z = (long long)T * ld_u; g.ldb_n = 1; g.ldb_k = ld_u; g.b_ncontig = 1;
        g.D = d_il_w; g.ldd_z = 0; g.ldd_m = O; g.ldd_n = 1; g.atomic = 1;
        if (part) {
            BM_CUDA(launch_gemm_planes(g, d_il_w, (long long)IL * O, part, st));
            if (int rc = sum_planes(part, g.nseg, (long long)IL * O, d_il_w, st)) return rc;
        } else {
            BM_CUDA(launch_gemm(g, st));
        }
    }
    if (d_il_b && part) {   // d_il_b[p] = sum dv, through the partials
        if (int rc = colsum(dv, (long long)B * T, IL, ld_dv, part, d_il_b, st)) return rc;
    } else if (d_il_b) {   // d_il_b[p] = sum dv
        BM_CUDA(cudaMemsetAsync(d_il_b, 0, sizeof(float) * IL, st));
        GemmP g = gemm_defaults();                      // column sums as a 1-row GEMM would waste a tile: dedicated kernel
        (void)g;
        long long rows = (long long)B * T;
        dim3 grid((unsigned)((rows + 255) / 256), (IL + 127) / 128);
        colsum_strided_kernel<<<grid, 128, 0, st>>>(dv, d_il_b, rows, IL, ld_dv, 256);
        BM_CHECK_LAUNCH();
    }
    if (du) {   // du[row][o] = sum_p dv[row][p] il_w[p][o]
        GemmP g = gemm_defaults();
        g.M = B * T; g.N = O; g.K = IL; g.kchunk = IL;
        g.A = dv; g.lda_m = ld_dv; g.lda_k = 1;
        g.B = il_w; g.ldb_n = 1; g.ldb_k = O; g.b_ncontig = 1;
        g.D = du; g.ldd_m = ld_du; g.ldd_n = 1;
        BM_CUDA(launch_gemm(g, st));
    }
    return 0;
}

extern "C" int bm_initial_linear_bwd(const float* dv, int ld_dv, const float* u, int ld_u, const float* il_w, int B, int T,
                                     int O, int IL, int ld_du, float* du, float* d_il_w, float* d_il_b,
                                     bm_stream_t stream) {
    return initial_linear_bwd(dv, ld_dv, u, ld_u, il_w, B, T, O, IL, ld_du, du, d_il_w, d_il_b, nullptr, ST(stream));
}
extern "C" long long bm_initial_linear_bwd_det_workspace(int B, int T, int O, int IL) {
    if (B <= 0 || T <= 0 || O <= 0 || IL <= 0) return 0;
    return std::max(colsum_ws_floats((long long)B * T, IL), planes_floats(B, IL, O));
}
extern "C" int bm_initial_linear_bwd_det(const float* dv, int ld_dv, const float* u, int ld_u, const float* il_w, int B, int T,
                                         int O, int IL, int ld_du, float* du, float* d_il_w, float* d_il_b, float* workspace,
                                         long long workspace_floats, bm_stream_t stream) {
    BM_CHECK_ARG(B > 0 && T > 0 && O > 0 && IL > 0);
    if (!d_il_w && !d_il_b)                      // the data gradient alone reduces nothing: no workspace
        return initial_linear_bwd(dv, ld_dv, u, ld_u, il_w, B, T, O, IL, ld_du, du, nullptr, nullptr, nullptr, ST(stream));
    BM_CHECK_WS(bm_initial_linear_bwd_det_workspace(B, T, O, IL));
    return initial_linear_bwd(dv, ld_dv, u, ld_u, il_w, B, T, O, IL, ld_du, du, d_il_w, d_il_b, workspace, ST(stream));
}

extern "C" int bm_sensor_mix_bwd(const float* du, int ld_du, const float* meg, const int* rec_order, const int* rec_off,
                                 int B, int C, int T, int O, int R, float* d_weights, bm_stream_t stream) {
    BM_CHECK_ARG(du && meg && rec_order && rec_off && d_weights && ld_du >= O);
    // dw[r][o][c] = sum_{b in r} sum_t du[b][t][o] meg[b][c][t]
    GemmP g = gemm_defaults();
    g.M = O; g.N = C; g.K = T; g.kchunk = T;
    g.Z = B; g.nseg = R; g.seg_off = rec_off; g.zlist = rec_order;
    g.A = du; g.lda_z = (long long)T * ld_du; g.lda_m = 1; g.lda_k = ld_du; g.a_mcontig = 1;
    g.B = meg; g.ldb_z = (long long)C * T; g.ldb_n = T; g.ldb_k = 1; g.b_ncontig = 0;
    g.D = d_weights; g.ldd_z = (long long)O * C; g.ldd_m = C; g.ldd_n = 1;
    BM_CUDA(launch_gemm(g, ST(stream)));
    return 0;
}

extern "C" int bm_sensor_mix_bwd_data(const float* du, int ld_du, const float* weights, const int* rec_of_sample,
                                      const float* mask, int B, int C, int T, int O, float* dmeg, bm_stream_t stream) {
    BM_CHECK_ARG(du && weights && rec_of_sample && dmeg && ld_du >= O && B > 0 && C > 0 && T > 0 && O > 0);
    // dmeg[b][c][t] = mask[c] sum_o du[b][t][o] w[rec_b][o][c]
    GemmP g = gemm_defaults();
    g.M = T; g.N = C; g.K = O; g.kchunk = O;
    g.Z = B; g.nseg = B; g.zchunk = 1;
    g.A = du; g.lda_z = (long long)T * ld_du; g.lda_m = ld_du; g.lda_k = 1;
    g.B = weights; g.bsel = rec_of_sample; g.ldb_z = (long long)O * C; g.ldb_n = 1; g.ldb_k = C; g.b_ncontig = 1;
    g.D = dmeg; g.ldd_z = (long long)C * T; g.ldd_m = 1; g.ldd_n = T;
    g.colscale = mask;
    BM_CUDA(launch_gemm(g, ST(stream)));
    return 0;
}

// det: the _det form (initial_linear's reductions through `workspace`).  Each stage runs only as far as its outputs are asked for:
// d_subj_w, d_il_w, d_il_b, d_weights NULL = frozen parameter; du NULL = no mix gradient and no meg gradient below (then
// d_weights must be NULL); dv NULL = nothing below the subject layer (then du, d_il_w, d_il_b must be NULL).
static int sensor_chain_bwd(const float* dx0, const float* meg, const float* il_w, const float* subj_w, const int* subject,
                            const float* u, const float* v, const int* subj_order, const int* subj_off, const int* rec_order,
                            const int* rec_off, int B, int C, int T, int O, int IL, int D, int ld_x0, int S, int R, float* dv,
                            float* du, float* d_subj_w, float* d_il_w, float* d_il_b, float* d_weights, float* workspace,
                            long long workspace_floats, bool det, bm_stream_t stream) {
    BM_CHECK_ARG(dx0 && ld_x0 >= D);
    BM_CHECK_ARG((dv || !(du || d_il_w || d_il_b)) && (du || !d_weights));
    BM_CHECK_ARG(!d_weights || (meg && rec_order && rec_off));
    // a short workspace is refused before any stage is enqueued, not after the subject-layer backward has written dv
    if (det && (d_il_w || d_il_b)) BM_CHECK_WS(bm_initial_linear_bwd_det_workspace(B, T, O, IL));
    // the subject and sensor-mix gradients reduce each segment inside one CTA: already fixed-order
    int rc = 0;
    if (dv || d_subj_w)
        rc = bm_subject_layers_bwd(dx0, ld_x0, v, IL, subj_w, subject, subj_order, subj_off, B, T, IL, D, S, IL, dv, d_subj_w,
                                   stream);
    if (!rc && (du || d_il_w || d_il_b))
        rc = det ? bm_initial_linear_bwd_det(dv, IL, u, O, il_w, B, T, O, IL, O, du, d_il_w, d_il_b, workspace,
                                             workspace_floats, stream)
                 : bm_initial_linear_bwd(dv, IL, u, O, il_w, B, T, O, IL, O, du, d_il_w, d_il_b, stream);
    if (!rc && d_weights) rc = bm_sensor_mix_bwd(du, O, meg, rec_order, rec_off, B, C, T, O, R, d_weights, stream);
    return rc;
}

extern "C" int bm_sensor_chain_bwd(const float* dx0, const float* meg, const float* il_w, const float* subj_w,
                                   const int* subject, const float* u, const float* v, const int* subj_order,
                                   const int* subj_off, const int* rec_order, const int* rec_off, int B, int C,
                                   int T, int O, int IL, int D, int ld_x0, int S, int R, float* dv, float* du,
                                   float* d_subj_w, float* d_il_w, float* d_il_b, float* d_weights,
                                   bm_stream_t stream) {
    return sensor_chain_bwd(dx0, meg, il_w, subj_w, subject, u, v, subj_order, subj_off, rec_order, rec_off, B, C, T, O, IL,
                            D, ld_x0, S, R, dv, du, d_subj_w, d_il_w, d_il_b, d_weights, nullptr, 0, false, stream);
}

extern "C" long long bm_sensor_chain_bwd_det_workspace(int B, int T, int O, int IL) {
    return bm_initial_linear_bwd_det_workspace(B, T, O, IL);
}
extern "C" int bm_sensor_chain_bwd_det(const float* dx0, const float* meg, const float* il_w, const float* subj_w,
                                       const int* subject, const float* u, const float* v, const int* subj_order,
                                       const int* subj_off, const int* rec_order, const int* rec_off, int B, int C,
                                       int T, int O, int IL, int D, int ld_x0, int S, int R, float* dv, float* du,
                                       float* d_subj_w, float* d_il_w, float* d_il_b, float* d_weights, float* workspace,
                                       long long workspace_floats, bm_stream_t stream) {
    return sensor_chain_bwd(dx0, meg, il_w, subj_w, subject, u, v, subj_order, subj_off, rec_order, rec_off, B, C, T, O, IL,
                            D, ld_x0, S, R, dv, du, d_subj_w, d_il_w, d_il_b, d_weights, workspace, workspace_floats, true,
                            stream);
}

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

// amax_out (nullable, every producer below): a device float that receives max |output| -- the scale source of the F16-pipe
// conv that consumes the tensor next (bm_tc_conv1d_f16's x_amax), folded into the producing kernel instead of a bm_amax pass
static int amax_begin(float* amax_out, cudaStream_t st) {
    if (amax_out) BM_CUDA(cudaMemsetAsync(amax_out, 0, sizeof(float), st));
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
        return tc::launch_wgrad_tc(G, cand, 1, Bc, Bn, (int)KT, (int)KT, 1, 1, dest, dest, passes, st);   // direct mode
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
        int rc = tc::launch_wgrad_tc(G, est, 1, Bn, Bc, (int)KT, (int)KT, 1, 1, dcand, dcand, passes, st);   // direct
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

// =================================================================================================
// Stand-alone ConvSequence epilogues (the forms of epi_fwd / epi_bwd above) + candidate-side ClipLoss gradient (SURVEY 8(f)
// row 3: DeepMel)
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

// =================================================================================================
// Retrieval evaluation (SURVEY 8(f) row 1)
// =================================================================================================
extern "C" int bm_retrieval_topk(const float* vals, long long ld, int Bn, int n_cols, const float* own_values,
                                 int own_col, int is_prob, int k, const long long* labels,
                                 const long long* own_labels, const long long* targets, long long* top_idx,
                                 float* top_prob, int* hit, float* soft, float* row_max, float* row_sum,
                                 bm_stream_t stream) {
    BM_CHECK_ARG(vals && Bn > 0 && n_cols > 0 && ld >= n_cols && k >= 0);
    BM_CHECK_ARG(!own_values || (own_col >= 0 && own_col < n_cols));
    BM_CHECK_ARG(!own_labels || (labels && own_col >= 0 && own_col < n_cols));
    BM_CHECK_ARG(!(hit || soft) || (labels && targets));
    BM_CHECK_ARG(k == 0 || top_idx || top_prob || hit);
    int threads = n_cols >= 4096 ? 512 : 256;
    retrieval_topk_kernel<<<Bn, threads, 0, ST(stream)>>>(vals, ld, n_cols, own_values, own_col, is_prob, k, labels,
                                                          own_labels, targets, top_idx, top_prob, hit, soft, row_max,
                                                          row_sum);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_retrieval_probs(const float* scores, long long ld, int Bn, int n_cols, float* probs,
                                  bm_stream_t stream) {
    BM_CHECK_ARG(scores && probs && Bn > 0 && n_cols > 0 && ld >= n_cols);
    softmax_rows_ld_kernel<<<Bn, 256, 0, ST(stream)>>>(scores, ld, n_cols, probs);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_retrieval_vocab_probs(const float* scores, long long ld, int Bn, const float* own_scores,
                                        const float* row_max, const float* row_sum, const int* perm, const int* seg,
                                        int V, const int* own_word, float* vocab, bm_stream_t stream) {
    BM_CHECK_ARG(scores && row_max && row_sum && perm && seg && vocab && Bn > 0 && V > 0);
    BM_CHECK_ARG(!own_scores || own_word);
    vocab_probs_kernel<<<Bn, 256, 0, ST(stream)>>>(scores, ld, own_scores, row_max, row_sum, perm, seg, V, own_word,
                                                   vocab);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_rowdot_scaled(const float* a, const float* c, int Bn, long long K, float* own,
                                bm_stream_t stream) {
    BM_CHECK_ARG(a && c && own && Bn > 0 && K > 0);
    rowdot_scaled_kernel<<<Bn, 512, 0, ST(stream)>>>(a, c, K, own);
    BM_CHECK_LAUNCH();
    return 0;
}

// =================================================================================================
// Batch preparation (SURVEY 8(f) row 2)
// =================================================================================================
extern "C" int bm_scale_clamp_crop(const float* x, const int* slot, const float* center, const float* scale, int B,
                                   int C, int T, int t0, int T_out, float limit, int clip, int inverse, float* y,
                                   unsigned int* peak_bits, bm_stream_t stream) {
    BM_CHECK_ARG(x && center && scale && y && B > 0 && C > 0 && T > 0);
    BM_CHECK_ARG(t0 >= 0 && T_out > 0 && t0 + T_out <= T);
    BM_CHECK_ARG(!clip || limit >= 0.f);
    cudaStream_t st = ST(stream);
    if (peak_bits) BM_CUDA(cudaMemsetAsync(peak_bits, 0, sizeof(unsigned) * B, st));
    long long rows = (long long)B * C;
    long long blocks = (rows + 7) / 8;                       // 8 warps (rows) per block
    long long cap = (long long)num_sms() * 8;                // one full wave of 2048-thread SMs, grid-stride beyond
    if (blocks > cap) blocks = cap;
    scale_clamp_crop_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, slot, center, scale, B, C, T, t0, T_out, limit, clip,
                                                             inverse, y, peak_bits);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_reject_compact(const unsigned int* peak_bits, const unsigned char* mask, long long mask_elems,
                                 float limit, int B, unsigned char* keep, int* keep_rows, int* n_keep,
                                 bm_stream_t stream) {
    BM_CHECK_ARG(peak_bits && keep && keep_rows && n_keep && B > 0);
    BM_CHECK_ARG(!mask || mask_elems > 0);
    reject_compact_kernel<<<1, 1024, 0, ST(stream)>>>(peak_bits, mask, mask_elems, limit, B, keep, keep_rows, n_keep);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_gather_rows(const float* x, const int* rows, int n_rows, long long row_elems, float* y,
                              bm_stream_t stream) {
    BM_CHECK_ARG(x && rows && y && n_rows > 0 && row_elems > 0);
    gather_rows_kernel<<<ew_grid((long long)n_rows * row_elems), 256, 0, ST(stream)>>>(x, rows, n_rows, row_elems, y);
    BM_CHECK_LAUNCH();
    return 0;
}

extern "C" int bm_scatter_rows(const float* x, const int* rows, int n_rows, long long row_elems, float* y,
                               bm_stream_t stream) {
    BM_CHECK_ARG(x && rows && y && n_rows > 0 && row_elems > 0);
    scatter_rows_kernel<<<ew_grid((long long)n_rows * row_elems), 256, 0, ST(stream)>>>(x, rows, n_rows, row_elems, y);
    BM_CHECK_LAUNCH();
    return 0;
}

// =================================================================================================
// tensor-core (wgmma) versions of K3/K4
// =================================================================================================
extern "C" int bm_tc_conv_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    return tc::conv_tc_supported(T, Cin, Ntot, Kw, glu) ? 1 : 0;
}

extern "C" int bm_tc_weight_split(const float* w, int Cout, int Cin, int Kw, float* f_hi, float* f_lo, float* g_hi,
                                  float* g_lo, bm_stream_t stream) {
    BM_CHECK_ARG(w && Cout > 0 && Cin > 0 && Kw > 0);
    BM_CHECK_ARG((f_hi || g_hi) && !(f_lo && !f_hi) && !(g_lo && !g_hi));
    tc::weight_split_kernel<<<ew_grid((long long)Cout * Cin * Kw), 256, 0, ST(stream)>>>(w, f_hi, f_lo, g_hi, g_lo,
                                                                                       Cout, Cin, Kw);
    BM_CHECK_LAUNCH();
    return 0;
}

// passes = 1 (the _tf32 form): w_hi alone is read, w_lo may be NULL; TC_BF16 (the _bf16 form): w_hi + w_lo is read,
// w_lo may be NULL (w_hi then holds the raw fp32 weights)
static int tc_conv1d(int passes, const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* addend,
                     int B, int T, int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                     float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(stats == nullptr);      // BatchNorm statistics in the epilogue: bm_tc_conv1d_persistent / bm_tc_conv1d_f16
    BM_CHECK_ARG(x && w_hi && (w_lo || passes != 3) && B > 0 && T > 0 && dilation >= 1 && (sign == 1 || sign == -1));
    BM_CHECK_ARG(glu ? (glu_out != nullptr) : (y != nullptr));
    BM_CHECK_ARG(B <= 65535);
    BM_CHECK_ARG(!(glu && (act || out_tmajor || aux)));
    BM_CHECK_ARG(tc::conv_tc_supported(T, Cin, Ntot, Kw, glu));
    tc::ConvOp o = tc::conv_op_defaults();
    o.x = x; o.w = w_hi; o.w_lo32 = passes == 1 ? nullptr : w_lo; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = Kw; o.dilation = dilation; o.sign = sign; o.glu = glu;
    o.bias = bias; o.addend = addend; o.y = y; o.aux = aux; o.glu_out = glu_out; o.act = act; o.out_tmajor = out_tmajor;
    o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_conv1d, tc_conv1d,
            (const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* addend, int B, int T,
             int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor, float* y, float* aux,
             float* glu_out, double* stats, int* status, bm_stream_t stream),
            (x, w_hi, w_lo, bias, addend, B, T, Cin, Ntot, Kw, dilation, sign, glu, act, out_tmajor, y, aux, glu_out, stats,
             status, stream))

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

// y = x * mask[c] over [B, C, T] (SimpleConv's subsample_meg_channels, simpleconv.py:97-102,200-203); y may alias x
extern "C" int bm_channel_mask(const float* x, const float* mask, int B, int C, int T, float* y, bm_stream_t stream) {
    BM_CHECK_ARG(x && mask && y && B > 0 && C > 0 && T > 0);
    const long long total = (long long)B * C * T;
    channel_mask_kernel<<<ew_grid(total), 256, 0, ST(stream)>>>(x, mask, y, C, T, total);
    BM_CHECK_LAUNCH();
    return 0;
}

// [Z, N, T] (channel-major) -> [Z, T, N] (channels-last)
extern "C" int bm_transpose_nt(const float* in, int Z, int N, int T, float* out, bm_stream_t stream) {
    BM_CHECK_ARG(in && out && Z > 0 && N > 0 && T > 0 && Z <= 65535);
    dim3 grid((T + 31) / 32, (N + 31) / 32, Z);
    transpose_nt_kernel<<<grid, dim3(32, 8), 0, ST(stream)>>>(in, out, N, T, N, N);
    BM_CHECK_LAUNCH();
    return 0;
}

// same with an output row stride ld_out >= N; the pad columns N..ld_out-1 are written as zeros
extern "C" int bm_transpose_nt_ld(const float* in, int Z, int N, int T, int ld_out, float* out, bm_stream_t stream) {
    BM_CHECK_ARG(in && out && Z > 0 && N > 0 && T > 0 && Z <= 65535 && ld_out >= N);
    dim3 grid((T + 31) / 32, (ld_out + 31) / 32, Z);
    transpose_nt_kernel<<<grid, dim3(32, 8), 0, ST(stream)>>>(in, out, N, T, ld_out, ld_out);
    BM_CHECK_LAUNCH();
    return 0;
}

// channel join / split (channel_join.cuh): the host describes each source once, the segments are laid out by column
namespace {
struct JoinSrc { float* p; int C, ld, cm, col; };

int channel_join_launch(bool split, float* packed, int B, int T, int Cp, int n, const JoinSrc* src, cudaStream_t st) {
    BM_CHECK_ARG(packed && B > 0 && T > 0 && Cp > 0 && n >= 1 && n <= 4 && B <= 65535);
    int order[4];
    for (int i = 0; i < n; ++i) {
        const JoinSrc& s = src[i];
        BM_CHECK_ARG(s.C > 0 && s.col >= 0 && s.col + s.C <= Cp && (s.cm == 0 || s.cm == 1));
        BM_CHECK_ARG(split || s.p);                               // a NULL split destination is not wanted
        BM_CHECK_ARG(!s.p || (s.cm ? s.ld >= T : s.ld >= s.C));
        order[i] = i;
    }
    std::sort(order, order + n, [&](int x, int y) { return src[x].col < src[y].col; });
    const bool packed_vec = (reinterpret_cast<uintptr_t>(packed) & 15) == 0 && Cp % 4 == 0;
    JoinArgs a{};
    a.T = T; a.Cp = Cp; a.packed = packed;
    int tiles = 0, end = 0;
    auto add = [&](float* p, int C, int ld, int cm, int col) {
        JoinSeg& g = a.s[a.n++];
        g.p = p; g.C = C; g.ld = ld; g.cm = cm; g.col = col; g.tile0 = tiles;
        g.vec = !cm && packed_vec && C % 4 == 0 && col % 4 == 0 && (!p || (ld % 4 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0));
        tiles += (C + (g.vec ? 128 : 32) - 1) / (g.vec ? 128 : 32);
    };
    for (int k = 0; k < n; ++k) {
        const JoinSrc& s = src[order[k]];
        BM_CHECK_ARG(s.col >= end);                              // column ranges do not overlap
        if (!split && s.col > end) add(nullptr, s.col - end, 0, 0, end);
        if (s.p) add(s.p, s.C, s.ld, s.cm, s.col);
        end = s.col + s.C;
    }
    if (!split && end < Cp) add(nullptr, Cp - end, 0, 0, end);
    if (a.n == 0) return 0;                                      // a split with every destination NULL
    dim3 grid(tiles, (T + 31) / 32, B);
    if (split) channel_join_kernel<true><<<grid, dim3(32, 8), 0, st>>>(a);
    else channel_join_kernel<false><<<grid, dim3(32, 8), 0, st>>>(a);
    BM_CHECK_LAUNCH();
    return 0;
}
}  // namespace

extern "C" int bm_channel_join(int B, int T, int Cp, int n, const float* src0, int C0, int ld0, int cm0, int col0,
                               const float* src1, int C1, int ld1, int cm1, int col1, const float* src2, int C2, int ld2,
                               int cm2, int col2, const float* src3, int C3, int ld3, int cm3, int col3, float* dst,
                               bm_stream_t stream) {
    const JoinSrc src[4] = {{const_cast<float*>(src0), C0, ld0, cm0, col0}, {const_cast<float*>(src1), C1, ld1, cm1, col1},
                            {const_cast<float*>(src2), C2, ld2, cm2, col2}, {const_cast<float*>(src3), C3, ld3, cm3, col3}};
    return channel_join_launch(false, dst, B, T, Cp, n, src, ST(stream));
}

extern "C" int bm_channel_split(const float* src, int B, int T, int Cp, int n, float* dst0, int C0, int ld0, int cm0,
                                int col0, float* dst1, int C1, int ld1, int cm1, int col1, float* dst2, int C2, int ld2,
                                int cm2, int col2, float* dst3, int C3, int ld3, int cm3, int col3, bm_stream_t stream) {
    const JoinSrc dst[4] = {{dst0, C0, ld0, cm0, col0}, {dst1, C1, ld1, cm1, col1}, {dst2, C2, ld2, cm2, col2},
                            {dst3, C3, ld3, cm3, col3}};
    return channel_join_launch(true, const_cast<float*>(src), B, T, Cp, n, dst, ST(stream));
}

extern "C" int bm_check_all_true(const unsigned char* mask, long long n, int code, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(status && n >= 0 && (mask || n == 0) && code != 0);
    if (n == 0) return 0;
    const bool vec = aligned16(mask);
    check_all_true_kernel<<<ew_grid(vec ? (n + 15) / 16 : n), 256, 0, ST(stream)>>>(mask, n, vec, code, status);
    BM_CHECK_LAUNCH();
    return 0;
}

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

// weight gradient of a (dilated) conv / pointwise layer on the tensor cores: dW[m][n][tap] = sum_{b,t} dY[b,t,m] X[b,t+s,n]
extern "C" int bm_tc_wgrad_supported(int M, int N) { return tc::wgrad_tc_supported(M, N) ? 1 : 0; }
extern "C" long long bm_tc_wgrad_workspace(int B, int M, int N, int Kw) {
    return (long long)tc::wgrad_workspace_floats(B, M, N, Kw);
}
static int tc_wgrad(int passes, const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                    float* workspace, float* dw, float* dbias, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(dy && x && workspace && dw && B > 0 && T > 0 && Kw >= 1 && Kw <= 3 && dilation >= 1);
    BM_CHECK_ARG(tc::wgrad_tc_supported(M, N) && Ntrue > 0 && Ntrue <= N);
    return tc::launch_wgrad_tc(dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, passes, ST(stream), dbias);
}
BM_TC_FORMS(bm_tc_wgrad, tc_wgrad,
            (const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation, float* workspace,
             float* dw, float* dbias, int* status, bm_stream_t stream),
            (dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, dbias, status, stream))

// weight gradient of a k-tap conv (csrc/tc_wgradp.cuh): output rows = (tap, x channel), reduction over the
// flattened rows; no bias gradient (use bm_col_sum on dy where the layer's bias gradient is not exactly zero)
extern "C" int bm_tc_wgrad_conv_supported(int T, int M, int N, int Kw) {
    return tc::wgradp_supported(T, M, N, Kw) ? 1 : 0;
}
extern "C" long long bm_tc_wgrad_conv_workspace(int B, int T, int M, int N, int Kw) {
    return (long long)tc::wgradp_workspace_floats(B, T, M, N, Kw);
}
static int tc_wgrad_conv(int passes, const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw,
                         int dilation, float* workspace, float* dw, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(dy && x && workspace && dw && B > 0 && T > 0 && dilation >= 1);
    BM_CHECK_ARG(tc::wgradp_supported(T, M, N, Kw) && Ntrue > 0 && Ntrue <= N);
    return tc::launch_wgrad_pp(dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, passes, status, ST(stream));
}
BM_TC_FORMS(bm_tc_wgrad_conv, tc_wgrad_conv,
            (const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation, float* workspace,
             float* dw, int* status, bm_stream_t stream),
            (dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, status, stream))

// the same weight gradient for callers that hold the operands' amax (csrc/tc_wgradp.cuh): dy_amax / x_amax = device floats with max |dy|, max |x|
// (bm_amax, or the amax_out of the kernels that produced the tensors); same shape gate and workspace as bm_tc_wgrad_conv
extern "C" int bm_tc_wgrad_conv_f16(const float* dy, const float* dy_amax, const float* x, const float* x_amax, int B, int T,
                                    int M, int N, int Ntrue, int Kw, int dilation, float* workspace, float* dw, int* status,
                                    bm_stream_t stream) {
    BM_CHECK_ARG(dy && dy_amax && x && x_amax && workspace && dw && B > 0 && T > 0 && dilation >= 1);
    BM_CHECK_ARG(tc::wgradp_supported(T, M, N, Kw) && Ntrue > 0 && Ntrue <= N);
    return tc::launch_wgrad_pp(dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, 3, status, ST(stream));
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

extern "C" int bm_tc_conv1d_persistent_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    return tc::conv_halves_supported(T, Cin, Ntot, Kw, glu) ? 1 : 0;
}
// w_raw = the RAW fp32 weights re-laid K-major [Kw][Ntot][Cin] (bm_tc_weight_split with f_lo / g_lo = NULL);
// accumulate=1: y += conv (in place)
static int tc_conv1d_persistent(int passes, const float* x, const float* w_raw, const float* bias, int accumulate, int B,
                                int T, int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                                float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(x && w_raw && B > 0 && T > 0 && dilation >= 1 && (sign == 1 || sign == -1));
    BM_CHECK_ARG(glu ? (glu_out != nullptr) : (y != nullptr));
    BM_CHECK_ARG(tc::conv_halves_supported(T, Cin, Ntot, Kw, glu));
    if (int rc = tc::conv_halves_epilogue_check(Ntot, glu, act, out_tmajor, accumulate, aux, stats, __func__)) return rc;
    tc::ConvOp o = tc::conv_op_defaults();
    o.x = x; o.w = w_raw; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = Kw; o.dilation = dilation; o.sign = sign; o.glu = glu;
    o.bias = bias; o.addend = accumulate ? y : nullptr; o.y = y; o.aux = act ? aux : nullptr; o.glu_out = glu_out;
    o.act = act; o.out_tmajor = out_tmajor; o.stats = stats; o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_conv1d_persistent, tc_conv1d_persistent,
            (const float* x, const float* w_raw, const float* bias, int accumulate, int B, int T, int Cin, int Ntot, int Kw,
             int dilation, int sign, int glu, int act, int out_tmajor, float* y, float* aux, float* glu_out, double* stats,
             int* status, bm_stream_t stream),
            (x, w_raw, bias, accumulate, B, T, Cin, Ntot, Kw, dilation, sign, glu, act, out_tmajor, y, aux, glu_out, stats,
             status, stream))

// ---- the same conv with fp16-piece weights: fp32 weights as two fp16 pieces of a power-of-two-scaled tensor.  bm_amax
// writes the largest magnitude of a tensor into a device float; bm_f16_split prepares the weights (w_raw [Kw][Ntot][Cin] ->
// fp16 hi / lo copies of w_raw * scale(amax)); the kernel scales x itself.
extern "C" int bm_amax(const float* x, long long n, float* amax, bm_stream_t stream) {
    BM_CHECK_ARG(x && amax && n > 0);
    return tc::launch_amax(x, n, amax, ST(stream));
}
extern "C" int bm_f16_split(const float* src, long long n, const float* amax, void* hi, void* lo, bm_stream_t stream) {
    BM_CHECK_ARG(src && amax && hi && lo && n > 0);
    return tc::launch_f16_split(src, n, amax, hi, lo, ST(stream));
}
extern "C" int bm_tc_weight_split_f16(const float* w, const float* w_amax, int Cout, int Cin, int Kw, void* f_hi, void* f_lo,
                                      void* g_hi, void* g_lo, bm_stream_t stream) {
    BM_CHECK_ARG(w && w_amax && Cout > 0 && Cin > 0 && Kw > 0);
    BM_CHECK_ARG((f_hi || g_hi) && (!f_hi == !f_lo) && (!g_hi == !g_lo));
    tc::weight_split_f16_kernel<<<ew_grid((long long)Cout * Cin * Kw), 256, 0, ST(stream)>>>(
        w, w_amax, reinterpret_cast<__half*>(f_hi), reinterpret_cast<__half*>(f_lo), reinterpret_cast<__half*>(g_hi),
        reinterpret_cast<__half*>(g_lo), Cout, Cin, Kw);
    BM_CHECK_LAUNCH();
    return 0;
}
extern "C" int bm_tc_conv1d_f16(const float* x, const float* x_amax, const void* w_hi, const void* w_lo, const float* w_amax,
                                const float* bias, int accumulate, int B, int T, int Cin, int Ntot, int Kw, int dilation,
                                int sign, int glu, int act, int out_tmajor, float* y, float* aux, float* glu_out,
                                double* stats, float* amax_out, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(x && x_amax && w_hi && w_lo && w_amax && B > 0 && T > 0 && dilation >= 1 && (sign == 1 || sign == -1));
    BM_CHECK_ARG(glu ? (glu_out != nullptr) : (y != nullptr));
    BM_CHECK_ARG(tc::conv_halves_supported(T, Cin, Ntot, Kw, glu));
    BM_CHECK_ARG(!amax_out || ((glu || act) && !out_tmajor));      // the outputs another conv consumes: GLU out, GELU out
    if (int rc = amax_begin(amax_out, ST(stream))) return rc;
    if (int rc = tc::conv_halves_epilogue_check(Ntot, glu, act, out_tmajor, accumulate, aux, stats, __func__)) return rc;
    tc::ConvOp o = tc::conv_op_defaults();          // passes = 3: the fp16 pieces have no single-pass form
    o.x = x; o.w_hi = reinterpret_cast<const __half*>(w_hi); o.w_lo = reinterpret_cast<const __half*>(w_lo); o.w_amax = w_amax;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = Kw; o.dilation = dilation; o.sign = sign; o.glu = glu;
    o.bias = bias; o.addend = accumulate ? y : nullptr; o.y = y; o.aux = act ? aux : nullptr; o.glu_out = glu_out;
    o.act = act; o.out_tmajor = out_tmajor; o.stats = stats; o.out_amax = reinterpret_cast<unsigned int*>(amax_out);
    o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}

// pointwise (1x1) contraction with a per-sample weight set (SubjectLayers.forward / its data gradient, common.py:55-58):
//   y[b,t,n] = sum_k x[b,t,k] W[wsel[b]][n][k];  w_hi/w_lo are the tf32-split K-major weight sets [S][Ntot][Cin]
static int tc_pointwise_sel(int passes, const float* x, const float* w_hi, const float* w_lo, const int* wsel, int n_sets,
                            int B, int T, int Cin, int Ntot, float* y, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(x && w_hi && (w_lo || passes != 3) && wsel && y && n_sets > 0 && B > 0 && B <= 65535 && T > 0);
    BM_CHECK_ARG(tc::conv_tc_supported(T, Cin, Ntot, 1, 0));
    tc::ConvOp o = tc::conv_op_defaults();
    o.x = x; o.w = w_hi; o.w_lo32 = passes == 1 ? nullptr : w_lo; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = 1; o.dilation = 1; o.sign = 1;
    o.n_wsets = n_sets; o.wsel = wsel; o.y = y; o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_pointwise_sel, tc_pointwise_sel,
            (const float* x, const float* w_hi, const float* w_lo, const int* wsel, int n_sets, int B, int T, int Cin,
             int Ntot, float* y, int* status, bm_stream_t stream),
            (x, w_hi, w_lo, wsel, n_sets, B, T, Cin, Ntot, y, status, stream))

// data gradient of the sensor mix on the tensor cores (ChannelMerger, common.py:358):
//   dmeg[b,c,t] = mask[c] sum_o du[b,t,o] W[wsel[b]][c][o], c < C;  w_hi / w_lo: tf32-split transposed weight sets [S][Cp][Op]
static int tc_sensor_mix_bwd_data(int passes, const float* du, const float* w_hi, const float* w_lo, const int* wsel,
                                  int n_sets, const float* mask, int B, int T, int Op, int Cp, int C, float* dmeg, int* status,
                                  bm_stream_t stream) {
    BM_CHECK_ARG(du && w_hi && (w_lo || passes != 3) && wsel && dmeg && n_sets > 0 && B > 0 && T > 0 && C > 0 && C <= Cp);
    BM_CHECK_ARG(tc::conv_tc_supported(T, Op, Cp, 1, 0));
    tc::SensorMixBwdOp o;
    memset(&o, 0, sizeof(o));
    o.x = du; o.w = w_hi; o.w_lo32 = passes == 1 ? nullptr : w_lo; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Op; o.Ntot = Cp; o.taps = 1; o.dilation = 1; o.sign = 1;
    o.n_wsets = n_sets; o.wsel = wsel; o.y = dmeg; o.err = status; o.C = C; o.mask = mask;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_sensor_mix_bwd_data, tc_sensor_mix_bwd_data,
            (const float* du, const float* w_hi, const float* w_lo, const int* wsel, int n_sets, const float* mask, int B,
             int T, int Op, int Cp, int C, float* dmeg, int* status, bm_stream_t stream),
            (du, w_hi, w_lo, wsel, n_sets, mask, B, T, Op, Cp, C, dmeg, status, stream))

// per-group pointwise weight gradient (SubjectLayers: dM[s] = sum over the samples of subject s), tensor cores:
//   out[g][m][n] = sum_{b in group g} sum_t dy[b,t,m] x[b,t,n];  out is [G][ceil(M/128)*128][N]
static int tc_wgrad_grouped(int passes, const float* dy, const float* x, const int* order, const int* seg_off, int G, int B,
                            int T, int M, int N, float* out, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(dy && x && order && seg_off && out && G > 0 && B > 0 && T > 0);
    BM_CHECK_ARG(tc::wgrad_tc_supported(M, N));
    return tc::launch_wgrad_tc_grouped(dy, x, order, seg_off, G, B, T, M, N, out, passes, ST(stream));
}
BM_TC_FORMS(bm_tc_wgrad_grouped, tc_wgrad_grouped,
            (const float* dy, const float* x, const int* order, const int* seg_off, int G, int B, int T, int M, int N,
             float* out, int* status, bm_stream_t stream),
            (dy, x, order, seg_off, G, B, T, M, N, out, status, stream))

// ---- K1 pieces, for callers that run the two attention contractions on the tensor cores -------------------------
extern "C" int bm_fourier_emb(const float* positions, const float* freq, int R, int C, int P, float* emb,
                              bm_stream_t stream) {
    BM_CHECK_ARG(positions && freq && emb && R > 0 && C > 0 && P > 0 && P % 2 == 0);
    int n = 0;
    while ((n + 1) * (n + 1) * 2 <= P) ++n;
    BM_CHECK_ARG(n * n * 2 == P);
    fourier_emb_kernel<<<ew_grid((long long)R * C * n * n), 256, 0, ST(stream)>>>(positions, freq, 0.2f, R * C, n, emb);
    BM_CHECK_LAUNCH();
    return 0;
}
// in-place: weights[r][o][:] = softmax_c(scores + mask), mask = -inf on INVALID / banned sensors (common.py:339-357)
extern "C" int bm_masked_softmax(float* weights, const float* positions, const float* ban_centre, float radius, int R,
                                 int O, int C, bm_stream_t stream) {
    BM_CHECK_ARG(weights && positions && R > 0 && O > 0 && C > 0);
    int rows = R * O;
    masked_softmax_kernel<<<(rows + 7) / 8, 256, 0, ST(stream)>>>(weights, positions, ban_centre, radius, -0.1f, R, O, C);
    BM_CHECK_LAUNCH();
    return 0;
}
// dscores = w * (dw - sum_c w dw), rows of length C
extern "C" int bm_softmax_bwd(const float* weights, const float* dweights, long long rows, int C, float* dscores,
                              bm_stream_t stream) {
    BM_CHECK_ARG(weights && dweights && dscores && rows > 0 && C > 0);
    softmax_bwd_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, ST(stream)>>>(weights, dweights, dscores, (int)rows, C);
    BM_CHECK_LAUNCH();
    return 0;
}
