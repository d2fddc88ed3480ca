// C-ABI entry points of the encoder's front on the FP32-FMA path: spatial attention (K1), sensor mix, initial linear,
// subject layers and the sensor chain (K2), and the K1 pieces (see include/bm_b200.h for the contract).
#include "api.cuh"
#include "elementwise.cuh"
#include "front.cuh"

using namespace bm;

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
