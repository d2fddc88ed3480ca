// C-ABI entry points of batch preparation, retrieval evaluation and the layout kernels: gathers, channel masks,
// transposes, channel join / split (see include/bm_b200.h for the contract).
#include "api.cuh"
#include "prep.cuh"
#include "retrieval.cuh"
#include "channel_join.cuh"

using namespace bm;

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
