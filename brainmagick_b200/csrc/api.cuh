// Plumbing shared by the C-ABI entry points of every *_api.cu (see include/bm_b200.h for the contract): the stream cast,
// the TF32 / bf16 forms, the workspace check, the deterministic reductions, and the launchers of kernels that one
// subsystem owns and others call.  Each of those launchers is defined once, beside its kernel.
#pragma once
#include <algorithm>
#include "../../include/bm_b200.h"
#include "common.cuh"
#include "gemm_simt.cuh"

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

#define BM_CHECK_WS(need)                                                                              \
    BM_CHECK_ARG(workspace && workspace_floats >= (need) && (reinterpret_cast<uintptr_t>(workspace) & 7) == 0)

namespace bm {

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
constexpr int COLSUM_RPB = 256;
inline long long blocks_of(long long rows, int rpb) { return (rows + rpb - 1) / rpb; }
inline long long colsum_ws_floats(long long rows, int C) { return blocks_of(rows, COLSUM_RPB) * C; }
// batch segments of the split weight-gradient GEMMs (the atomic form's count); planes = segments x output elements
inline int wgrad_segments(int B, int tiles) {
    const int zchunk = (B + pick_chunks(B, tiles) - 1) / pick_chunks(B, tiles);
    return (B + zchunk - 1) / zchunk;
}
inline long long planes_floats(int B, int M, int N, int taps = 1) {
    return (long long)wgrad_segments(B, tiles_of(M, N) * taps) * M * N * taps;
}

// out[c] = sum_{r < n} part[r][c] by reduce_rows_kernel, for T = float and double (convseq_api.cu)
template <class T>
int reduce_rows(const T* part, long long n, int W, T* out, cudaStream_t st);

// out[c] = sum_r X[r*ld + c] over `rows` rows through the colsum_ws_floats(rows, C) partials `part` (convseq_api.cu)
int colsum(const float* X, long long rows, int C, int ld, float* part, float* out, cudaStream_t st);

// the split GEMM g (atomic form: g.D inside the output `out` of `elems` elements, g.atomic = 1) with one partial plane per
// segment: segment s writes part[s * elems + (g.D - out) + ...]; sum_planes adds the planes in segment order
inline cudaError_t launch_gemm_planes(GemmP g, const float* out, long long elems, float* part, cudaStream_t st) {
    g.D = part + (g.D - out);
    g.ldd_z = elems;
    g.atomic = 0;
    return launch_gemm(g, st);
}
inline int sum_planes(const float* part, int nseg, long long elems, float* out, cudaStream_t st) {
    return reduce_rows(part, (long long)nseg, (int)elems, out, st);
}

// amax_out (nullable, every producer that takes it): a device float that receives max |output| -- the scale source of the
// F16-pipe conv that consumes the tensor next (bm_tc_conv1d_f16's x_amax), folded into the producing kernel instead of a
// bm_amax pass
inline int amax_begin(float* amax_out, cudaStream_t st) {
    if (amax_out) BM_CUDA(cudaMemsetAsync(amax_out, 0, sizeof(float), st));
    return 0;
}

namespace tc {
// tensor-core launchers that tc_conv_api.cu owns and the epilogue / CLIP entry points call
int launch_amax(const float* x, long long n, float* cell, cudaStream_t st);                             // tc_conv.cuh
bool wgrad_tc_supported(int M, int N);                                                                  // tc_wgrad.cuh
int launch_wgrad_tc(const float* dY, const float* X, int B, int T, int M, int N, int Ntrue, int taps, int dilation,
                    float* ws, float* dW, int passes, cudaStream_t st, float* dbias);
}  // namespace tc

}  // namespace bm
