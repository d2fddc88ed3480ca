// Generic FP32-FMA tiled GEMM: the workhorse for every *small* contraction of the hot path (spatial attention, sensor
// chain, per-subject layers, parameter gradients) and for the shapes outside the tensor-core shape gates (the small unit-test
// models).
//
//   D[g][m][n] (+)= epi( sum_{z in seg(g)} sum_{tap} sum_{k in krange} A(z, m + a_shift_m[tap], k) * B(bz(z), tap, n, k + b_shift_k[tap]) )
//
// * strides are in elements and arbitrary; `a_mcontig` / `b_ncontig` only pick the coalescing-friendly
//   thread->element mapping of the tile loaders.
// * rows of A shifted outside [0,M) and k of B shifted outside [0,K) read 0: that is the zero padding of the
//   dilated Conv1d (bm/models/common.py:112-114) without materialising padded tensors.
// * segments: either fixed chunks of `zchunk` items, or CSR (`seg_off`, `zlist`) for per-subject /
//   per-recording reductions (dM[s] = sum over samples of subject s, appendix A.2 of SURVEY.md).
// * epilogue: column scale, bias, addend (skip/residual gradient), pre-activation store, exact GELU, GLU
//   pairing of column n with n + N/2 (common.py:133-138), per-column (sum, sumsq) in fp64 for train-mode
//   BatchNorm statistics (common.py:118-119), atomic accumulation for split reductions.
#pragma once
#include "common.cuh"

namespace bm {

struct GemmP {
    int M, N, K, taps;
    int Z, zchunk, nseg, ksplit, kchunk;
    const int* seg_off;
    const int* zlist;
    const float* A;
    long long lda_z, lda_m, lda_k;
    int a_mcontig;
    int a_shift_m[3];
    const float* B;
    long long ldb_z, ldb_tap, ldb_n, ldb_k;
    int b_ncontig;
    const int* bsel;
    int b_shift_k[3];
    float* D;
    long long ldd_z, ldd_m, ldd_n;
    int atomic;
    const float* bias;
    const float* colscale;
    const float* addend;
    float* aux;
    int act;
    int glu;
    float* glu_out;
    long long ldg_z, ldg_m, ldg_n;
    double* stats;
};

inline GemmP gemm_defaults() {
    GemmP p;
    memset(&p, 0, sizeof(p));
    p.taps = 1;
    p.Z = 1;
    p.zchunk = 1;
    p.nseg = 1;
    p.ksplit = 1;
    return p;
}

constexpr int GBM = 128, GBN = 128, GBK = 16, GNT = 256, GPAD = 4;

// launches gemm_simt_kernel (gemm_simt.cu) over the output tiles of p
cudaError_t launch_gemm(const GemmP& p, cudaStream_t st);

}  // namespace bm
