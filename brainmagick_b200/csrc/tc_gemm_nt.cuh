// ClipLoss backward contractions (bm/losses.py:91-114 differentiated, SURVEY.md A.6) on the 3xTF32 wgmma engine (or its
// single-pass TF32 / bf16 forms: passes = 1 / TC_BF16):
//
//     D[m][n] = sum_k A[m][k] * B[k][n]        A [M][K] row-major (K contiguous), B [K][N] row-major (N contiguous)
//
//   dE = G C      (M = estimates, K = candidates,  N = F*T = 368 640):  A = G   [Bn][Bc], B = candidates [Bc][F*T]
//   dC = G^T E    (M = candidates, K = estimates,  N = F*T):            A = G^T [Bc][Bn], B = estimates  [Bn][F*T]
#pragma once
#include "tc_common.cuh"

namespace bm {
namespace tc {

struct GemmNTOp {
    static constexpr bool A_KCONTIG = true, B_KCONTIG = false;
    const float* A; const float* B; float* D;
    int M, N, K;
    struct Cta { int m0, n0; };
    template <int BN> __device__ Cta cta() const { return Cta{(int)blockIdx.y * HG_BM, (int)blockIdx.x * BN}; }
    __device__ int kblocks(const Cta&) const { return (K + HG_BK - 1) / HG_BK; }
    __device__ float4 a4(const Cta& c, int kb, int r, int q) const {
        const int m = c.m0 + r, k = kb * HG_BK + 4 * q;
        if (m >= M || k >= K) return make_float4(0.f, 0.f, 0.f, 0.f);
        return __ldg(reinterpret_cast<const float4*>(A + (long long)m * K + k));
    }
    __device__ float4 b4(const Cta& c, int kb, int k, int q) const {
        const int kk = kb * HG_BK + k, n = c.n0 + 4 * q;
        if (kk >= K || n >= N) return make_float4(0.f, 0.f, 0.f, 0.f);
        return __ldg(reinterpret_cast<const float4*>(B + (long long)kk * N + n));
    }
    template <int BN> __device__ void epilogue(const Cta& c, const float* acc, int m0) const {
        HgStore s{D, N, M, N};
        s.store<BN>(acc, c.m0 + m0, c.n0);
    }
};

// dE = G C over pooled candidates (ClipPooledOp's rows): B row kk is B + kk*N for kk < Bb, else arena + slots[kk - Bb]*N,
// and zero for Bc <= kk < K (K: G's row pitch, Bc rounded up to a multiple of 4 floats)
struct GemmNTPooledOp : GemmNTOp {
    const float* arena; const int* slots;
    int Bb, Bc;
    __device__ float4 b4(const Cta& c, int kb, int k, int q) const {
        const int kk = kb * HG_BK + k, n = c.n0 + 4 * q;
        if (kk >= Bc || n >= N) return make_float4(0.f, 0.f, 0.f, 0.f);
        const float* row = kk < Bb ? B + (long long)kk * N : arena + (long long)__ldg(slots + (kk - Bb)) * N;
        return __ldg(reinterpret_cast<const float4*>(row + n));
    }
};

inline bool gemm_nt_pp_supported(int M, int N, int K) {
    return M > 0 && N >= 32 && K >= 8 && K % 4 == 0 && N % 4 == 0;
}

// D [M][N] = A [M][K] * B [K][N], all row-major fp32
inline int launch_gemm_nt_pp(const float* A, const float* B, float* D, int M, int N, int K, int passes, int* err,
                             cudaStream_t st) {
    (void)err;
    GemmNTOp o{A, B, D, M, N, K};
    return hg_launch<HG_BN>(o, dim3((N + HG_BN - 1) / HG_BN, (M + HG_BM - 1) / HG_BM, 1), passes, st, __func__);
}

// D [M][N] = G [M][ldg] * pooled candidates [Bc][N] (GemmNTPooledOp); ldg % 4 == 0, the columns Bc..ldg-1 of G zero
inline int launch_gemm_nt_pooled(const float* G, int ldg, const float* cand, int Bb, const float* arena, const int* slots,
                                 int Bc, float* D, int M, int N, int passes, cudaStream_t st) {
    GemmNTPooledOp o;
    o.A = G; o.B = cand; o.D = D; o.M = M; o.N = N; o.K = ldg;
    o.arena = arena; o.slots = slots; o.Bb = Bb; o.Bc = Bc;
    return hg_launch<HG_BN>(o, dim3((N + HG_BN - 1) / HG_BN, (M + HG_BM - 1) / HG_BM, 1), passes, st, __func__);
}

}  // namespace tc
}  // namespace bm
