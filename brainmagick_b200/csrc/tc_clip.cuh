// K6: ClipLoss.get_scores (bm/losses.py:91-94) as ONE split-K tensor-core GEMM (3xTF32 wgmma engine of tc_common.cuh, or
// its single-pass TF32 form: passes = 1, or its bf16 form: passes = TC_BF16; the candidate norms stay fp64 sums of squares
// of the fp32 values either way)
// followed by ONE finalize kernel (split reduction + 1/norm scale + row softmax / cross-entropy + batch mean,
// bm/losses.py:97-114).
//
//     S[b][o] = sum_k E[b][k] C[o][k]          E = estimates [Bn][K], C = candidates [Bc][K], K = F*T (368 640)
//
// K is long: a self dot product chained through the tensor core's truncating accumulator would come out ~1e-4 low; the
// engine adds every 32-wide K block into a round-to-nearest fp32 sum instead.  The candidate norms (the 1/||c|| of
// losses.py:91) come from a fp64 row sum of squares beside the GEMM.
//   grid: 128-estimate x 128-candidate tiles x K slices; outputs: partial scores [ks][Bn][Bc] and [ks][Bc] fp64 partial sums
//   of squares (slice 0 holds the full sums); `clip_finalize_kernel` reduces both in a fixed order.  The sums of squares in
//   slot 0 come from up to 32 K splits per candidate added with fp64 atomics, so their last bits depend on block order; the
//   deterministic form (`det`) computes each candidate's sum in one block, which adds onto its zeroed slot exactly once.
#pragma once
#include "tc_common.cuh"
#include "clip.cuh"

namespace bm {
namespace tc {

constexpr int CL_BK = HG_BK;

struct ClipOp {
    static constexpr bool A_KCONTIG = true, B_KCONTIG = true;
    const float* E; const float* C;
    int Bn, Bc, chunks, per_split;
    long long KT;
    float* P;                   // [ks][Bn][Bc]
    struct Cta { int m0, n0, c0, c1; };
    template <int BN> __device__ Cta cta() const {
        Cta c;
        c.n0 = blockIdx.x * BN;
        c.m0 = blockIdx.y * HG_BM;
        c.c0 = blockIdx.z * per_split;
        c.c1 = min(chunks, c.c0 + per_split);
        return c;
    }
    __device__ int kblocks(const Cta& c) const { return max(0, c.c1 - c.c0); }
    __device__ float4 a4(const Cta& c, int kb, int r, int q) const {
        const int m = c.m0 + r;
        const long long k = (long long)(c.c0 + kb) * HG_BK + 4 * q;
        if (m >= Bn || k >= KT) return make_float4(0.f, 0.f, 0.f, 0.f);
        return __ldg(reinterpret_cast<const float4*>(E + m * KT + k));
    }
    __device__ float4 b4(const Cta& c, int kb, int r, int q) const {
        const int n = c.n0 + r;
        const long long k = (long long)(c.c0 + kb) * HG_BK + 4 * q;
        if (n >= Bc || k >= KT) return make_float4(0.f, 0.f, 0.f, 0.f);
        return __ldg(reinterpret_cast<const float4*>(C + n * KT + k));
    }
    template <int BN> __device__ void epilogue(const Cta& c, const float* acc, int m0) const {
        HgStore s{P + (long long)blockIdx.z * Bn * Bc, Bc, Bn, Bc};
        s.store<BN>(acc, c.m0 + m0, c.n0);
    }
};

// ClipOp over pooled candidates: candidate n is C + n*KT for n < Bb (the batch rows, read in place), else
// arena + slots[n - Bb]*KT (a row of the negative pool's device storage); one more load per row than ClipOp
struct ClipPooledOp : ClipOp {
    const float* arena; const int* slots;
    int Bb;
    __device__ float4 b4(const Cta& c, int kb, int r, int q) const {
        const int n = c.n0 + r;
        const long long k = (long long)(c.c0 + kb) * HG_BK + 4 * q;
        if (n >= Bc || k >= KT) return make_float4(0.f, 0.f, 0.f, 0.f);
        const float* row = n < Bb ? C + n * KT : arena + __ldg(slots + (n - Bb)) * KT;
        return __ldg(reinterpret_cast<const float4*>(row + k));
    }
};

// ---- finalize: fixed-order reduction of the K slices, 1/norm, scores, optional softmax / cross-entropy / batch mean ----
// one block per estimate row b.  `counter` (zeroed by the launcher) elects the last block, which averages row_loss in a
// fixed order.
__global__ void clip_finalize_kernel(const float* __restrict__ P, const double* __restrict__ ssp, int ks, int Bn, int Bc,
                                     int target_offset, float* __restrict__ inv_norm, float* __restrict__ scores,
                                     float* __restrict__ probs, float* __restrict__ row_loss, float* __restrict__ loss,
                                     unsigned int* __restrict__ counter) {
    __shared__ float red[32];
    __shared__ float bcast;
    __shared__ unsigned int ticket;
    const int b = blockIdx.x;
    const long long plane = (long long)Bn * Bc;
    float* srow = scores + (long long)b * Bc;
    float mx = -INFINITY;
    for (int o = threadIdx.x; o < Bc; o += blockDim.x) {
        float n;
        if (ssp) {
            double ss = 0.0;
            for (int k = 0; k < ks; ++k) ss += ssp[(long long)k * Bc + o];
            n = 1.f / (1e-8f + (float)sqrt(ss));                  // losses.py:91
            if (b == 0) inv_norm[o] = n;
        } else {
            n = inv_norm[o];
        }
        float s = 0.f;
        const float* src = P + (long long)b * Bc + o;
        for (int k = 0; k < ks; ++k) s += src[(long long)k * plane];
        s *= n;
        srow[o] = s;
        mx = fmaxf(mx, s);
    }
    if (!probs && !row_loss) return;
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : -INFINITY;
        v = warp_max(v);
        if (threadIdx.x == 0) bcast = v;
    }
    __syncthreads();
    mx = bcast;
    __syncthreads();
    float sum = 0.f;
    for (int o = threadIdx.x; o < Bc; o += blockDim.x) sum += expf(srow[o] - mx);   // own columns: written by this thread
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) bcast = v;
    }
    __syncthreads();
    sum = bcast;
    if (probs) {
        const float inv = 1.f / sum;
        for (int o = threadIdx.x; o < Bc; o += blockDim.x) probs[(long long)b * Bc + o] = expf(srow[o] - mx) * inv;
    }
    if (!row_loss) return;
    __syncthreads();                                              // srow[b + target_offset] may belong to another thread
    if (threadIdx.x == 0) {
        row_loss[b] = (logf(sum) + mx) - srow[b + target_offset];
        __threadfence();
        ticket = loss ? atomicAdd(counter, 1u) : 0u;
    }
    __syncthreads();
    if (!loss || ticket != (unsigned)(Bn - 1)) return;
    __threadfence();
    __shared__ double dred[32];
    double acc = 0.0;
    for (int i = threadIdx.x; i < Bn; i += blockDim.x) acc += (double)__ldcg(row_loss + i);
    acc = warp_sum_d(acc);
    if ((threadIdx.x & 31) == 0) dred[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = threadIdx.x < (blockDim.x >> 5) ? dred[threadIdx.x] : 0.0;
        v = warp_sum_d(v);
        if (threadIdx.x == 0) loss[0] = (float)(v / Bn);
    }
}

// ---- geometry / workspace -------------------------------------------------------------------------------------------
struct ClipGeom { int ks, chunks, per_split; };

inline bool clip_tc_supported(int Bn, int Bc, long long KT) {
    return Bn > 0 && Bc > 0 && KT >= CL_BK && KT % 4 == 0 && KT < (1ll << 31);
}
inline ClipGeom clip_geometry(int Bn, int Bc, long long KT) {
    ClipGeom g;
    g.chunks = (int)((KT + CL_BK - 1) / CL_BK);
    const int tiles = ((Bc + HG_BN - 1) / HG_BN) * ((Bn + HG_BM - 1) / HG_BM);
    int ks = num_sms() / tiles;                                   // one wave of 128 x 128 tiles
    if (ks < 1) ks = 1;
    if (ks > g.chunks) ks = g.chunks;
    g.per_split = (g.chunks + ks - 1) / ks;
    g.ks = (g.chunks + g.per_split - 1) / g.per_split;            // no empty slice
    return g;
}
// floats: partial scores, then fp64 partial sums of squares (8-byte aligned), then the finalize ticket
inline long long clip_ws_floats(int Bn, int Bc, long long KT) {
    const ClipGeom g = clip_geometry(Bn, Bc, KT);
    long long n = (long long)g.ks * Bn * Bc;
    n += n & 1;
    return n + 2ll * g.ks * Bc + 2;
}

// scores [Bn][Bc] (+ inv_norm when !norms_given, + probs / row_loss / loss when requested).  slots != NULL: pooled
// candidates (ClipPooledOp): candidates Bb..Bc-1 are the arena rows slots[0..Bc-Bb-1]
inline int launch_clip_scores(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given,
                              int target_offset, float* inv_norm, float* scores, float* probs, float* row_loss,
                              float* loss, float* ws, int passes, int* err, cudaStream_t st, bool det = false,
                              int Bb = 0, const float* arena = nullptr, const int* slots = nullptr) {
    (void)err;
    const ClipGeom g = clip_geometry(Bn, Bc, KT);
    long long nP = (long long)g.ks * Bn * Bc;
    nP += nP & 1;
    double* ssp = norms_given ? nullptr : reinterpret_cast<double*>(ws + nP);
    unsigned int* counter = reinterpret_cast<unsigned int*>(ws + nP + 2ll * g.ks * Bc);
    if (loss) {
        cudaError_t em = cudaMemsetAsync(counter, 0, sizeof(unsigned int), st);
        if (em != cudaSuccess) return set_error(3, "%s: memset: %s", __func__, cudaGetErrorString(em));
    }
    if (ssp) {
        cudaError_t em = cudaMemsetAsync(ssp, 0, sizeof(double) * g.ks * Bc, st);
        if (em != cudaSuccess) return set_error(3, "%s: memset: %s", __func__, cudaGetErrorString(em));
        int splits = (int)((KT + 65535) / 65536);
        if (splits > 32) splits = 32;
        if (det) splits = 1;                                      // one add per slot: independent of block order
        if (slots) row_sumsq_pooled_kernel<<<dim3(Bc, splits), 256, 0, st>>>(cand, Bb, arena, slots, ssp, KT);
        else row_sumsq_kernel<<<dim3(Bc, splits), 256, 0, st>>>(cand, ssp, KT);
        ++g_launches;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return set_error(3, "%s: norm launch failed: %s", __func__, cudaGetErrorString(e));
    }
    const dim3 grid((Bc + HG_BN - 1) / HG_BN, (Bn + HG_BM - 1) / HG_BM, g.ks);
    if (slots) {
        ClipPooledOp o;
        o.E = est; o.C = cand; o.Bn = Bn; o.Bc = Bc; o.chunks = g.chunks; o.per_split = g.per_split; o.KT = KT; o.P = ws;
        o.arena = arena; o.slots = slots; o.Bb = Bb;
        if (int rc = hg_launch<HG_BN>(o, grid, passes, st, __func__)) return rc;
    } else {
        ClipOp o;
        o.E = est; o.C = cand; o.Bn = Bn; o.Bc = Bc; o.chunks = g.chunks; o.per_split = g.per_split; o.KT = KT; o.P = ws;
        if (int rc = hg_launch<HG_BN>(o, grid, passes, st, __func__)) return rc;
    }
    clip_finalize_kernel<<<Bn, 256, 0, st>>>(ws, ssp, g.ks, Bn, Bc, target_offset, inv_norm, scores, probs, row_loss,
                                             loss, counter);
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: finalize launch failed: %s", __func__, cudaGetErrorString(e));
    return 0;
}

}  // namespace tc
}  // namespace bm
