// Channel join / split of SimpleConv's input streams and encoder outputs (bm/models/simpleconv.py:234-243): up to four
// sources placed side by side in the columns of one channels-last [B, T, Cp] tensor, and the reverse for the gradients.
// A source is channels-last (rows of stride ld) or channel-major [B, C, T] (channel stride ld >= T, i.e. possibly a view
// cropped in time), transposed through a shared-memory tile on the way.  Pure copies: deterministic, identical under TF32.
#pragma once
#include "common.cuh"

namespace bm {

constexpr int JOIN_MAX_SEGS = 9;     // 4 sources and the 5 zero-filled gaps around them

struct JoinSeg {
    float* p;       // the source (join) / destination (split); nullptr on join: a zero-filled gap
    int C;          // columns
    int ld;         // channels-last: row stride; channel-major: channel stride (sample stride C * ld)
    int cm;         // 1: channel-major [B, C, T]
    int col;        // first column in the packed tensor
    int vec;        // channels-last with 16-byte aligned rows and C, ld, col multiples of 4: float4 accesses
    int tile0;      // first blockIdx.x of this segment
};

struct JoinArgs {
    JoinSeg s[JOIN_MAX_SEGS];
    int n;
    int T, Cp;
    float* packed;  // [B, T, Cp]
};

// grid (sum of the segments' column tiles, ceil(T / 32), B), block (32, 8).  A column tile is 32 columns (128 with float4).
template <bool SPLIT>
__global__ void channel_join_kernel(const JoinArgs a) {
    __shared__ float tile[32][33];
    int si = 0;
    while (si + 1 < a.n && (int)blockIdx.x >= a.s[si + 1].tile0) ++si;
    const JoinSeg s = a.s[si];
    const int b = blockIdx.z, t0 = blockIdx.y * 32, T = a.T;
    float* packed = a.packed + (long long)b * T * a.Cp + s.col;
    if (s.cm) {
        const int c0 = ((int)blockIdx.x - s.tile0) * 32;
        float* cm = s.p + (long long)b * s.C * s.ld;
        if (!SPLIT) {
#pragma unroll
            for (int i = threadIdx.y; i < 32; i += 8) {
                const int c = c0 + i, t = t0 + threadIdx.x;
                tile[i][threadIdx.x] = (c < s.C && t < T) ? cm[(long long)c * s.ld + t] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int i = threadIdx.y; i < 32; i += 8) {
                const int t = t0 + i, c = c0 + threadIdx.x;
                if (t < T && c < s.C) packed[(long long)t * a.Cp + c] = tile[threadIdx.x][i];
            }
        } else {
#pragma unroll
            for (int i = threadIdx.y; i < 32; i += 8) {
                const int t = t0 + i, c = c0 + threadIdx.x;
                tile[threadIdx.x][i] = (t < T && c < s.C) ? packed[(long long)t * a.Cp + c] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int i = threadIdx.y; i < 32; i += 8) {
                const int c = c0 + i, t = t0 + threadIdx.x;
                if (c < s.C && t < T) cm[(long long)c * s.ld + t] = tile[i][threadIdx.x];
            }
        }
        return;
    }
    const int V = s.vec ? 4 : 1;
    const int c = ((int)blockIdx.x - s.tile0) * 32 * V + threadIdx.x * V;
    if (c >= s.C) return;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int t = t0 + i;
        if (t >= T) break;
        float* pk = packed + (long long)t * a.Cp + c;
        float* cl = s.p ? s.p + ((long long)b * T + t) * s.ld + c : nullptr;
        if (s.vec) {
            if (SPLIT) *reinterpret_cast<float4*>(cl) = *reinterpret_cast<const float4*>(pk);
            else *reinterpret_cast<float4*>(pk) = cl ? *reinterpret_cast<const float4*>(cl) : make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            if (SPLIT) *cl = *pk;
            else *pk = cl ? *cl : 0.f;
        }
    }
}

}  // namespace bm
