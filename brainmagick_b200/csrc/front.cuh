// The spatial attention's elementwise kernels (front_api.cu).
#pragma once
#include "common.cuh"

namespace bm {

// ------------------------------------------------------------------------------------------------
// K1 pieces: Fourier embedding of sensor positions and the masked softmax (common.py:254-271,339-357)
// ------------------------------------------------------------------------------------------------
// emb[rc][k*n+l] = cos(loc), emb[rc][P/2 + k*n+l] = sin(loc), loc = (x+margin)*f[k] + (y+margin)*f[l]
// `freq` is the table 2*pi*arange(n)/(1+2*margin) built by the host with the reference's own op order, and
// the products/sum are rounded separately (no FMA contraction) so that `loc` is bit-identical to torch's.
__global__ void fourier_emb_kernel(const float* __restrict__ pos, const float* __restrict__ freq, float margin,
                                   int RC, int n, float* __restrict__ emb) {
    const int P2 = n * n;
    long long total = (long long)RC * P2;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        int rc = (int)(idx / P2);
        int kl = (int)(idx - (long long)rc * P2);
        int k = kl / n, l = kl - k * n;
        float x = __fadd_rn(pos[2 * rc], margin), y = __fadd_rn(pos[2 * rc + 1], margin);
        float loc = __fadd_rn(__fmul_rn(x, freq[k]), __fmul_rn(y, freq[l]));
        float s, c;
        sincosf(loc, &s, &c);
        emb[(long long)rc * 2 * P2 + kl] = c;
        emb[(long long)rc * 2 * P2 + P2 + kl] = s;
    }
}

// in-place softmax over c of scores[r][o][:] with -inf on invalid (pos == INVALID) and banned sensors
// (||pos - centre|| <= radius, training only).  One warp per (r, o) row.
__global__ void masked_softmax_kernel(float* __restrict__ w, const float* __restrict__ pos,
                                      const float* __restrict__ centre, float radius, float invalid, int R, int O,
                                      int C) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= R * O) return;
    int r = row / O;
    float* s = w + (long long)row * C;
    const float* pr = pos + (long long)r * C * 2;
    float cx = 0.f, cy = 0.f;
    if (centre) { cx = centre[0]; cy = centre[1]; }
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) {
        float x = pr[2 * c], y = pr[2 * c + 1];
        bool masked = (x == invalid) && (y == invalid);
        if (centre) {
            float dx = x - cx, dy = y - cy;
            masked = masked || (sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) <= radius);
        }
        float v = masked ? -INFINITY : s[c];
        s[c] = v;
        mx = fmaxf(mx, v);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) {
        float e = expf(s[c] - mx);
        s[c] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    float inv = 1.f / sum;
    for (int c = lane; c < C; c += 32) s[c] *= inv;
}

// dscore = w * (dw - sum_c w*dw)   (softmax backward, one warp per row)
__global__ void softmax_bwd_kernel(const float* __restrict__ w, const float* __restrict__ dw,
                                   float* __restrict__ ds, int rows, int C) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* wr = w + (long long)row * C;
    const float* dr = dw + (long long)row * C;
    float dot = 0.f;
    for (int c = lane; c < C; c += 32) dot += wr[c] * dr[c];
    dot = warp_sum(dot);
    for (int c = lane; c < C; c += 32) ds[(long long)row * C + c] = wr[c] * (dr[c] - dot);
}

}  // namespace bm
