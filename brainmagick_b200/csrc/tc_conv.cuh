// K3/K4/K5 on the Hopper tensor cores: dilated Conv1d (and its data gradient, and the 1x1 head / subject layers) as an
// implicit GEMM on the 3xTF32 wgmma engine of tc_common.cuh (or its single-pass TF32 form: ConvOp::passes = 1).
//
//   y[b, t, n] = bias[n] + sum_{tap} sum_{k} x[b, t + shift(tap), k] * W[wset(b)][tap][n][k]      (channels-last x, y)
//
// shift(tap) = sign * (tap - taps/2) * dilation; a shifted time outside [0, T) reads zeros (the conv's zero padding, never
// the neighbouring sample: the activation tile is a TMA box of one sample).  Runs on hc_conv_kernel of tc_common.cuh, whose
// persistent CTAs walk the tiles: one tile = 128 times of one sample x BN output columns, BN = hg_pick_bn(Ntot): 160 for the
// 320- and 640-wide layers, 128 for 1024 (GLU: BN/2 'a' columns and the BN/2 gate columns they pair with, so that
// a * sigmoid(gate) is formed in registers).  Tiles are numbered column tile fastest, then time tile, then sample.
// The weights arrive as raw fp32 [sets][taps][Ntot][Cin], as its two tf32 pieces (bm_tc_weight_split) or as the two fp16
// pieces of a power-of-two-scaled copy (bm_tc_weight_split_f16); the pieces are summed back on load (fp16: ~22 significant
// bits of the weight, the precision the pieces carry).  Fused epilogue: bias, addend (skip gradient / in-place accumulate),
// pre-activation copy, exact GELU, channel-major store, GLU, BatchNorm column statistics (fp64), max |output|.
#pragma once
#include <cuda_fp16.h>
#include <cstring>
#include "tc_common.cuh"

namespace bm {
namespace tc {

constexpr int HP_TARGET_EXP = 14;                                    // scaled maximum in [2^14, 2^15)

// The power of two that puts a tensor whose largest magnitude is `amax` into [2^14, 2^15) (where both fp16 pieces of a
// value are exact); 1 for an all-zero / non-finite tensor.  Identical on every thread that evaluates it (bit arithmetic).
__host__ __device__ __forceinline__ float f16_scale_of(float amax) {
#ifdef __CUDA_ARCH__
    const uint32_t bits = __float_as_uint(amax);
#else
    uint32_t bits; memcpy(&bits, &amax, 4);
#endif
    const int e = (int)((bits >> 23) & 0xFF);
    if (e == 0 || e == 255) return 1.0f;
    int se = 127 + HP_TARGET_EXP - (e - 127);             // exponent field of the scale
    se = se < 1 ? 1 : (se > 254 ? 254 : se);
    const uint32_t sb = (uint32_t)se << 23;
#ifdef __CUDA_ARCH__
    return __uint_as_float(sb);
#else
    float s; memcpy(&s, &sb, 4); return s;
#endif
}

struct ConvOp {
    const float* x;                       // [B, T, Cin]
    const float* w;                       // fp32 weights [sets][taps][Ntot][Cin], or null: fp16 pieces below
    const float* w_lo32;                  // nullable: second tf32 piece of w (bm_tc_weight_split), added back on load
    const __half* w_hi; const __half* w_lo; const float* w_amax;
    int B, T, Cin, Ntot, taps, dilation, sign, glu, ttiles, ncols;     // ttiles / ncols: time / column tiles
    int n_wsets; const int* wsel;         // per-sample weight set (SubjectLayers) or null
    const float* bias;                    // [Ntot] or null
    const float* addend;                  // [B,T,Ntot] or null (may alias y: in-place accumulate)
    float* y;                             // [B,T,Ntot], [B,Ntot,T] when out_tmajor; GLU: the pre-GLU h (nullable)
    float* aux;                           // pre-activation copy or null
    float* glu_out;                       // GLU: [B,T,Ntot/2]
    double* stats;                        // [2*Ntot] column sum / sum of squares of y (zeroed by the launcher) or null
    unsigned int* out_amax;               // max |GELU / GLU output| (float bits) or null
    int act, out_tmajor;
    int* err;
    int passes;                           // 3: 3xTF32, 1: single-pass TF32 (reads w alone; not with the fp16 pieces)

    struct Cta { int b, t0, n_tile, wbase; float w_inv; };
    template <int BN> __device__ Cta cta(int tile) const {
        Cta c;
        const int bt = tile / ncols;
        c.n_tile = tile - bt * ncols;
        c.b = bt / ttiles;
        c.t0 = (bt - c.b * ttiles) * HG_BM;
        int s = wsel ? wsel[c.b] : 0;
        if (s < 0 || s >= n_wsets) {                 // a subject / recording index outside the weight sets: report it like
            if (err && threadIdx.x == 0) atomicCAS(err, 0, 900);     // the reference's gather would raise (thread 0: the
                                                                     // producer, which evaluates every tile)
            s = 0;
        }
        c.wbase = s * taps;
        c.w_inv = w ? 1.f : 1.f / f16_scale_of(__ldg(w_amax));
        return c;
    }
    __device__ int kblocks(const Cta&) const { return taps * (Cin / HG_BK); }
    // TMA box (channel k0, time, sample) of the A tile of K block kb: the tile's times shifted by the tap.  Shifted times
    // outside [0, T) arrive as zeros; tile rows t >= T may read live times, but their outputs are never stored.
    __device__ int3 a_box(const Cta& c, int kb) const {
        const int kch = Cin / HG_BK, tap = kb / kch, k0 = (kb - tap * kch) * HG_BK;
        return make_int3(k0, c.t0 + sign * (tap - taps / 2) * dilation, c.b);
    }
    // output column of tile column j (GLU: j < BN/2 'a' columns, j >= BN/2 their gates), -1 past the end
    template <int BN> __device__ int col_of(const Cta& c, int j) const {
        if (glu) {
            const int H = Ntot / 2, cc = c.n_tile * (BN / 2) + (int)((unsigned)j % (BN / 2));
            return cc < H ? cc + (j >= BN / 2 ? H : 0) : -1;
        }
        const int n = c.n_tile * BN + j;
        return n < Ntot ? n : -1;
    }
    // B operand, in steps so that the producer can issue a whole tile's loads back to back and ahead of their use:
    //   b_col: element offset of (tile column j, k quad q) within a K block, -1 past the end (the same for every block);
    //   b_base: element offset of K block kb;  b_load<FMT>: the loads of the 4 fp32 weights at element offset `off`, as
    //   they arrive;  b_value<FMT>: the 4 weights from them
    enum { B_RAW, B_SPLIT, B_F16 };
    __device__ int b_format() const { return w ? (w_lo32 ? B_SPLIT : B_RAW) : B_F16; }
    template <int BN> __device__ int b_col(const Cta& c, int j, int q) const {
        const int n = col_of<BN>(c, j);
        return n < 0 ? -1 : n * Cin + 4 * q;
    }
    __device__ long long b_base(const Cta& c, int kb) const {
        const int kch = Cin / HG_BK, tap = kb / kch, k0 = (kb - tap * kch) * HG_BK;
        return (long long)(c.wbase + tap) * Ntot * Cin + k0;
    }
    template <int FMT> __device__ HcB b_load(long long off) const {
        HcB r;
        if (FMT == B_F16) {                          // h = the fp16 hi and lo pieces' bits
            const uint2 h = __ldg(reinterpret_cast<const uint2*>(w_hi + off));
            const uint2 l = __ldg(reinterpret_cast<const uint2*>(w_lo + off));
            r.h = make_float4(__uint_as_float(h.x), __uint_as_float(h.y), __uint_as_float(l.x), __uint_as_float(l.y));
            return r;
        }
        r.h = __ldg(reinterpret_cast<const float4*>(w + off));
        if (FMT == B_SPLIT) r.l = __ldg(reinterpret_cast<const float4*>(w_lo32 + off));
        return r;
    }
    template <int FMT> __device__ float4 b_value(const Cta& c, const HcB& r) const {
        if (FMT != B_F16) {
            float4 v = r.h;
            if (FMT == B_SPLIT) { v.x += r.l.x; v.y += r.l.y; v.z += r.l.z; v.w += r.l.w; }
            return v;
        }
        const uint32_t hx = __float_as_uint(r.h.x), hy = __float_as_uint(r.h.y);
        const uint32_t lx = __float_as_uint(r.h.z), ly = __float_as_uint(r.h.w);
        const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&hx)), h1 = __half22float2(*reinterpret_cast<const __half2*>(&hy));
        const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&lx)), l1 = __half22float2(*reinterpret_cast<const __half2*>(&ly));
        return make_float4((h0.x + l0.x) * c.w_inv, (h0.y + l0.y) * c.w_inv, (h1.x + l1.x) * c.w_inv, (h1.y + l1.y) * c.w_inv);
    }

    // run by the 256 consumer threads of hc_conv_kernel, once per tile; PASSES only gives each kernel instantiation its own
    // col_sums (a static shared array shared by the 3- and 1-pass kernels would change the shared-memory layout of both)
    template <int BN, int PASSES> __device__ void epilogue(const Cta& c, const float* acc, int m0) const {
        __shared__ double col_sums[2 * BN];
        float am = 0.f;
        if (glu) {
            const int H = Ntot / 2;
#pragma unroll
            for (int i = 0; i < BN / 4; ++i) {           // tile columns 0..BN/2-1; the gate of column j is column j + BN/2
                const int t = c.t0 + m0 + hg_row(i), cc = c.n_tile * (BN / 2) + hg_col(i);
                if (t >= T || cc >= H) continue;
                const long long row = (long long)c.b * T + t;
                float a = acc[i], g = acc[i + BN / 4];
                if (bias) { a += bias[cc]; g += bias[H + cc]; }
                if (y) { y[row * Ntot + cc] = a; y[row * Ntot + H + cc] = g; }
                const float o = a * sigmoid_f(g);
                glu_out[row * H + cc] = o;
                am = fmaxf(am, fabsf(o));
            }
        } else {
            if (stats) {
                hc_consumer_sync();                      // the previous tile's reads of col_sums, before they are cleared
                for (int i = hc_consumer_tid(); i < 2 * BN; i += HC_CONSUMERS) col_sums[i] = 0.0;
                hc_consumer_sync();
            }
#pragma unroll
            for (int g = 0; g < BN / 8; ++g) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float s1 = 0.f, s2 = 0.f;
                    const int j = 8 * g + 2 * (threadIdx.x & 3) + e, n = c.n_tile * BN + j;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i = 4 * g + 2 * h + e;
                        const int t = c.t0 + m0 + hg_row(i);
                        if (t >= T || n >= Ntot) continue;
                        const long long row = (long long)c.b * T + t;
                        float v = acc[i];
                        if (bias) v += bias[n];
                        if (addend) v += addend[row * Ntot + n];
                        if (aux) aux[row * Ntot + n] = v;
                        if (act) { v = gelu_f(v); am = fmaxf(am, fabsf(v)); }
                        if (out_tmajor) y[((long long)c.b * Ntot + n) * T + t] = v;
                        else y[row * Ntot + n] = v;
                        s1 += v;
                        s2 = fmaf(v, v, s2);
                    }
                    if (stats) {
#pragma unroll
                        for (int o = 4; o < 32; o <<= 1) {
                            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                            s2 += __shfl_xor_sync(0xffffffffu, s2, o);
                        }
                        if ((threadIdx.x & 31) < 4 && n < Ntot) {
                            atomicAdd(&col_sums[j], (double)s1);
                            atomicAdd(&col_sums[BN + j], (double)s2);
                        }
                    }
                }
            }
            if (stats) {
                hc_consumer_sync();
                for (int j = hc_consumer_tid(); j < BN; j += HC_CONSUMERS) {
                    const int n = c.n_tile * BN + j;
                    if (n < Ntot) {
                        atomicAdd(stats + n, col_sums[j]);
                        atomicAdd(stats + Ntot + n, col_sums[BN + j]);
                    }
                }
            }
        }
        if (out_amax) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
            if ((threadIdx.x & 31) == 0 && am > 0.f) atomicMax(out_amax, __float_as_uint(am));
        }
    }
};

// Data gradient of the sensor mix (ChannelMerger, common.py:358) as a pointwise ConvOp with one weight set per recording:
//   dmeg[b, c, t] = mask[c] * sum_o du[b, t, o] * W[wsel[b]][c][o]
// x = du [B,T,Cin=Op], w = the transposed attention weights [R][Ntot=Cp][Op].  Its own epilogue stores only the C live sensor
// rows, channel-major [B,C,T], times the channel mask (nullable); the ConvOp epilogue itself is untouched.
struct SensorMixBwdOp : ConvOp {
    int C;
    const float* mask;
    template <int BN, int PASSES> __device__ void epilogue(const Cta& c, const float* acc, int m0) const {
#pragma unroll
        for (int g = 0; g < BN / 8; ++g) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = c.n_tile * BN + 8 * g + 2 * (threadIdx.x & 3) + e;
                if (n >= C) continue;
                const float m = mask ? mask[n] : 1.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = 4 * g + 2 * h + e;
                    const int t = c.t0 + m0 + hg_row(i);
                    if (t < T) y[((long long)c.b * C + n) * T + t] = acc[i] * m;
                }
            }
        }
    }
};

inline ConvOp conv_op_defaults() {
    ConvOp o;
    memset(&o, 0, sizeof(o));
    o.n_wsets = 1;
    o.passes = 3;
    return o;
}

inline int launch_conv_op(ConvOp o, cudaStream_t st, const char* who) {
    if ((long long)o.B * o.T >= (1ll << 31)) return set_error(2, "%s: too many rows%s", who);
    o.ttiles = (o.T + HG_BM - 1) / HG_BM;
    const int bn = hg_pick_bn(o.Ntot);                   // GLU: BN/2 'a' columns and their gates per tile
    o.ncols = o.glu ? (o.Ntot / 2 + bn / 2 - 1) / (bn / 2) : (o.Ntot + bn - 1) / bn;
    if (o.stats) {
        cudaError_t em = cudaMemsetAsync(o.stats, 0, sizeof(double) * 2 * o.Ntot, st);
        if (em != cudaSuccess) return set_error(3, "%s: memset: %s", who, cudaGetErrorString(em));
    }
    return hc_launch_bn(bn, o, (long long)o.B * o.ttiles * o.ncols, st, who);
}

// W[o][i][j] (nn.Conv1d layout) -> tf32-split K-major operands:
//   fwd  operand: F[j][o][i]   (n = o, k = i)        data-gradient operand: G[j][i][o]   (n = i, k = o)
__global__ void weight_split_kernel(const float* __restrict__ W, float* __restrict__ f_hi, float* __restrict__ f_lo,
                                    float* __restrict__ g_hi, float* __restrict__ g_lo, int O, int I, int Kw) {
    long long total = (long long)O * I * Kw;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        int j = (int)(idx % Kw);
        long long oi = idx / Kw;
        int i = (int)(oi % I), o = (int)(oi / I);
        float v = W[idx];
        float h = tf32_rna(v), l = tf32_rna(v - h);
        long long fi = ((long long)j * O + o) * I + i, gi = ((long long)j * I + i) * O + o;
        // a NULL lo pointer asks for the RAW fp32 value in the re-laid array (the v2 kernel splits in shared memory)
        if (f_hi) { if (f_lo) { f_hi[fi] = h; f_lo[fi] = l; } else f_hi[fi] = v; }
        if (g_hi) { if (g_lo) { g_hi[gi] = h; g_lo[gi] = l; } else g_hi[gi] = v; }
    }
}

// Shape gate of bm_tc_conv1d / bm_tc_pointwise_sel: Ntot a multiple of 16 with a divisor in [64, 160] (GLU: H a multiple
// of 80), K chunks of 32 input channels.  The kernel itself handles any N; the gate is the library's published contract.
inline bool conv_tc_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    if (Kw < 1 || Kw > 3 || (Kw & 1) == 0) return false;
    if (Cin % HG_BK != 0) return false;
    if (glu) return Ntot % 2 == 0 && (Ntot / 2) % 80 == 0;
    for (int bn = 160; bn >= 64; bn -= 16)
        if (Ntot % bn == 0) return true;
    return false;
}

// x [B,T,Cin]; w_hi / w_lo [Kw][Ntot][Cin] (wsel: [n_wsets][Kw][Ntot][Cin]), the tf32 pieces of bm_tc_weight_split
// (passes = 1: w_hi alone is read, w_lo may be null)
struct ConvTcP {
    int B, T, Cin, Ntot, taps, dilation, sign, glu, act, out_tmajor, passes;
    const float* bias; const float* addend;
    float* y; float* aux; float* glu_out;
    int n_wsets; const int* wsel;
    int* err;
};
inline int launch_conv_tc(const float* x, const float* w_hi, const float* w_lo, const ConvTcP& p, cudaStream_t st) {
    ConvOp o = conv_op_defaults();
    o.x = x; o.w = w_hi; o.w_lo32 = w_lo; o.B = p.B; o.T = p.T; o.Cin = p.Cin; o.Ntot = p.Ntot; o.taps = p.taps; o.dilation = p.dilation;
    o.sign = p.sign; o.glu = p.glu; o.n_wsets = p.wsel ? p.n_wsets : 1; o.wsel = p.wsel; o.bias = p.bias;
    o.addend = p.addend; o.y = p.y; o.aux = p.aux; o.glu_out = p.glu_out; o.act = p.act; o.out_tmajor = p.out_tmajor;
    o.err = p.err; o.passes = p.passes;
    return launch_conv_op(o, st, __func__);
}

// du [B,T,Op]; w_hi / w_lo [n_sets][Cp][Op] (tf32 pieces; passes = 1: w_hi alone); dmeg [B,C,T] with C <= Cp; mask [C]
// or null
inline int launch_sensor_mix_bwd_tc(const float* du, const float* w_hi, const float* w_lo, const int* wsel, int n_sets,
                                    const float* mask, int B, int T, int Op, int Cp, int C, float* dmeg, int passes,
                                    int* err, cudaStream_t st) {
    SensorMixBwdOp o;
    memset(&o, 0, sizeof(o));
    o.x = du; o.w = w_hi; o.w_lo32 = w_lo; o.B = B; o.T = T; o.Cin = Op; o.Ntot = Cp; o.taps = 1; o.dilation = 1; o.sign = 1;
    o.n_wsets = n_sets; o.wsel = wsel; o.y = dmeg; o.err = err; o.C = C; o.mask = mask; o.passes = passes;
    if ((long long)B * T >= (1ll << 31)) return set_error(2, "%s: too many rows%s", __func__);
    o.ttiles = (T + HG_BM - 1) / HG_BM;
    const int bn = hg_pick_bn(Cp);
    o.ncols = (Cp + bn - 1) / bn;
    return hc_launch_bn(bn, o, (long long)B * o.ttiles * o.ncols, st, __func__);
}

}  // namespace tc
}  // namespace bm
