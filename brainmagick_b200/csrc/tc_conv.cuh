// K3/K4/K5 on the Hopper tensor cores: dilated Conv1d (and its data gradient, and the 1x1 head / subject layers) as an
// implicit GEMM on the 3xTF32 wgmma engine of tc_common.cuh (or its single-pass TF32 form: ConvOp::passes = 1, or its bf16
// form: ConvOp::passes = TC_BF16).
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
// Every conv entry point of tc_conv_api.cu fills its op and launches it through launch_conv.
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
    int passes;                           // 3: 3xTF32, 1: single-pass TF32 (reads w alone), TC_BF16: bf16 (w + w_lo32
                                          // rounded once); not with the fp16 pieces

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

    // Run by the 256 consumer threads of hc_conv_kernel, once per tile.  Element i of the thread's fragment is row
    // t0 + m0 + hg_row(i) (two rows per thread: r and r + 8) and tile column hg_col(i); elements i and i + 1 (i even) are
    // two adjacent columns, so the row-major outputs are stored as float2 (Ntot, H and every column offset are even; the
    // launcher checks the pointers' 8-byte alignment).  A column group's loads (bias, addend) are all issued before its
    // first store: `addend` may alias `y`, so a load behind a store would wait for it, one L2 round trip per element.
    // Hoisting the addend above the y stores is legal: each element is read and then written by this thread alone.
    // BatchNorm statistics: each warp's per-column fp32 sums of d = y - bias and d^2 over its 16 rows (shuffle tree over the
    // 8 row lanes) go to `partial` with plain stores; after a consumer barrier one thread per column adds the 8 warps'
    // partials in fixed order in fp64, adds the bias back in fp64 and issues the global fp64 atomics.  Unshifted fp32 sums
    // of y^2 would cancel the variance away in bn_finalize_kernel's E[y^2] - E[y]^2 once the bias puts a channel's mean
    // ~100x above its standard deviation.  PASSES only gives each kernel instantiation its own `partial` (a static
    // shared array shared by the 3- and 1-pass kernels would change the shared-memory layout of both).
    template <int BN, int PASSES> __device__ void epilogue(const Cta& c, const float* acc, int m0, HcProbe& pr) const {
        constexpr int NW = HC_CONSUMERS / 32, NG = BN / 8;    // consumer warps; 8-column groups of the fragment
        __shared__ __align__(8) float partial[NW][2][BN];
        const int tq = threadIdx.x & 3, t = c.t0 + m0 + hg_row(0);
        const bool r_ok[2] = {t < T, t + 8 < T};
        const long long row = (long long)c.b * T + t;          // the thread's rows: row and row + 8
        float am = 0.f;
        if (glu) {
            const int H = Ntot / 2, c0 = c.n_tile * (BN / 2) + 2 * tq;   // 'a' columns c0 + 8 g (+1); gates at + H
            float2 ba[NG / 2], bg[NG / 2];
#pragma unroll
            for (int g = 0; g < NG / 2; ++g) {
                const int cc = c0 + 8 * g;
                ba[g] = bg[g] = make_float2(0.f, 0.f);
                if (bias && cc < H) {
                    ba[g] = __ldg(reinterpret_cast<const float2*>(bias + cc));
                    bg[g] = __ldg(reinterpret_cast<const float2*>(bias + H + cc));
                }
            }
            pr.mark(HP_EPI_LOAD);
#pragma unroll
            for (int g = 0; g < NG / 2; ++g) {             // tile columns 0..BN/2-1; the gate of column j is column j + BN/2
                const int cc = c0 + 8 * g;
                if (cc >= H) continue;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!r_ok[h]) continue;
                    const int i = 4 * g + 2 * h;
                    const long long r = row + 8 * h;
                    float2 a = make_float2(acc[i], acc[i + 1]), gt = make_float2(acc[i + BN / 4], acc[i + 1 + BN / 4]);
                    if (bias) { a.x += ba[g].x; a.y += ba[g].y; gt.x += bg[g].x; gt.y += bg[g].y; }
                    if (y) {
                        *reinterpret_cast<float2*>(y + r * Ntot + cc) = a;
                        *reinterpret_cast<float2*>(y + r * Ntot + H + cc) = gt;
                    }
                    const float2 o = make_float2(a.x * sigmoid_f(gt.x), a.y * sigmoid_f(gt.y));
                    *reinterpret_cast<float2*>(glu_out + r * H + cc) = o;
                    am = fmaxf(am, fmaxf(fabsf(o.x), fabsf(o.y)));
                }
            }
            pr.mark(HP_EPI_STORE);
        } else {
            // One copy of the row loop per combination of fused outputs the launchers use, each compiled with only the
            // code its outputs need, and the general loop for any other combination.  Every copy computes each output
            // element with the same expression, so the outputs are bitwise those of the general loop.  The general loop
            // is fully unrolled with every output behind a runtime branch: at BN = 160 the kernel's consumer code was
            // ~140 KB of SASS, most of it branched over by any one combination, and the specialised copies ran the
            // epilogues of the step's convs 5-37 % faster (DESIGN §4.2).
            using F = std::false_type;
            using Tr = std::true_type;
            const bool plain = !addend && !aux && !act && !out_tmajor;
            if (stats && plain) epilogue_rows<BN>(c, acc, m0, partial, pr, am, Tr(), F(), F(), F());
            else if (stats) epilogue_rows<BN>(c, acc, m0, partial, pr, am, Tr(), Tr(), Tr(), Tr());
            else if (plain) epilogue_rows<BN>(c, acc, m0, partial, pr, am, F(), F(), F(), F());
            else if (out_tmajor && !addend && !aux && !act) epilogue_rows<BN>(c, acc, m0, partial, pr, am, F(), F(), F(), Tr());
            else if ((aux || act) && !addend && !out_tmajor) epilogue_rows<BN>(c, acc, m0, partial, pr, am, F(), F(), Tr(), F());
            else if (addend && !aux && !act && !out_tmajor) epilogue_rows<BN>(c, acc, m0, partial, pr, am, F(), Tr(), F(), F());
            else epilogue_rows<BN>(c, acc, m0, partial, pr, am, F(), Tr(), Tr(), Tr());
        }
        if (out_amax) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
            if ((threadIdx.x & 31) == 0 && am > 0.f) atomicMax(out_amax, __float_as_uint(am));
        }
    }
    // The non-GLU epilogue of `epilogue`: STATS / ADD / ACT / TMAJ compile in the BatchNorm statistics, the addend, the
    // pre-activation copy with GELU, and the channel-major store (each still taken only where its pointer or flag is set).
    template <int BN, class STATS, class ADD, class ACT, class TMAJ>
    __device__ __forceinline__ void epilogue_rows(const Cta& c, const float* acc, int m0, float (*partial)[2][BN],
                                                  HcProbe& pr, float& am, STATS, ADD, ACT, TMAJ) const {
        constexpr int NW = HC_CONSUMERS / 32, NG = BN / 8;    // consumer warps; 8-column groups of the fragment
        constexpr int GS = NG / 2;                           // column groups per load batch (registers: acc + 60)
        constexpr bool S_ = STATS::value, A_ = ADD::value, G_ = ACT::value, M_ = TMAJ::value;
        const int tq = threadIdx.x & 3, t = c.t0 + m0 + hg_row(0);
        const bool r_ok[2] = {t < T, t + 8 < T};
        const long long row = (long long)c.b * T + t;          // the thread's rows: row and row + 8
        {
            const int n0 = c.n_tile * BN + 2 * tq;            // the thread's columns: n0 + 8 g (+1)
            const int warp = hc_consumer_tid() >> 5;
#pragma unroll
            for (int g0 = 0; g0 < NG; g0 += GS) {
                float2 bv[GS], av[GS][2];
#pragma unroll
                for (int k = 0; k < GS; ++k) {
                    const int n = n0 + 8 * (g0 + k);
                    bv[k] = av[k][0] = av[k][1] = make_float2(0.f, 0.f);
                    if (n >= Ntot) continue;
                    if (bias) bv[k] = __ldg(reinterpret_cast<const float2*>(bias + n));
                    if (A_ && addend) {
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            if (r_ok[h]) av[k][h] = *reinterpret_cast<const float2*>(addend + (row + 8 * h) * Ntot + n);
                    }
                }
                pr.mark(HP_EPI_LOAD);
#pragma unroll
                for (int k = 0; k < GS; ++k) {
                    const int g = g0 + k, n = n0 + 8 * g;
                    float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};     // columns n and n + 1, summed over rows r, r + 8
                    if (n < Ntot) {
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            if (!r_ok[h]) continue;
                            const long long r = row + 8 * h;
                            float v[2] = {acc[4 * g + 2 * h], acc[4 * g + 2 * h + 1]};
                            if (bias) { v[0] += bv[k].x; v[1] += bv[k].y; }
                            if (A_ && addend) { v[0] += av[k][h].x; v[1] += av[k][h].y; }
                            if (G_ && aux) *reinterpret_cast<float2*>(aux + r * Ntot + n) = make_float2(v[0], v[1]);
                            if (G_ && act) {
                                v[0] = gelu_f(v[0]);
                                v[1] = gelu_f(v[1]);
                                am = fmaxf(am, fmaxf(fabsf(v[0]), fabsf(v[1])));
                            }
                            if (M_ && out_tmajor) {
                                y[((long long)c.b * Ntot + n) * T + t + 8 * h] = v[0];
                                y[((long long)c.b * Ntot + n + 1) * T + t + 8 * h] = v[1];
                            } else {
                                *reinterpret_cast<float2*>(y + r * Ntot + n) = make_float2(v[0], v[1]);
                            }
                            if (S_ && stats) {
                                // about the bias: exact (Sterbenz) while the bias dominates, and what is left is centred
                                const float d[2] = {v[0] - bv[k].x, v[1] - bv[k].y};
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    s1[e] += d[e];
                                    s2[e] = fmaf(d[e], d[e], s2[e]);
                                }
                            }
                        }
                    }
                    if (S_ && stats) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
#pragma unroll
                            for (int o = 4; o < 32; o <<= 1) {
                                s1[e] += __shfl_xor_sync(0xffffffffu, s1[e], o);
                                s2[e] += __shfl_xor_sync(0xffffffffu, s2[e], o);
                            }
                        }
                        if ((threadIdx.x & 31) < 4) {
                            const int j = 8 * g + 2 * tq;
                            *reinterpret_cast<float2*>(&partial[warp][0][j]) = make_float2(s1[0], s1[1]);
                            *reinterpret_cast<float2*>(&partial[warp][1][j]) = make_float2(s2[0], s2[1]);
                        }
                    }
                }
                pr.mark(HP_EPI_STORE);
            }
            if (S_ && stats) {
                hc_consumer_sync();                      // every warp's partials of this tile are in `partial`
                const int j = hc_consumer_tid(), n = c.n_tile * BN + j;
                if (j < BN && n < Ntot) {
                    double d1 = 0.0, d2 = 0.0;
#pragma unroll
                    for (int w = 0; w < NW; ++w) {
                        d1 += (double)partial[w][0][j];
                        d2 += (double)partial[w][1][j];
                    }
                    // back from the bias-shifted sums over the tile's rows: sum (d + b) and sum (d + b)^2
                    const double b = bias ? (double)__ldg(bias + n) : 0.0, rows = (double)min(HG_BM, T - c.t0);
                    atomicAdd(stats + n, fma(rows, b, d1));
                    atomicAdd(stats + Ntot + n, d2 + b * fma(rows, b, 2.0 * d1));
                }
                hc_consumer_sync();                      // the reads, before the next tile's partials overwrite them
            }
        }
    }
};

// Data gradient of the sensor mix (ChannelMerger, common.py:358) as a pointwise ConvOp with one weight set per recording:
//   dmeg[b, c, t] = mask[c] * sum_o du[b, t, o] * W[wsel[b]][c][o]
// x = du [B,T,Cin=Op], w = the transposed attention weights [R][Ntot=Cp][Op].  Its own epilogue stores only the C live sensor
// rows, channel-major [B,C,T], times the channel mask (nullable; its columns are loaded before the first store); the
// ConvOp epilogue itself is untouched.
struct SensorMixBwdOp : ConvOp {
    int C;
    const float* mask;
    template <int BN, int PASSES> __device__ void epilogue(const Cta& c, const float* acc, int m0, HcProbe& pr) const {
        const int n0 = c.n_tile * BN + 2 * (threadIdx.x & 3), t = c.t0 + m0 + hg_row(0);   // columns n0 + 8 g + e
        float m[BN / 8][2];
#pragma unroll
        for (int g = 0; g < BN / 8; ++g)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = n0 + 8 * g + e;
                m[g][e] = mask && n < C ? __ldg(mask + n) : 1.f;
            }
        pr.mark(HP_EPI_LOAD);
#pragma unroll
        for (int g = 0; g < BN / 8; ++g) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = n0 + 8 * g + e;
                if (n >= C) continue;
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (t + 8 * h < T) y[((long long)c.b * C + n) * T + t + 8 * h] = acc[4 * g + 2 * h + e] * m[g][e];
            }
        }
        pr.mark(HP_EPI_STORE);
    }
};

inline ConvOp conv_op_defaults() {
    ConvOp o;
    memset(&o, 0, sizeof(o));
    o.n_wsets = 1;
    o.passes = 3;
    return o;
}

// The launch every conv entry point ends in, once it has filled its ConvOp (or SensorMixBwdOp): the time and column
// tiling, the zeroed BatchNorm statistics and the kernel.  `who` is the entry point, for the error messages.
template <class Op> inline int launch_conv(Op o, cudaStream_t st, const char* who) {
    if ((long long)o.B * o.T >= (1ll << 31)) return set_error(2, "%s: too many rows%s", who);
    if (std::is_same<Op, ConvOp>::value) {    // ConvOp's epilogue accesses float2; SensorMixBwdOp's stores scalars
        auto a8 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; };
        if (!a8(o.bias) || !a8(o.addend) || !a8(o.aux) || !a8(o.glu_out) || (!o.out_tmajor && !a8(o.y)))
            return set_error(2, "%s: bias, addend and the row-major outputs must be 8-byte aligned%s", who);
    }
    o.ttiles = (o.T + HG_BM - 1) / HG_BM;
    const int bn = hg_pick_bn(o.Ntot);                   // GLU: BN/2 'a' columns and their gates per tile
    o.ncols = o.glu ? (o.Ntot / 2 + bn / 2 - 1) / (bn / 2) : (o.Ntot + bn - 1) / bn;
    if (o.stats) {
        cudaError_t em = cudaMemsetAsync(o.stats, 0, sizeof(double) * 2 * o.Ntot, st);
        if (em != cudaSuccess) return set_error(3, "%s: memset: %s", who, cudaGetErrorString(em));
    }
    return hc_launch_bn(bn, o, (long long)o.B * o.ttiles * o.ncols, st, who);
}

// ---- the published shape gates and epilogue rules ---------------------------------------------------------------------
// The kernel itself handles any N; the gates are the library's contract.
// bm_tc_conv1d / bm_tc_pointwise_sel: Ntot a multiple of 16 with a divisor in [64, 160] (GLU: H a multiple of 80), K chunks
// of 32 input channels.
inline bool conv_tc_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    if (Kw < 1 || Kw > 3 || (Kw & 1) == 0) return false;
    if (Cin % HG_BK != 0) return false;
    if (glu) return Ntot % 2 == 0 && (Ntot / 2) % 80 == 0;
    for (int bn = 160; bn >= 64; bn -= 16)
        if (Ntot % bn == 0) return true;
    return false;
}

// bm_tc_conv1d_persistent / bm_tc_conv1d_f16: the output columns split into pairs of column halves of nh = 160 or 128
// (Ntot a multiple of 2 nh; GLU: H a multiple of nh), K chunks of 32 input channels.  conv_half_width: nh, 0 if none.
inline int conv_half_width(int Ntot, int glu) {
    if (glu && (Ntot % 2)) return 0;
    const int n = glu ? Ntot / 2 : Ntot;
    for (int nh = 160; nh >= 128; nh -= 32)
        if (n % (glu ? nh : 2 * nh) == 0) return nh;
    return 0;
}
inline bool conv_halves_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    if (Kw < 1 || Kw > 3 || (Kw & 1) == 0) return false;
    if (Cin % HG_BK != 0) return false;
    return conv_half_width(Ntot, glu) != 0;
}
// The epilogue combinations bm_tc_conv1d_persistent* and bm_tc_conv1d_f16 accept (accumulate: y += conv in place), for a
// shape that passed conv_halves_supported: 0, or 2 with the reason.  BatchNorm statistics need a plain conv of one pair of
// column halves (Ntot = 2 nh).
inline int conv_halves_epilogue_check(int Ntot, int glu, int act, int out_tmajor, int accumulate, const float* aux,
                                      const double* stats, const char* who) {
    if (stats && (glu || out_tmajor || act || accumulate || Ntot != 2 * conv_half_width(Ntot, 0)))
        return set_error(2, "%s: statistics need a plain single-N-tile conv%s", who);
    if (glu && (act || out_tmajor || aux || accumulate)) return set_error(2, "%s: GLU excludes the other epilogues%s", who);
    if (out_tmajor && (act || accumulate)) return set_error(2, "%s: channel-major output is a plain store%s", who);
    if (act && accumulate) return set_error(2, "%s: accumulate excludes the activation%s", who);
    return 0;
}

// ---- weight preparation -------------------------------------------------------------------------------------------------
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
        // a NULL lo pointer asks for the RAW fp32 value in the re-laid array (bm_tc_conv1d_persistent's weights: the
        // kernel splits them on load)
        if (f_hi) { if (f_lo) { f_hi[fi] = h; f_lo[fi] = l; } else f_hi[fi] = v; }
        if (g_hi) { if (g_lo) { g_hi[gi] = h; g_lo[gi] = l; } else g_hi[gi] = v; }
    }
}

// The fp16 pieces of bm_tc_conv1d_f16's weights: w*s = hi + lo (11 + 11 significant bits) with s = f16_scale_of(amax).
// largest |x| of a tensor into `cell` (a float whose bits compare like an unsigned integer because it is non-negative);
// NaNs are ignored by fmaxf, +-inf gives inf (=> scale 1: the conv then propagates the non-finite values like fp32 would).
// x need only be float-aligned (the generic epilogue and GLU forms run on misaligned views): the `head` elements before its
// first 16-byte boundary and the tail after the last whole float4 are read one by one.
__global__ void __launch_bounds__(256) amax_kernel(const float* __restrict__ x, long long n, unsigned int* __restrict__ cell) {
    float m = 0.f;
    const long long head = min(n, (long long)(((16 - (reinterpret_cast<uintptr_t>(x) & 15)) & 15) >> 2));
    const long long n4 = (n - head) >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x + head);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(x4 + i);
        m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
    }
    if (blockIdx.x == 0) {
        for (long long i = threadIdx.x; i < head; i += blockDim.x) m = fmaxf(m, fabsf(x[i]));
        for (long long i = head + (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(x[i]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float wm[8];
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) m = fmaxf(m, wm[w]);
        if (m > 0.f) atomicMax(cell, __float_as_uint(m));
    }
}
// src * scale(amax) -> fp16 hi and lo copies (same element order)
__global__ void __launch_bounds__(256) f16_split_kernel(const float* __restrict__ src, long long n,
                                                        const float* __restrict__ amax, __half* __restrict__ hi,
                                                        __half* __restrict__ lo) {
    const float s = f16_scale_of(__ldg(amax));
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = src[i] * s;
        const __half h = __float2half_rn(v);
        hi[i] = h;
        lo[i] = __float2half_rn(v - __half2float(h));
    }
}

// W[o][i][j] (nn.Conv1d layout) * scale(amax) -> fp16 hi / lo pieces in the K-major layouts of bm_tc_weight_split:
//   forward operand F[j][o][i], data-gradient operand G[j][i][o]; either pair may be NULL.  One launch per layer and step
//   instead of re-layout + two splits.
__global__ void __launch_bounds__(256) weight_split_f16_kernel(const float* __restrict__ W, const float* __restrict__ amax,
                                                               __half* __restrict__ f_hi, __half* __restrict__ f_lo,
                                                               __half* __restrict__ g_hi, __half* __restrict__ g_lo, int O, int I,
                                                               int Kw) {
    const float s = f16_scale_of(__ldg(amax));
    const long long total = (long long)O * I * Kw;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(idx % Kw);
        const long long oi = idx / Kw;
        const int i = (int)(oi % I), o = (int)(oi / I);
        const float v = W[idx] * s;
        const __half h = __float2half_rn(v);
        const __half l = __float2half_rn(v - __half2float(h));
        const long long fi = ((long long)j * O + o) * I + i, gi = ((long long)j * I + i) * O + o;
        if (f_hi) { f_hi[fi] = h; f_lo[fi] = l; }
        if (g_hi) { g_hi[gi] = h; g_lo[gi] = l; }
    }
}

int launch_amax(const float* x, long long n, float* cell, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(cell, 0, 4, st);
    if (e != cudaSuccess) return set_error(3, "%s: memset: %s", __func__, cudaGetErrorString(e));
    long long blocks = (n / 4 + 255) / 256;
    const long long cap = (long long)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    amax_kernel<<<(int)blocks, 256, 0, st>>>(x, n, reinterpret_cast<unsigned int*>(cell));
    ++g_launches;
    e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: launch failed: %s", __func__, cudaGetErrorString(e));
    return 0;
}
inline int launch_f16_split(const float* src, long long n, const float* amax, void* hi, void* lo, cudaStream_t st) {
    f16_split_kernel<<<ew_grid(n), 256, 0, st>>>(src, n, amax, reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo));
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: launch failed: %s", __func__, cudaGetErrorString(e));
    return 0;
}

}  // namespace tc
}  // namespace bm
