// K3/K4/K5 (dilated Conv1d / Conv1d+GLU / head 1x1, forward and data gradient) with the RAW fp32 weights re-laid K-major
// [Kw][Ntot][Cin] (bm_tc_weight_split with NULL lo pointers): the ConvOp GEMM of tc_conv.cuh, whose producer warps split the
// weights into tf32 pieces on their way into shared memory.
//
//   y[p, n] = bias[n] + sum_tap sum_k x[p + shift(tap), k] * W[tap][n][k]        p = b*T + t (channels-last rows)
//
// Epilogue modes: store y | y += conv (accumulate, in place) | aux = pre-activation (nullable), y = GELU |
// GLU: y = h (nullable), glu_out = a * sigmoid(gate) | y channel-major [B][Ntot][T]; BatchNorm statistics of y (plain store).
#pragma once
#include "tc_conv.cuh"
#include "tc_pair.cuh"

namespace bm {
namespace tc {

inline int conv_pp_pick_nh(int Ntot, int glu) { return pair_pick_nh(Ntot, glu); }
inline bool conv_pp_supported(int T, int Cin, int Ntot, int Kw, int glu) { return pair_conv_supported(T, Cin, Ntot, Kw, glu); }

// x [R = B*T, Cin] channels-last rows; w_raw [Kw][Ntot][Cin] (fp32, K-major re-layout of the nn.Conv1d weight)
struct ConvPPArgs {
    const float* x; const float* w_raw; const float* bias;
    int B, T, Cin, Ntot, taps, dilation, sign;
    int glu, act, out_tmajor, accumulate;     // accumulate: y += conv (in place)
    int passes;                               // 3: 3xTF32, 1: single-pass TF32
    float* y; float* aux; float* glu_out; double* stats; int* err;
};

inline ConvOp conv_pp_op(const ConvPPArgs& a) {
    ConvOp o = conv_op_defaults();
    o.x = a.x; o.w = a.w_raw; o.bias = a.bias; o.B = a.B; o.T = a.T; o.Cin = a.Cin; o.Ntot = a.Ntot; o.taps = a.taps;
    o.dilation = a.dilation; o.sign = a.sign; o.glu = a.glu; o.act = a.act; o.out_tmajor = a.out_tmajor;
    o.addend = a.accumulate ? a.y : nullptr; o.y = a.y; o.aux = a.act ? a.aux : nullptr; o.glu_out = a.glu_out;
    o.stats = a.stats; o.err = a.err; o.passes = a.passes;
    return o;
}

inline int launch_conv_pp(const ConvPPArgs& a, cudaStream_t st) {
    const int nh = conv_pp_pick_nh(a.Ntot, a.glu);
    if (nh == 0 || nh % 32 != 0) return set_error(2, "%s: unsupported N%s", __func__);
    const int ntn = a.glu ? (a.Ntot / 2) / nh : a.Ntot / (2 * nh);
    if (a.stats && (a.glu || a.out_tmajor || a.act || a.accumulate || ntn != 1))
        return set_error(2, "%s: statistics need a plain single-N-tile conv%s", __func__);
    if (a.glu && (a.act || a.out_tmajor || a.aux || a.accumulate)) return set_error(2, "%s: GLU excludes the other epilogues%s", __func__);
    if (a.out_tmajor && (a.act || a.accumulate)) return set_error(2, "%s: channel-major output is a plain store%s", __func__);
    if (a.act && a.accumulate) return set_error(2, "%s: accumulate excludes the activation%s", __func__);

    return launch_conv_op(conv_pp_op(a), st, __func__);
}

}  // namespace tc
}  // namespace bm
