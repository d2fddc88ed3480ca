// C-ABI entry points of the tensor-core convs and weight gradients (see include/bm_b200.h for the contract).
#include "api.cuh"
#include "tc_conv.cuh"
#include "tc_wgrad.cuh"
#include "tc_wgradp.cuh"

using namespace bm;

#ifdef BM_HC_PHASES
// the per-phase probe's counters (tc_common.cuh HcPhase): out[kernel * HP_N + phase] after the device is idle; reset: zero
// them.  Only in the probe build of profiles/conv_phase_probe.py, not part of the ABI.
extern "C" int bm_hc_phases(unsigned long long* out, int reset) {
    BM_CUDA(cudaDeviceSynchronize());
    BM_CUDA(cudaMemcpyFromSymbol(out, tc::g_hc_phases, sizeof(tc::g_hc_phases)));
    if (reset) {
        static const unsigned long long zeros[2 * tc::HP_N] = {};
        BM_CUDA(cudaMemcpyToSymbol(tc::g_hc_phases, zeros, sizeof(zeros)));
    }
    return 0;
}
#endif

// =================================================================================================
// tensor-core (wgmma) versions of K3/K4
// =================================================================================================
extern "C" int bm_tc_conv_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    return tc::conv_tc_supported(T, Cin, Ntot, Kw, glu) ? 1 : 0;
}

extern "C" int bm_tc_weight_split(const float* w, int Cout, int Cin, int Kw, float* f_hi, float* f_lo, float* g_hi,
                                  float* g_lo, bm_stream_t stream) {
    BM_CHECK_ARG(w && Cout > 0 && Cin > 0 && Kw > 0);
    BM_CHECK_ARG((f_hi || g_hi) && !(f_lo && !f_hi) && !(g_lo && !g_hi));
    tc::weight_split_kernel<<<ew_grid((long long)Cout * Cin * Kw), 256, 0, ST(stream)>>>(w, f_hi, f_lo, g_hi, g_lo,
                                                                                       Cout, Cin, Kw);
    BM_CHECK_LAUNCH();
    return 0;
}

// passes = 1 (the _tf32 form): w_hi alone is read, w_lo may be NULL; TC_BF16 (the _bf16 form): w_hi + w_lo is read,
// w_lo may be NULL (w_hi then holds the raw fp32 weights)
static int tc_conv1d(int passes, const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* addend,
                     int B, int T, int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                     float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(stats == nullptr);      // BatchNorm statistics in the epilogue: bm_tc_conv1d_persistent / bm_tc_conv1d_f16
    BM_CHECK_ARG(x && w_hi && (w_lo || passes != 3) && B > 0 && T > 0 && dilation >= 1 && (sign == 1 || sign == -1));
    BM_CHECK_ARG(glu ? (glu_out != nullptr) : (y != nullptr));
    BM_CHECK_ARG(B <= 65535);
    BM_CHECK_ARG(!(glu && (act || out_tmajor || aux)));
    BM_CHECK_ARG(tc::conv_tc_supported(T, Cin, Ntot, Kw, glu));
    tc::ConvOp o = tc::conv_op_defaults();
    o.x = x; o.w = w_hi; o.w_lo32 = passes == 1 ? nullptr : w_lo; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = Kw; o.dilation = dilation; o.sign = sign; o.glu = glu;
    o.bias = bias; o.addend = addend; o.y = y; o.aux = aux; o.glu_out = glu_out; o.act = act; o.out_tmajor = out_tmajor;
    o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_conv1d, tc_conv1d,
            (const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* addend, int B, int T,
             int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor, float* y, float* aux,
             float* glu_out, double* stats, int* status, bm_stream_t stream),
            (x, w_hi, w_lo, bias, addend, B, T, Cin, Ntot, Kw, dilation, sign, glu, act, out_tmajor, y, aux, glu_out, stats,
             status, stream))

// weight gradient of a (dilated) conv / pointwise layer on the tensor cores: dW[m][n][tap] = sum_{b,t} dY[b,t,m] X[b,t+s,n]
extern "C" int bm_tc_wgrad_supported(int M, int N) { return tc::wgrad_tc_supported(M, N) ? 1 : 0; }
extern "C" long long bm_tc_wgrad_workspace(int B, int M, int N, int Kw) {
    return (long long)tc::wgrad_workspace_floats(B, M, N, Kw);
}
static int tc_wgrad(int passes, const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                    float* workspace, float* dw, float* dbias, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(dy && x && workspace && dw && B > 0 && T > 0 && Kw >= 1 && Kw <= 3 && dilation >= 1);
    BM_CHECK_ARG(tc::wgrad_tc_supported(M, N) && Ntrue > 0 && Ntrue <= N);
    return tc::launch_wgrad_tc(dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, passes, ST(stream), dbias);
}
BM_TC_FORMS(bm_tc_wgrad, tc_wgrad,
            (const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation, float* workspace,
             float* dw, float* dbias, int* status, bm_stream_t stream),
            (dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, dbias, status, stream))

// weight gradient of a k-tap conv (csrc/tc_wgradp.cuh): output rows = (tap, x channel), reduction over the
// flattened rows; no bias gradient (use bm_col_sum on dy where the layer's bias gradient is not exactly zero)
extern "C" int bm_tc_wgrad_conv_supported(int T, int M, int N, int Kw) {
    return tc::wgradp_supported(T, M, N, Kw) ? 1 : 0;
}
extern "C" long long bm_tc_wgrad_conv_workspace(int B, int T, int M, int N, int Kw) {
    return (long long)tc::wgradp_workspace_floats(B, T, M, N, Kw);
}
static int tc_wgrad_conv(int passes, const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw,
                         int dilation, float* workspace, float* dw, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(dy && x && workspace && dw && B > 0 && T > 0 && dilation >= 1);
    BM_CHECK_ARG(tc::wgradp_supported(T, M, N, Kw) && Ntrue > 0 && Ntrue <= N);
    return tc::launch_wgrad_pp(dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, passes, status, ST(stream));
}
BM_TC_FORMS(bm_tc_wgrad_conv, tc_wgrad_conv,
            (const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation, float* workspace,
             float* dw, int* status, bm_stream_t stream),
            (dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, status, stream))

// the same weight gradient for callers that hold the operands' amax (csrc/tc_wgradp.cuh): dy_amax / x_amax = device floats with max |dy|, max |x|
// (bm_amax, or the amax_out of the kernels that produced the tensors); same shape gate and workspace as bm_tc_wgrad_conv
extern "C" int bm_tc_wgrad_conv_f16(const float* dy, const float* dy_amax, const float* x, const float* x_amax, int B, int T,
                                    int M, int N, int Ntrue, int Kw, int dilation, float* workspace, float* dw, int* status,
                                    bm_stream_t stream) {
    BM_CHECK_ARG(dy && dy_amax && x && x_amax && workspace && dw && B > 0 && T > 0 && dilation >= 1);
    BM_CHECK_ARG(tc::wgradp_supported(T, M, N, Kw) && Ntrue > 0 && Ntrue <= N);
    return tc::launch_wgrad_pp(dy, x, B, T, M, N, Ntrue, Kw, dilation, workspace, dw, 3, status, ST(stream));
}

extern "C" int bm_tc_conv1d_persistent_supported(int T, int Cin, int Ntot, int Kw, int glu) {
    return tc::conv_halves_supported(T, Cin, Ntot, Kw, glu) ? 1 : 0;
}
// w_raw = the RAW fp32 weights re-laid K-major [Kw][Ntot][Cin] (bm_tc_weight_split with f_lo / g_lo = NULL);
// accumulate=1: y += conv (in place)
static int tc_conv1d_persistent(int passes, const float* x, const float* w_raw, const float* bias, int accumulate, int B,
                                int T, int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                                float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(x && w_raw && B > 0 && T > 0 && dilation >= 1 && (sign == 1 || sign == -1));
    BM_CHECK_ARG(glu ? (glu_out != nullptr) : (y != nullptr));
    BM_CHECK_ARG(tc::conv_halves_supported(T, Cin, Ntot, Kw, glu));
    if (int rc = tc::conv_halves_epilogue_check(Ntot, glu, act, out_tmajor, accumulate, aux, stats, __func__)) return rc;
    tc::ConvOp o = tc::conv_op_defaults();
    o.x = x; o.w = w_raw; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = Kw; o.dilation = dilation; o.sign = sign; o.glu = glu;
    o.bias = bias; o.addend = accumulate ? y : nullptr; o.y = y; o.aux = act ? aux : nullptr; o.glu_out = glu_out;
    o.act = act; o.out_tmajor = out_tmajor; o.stats = stats; o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_conv1d_persistent, tc_conv1d_persistent,
            (const float* x, const float* w_raw, const float* bias, int accumulate, int B, int T, int Cin, int Ntot, int Kw,
             int dilation, int sign, int glu, int act, int out_tmajor, float* y, float* aux, float* glu_out, double* stats,
             int* status, bm_stream_t stream),
            (x, w_raw, bias, accumulate, B, T, Cin, Ntot, Kw, dilation, sign, glu, act, out_tmajor, y, aux, glu_out, stats,
             status, stream))

// ---- the same conv with fp16-piece weights: fp32 weights as two fp16 pieces of a power-of-two-scaled tensor.  bm_amax
// writes the largest magnitude of a tensor into a device float; bm_f16_split prepares the weights (w_raw [Kw][Ntot][Cin] ->
// fp16 hi / lo copies of w_raw * scale(amax)); the kernel scales x itself.
extern "C" int bm_amax(const float* x, long long n, float* amax, bm_stream_t stream) {
    BM_CHECK_ARG(x && amax && n > 0);
    return tc::launch_amax(x, n, amax, ST(stream));
}
extern "C" int bm_f16_split(const float* src, long long n, const float* amax, void* hi, void* lo, bm_stream_t stream) {
    BM_CHECK_ARG(src && amax && hi && lo && n > 0);
    return tc::launch_f16_split(src, n, amax, hi, lo, ST(stream));
}
extern "C" int bm_tc_weight_split_f16(const float* w, const float* w_amax, int Cout, int Cin, int Kw, void* f_hi, void* f_lo,
                                      void* g_hi, void* g_lo, bm_stream_t stream) {
    BM_CHECK_ARG(w && w_amax && Cout > 0 && Cin > 0 && Kw > 0);
    BM_CHECK_ARG((f_hi || g_hi) && (!f_hi == !f_lo) && (!g_hi == !g_lo));
    tc::weight_split_f16_kernel<<<ew_grid((long long)Cout * Cin * Kw), 256, 0, ST(stream)>>>(
        w, w_amax, reinterpret_cast<__half*>(f_hi), reinterpret_cast<__half*>(f_lo), reinterpret_cast<__half*>(g_hi),
        reinterpret_cast<__half*>(g_lo), Cout, Cin, Kw);
    BM_CHECK_LAUNCH();
    return 0;
}
extern "C" int bm_tc_conv1d_f16(const float* x, const float* x_amax, const void* w_hi, const void* w_lo, const float* w_amax,
                                const float* bias, int accumulate, int B, int T, int Cin, int Ntot, int Kw, int dilation,
                                int sign, int glu, int act, int out_tmajor, float* y, float* aux, float* glu_out,
                                double* stats, float* amax_out, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(x && x_amax && w_hi && w_lo && w_amax && B > 0 && T > 0 && dilation >= 1 && (sign == 1 || sign == -1));
    BM_CHECK_ARG(glu ? (glu_out != nullptr) : (y != nullptr));
    BM_CHECK_ARG(tc::conv_halves_supported(T, Cin, Ntot, Kw, glu));
    BM_CHECK_ARG(!amax_out || ((glu || act) && !out_tmajor));      // the outputs another conv consumes: GLU out, GELU out
    if (int rc = amax_begin(amax_out, ST(stream))) return rc;
    if (int rc = tc::conv_halves_epilogue_check(Ntot, glu, act, out_tmajor, accumulate, aux, stats, __func__)) return rc;
    tc::ConvOp o = tc::conv_op_defaults();          // passes = 3: the fp16 pieces have no single-pass form
    o.x = x; o.w_hi = reinterpret_cast<const __half*>(w_hi); o.w_lo = reinterpret_cast<const __half*>(w_lo); o.w_amax = w_amax;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = Kw; o.dilation = dilation; o.sign = sign; o.glu = glu;
    o.bias = bias; o.addend = accumulate ? y : nullptr; o.y = y; o.aux = act ? aux : nullptr; o.glu_out = glu_out;
    o.act = act; o.out_tmajor = out_tmajor; o.stats = stats; o.out_amax = reinterpret_cast<unsigned int*>(amax_out);
    o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}

// pointwise (1x1) contraction with a per-sample weight set (SubjectLayers.forward / its data gradient, common.py:55-58):
//   y[b,t,n] = sum_k x[b,t,k] W[wsel[b]][n][k];  w_hi/w_lo are the tf32-split K-major weight sets [S][Ntot][Cin]
static int tc_pointwise_sel(int passes, const float* x, const float* w_hi, const float* w_lo, const int* wsel, int n_sets,
                            int B, int T, int Cin, int Ntot, float* y, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(x && w_hi && (w_lo || passes != 3) && wsel && y && n_sets > 0 && B > 0 && B <= 65535 && T > 0);
    BM_CHECK_ARG(tc::conv_tc_supported(T, Cin, Ntot, 1, 0));
    tc::ConvOp o = tc::conv_op_defaults();
    o.x = x; o.w = w_hi; o.w_lo32 = passes == 1 ? nullptr : w_lo; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Cin; o.Ntot = Ntot; o.taps = 1; o.dilation = 1; o.sign = 1;
    o.n_wsets = n_sets; o.wsel = wsel; o.y = y; o.err = status;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_pointwise_sel, tc_pointwise_sel,
            (const float* x, const float* w_hi, const float* w_lo, const int* wsel, int n_sets, int B, int T, int Cin,
             int Ntot, float* y, int* status, bm_stream_t stream),
            (x, w_hi, w_lo, wsel, n_sets, B, T, Cin, Ntot, y, status, stream))

// data gradient of the sensor mix on the tensor cores (ChannelMerger, common.py:358):
//   dmeg[b,c,t] = mask[c] sum_o du[b,t,o] W[wsel[b]][c][o], c < C;  w_hi / w_lo: tf32-split transposed weight sets [S][Cp][Op]
static int tc_sensor_mix_bwd_data(int passes, const float* du, const float* w_hi, const float* w_lo, const int* wsel,
                                  int n_sets, const float* mask, int B, int T, int Op, int Cp, int C, float* dmeg, int* status,
                                  bm_stream_t stream) {
    BM_CHECK_ARG(du && w_hi && (w_lo || passes != 3) && wsel && dmeg && n_sets > 0 && B > 0 && T > 0 && C > 0 && C <= Cp);
    BM_CHECK_ARG(tc::conv_tc_supported(T, Op, Cp, 1, 0));
    tc::SensorMixBwdOp o;
    memset(&o, 0, sizeof(o));
    o.x = du; o.w = w_hi; o.w_lo32 = passes == 1 ? nullptr : w_lo; o.passes = passes;
    o.B = B; o.T = T; o.Cin = Op; o.Ntot = Cp; o.taps = 1; o.dilation = 1; o.sign = 1;
    o.n_wsets = n_sets; o.wsel = wsel; o.y = dmeg; o.err = status; o.C = C; o.mask = mask;
    return tc::launch_conv(o, ST(stream), __func__);
}
BM_TC_FORMS(bm_tc_sensor_mix_bwd_data, tc_sensor_mix_bwd_data,
            (const float* du, const float* w_hi, const float* w_lo, const int* wsel, int n_sets, const float* mask, int B,
             int T, int Op, int Cp, int C, float* dmeg, int* status, bm_stream_t stream),
            (du, w_hi, w_lo, wsel, n_sets, mask, B, T, Op, Cp, C, dmeg, status, stream))

// per-group pointwise weight gradient (SubjectLayers: dM[s] = sum over the samples of subject s), tensor cores:
//   out[g][m][n] = sum_{b in group g} sum_t dy[b,t,m] x[b,t,n];  out is [G][ceil(M/128)*128][N]
static int tc_wgrad_grouped(int passes, const float* dy, const float* x, const int* order, const int* seg_off, int G, int B,
                            int T, int M, int N, float* out, int* status, bm_stream_t stream) {
    BM_CHECK_ARG(dy && x && order && seg_off && out && G > 0 && B > 0 && T > 0);
    BM_CHECK_ARG(tc::wgrad_tc_supported(M, N));
    return tc::launch_wgrad_tc_grouped(dy, x, order, seg_off, G, B, T, M, N, out, passes, ST(stream));
}
BM_TC_FORMS(bm_tc_wgrad_grouped, tc_wgrad_grouped,
            (const float* dy, const float* x, const int* order, const int* seg_off, int G, int B, int T, int M, int N,
             float* out, int* status, bm_stream_t stream),
            (dy, x, order, seg_off, G, B, T, M, N, out, status, stream))
