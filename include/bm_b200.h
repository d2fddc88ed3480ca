/* brainmagick_b200 -- C ABI of the H100-native (sm_90a) contrastive training step (SimpleConv + ClipLoss).
 *
 * The reference (facebookresearch/brainmagick) has no FFI: its boundary for this path is the Python object
 * surface of `bm.models.SimpleConv` (bm/models/simpleconv.py:22-249) and `bm.losses.ClipLoss`
 * (bm/losses.py:29-114), called from bm/solver.py:297,373 and bm/train.py:84-86.  The drop-in modules in
 * `brainmagick_b200/` keep that surface and call THIS library through ctypes; INTEGRATION.md shows the binding.
 *
 * Conventions (all entry points):
 *   - plain pointers and sizes only; every pointer is DEVICE memory unless stated; fp32 data, int32 indices,
 *     fp64 only for the small statistics scratch buffers;
 *   - the caller owns every buffer (inputs, outputs, saved activations, scratch); the library never allocates;
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*); no entry point synchronises;
 *   - returns 0 on success, non-zero on error; `bm_last_error()` gives the message (thread local);
 *   - activations inside the encoder are channels-last [B, T, C]; the model input `meg` [B, C, T], the encoder
 *     output `estimate` [B, F, T] and the `candidates` [B', F, T] keep the reference's channel-major layout.
 * There is no CPU fallback anywhere in this library.
 */
#ifndef BM_B200_H_
#define BM_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef void* bm_stream_t;

const char* bm_last_error(void);
int bm_abi_version(void);
/* number of CUDA kernels this library has launched since it was loaded (bench.py's `gpu_launches`). */
unsigned long long bm_launch_count(void);
/* experiment switches (returns the previous value).  No switch is defined: every kernel ignores the flags (kept for
 * ABI compatibility). */
int bm_set_debug_flags(int flags);
/* profiling aid (process-wide, NOT part of the product path): device buffer for per-CTA cycle counters; the current
 * kernels record none.  NULL (default). */
int bm_set_debug_buffer(long long* buf);

/* ---- K1: spatial-attention weights, once per recording ------------------------------------------------
 * replaces FourierEmb.forward (bm/models/common.py:254-271) + the score/softmax half of ChannelMerger.forward
 * (common.py:337-357).  positions [R,C,2] (INVALID=-0.1 marks padded sensors), freq [n] = 2*pi*arange(n)/1.4
 * with n = sqrt(P/2), heads [O,P], ban_centre [2] or NULL (eval / dropout 0).
 * out: emb [R,C,P] (saved for backward), weights [R,O,C] = softmax over C. */
int bm_attention_weights_fwd(const float* positions, const float* freq, const float* heads,
                             const float* ban_centre, float radius, int R, int C, int O, int P, float* emb,
                             float* weights, bm_stream_t stream);
/* dweights [R,O,C] -> dheads [O,P]; dscores is [R,O,C] scratch. */
int bm_attention_weights_bwd(const float* dweights, const float* weights, const float* emb, int R, int C, int O,
                             int P, float* dscores, float* dheads, bm_stream_t stream);

/* K1 in pieces (the two contractions -- scores = emb heads^T and dheads = dscores^T emb -- then run on the tensor-core
 * kernels bm_tc_conv1d_persistent(out_tmajor) / bm_tc_wgrad): Fourier embedding, in-place masked softmax, softmax backward. */
int bm_fourier_emb(const float* positions, const float* freq, int R, int C, int P, float* emb, bm_stream_t stream);
int bm_masked_softmax(float* weights, const float* positions, const float* ban_centre, float radius, int R, int O, int C,
                      bm_stream_t stream);
int bm_softmax_bwd(const float* weights, const float* dweights, long long rows, int C, float* dscores,
                   bm_stream_t stream);

/* ---- K2: sensor chain ----------------------------------------------------------------------------------
 * replaces the mixing einsum of ChannelMerger.forward (common.py:358), `initial_linear` (simpleconv.py:113-120,
 * 213-214) and SubjectLayers.forward (common.py:55-58):
 *   u[b,t,o] = sum_c weights[rec[b],o,c] meg[b,c,t];  v = il_w u + il_b;  x0[b,t,d] = sum_p subj_w[subj[b],p,d] v[b,t,p]
 * meg [B,C,T]; il_w [IL,O]; subj_w [S,IL,D]; out u [B,T,O], v [B,T,IL], x0 [B,T,ld_x0] (channels-last; ld_x0 >= D
 * lets the caller keep x0 zero-padded to a multiple of 32 channels for the tensor-core conv that follows). */
int bm_sensor_chain_fwd(const float* meg, const float* weights, const int* rec_of_sample, const float* il_w,
                        const float* il_b, const float* subj_w, const int* subject, int B, int C, int T, int O,
                        int IL, int D, int ld_x0, float* u, float* v, float* x0, bm_stream_t stream);
/* dx0 [B,T,D] -> d_subj_w [S,IL,D], d_il_w [IL,O], d_il_b [IL], d_weights [R,O,C].
 * (subj_order, subj_off[S+1]) and (rec_order, rec_off[R+1]) are CSR groupings of the samples by subject and by
 * recording; dv [B,T,IL] and du [B,T,O] are scratch (du also out: the gradient at the mix output).
 * Frozen parameters: d_subj_w, d_il_w, d_il_b, d_weights may each be NULL; its GEMM / reduction is skipped.  du may be
 * NULL when d_weights is (nothing below needs it), dv when du, d_il_w and d_il_b are; a stage with no output left is not
 * run.  With every pointer non-NULL the call is the full backward. */
int bm_sensor_chain_bwd(const float* dx0, const float* meg, const float* il_w, const float* subj_w,
                        const int* subject, const float* u, const float* v, const int* subj_order,
                        const int* subj_off, const int* rec_order, const int* rec_off, int B, int C, int T, int O,
                        int IL, int D, int ld_x0, int S, int R, float* dv, float* du, float* d_subj_w, float* d_il_w,
                        float* d_il_b, float* d_weights, bm_stream_t stream);

/* The same chain as separate stages with explicit leading dimensions (u / v / dv / du / x0 may be kept zero-padded to a
 * multiple of 64 channels so that `initial_linear` runs on the tensor-core pointwise kernel, bm_tc_conv1d_persistent Kw=1). */
int bm_sensor_mix_fwd(const float* meg, const float* weights, const int* rec_of_sample, int B, int C, int T, int O,
                      int ld_u, float* u, bm_stream_t stream);
int bm_initial_linear_fwd(const float* u, int ld_u, const float* il_w, const float* il_b, int B, int T, int O, int IL,
                          int ld_v, float* v, bm_stream_t stream);
int bm_subject_layers_fwd(const float* v, int ld_v, const float* subj_w, const int* subject, int B, int T, int IL, int D,
                          int ld_x0, float* x0, bm_stream_t stream);
/* bm_subject_layers_bwd: dv (the data gradient) and d_subj_w may each be NULL -- NULL dv: nothing below needs it (v, the
 * CSR grouping are then read only for d_subj_w); NULL d_subj_w: frozen weights (v and the grouping may be NULL).
 * bm_initial_linear_bwd (and its _det form): du, d_il_w and d_il_b may each be NULL and skip their GEMM / column sum; the
 * _det form needs no workspace (NULL, 0) when d_il_w and d_il_b are both NULL. */
int bm_subject_layers_bwd(const float* dx0, int ld_x0, const float* v, int ld_v, const float* subj_w, const int* subject,
                          const int* subj_order, const int* subj_off, int B, int T, int IL, int D, int S, int ld_dv,
                          float* dv, float* d_subj_w, bm_stream_t stream);
int bm_initial_linear_bwd(const float* dv, int ld_dv, const float* u, int ld_u, const float* il_w, int B, int T, int O,
                          int IL, int ld_du, float* du, float* d_il_w, float* d_il_b, bm_stream_t stream);
int bm_sensor_mix_bwd(const float* du, int ld_du, const float* meg, const int* rec_order, const int* rec_off, int B, int C,
                      int T, int O, int R, float* d_weights, bm_stream_t stream);
/* Data gradient of the sensor mix, for callers that backpropagate to `meg` (gradient-based attribution, input
 * optimisation): dmeg[b,c,t] = mask[c] * sum_o weights[rec[b],o,c] du[b,t,o].  du [B,T,ld_du]; weights [R,O,C]; mask [C]
 * (nullable = all ones: SimpleConv's subsample_meg_channels mask, simpleconv.py:200-203); dmeg [B,C,T] channel-major.
 * Sensors with attention weight 0 (INVALID / banned) receive exactly 0. */
int bm_sensor_mix_bwd_data(const float* du, int ld_du, const float* weights, const int* rec_of_sample, const float* mask, int B,
                           int C, int T, int O, float* dmeg, bm_stream_t stream);

/* ---- K3: dilated Conv1d + train-mode BatchNorm + GELU + skip (ConvSequence, common.py:98-151) ------------
 * w [Cout,Cin,Kw] -> wf [Kw,Cin,Cout] (forward operand), wb [Kw,Cout,Cin] (data-gradient operand). */
int bm_conv_weight_prep(const float* w, int Cout, int Cin, int Kw, float* wf, float* wb, bm_stream_t stream);
/* y[b,t,o] = bias[o] + sum_{i,j} w[o,i,j] x[b, t+(j-Kw/2)*dilation, i]  (zero outside [0,T)); x,y channels-last.
 * stats (nullable): fp64 [2*Cout] receiving sum(y), sum(y^2) over (b,t) -- zeroed by this call. */
int bm_conv1d_fwd(const float* x, const float* wf, const float* bias, int B, int T, int Cin, int Cout, int Kw,
                  int dilation, float* y, double* stats, bm_stream_t stream);
/* batch statistics -> mean, invstd; updates running stats (nullable) like nn.BatchNorm1d(momentum). */
int bm_bn_stats_finalize(const double* stats, long long n, float eps, float momentum, float* running_mean,
                         float* running_var, float* mean, float* invstd, int C, bm_stream_t stream);
/* bm_bn_stats_finalize with n read on the device from stats[2C] (stats fp64 [2C + 1]): the SyncBatchNorm form, whose sums
 * and row count are all-reduced over the group in one buffer without a host read of the count. */
int bm_bn_stats_finalize_counted(const double* stats, float eps, float momentum, float* running_mean, float* running_var,
                                 float* mean, float* invstd, int C, bm_stream_t stream);
/* Cumulative-average forms of the two above (nn.BatchNorm1d with momentum=None): the running statistics are updated with
 * factor 1 / num_batches_tracked, read on the device from the layer's int64 counter, which the caller has already
 * incremented for this batch on the same stream (torch's order: increment, then factor).  The host never reads the count.
 * running_mean / running_var are required. */
int bm_bn_stats_finalize_cumulative(const double* stats, long long n, float eps, const long long* num_batches_tracked,
                                    float* running_mean, float* running_var, float* mean, float* invstd, int C,
                                    bm_stream_t stream);
int bm_bn_stats_finalize_counted_cumulative(const double* stats, float eps, const long long* num_batches_tracked,
                                            float* running_mean, float* running_var, float* mean, float* invstd, int C,
                                            bm_stream_t stream);
int bm_bn_eval_stats(const float* running_mean, const float* running_var, float eps, float* mean, float* invstd,
                     int C, bm_stream_t stream);
/* x_new = GELU(gamma*(y-mean)*invstd + beta) (+ x_old if not NULL); rows = B*T.
 * amax_out (nullable; the same argument on bm_bn_gelu_skip_bwd, bm_glu_bwd, bm_tc_conv1d_f16): a device float that receives
 * max |output| -- the x_amax of the F16-pipe conv (bm_tc_conv1d_f16) that consumes the tensor next, produced by the kernel
 * that writes the tensor instead of a separate bm_amax pass over it. */
int bm_bn_gelu_skip_fwd(const float* y, const float* mean, const float* invstd, const float* gamma,
                        const float* beta, const float* x_old, float* x_new, long long rows, int C, float* amax_out,
                        bm_stream_t stream);
/* g = dL/dx_new -> dy (through GELU and BN), dgamma, dbeta.  batch_stats=1: training-mode BN backward.
 * sums: fp64 [2*C] scratch.
 * batch_stats=0 with dgamma == dbeta == NULL (an eval-mode BatchNorm whose affine parameters are frozen): sums may be NULL
 * too, and the call is one elementwise pass over g and y -- no column reduction, no fp64 scratch, and no workspace in the
 * _det form (NULL, 0).  Its dy is bitwise the reducing form's.  With batch_stats=1, sums / dgamma / dbeta stay required:
 * the data gradient needs the sums.  The same holds for bm_bn_act_skip_bwd(_det) with a BatchNorm (mean != NULL). */
int bm_bn_gelu_skip_bwd(const float* g, const float* y, const float* mean, const float* invstd,
                        const float* gamma, const float* beta, int batch_stats, long long rows, int C,
                        double* sums, float* dy, float* dgamma, float* dbeta, float* amax_out /* of dy */,
                        bm_stream_t stream);
/* bm_bn_gelu_skip_bwd with batch_stats=1 in two calls, so that a SyncBatchNorm caller can all-reduce the sums between them:
 * _reduce writes sums [2C] = (sum dz, sum dz*yhat) over its rows and the local dbeta / dgamma (their float roundings);
 * _apply writes dy from sums fp64 [2C + 1], the group's sums with the group's row count n in sums[2C] (read on the device).
 * With the local sums and n = rows the pair gives bm_bn_gelu_skip_bwd's bits. */
int bm_bn_gelu_skip_bwd_reduce(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                               const float* beta, long long rows, int C, double* sums, float* dgamma, float* dbeta,
                               bm_stream_t stream);
int bm_bn_gelu_skip_bwd_apply(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                              const float* beta, long long rows, int C, const double* sums, float* dy, bm_stream_t stream);
/* dx = conv_transpose(dy) (+ addend, the skip-path gradient, if not NULL). */
int bm_conv1d_bwd_data(const float* dy, const float* wb, const float* addend, int B, int T, int Cin, int Cout,
                       int Kw, int dilation, float* dx, bm_stream_t stream);
/* dw [Cout,Cin,Kw] (reference layout), dbias [Cout]. */
int bm_conv1d_bwd_weight(const float* dy, const float* x, int B, int T, int Cin, int Cout, int Kw, int dilation,
                         float* dw, float* dbias, bm_stream_t stream);

/* ---- K4: Conv1d(H -> 2H, Kw, pad=Kw/2) + GLU (common.py:133-138) ----------------------------------------
 * wf [Kw,Cin,2H]; h (nullable, saved for backward) [B,T,2H]; out [B,T,H] = h[:, :H] * sigmoid(h[:, H:]). */
int bm_conv1d_glu_fwd(const float* x, const float* wf, const float* bias, int B, int T, int Cin, int H, int Kw,
                      float* h, float* out, bm_stream_t stream);
int bm_glu_bwd(const float* g, const float* h, long long rows, int H, float* dh,
               float* dbias /* nullable [2H]: sum over rows of dh = the GLU conv's bias gradient, from the same pass */,
               float* amax_out /* of dh */, bm_stream_t stream);
/* (bm_glu_bwd_det with dbias == NULL reduces nothing and needs no workspace: NULL, 0.) */

/* ---- K5: head Conv1d(H,2H,1) -> GELU -> ConvTranspose1d(2H,F,1) (simpleconv.py:185-189,246-249) --------
 * x [B,T,H]; w0 [2H,H]; w2 [2H,F] (ConvTranspose1d weight is input-major); out h1,q [B,T,2H], est [B,F,T]. */
int bm_head_fwd(const float* x, const float* w0, const float* b0, const float* w2, const float* b2, int B, int T,
                int H, int F, float* h1, float* q, float* est, bm_stream_t stream);
/* dest [B,F,T] -> dx [B,T,H], dw0 [2H,H], db0 [2H], dw2 [2H,F], db2 [F]; dq [B,T,2H] scratch.
 * dw0, db0, dw2, db2 (frozen head parameters) and dx (nothing below needs it) may each be NULL and skip their GEMM /
 * reduction; with dx, dw0 and db0 all NULL neither dq nor GELU'(h1) is computed (dq, h1, w2 may then be NULL).  The _det
 * form needs no workspace (NULL, 0) when all four parameter gradients are NULL. */
int bm_head_bwd(const float* dest, const float* x, const float* w0, const float* w2, const float* h1,
                const float* q, int B, int T, int H, int F, float* dq, float* dx, float* dw0, float* db0,
                float* dw2, float* db2, bm_stream_t stream);

/* parameter-gradient half of bm_head_bwd, for callers that compute dq and dx themselves (tensor-core path):
 * in: dq = d(loss)/dq [B,T,2H]; out: dw2, db2, dq <- dq*GELU'(h1) (in place), dw0, db0.  dw0, db0, dw2, db2 may each be
 * NULL (x is read only for dw0, q only for dw2); dq always becomes dh1. */
int bm_head_bwd_params(const float* dest, const float* x, const float* h1, const float* q, int B, int T, int H, int F,
                       float* dq, float* dw0, float* db0, float* dw2, float* db2, bm_stream_t stream);

/* ---- K6: ClipLoss (bm/losses.py:77-114) -----------------------------------------------------------------
 * est [Bn,KT], cand [Bc,KT] (KT = F*T, any consistent flattening).
 * bm_clip_scores = ClipLoss.get_scores (+ get_probabilities when probs != NULL):
 *   inv_norm[o] = 1/(1e-8+||cand_o||), scores[b,o] = inv_norm[o] <est_b, cand_o>, probs = softmax_o(scores).
 *   norms_given = 1: inv_norm is an INPUT (a fixed candidate set is normed once, see bm_candidate_inv_norms).
 * One split-K wgmma GEMM (3xTF32; every 32-wide K block is accumulated into an fp32 round-to-nearest running sum,
 * because the tensor core's accumulator truncates), a row sum of squares for the candidate norms, + one finalize kernel (slice reduction in a fixed order, norm scale, row softmax / cross-entropy / batch mean).
 * workspace: bm_clip_workspace(Bn,Bc,KT) floats of caller-owned scratch, 8-byte aligned; status: device int set on a
 * kernel failure (reserved; never hangs).  KT % 4 != 0 (no 16-byte row pitch) falls to the FP32-FMA GEMM of this library. */
long long bm_clip_workspace(int Bn, int Bc, long long KT);
int bm_clip_scores(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given, float* inv_norm,
                   float* scores, float* probs, float* workspace, long long workspace_floats, int* status,
                   bm_stream_t stream);
/* inv_norm[o] = 1/(1e-8+||cand_o||) alone (losses.py:91); ss fp64 [Bc] scratch. */
int bm_candidate_inv_norms(const float* cand, int Bc, long long KT, double* ss, float* inv_norm, bm_stream_t stream);
/* ClipLoss.forward: loss = mean_b CE(scores[b,:], target_offset + b).  target_offset = 0 is the reference;
 * rank*Bn is the multi-GPU extension with all-gathered candidates.  row_loss [Bn], loss [1]; inv_norm, scores, probs
 * are outputs kept for the backward. */
int bm_clip_loss_fwd(const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset,
                     float* inv_norm, float* scores, float* probs, float* row_loss, float* loss, float* workspace,
                     long long workspace_floats, int* status, bm_stream_t stream);
/* dL/dest [Bn,KT] = gout * ((probs - onehot)/Bn * inv_norm) @ cand ; G [Bn,Bc] scratch; gout [1] on device. */
int bm_clip_loss_bwd(const float* probs, const float* inv_norm, const float* cand, const float* gout, int Bn,
                     int Bc, long long KT, int target_offset, float* G, float* dest, int* status, bm_stream_t stream);
/* The same over pooled candidates (the solver's `optim.negatives` pool, bm/solver.py:358-371): candidate o is cand[o] for
 * o < Bb (the batch, read in place) and arena[slots[o - Bb]] for Bb <= o < Bc (a row of the pool's device storage, slots
 * int32 [Bc - Bb] on the device; arena and slots may be NULL when Bb == Bc).  The contiguous forms' arithmetic, bit for bit:
 * the forward runs the same kernels with one more load per pool row; the backward always runs the wgmma GEMM of
 * bm_clip_loss_bwd's Bn >= 192 form, over G [Bn, ldg] scratch with ldg = Bc rounded up to a multiple of 4 (zero columns).
 * Requires KT % 4 == 0 and KT >= 32.  The `_det`, `_tf32` and `_bf16` forms are those of bm_clip_loss_fwd. */
int bm_clip_loss_fwd_pooled(const float* est, const float* cand, int Bb, const float* arena, const int* slots, int Bn,
                            int Bc, long long KT, int target_offset, float* inv_norm, float* scores, float* probs,
                            float* row_loss, float* loss, float* workspace, long long workspace_floats, int* status,
                            bm_stream_t stream);
int bm_clip_loss_bwd_pooled(const float* probs, const float* inv_norm, const float* cand, int Bb, const float* arena,
                            const int* slots, const float* gout, int Bn, int Bc, long long KT, int target_offset, float* G,
                            float* dest, int* status, bm_stream_t stream);

/* ---- Stand-alone ConvSequence / DeepMel (SURVEY 8(f) row 3): bm/models/common.py:79-151, bm/models/features.py:15-35 --
 * Layer epilogue x_new = act(bn(y)) (+ x_old) over channels-last rows [rows, C] and its backward, for any activation:
 * act 0 = GELU, 1 = LeakyReLU(slope) (common.py:95), 2 = none; mean == NULL = no BatchNorm (the layer then only applies the
 * activation / the skip).  bm_bn_gelu_skip_*, bm_bn_act_skip_* and bm_bn_act_gain_skip_* are forms of one epilogue: where
 * their contracts overlap (BatchNorm + GELU, no gain) they give the same bits.
 * bm_bn_act_skip_bwd: dy = d/dy of the above given g = dL/dx_new (the skip branch's gradient is g itself);
 * batch_stats=1: training-mode BatchNorm (dgamma, dbeta, fp64 sums [2C] scratch), 0: eval statistics. */
int bm_bn_act_skip_fwd(const float* y, const float* mean, const float* invstd, const float* gamma, const float* beta,
                       const float* x_old, float* x_new, long long rows, int C, int act, float slope,
                       bm_stream_t stream);
int bm_bn_act_skip_bwd(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                       const float* beta, int batch_stats, long long rows, int C, int act, float slope, double* sums,
                       float* dy, float* dgamma, float* dbeta, bm_stream_t stream);
/* bm_bn_act_skip_bwd with a training-mode BatchNorm in two calls, as bm_bn_gelu_skip_bwd_reduce / _apply. */
int bm_bn_act_skip_bwd_reduce(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                              const float* beta, long long rows, int C, int act, float slope, double* sums, float* dgamma,
                              float* dbeta, bm_stream_t stream);
int bm_bn_act_skip_bwd_apply(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                             const float* beta, long long rows, int C, int act, float slope, const double* sums, float* dy,
                             bm_stream_t stream);
/* Residual gain of a ConvSequence layer (LayerScale and post_skip, common.py:65-76,126-130):
 * x_new = post[c] * ((boost * scale[c]) * branch) (+ x_old), branch = act(bn(y)) as in bm_bn_act_skip_fwd; scale [C]
 * (LayerScale's parameter, boost its factor 5) and post [C] (the depthwise 1x1 conv's weight) are each nullable (gain 1).
 * bm_bn_act_gain_skip_bwd: dy = d/dy of the branch given gain(g), g = dL/dx_new, with the BatchNorm cases of
 * bm_bn_act_skip_bwd, and in the same reduction pass S[c] = sum_rows g*branch (branch recomputed from y; fp32 per thread, fp64
 * across threads and blocks, as the BatchNorm sums):
 * dscale = boost*post*S, dpost = (boost*scale)*S, each nullable (frozen: not reduced).  sums: fp64 scratch [3C], needed
 * when anything is reduced (a BatchNorm in training mode, dgamma / dbeta, dscale or dpost). */
int bm_bn_act_gain_skip_fwd(const float* y, const float* mean, const float* invstd, const float* gamma, const float* beta,
                            const float* x_old, float* x_new, long long rows, int C, int act, float slope,
                            const float* scale, float boost, const float* post, bm_stream_t stream);
int bm_bn_act_gain_skip_bwd(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                            const float* beta, int batch_stats, long long rows, int C, int act, float slope,
                            const float* scale, float boost, const float* post, double* sums, float* dy, float* dgamma,
                            float* dbeta, float* dscale, float* dpost, bm_stream_t stream);
/* Gradient of ClipLoss.forward w.r.t. the CANDIDATES (a trainable feature model, solver.py:304-320): with G as in
 * bm_clip_loss_bwd, dcand[o] = sum_b G[b,o] est[b] - coef[o] cand[o], coef[o] = (sum_b G[b,o] scores[b,o]) / ||cand_o||
 * (the derivative of the 1/(1e-8+||.||) normalisation, losses.py:91).  G [Bn,Bc], coef [Bc]: scratch. */
int bm_clip_loss_bwd_cand(const float* probs, const float* scores, const float* inv_norm, const float* est,
                          const float* cand, const float* gout, int Bn, int Bc, long long KT, int target_offset,
                          float* G, float* coef, float* dcand, int* status, bm_stream_t stream);
/* Backward of ClipLoss.get_scores (losses.py:91-94) for an arbitrary upstream gradient dscores [Bn,Bc]: with
 * G = dscores * inv_norm (per column), dest [Bn,KT] = G @ cand and dcand [Bc,KT] = G^T est - coef * cand, coef as in
 * bm_clip_loss_bwd_cand (0 for a zero candidate, as autograd's norm backward defines it).  The same GEMMs as
 * bm_clip_loss_bwd / bm_clip_loss_bwd_cand.  dest and dcand are each nullable; scores [Bn,Bc], est and coef [Bc] (scratch)
 * are needed for dcand only.  G [Bn,Bc]: scratch.  get_probabilities: dscores = bm_softmax_bwd(probs, dprobs) first. */
int bm_clip_scores_bwd(const float* dscores, const float* scores, const float* inv_norm, const float* est, const float* cand,
                       int Bn, int Bc, long long KT, float* G, float* coef, float* dest, float* dcand, int* status,
                       bm_stream_t stream);

/* ---- Retrieval evaluation (SURVEY 8(f) row 1): scripts/run_eval_probs.py:237-307, bm/wer.py:80-116 ---------
 * The score matrix comes from bm_clip_scores (queries x candidates, candidate axis optionally zero-padded to the
 * tensor-core tile: ld >= n_cols); these entry points replace the host-side softmax / topk / scatter_add / label
 * comparison the reference runs per query (wer.py) or per query batch on the CPU copy (run_eval_probs.py).
 * bm_retrieval_topk, one row b of `vals` (stride ld) at a time:
 *   is_prob=0: vals are scores, p = softmax over the n_cols columns (row_max/row_sum, nullable, receive its stats);
 *   is_prob=1: vals are probabilities already, negative entries are holes;
 *   own_values [Bn] (nullable): per-row value standing in column own_col -- wer.py:93 overwrites the last negative
 *     with the query's own true output; own_labels [Bn] likewise for that column's label (wer.py:94);
 *   top_idx/top_prob [Bn,k] (nullable): the k best columns, best first, ties -> lower column (-1 / 0 if fewer);
 *   hit[b] = rank (0 = best) of the first of the k selected columns whose label is targets[b], -1 if none: a top-k'
 *     hit for any k' <= k is 0 <= hit[b] < k' (run_eval_probs.py:253-259, wer.py:107-111);
 *   soft[b] = sum of p over the columns whose label is targets[b] (wer.py:114-115).
 * bm_retrieval_probs: probs [Bn,n_cols] = softmax(scores[:, :n_cols])  (ClipLoss.get_probabilities, losses.py:97-102).
 * bm_retrieval_vocab_probs: per-word probabilities (wer.py:101-104) without atomics: vocab [Bn,V+1],
 *   vocab[b][w] = sum_{j in seg[w]..seg[w+1]} p[b][perm[j]] (+ the own candidate's p when own_word[b] == w);
 *   column V = own p when own_word[b] == V (a word no shared negative carries), else -1 (a hole for bm_retrieval_topk).
 * bm_rowdot_scaled: own[b] = <a_b, c_b> / (1e-8 + ||c_b||): the score of a query against its own true output. */
int bm_retrieval_topk(const float* vals, long long ld, int Bn, int n_cols, const float* own_values, int own_col,
                      int is_prob, int k, const long long* labels, const long long* own_labels,
                      const long long* targets, long long* top_idx, float* top_prob, int* hit, float* soft,
                      float* row_max, float* row_sum, bm_stream_t stream);
int bm_retrieval_probs(const float* scores, long long ld, int Bn, int n_cols, float* probs, bm_stream_t stream);
int bm_retrieval_vocab_probs(const float* scores, long long ld, int Bn, const float* own_scores, const float* row_max,
                             const float* row_sum, const int* perm, const int* seg, int V, const int* own_word,
                             float* vocab, bm_stream_t stream);
int bm_rowdot_scaled(const float* a, const float* c, int Bn, long long K, float* own, bm_stream_t stream);

/* ---- Batch preparation (SURVEY 8(f) row 2): bm/norm.py:239-275, 325-341; bm/solver.py:262-274 ---------------
 * bm_scale_clamp_crop: y [B,C,T_out] = op(x [B,C,T])[..., t0:t0+T_out] with op = (x - center[slot[b]][c]) / scale[..]
 *   (BatchScaler.transform; inverse=1: x*scale + center), then clamp to +-limit when clip (ScaleReject, norm.py:332-333)
 *   -- one pass, bit-identical to the reference's fp32 arithmetic.  center/scale: [R,C] tables (RobustScaler per
 *   recording, or one row of per-channel StandardScaler constants with slot = NULL).  peak_bits [B] (nullable): bit
 *   pattern of max |op(x)| over the whole uncropped sample (what ScaleReject tests, norm.py:334).
 * bm_reject_compact: keep[b] = !(peak > limit) && (mask == NULL || any(mask[b])) (norm.py:335-339);
 *   keep_rows = kept sample indices in order, n_keep[0] their count.
 * bm_gather_rows: y[i] = x[rows[i]] over rows of row_elems floats (batch[keep], norm.py:340).
 * bm_scatter_rows: y[rows[i]] = x[i], its inverse (rows distinct): a batch written into free rows of the negative pool. */
int bm_scale_clamp_crop(const float* x, const int* slot, const float* center, const float* scale, int B, int C, int T,
                        int t0, int T_out, float limit, int clip, int inverse, float* y, unsigned int* peak_bits,
                        bm_stream_t stream);
int bm_reject_compact(const unsigned int* peak_bits, const unsigned char* mask, long long mask_elems, float limit,
                      int B, unsigned char* keep, int* keep_rows, int* n_keep, bm_stream_t stream);
int bm_gather_rows(const float* x, const int* rows, int n_rows, long long row_elems, float* y, bm_stream_t stream);
int bm_scatter_rows(const float* x, const int* rows, int n_rows, long long row_elems, float* y, bm_stream_t stream);

/* ---- tensor-core (wgmma) versions of K3/K4: 3xTF32 implicit-GEMM conv ------------------------------------
 * Same arithmetic contract as bm_conv1d_fwd / bm_conv1d_bwd_data / bm_conv1d_glu_fwd (fp32-faithful: every
 * product is hi*hi + lo*hi + hi*lo of tf32 splits, fp32 accumulation per 32-wide K block).
 * bm_tc_weight_split: w [Cout,Cin,Kw] -> forward operand f_hi/f_lo [Kw,Cout,Cin] and data-gradient operand
 * g_hi/g_lo [Kw,Cin,Cout] (either pair may be NULL).
 * bm_tc_conv1d: x [B,T,Cin], w_hi/w_lo [Kw,Ntot,Cin]; sign=+1 forward taps, -1 data gradient; glu=1: Ntot = 2H,
 * y (nullable) receives h, glu_out [B,T,H].  status: device int (nullable) set non-zero if the kernel's pipeline
 * timed out (never hangs).  bm_tc_conv_supported: shape gate (Cin % 32, Ntot % 160 or H % 80). */
int bm_tc_conv_supported(int T, int Cin, int Ntot, int Kw, int glu);
int bm_tc_weight_split(const float* w, int Cout, int Cin, int Kw, float* f_hi, float* f_lo, float* g_hi,
                       float* g_lo, bm_stream_t stream);
int bm_tc_conv1d(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* addend,
                 int B, int T, int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                 float* y, float* aux, float* glu_out, double* stats /* must be NULL: see bm_tc_conv1d_persistent */,
                 int* status, bm_stream_t stream);
/* act=1: y = GELU(.) and aux (nullable) receives the pre-activation; out_tmajor=1: y is [B,Ntot,T] (the head's
 * channel-major `estimate`).  With Kw=1 this is the pointwise (1x1) contraction of the head (K5).
 * bm_col_stats: stats[0:C] = sum_r y[r,c], stats[C:2C] = sum_r y[r,c]^2 (fp64), the BatchNorm batch statistics. */
int bm_col_stats(const float* y, long long rows, int C, double* stats, bm_stream_t stream);
/* bm_tc_conv1d_persistent: the same conv from the RAW fp32 weights re-laid K-major [Kw][Ntot][Cin] (bm_tc_weight_split with
 * f_lo / g_lo = NULL); the kernel splits them into tf32 pieces itself (taps that would cross a sample edge read zeros =
 * the conv padding).  accumulate=1: y += conv(x) in place (the skip-path gradient).  glu / act / out_tmajor / aux / glu_out as
 * bm_tc_conv1d.  stats (nullable; plain forward only): BatchNorm batch statistics stats[0:Ntot] = sum(y), stats[Ntot:2Ntot]
 * = sum(y^2) (fp64, zeroed by the call) reduced per tile in shared memory -- replaces bm_col_stats.
 * Shape gate (bm_tc_conv1d_persistent_supported): Cin % 32 == 0 and Ntot % 320 == 0 or Ntot % 256 == 0 (GLU: halves). */
int bm_tc_conv1d_persistent_supported(int T, int Cin, int Ntot, int Kw, int glu);
int bm_tc_conv1d_persistent(const float* x, const float* w_raw, const float* bias, int accumulate, int B, int T, int Cin,
                            int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor, float* y,
                            float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream);

/* The same conv with the weights as fp16 pieces (bm_tc_conv1d_f16; replaces the same reference lines as
 * bm_tc_conv1d_persistent: nn.Conv1d / GLU in bm/models/common.py:107-151, the head's 1x1 convs simpleconv.py:153-168).
 * The weights are carried as two fp16 pieces (11 + 11 significant bits) of the tensor times a power of two that puts its
 * largest magnitude in [2^14, 2^15); the kernel sums the pieces back (hi + lo: ~22 significant bits of the weight, the
 * precision of the pieces) and runs the same 3xTF32 GEMM (x_amax is accepted and not needed).  bm_amax: amax[0] =
 * max |x[i]| (device float; one HBM pass).  bm_f16_split: hi/lo = fp16 pieces of
 * src * scale(amax[0]) in the same element order (the weights, once per step, from bm_tc_weight_split's raw K-major
 * re-layout).  bm_tc_conv1d_f16: arguments as bm_tc_conv1d_persistent with (w_hi, w_lo, w_amax) in place of w_raw and
 * x_amax = the device float bm_amax wrote for x; same shape gate. */
int bm_amax(const float* x, long long n, float* amax, bm_stream_t stream);
int bm_f16_split(const float* src, long long n, const float* amax, void* hi, void* lo, bm_stream_t stream);
/* bm_tc_weight_split_f16: bm_tc_weight_split + bm_f16_split in one launch: w [Cout,Cin,Kw] (nn.Conv1d layout) times
 * scale(w_amax[0]) -> fp16 pieces of the forward operand f [Kw,Cout,Cin] and of the data-gradient operand g [Kw,Cin,Cout]
 * (either pair may be NULL); w_amax = bm_amax over w. */
int bm_tc_weight_split_f16(const float* w, const float* w_amax, int Cout, int Cin, int Kw, void* f_hi, void* f_lo, void* g_hi,
                           void* g_lo, bm_stream_t stream);
int bm_tc_conv1d_f16(const float* x, const float* x_amax, const void* w_hi, const void* w_lo, const float* w_amax,
                     const float* bias, int accumulate, int B, int T, int Cin, int Ntot, int Kw, int dilation, int sign,
                     int glu, int act, int out_tmajor, float* y, float* aux, float* glu_out, double* stats,
                     float* amax_out /* nullable: max |glu_out| (glu) or max |y| (act), see bm_bn_gelu_skip_fwd */, int* status,
                     bm_stream_t stream);

/* bm_tc_wgrad: weight gradient on the tensor cores (3xTF32): dw[m][n][tap] = sum_{b,t} dy[b,t,m] x[b,t+(tap-Kw/2)*dil,n]
 * for n < Ntrue (x may be channel-padded to N); dy [B,T,M], x [B,T,N] channels-last; dw in nn.Conv1d layout
 * [M][Ntrue][Kw].  workspace: bm_tc_wgrad_workspace() floats (per-batch-slice partial tiles, reduced in a fixed
 * order => deterministic).  dbias (nullable) [M] receives the bias gradient sum_{b,t} dy[b,t,m], accumulated from the dy
 * values (one column-sum pass).  bm_col_sum: out[c] = sum_r x[r,c] (other bias gradients). */
int bm_tc_wgrad_supported(int M, int N);
long long bm_tc_wgrad_workspace(int B, int M, int N, int Kw);
int bm_tc_wgrad(const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                float* workspace, float* dw, float* dbias, int* status, bm_stream_t stream);
/* bm_tc_wgrad_conv: the same weight gradient as ONE GEMM (csrc/tc_wgradp.cuh) whose output rows are the (tap, x-channel)
 * pairs, reduced over the flattened rows b*T + t in exact chunks of 32 (the tap shift is applied to the x side; a shifted
 * row across a sample edge reads 0).  No dbias output.  T >= 32; M % 64 == 0; N % 4 == 0. */
int bm_tc_wgrad_conv_supported(int T, int M, int N, int Kw);
long long bm_tc_wgrad_conv_workspace(int B, int T, int M, int N, int Kw);
int bm_tc_wgrad_conv(const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                     float* workspace, float* dw, int* status, bm_stream_t stream);
/* bm_tc_wgrad_conv_f16: the same for callers that hold dy_amax / x_amax (device floats: bm_amax or a producer's
 * amax_out); the result is bm_tc_wgrad_conv's (the amax values are not needed by the 3xTF32 arithmetic).  Same gate and
 * workspace. */
int bm_tc_wgrad_conv_f16(const float* dy, const float* dy_amax, const float* x, const float* x_amax, int B, int T, int M,
                         int N, int Ntrue, int Kw, int dilation, float* workspace, float* dw, int* status,
                         bm_stream_t stream);
int bm_col_sum(const float* x, long long rows, int C, float* out, bm_stream_t stream);
/* SubjectLayers (common.py:55-58) on the tensor cores.
 * bm_tc_pointwise_sel: y[b,t,n] = sum_k x[b,t,k] W[wsel[b]][n][k] with tf32-split weight sets w_hi/w_lo [S][Ntot][Cin].
 * bm_tc_wgrad_grouped: out[g][m][n] = sum_{b in group g} sum_t dy[b,t,m] x[b,t,n], groups as CSR (order, seg_off[G+1]);
 * out is [G][ceil(M/128)*128][N] (rows >= M are zero). */
int bm_tc_pointwise_sel(const float* x, const float* w_hi, const float* w_lo, const int* wsel, int n_sets, int B, int T,
                        int Cin, int Ntot, float* y, int* status, bm_stream_t stream);
int bm_tc_wgrad_grouped(const float* dy, const float* x, const int* order, const int* seg_off, int G, int B, int T, int M,
                        int N, float* out, int* status, bm_stream_t stream);
/* bm_sensor_mix_bwd_data on the tensor cores: the pointwise contraction of bm_tc_pointwise_sel with du [B,T,Op] as x and
 * the TRANSPOSED attention weights as the per-recording weight sets, w_hi/w_lo [S][Cp][Op] (tf32 pieces, zero-padded;
 * wsel = rec_of_sample).  The epilogue stores only the C <= Cp live sensor rows, channel-major dmeg [B,C,T], times mask [C]
 * (nullable).  Shape gate: bm_tc_conv_supported(T, Op, Cp, 1, 0). */
int bm_tc_sensor_mix_bwd_data(const float* du, const float* w_hi, const float* w_lo, const int* wsel, int n_sets,
                              const float* mask, int B, int T, int Op, int Cp, int C, float* dmeg, int* status,
                              bm_stream_t stream);
/* dh = dq * GELU'(h), elementwise over n values (dh may alias dq): the head's activation backward. */
int bm_gelu_bwd(const float* dq, const float* h, long long n, float* dh, bm_stream_t stream);
/* y[b,c,t] = x[b,c,t] * mask[c]: SimpleConv(subsample_meg_channels=n) keeps n sensors drawn with random.Random(1234)
 * and zeroes the others before the merger (bm/models/simpleconv.py:97-102, 200-203).  y may alias x. */
int bm_channel_mask(const float* x, const float* mask, int B, int C, int T, float* y, bm_stream_t stream);
/* in [Z,N,T] (channel-major) -> out [Z,T,N] (channels-last): the gradient of `estimate` enters the head backward. */
int bm_transpose_nt(const float* in, int Z, int N, int T, float* out, bm_stream_t stream);
/* same with an output row stride ld_out >= N (pad columns written as zeros): meg [B,C,T] -> channels-last, channel-padded. */
int bm_transpose_nt_ld(const float* in, int Z, int N, int T, int ld_out, float* out, bm_stream_t stream);
/* Channel join of SimpleConv's input streams / encoder outputs (bm/models/simpleconv.py:234-243): dst [B,T,Cp]
 * channels-last receives n (1..4) sources side by side, source i in columns [col_i, col_i + C_i) (ranges must not
 * overlap); every column no source covers is written as zero.  Source i is channels-last (cm_i = 0: rows of stride
 * ld_i >= C_i, an encoder output or the front's x0) or channel-major (cm_i = 1: [B, C_i, T] with channel stride ld_i >= T
 * and sample stride C_i * ld_i, e.g. a raw input stream cropped in time), transposed on the way.  Slots i >= n are
 * ignored.  An exact copy: deterministic, the same under TF32.  B <= 65535. */
int bm_channel_join(int B, int T, int Cp, int n, const float* src0, int C0, int ld0, int cm0, int col0,
                    const float* src1, int C1, int ld1, int cm1, int col1, const float* src2, int C2, int ld2, int cm2,
                    int col2, const float* src3, int C3, int ld3, int cm3, int col3, float* dst, bm_stream_t stream);
/* The reverse, for the gradients: src [B,T,Cp]; dst_i receives columns [col_i, col_i + C_i) in the layout (cm_i, ld_i)
 * of bm_channel_join's sources.  dst_i NULL: that range is not wanted. */
int bm_channel_split(const float* src, int B, int T, int Cp, int n, float* dst0, int C0, int ld0, int cm0, int col0,
                     float* dst1, int C1, int ld1, int cm1, int col1, float* dst2, int C2, int ld2, int cm2, int col2,
                     float* dst3, int C3, int ld3, int cm3, int col3, bm_stream_t stream);
/* ClipLoss's `assert mask.all()` (bm/losses.py:110) on the device, for a step captured in a CUDA graph where the host cannot
 * read the mask: *status <- code (code != 0; only if *status is still 0) when any of the n bytes of `mask` (a bool tensor)
 * is 0.  Nothing is written otherwise; n = 0 enqueues nothing.  The caller raises at its next read of the status word. */
int bm_check_all_true(const unsigned char* mask, long long n, int code, int* status, bm_stream_t stream);

/* ---- Masked regression losses L1Loss / L2Loss (bm/losses.py:11-26) ---------------------------------------------------
 * kind 0 (L1): loss = mean |est - out|, kind 1 (L2): loss = mean (est - out)^2, both over the N entries (b, c, t) where
 * mask[b, c, t] != 0 -- torch.nn.L1Loss() / MSELoss() of est[mask] and out[mask].
 * est and out are [B, C, T] fp32 with t-stride 1 and (b, c) strides est_sb / est_sc and out_sb / out_sc in elements, at any
 * element offset (a view cropped in time is read in place); mask is one byte per entry read at
 * mask[b*mask_sb + c*mask_sc + t*mask_st] (stride 0 along a broadcast dimension).
 * bm_masked_loss_fwd: loss [1] and inv_n [1] = 1 / N on the device; N = 0 gives loss NaN (the mean of nothing).  The sum is
 * taken in fp64 in a fixed order on a grid set by the shape and the SM count: bitwise repeatable, no atomics.  workspace:
 * bm_masked_loss_workspace(B, C, T) floats of caller-owned scratch, 8-byte aligned.
 * bm_masked_loss_bwd: gout [1] the loss's upstream gradient and inv_n [1] from the forward, both read on the device ->
 * d_est = sign(est - out) gout inv_n (L1; sign(0) = 0) or 2 (est - out) gout inv_n (L2) where the mask is set, 0 elsewhere,
 * and d_out = -d_est, each a contiguous [B, C, T] buffer or NULL (not computed). */
long long bm_masked_loss_workspace(int B, int C, int T);
int bm_masked_loss_fwd(int kind, const float* est, long long est_sb, long long est_sc, const float* out, long long out_sb,
                       long long out_sc, const unsigned char* mask, long long mask_sb, long long mask_sc, long long mask_st,
                       int B, int C, int T, float* workspace, long long workspace_floats, float* loss, float* inv_n,
                       bm_stream_t stream);
int bm_masked_loss_bwd(int kind, const float* gout, const float* inv_n, const float* est, long long est_sb, long long est_sc,
                       const float* out, long long out_sb, long long out_sc, const unsigned char* mask, long long mask_sb,
                       long long mask_sc, long long mask_st, int B, int C, int T, float* d_est, float* d_out,
                       bm_stream_t stream);

/* ---- FeatureDecodingLoss (bm/losses.py:117-173) --------------------------------------------------------------------
 * loss = the sum, in feature order, of one fp32 term per feature f = 0..F-1 of a device table of 6 ints per feature:
 * (kind, est_start, width, out_start, weight_offset, lse_slot).
 *   kind 0 (regression): mean (est - out)^2 over the masked entries of est channels [est_start, est_start + width) and out
 *     channels [out_start, out_start + width), the mask's channel c - est_start (mask_sc 0: one channel for all).
 *   kind 1 (categorical, K = width): torch's F.cross_entropy of the logits est[b, est_start + k, t], k < K, against the
 *     target (long) out[b, out_start, t] over the (b, t) where mask[b, 0, t] != 0: sum w_y (lse - z_y) / sum w_y with
 *     w = weights[weight_offset + y] (weight_offset -1: w = 1), ignore_index -100.  lse_slot s: the forward stores the
 *     log-sum-exp of every (b, t) at lse[(s * B + b) * T + t].
 * est and out are fp32 with t-stride 1 and (b, c) strides in elements, at any element offset; mask is one byte per entry
 * read at mask[b*mask_sb + c*mask_sc + t*mask_st].  1 <= F <= 15.
 * bm_decoding_loss_fwd: loss [1] and scale [F] (2 / N_f, or 1 / W_f) on the device; partials in fp64 in a fixed order on a
 * grid set by the shape and the SM count: bitwise repeatable, no atomics.  flag [1] <- 0, or the reference's first error
 * as code | (feature << 16): 904 no mask entry is set (assert mask.any()), 905 a categorical target >= K or NaN at any
 * (b, t) (assert K > output[:, start].max()), 906 a masked target that is negative and not -100 (torch's "target out of
 * bounds").  status (NULL: none) <- the code if it is still 0.  A bad target contributes nothing and indexes nothing.
 * workspace: bm_decoding_loss_workspace(B, T, F) floats of caller-owned scratch, 8-byte aligned.
 * bm_decoding_loss_bwd: gout [1], scale and lse from the forward -> d_est [B, est_C, T] (regression: 2 (est - out) gout /
 * N_f; categorical: gout w_y / W_f (softmax - onehot(y)); 0 where the mask is 0, at ignored or bad targets and on channels
 * no feature holds) and d_out [B, out_C, T] (regression: -d_est of the channel; 0 elsewhere), contiguous, or NULL. */
long long bm_decoding_loss_workspace(int B, int T, int F);
int bm_decoding_loss_fwd(const float* est, long long est_sb, long long est_sc, const float* out, long long out_sb,
                         long long out_sc, const unsigned char* mask, long long mask_sb, long long mask_sc, long long mask_st,
                         int B, int T, const int* table, int F, const float* weights, float* lse, float* workspace,
                         long long workspace_floats, float* loss, float* scale, int* flag, int* status, bm_stream_t stream);
int bm_decoding_loss_bwd(const float* gout, const float* scale, const float* lse, const float* est, long long est_sb,
                         long long est_sc, const float* out, long long out_sb, long long out_sc, const unsigned char* mask,
                         long long mask_sb, long long mask_sc, long long mask_st, int B, int T, int est_C, int out_C,
                         const int* table, int F, const float* weights, float* d_est, float* d_out, bm_stream_t stream);

/* ---- Test metrics (bm/metrics.py: OnlineCorrelation, L1Reg, L2Reg, ClassificationAcc) --------------------------------
 * kind 0 correlation, 1 L1Reg, 2 L2Reg, 3 ClassificationAcc.  dtype / out_dtype 0 fp32, 1 fp64.
 * bm_metric_update adds one update's per-column sums over n < N into acc, fp64 [NP, C*T] on the device (NP = 6 for the
 * correlation: Σ l·r·m, Σ l·m, Σ r·m, Σ (l·m)², Σ (r·m)², count; NP = 2 otherwise: the sum, count), column c*T + t:
 *   kinds 0-2: left and right [N, C, T] read at left[n*left_sn + c*left_sc + t*left_st] (the same for right), any element
 *     offset; L1Reg sums |(l - r)·m|, L2Reg ((l - r)·m)², l - r formed in the operands' dtype.
 *   kind 3 (C = 1): the first index of the maximum (NaN maximal) over the K channels left[n*left_sn + k*left_sc +
 *     t*left_st] compared, as fp64 values, with right[n*right_sn + t*right_st]; the sum counts the equal masked (n, t).
 * m is the mask byte mask[n*mask_sn + c*mask_sc + t*mask_st] (stride 0 along a broadcast dimension) as 0 or 1, multiplied
 * in (a masked-out inf or NaN still gives NaN).  The count adds the mask over its own first dimension mask_n (1 or N).
 * seen [2] int32 on the device: the update reads seen[parity]; while it is 0 the accumulators are overwritten instead of
 * added to.  It stores 1 into seen[parity ^ 1] when seen[parity] is set or a mask entry was True, and nothing else; the
 * caller flips parity after every update.  Sums are fp64 FMAs in a fixed row order; when the columns do not fill the GPU
 * the rows are split into a fixed number of chunks (shape and SM count only) whose partials are added in order by a second
 * launch: one or two launches per update, bitwise repeatable, no atomics.  workspace: bm_metric_workspace(N, C, T) floats
 * of caller-owned scratch, 8-byte aligned (0: none needed; NULL is then accepted).  C*T = 0 (an empty slice or time
 * crop) launches nothing, reads no pointer and leaves seen as it is.
 * bm_metric_finalize: out [C*T] in out_dtype -- the correlation (the reference's get() formula, order and tol) or sum /
 * count -- and flag [1]: bit 1 left norm² < -tol, 2 a left norm² is NaN, 4 and 8 the same for the right, 16 a NaN result,
 * 32 a nonzero count.  With C*T = 0, acc and out may be NULL and flag gets 0. */
long long bm_metric_workspace(int N, int C, int T);
int bm_metric_update(int kind, int dtype, const void* left, long long left_sn, long long left_sc, long long left_st,
                     const void* right, long long right_sn, long long right_sc, long long right_st, const unsigned char* mask,
                     long long mask_sn, long long mask_sc, long long mask_st, int mask_n, int N, int C, int T, int K,
                     double* acc, int* seen, int parity, float* workspace, long long workspace_floats, bm_stream_t stream);
int bm_metric_finalize(int kind, const double* acc, int C, int T, double tol, void* out, int out_dtype, int* flag,
                       bm_stream_t stream);

/* ---- Spectral-norm penalty (bm/svd.py: svd_penalty) -----------------------------------------------------------------
 * For W weights, each the row-major fp32 matrix P [rows_p, cols_p] (a weight viewed as [shape[0], -1]) read in place in its
 * tall orientation A [m, n], m >= n (A = Pᵀ when rows_p < cols_p): the estimate λ of torch.svd_lowrank(P, q, niter)'s
 * S[0]², i.e. the top eigenvalue of Qᵀ A Aᵀ Q where Q spans A (AᵀA)^niter R for the draw R [n, q] (randomized subspace
 * iteration with an orthonormalisation after every product; only the spans enter); when n <= q the span is A's whole range
 * and λ is σ₁(A)² exactly.  Columns of a panel whose Cholesky pivot is at or below 1e-8 of its Gram matrix's largest
 * diagonal are dropped, so a weight of rank below q gives a finite value and gradient (DESIGN §4.10).  Everything is FP32
 * FMA with fp64 Gram matrices and eigenproblems, whatever the TF32 flag or autocast; no atomics and a fixed order everywhere, so repeated calls are bitwise identical.  q = 1..32, niter >= 0.
 * bm_svd_table (host only, no launch) fills table int64 [W, 12] from the weights' device addresses ptrs, shapes and grad
 * flags (nonzero: the weight gets a gradient), and sizes int64 [7]: the float workspace, the double workspace, the draw
 * buffer R and the gradient buffer in elements, then the grouped tile counts tiles_m, tiles_n and tiles_w.  The caller
 * copies the table to the device once and passes it, with those counts, to every call for the same weights and settings.
 * Weight i's draw is R[table[i][7] ...] as an [n_i, q] row-major block, n_i = min(rows_p, cols_p).
 * bm_svd_penalty_fwd: out [1] fp32 = Σ λ_i / proba (fp64 sum in weight order), all on the device; it leaves in ws / ws64
 * (sizes[0] floats / sizes[1] doubles, caller-owned) what the backward of the same call reads.  13 launches at niter = 2
 * (2 niter + 5 at most, fewer when no weight has n > q), whatever W.
 * bm_svd_penalty_bwd: after the forward with the same buffers, writes the gradient gout[0] / proba · dλ_i/dP_i of every
 * weight with a gradient into grad (sizes[3] floats; weight i's [rows_p, cols_p] block at table[i][8]), every element once:
 * for n <= q 2 σ₁ u₁ v₁ᵀ, else the derivative through the spans (DESIGN §4.10).  At most 2 niter + 5 launches, whatever W. */
int bm_svd_table(int W, const long long* ptrs, const long long* rows_p, const long long* cols_p, const int* grad, int q,
                 int niter, long long* table, long long* sizes);
int bm_svd_penalty_fwd(const long long* table, int W, int q, int niter, long long tiles_m, long long tiles_n, const float* R,
                       float* ws, double* ws64, double proba, float* out, bm_stream_t stream);
int bm_svd_penalty_bwd(const long long* table, int W, int q, int niter, long long tiles_m, long long tiles_n,
                       long long tiles_w, const float* R, float* ws, const double* ws64, const float* gout, double proba,
                       float* grad, bm_stream_t stream);

/* ---- Deterministic forms (torch.use_deterministic_algorithms(True) in the drop-in modules) -------------------------
 * Every `_det` entry point computes what its default form computes, with the same arguments plus (where noted) a
 * caller-owned workspace of bm_<op>_det_workspace(dims) floats, 8-byte aligned, checked against `workspace_floats`.  Its
 * floating-point reductions run in a fixed order: each block stores its partial row into the workspace ([n_blocks][width],
 * fp64 where the default form accumulates in fp64) and one more kernel sums the rows in index order; the FP32-FMA
 * split-batch weight-gradient GEMMs store one partial plane per batch segment and sum the planes in segment order (the
 * segment count follows the SM count, so these workspace sizes depend on the device), and the other split GEMMs (dheads,
 * the FP32-FMA CLIP scores) run unsplit.  Repeated calls on the same inputs give bitwise-identical outputs on the same
 * device model and library build; the bits may differ from the default form's.  The entry points of this header that are
 * not listed here have no order-dependent floating-point reduction (or only atomicMax on amax cells, which is exact).
 * With the default form, bm_tc_conv1d_persistent / bm_tc_conv1d_f16 / bm_conv1d_fwd fold the BatchNorm statistics into
 * the conv with atomics; a deterministic caller passes stats = NULL and calls bm_col_stats_det on the output instead, and
 * bm_tc_wgrad callers pass dbias = NULL and call bm_col_sum_det. */
long long bm_col_stats_det_workspace(long long rows, int C);
int bm_col_stats_det(const float* y, long long rows, int C, float* workspace, long long workspace_floats, double* stats,
                     bm_stream_t stream);
long long bm_col_sum_det_workspace(long long rows, int C);
int bm_col_sum_det(const float* x, long long rows, int C, float* workspace, long long workspace_floats, float* out,
                   bm_stream_t stream);
long long bm_bn_gelu_skip_bwd_det_workspace(long long rows, int C);
int bm_bn_gelu_skip_bwd_det(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                            const float* beta, int batch_stats, long long rows, int C, double* sums, float* dy, float* dgamma,
                            float* dbeta, float* amax_out, float* workspace, long long workspace_floats, bm_stream_t stream);
/* workspace unused (may be NULL) when mean == NULL, or batch_stats == 0 with dgamma == dbeta == NULL */
long long bm_bn_act_skip_bwd_det_workspace(long long rows, int C);
int bm_bn_act_skip_bwd_det(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                           const float* beta, int batch_stats, long long rows, int C, int act, float slope, double* sums,
                           float* dy, float* dgamma, float* dbeta, float* workspace, long long workspace_floats,
                           bm_stream_t stream);
long long bm_bn_gelu_skip_bwd_reduce_det_workspace(long long rows, int C);
int bm_bn_gelu_skip_bwd_reduce_det(const float* g, const float* y, const float* mean, const float* invstd,
                                   const float* gamma, const float* beta, long long rows, int C, double* sums, float* dgamma,
                                   float* dbeta, float* workspace, long long workspace_floats, bm_stream_t stream);
long long bm_bn_act_skip_bwd_reduce_det_workspace(long long rows, int C);
int bm_bn_act_skip_bwd_reduce_det(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                                  const float* beta, long long rows, int C, int act, float slope, double* sums, float* dgamma,
                                  float* dbeta, float* workspace, long long workspace_floats, bm_stream_t stream);
/* workspace unused (may be NULL) when nothing is reduced (see bm_bn_act_gain_skip_bwd) */
long long bm_bn_act_gain_skip_bwd_det_workspace(long long rows, int C);
int bm_bn_act_gain_skip_bwd_det(const float* g, const float* y, const float* mean, const float* invstd, const float* gamma,
                                const float* beta, int batch_stats, long long rows, int C, int act, float slope,
                                const float* scale, float boost, const float* post, double* sums, float* dy, float* dgamma,
                                float* dbeta, float* dscale, float* dpost, float* workspace, long long workspace_floats,
                                bm_stream_t stream);
long long bm_glu_bwd_det_workspace(long long rows, int H);
int bm_glu_bwd_det(const float* g, const float* h, long long rows, int H, float* dh, float* dbias, float* amax_out,
                   float* workspace, long long workspace_floats, bm_stream_t stream);
long long bm_conv1d_bwd_weight_det_workspace(int B, int T, int Cin, int Cout, int Kw);
int bm_conv1d_bwd_weight_det(const float* dy, const float* x, int B, int T, int Cin, int Cout, int Kw, int dilation,
                             float* dw, float* dbias, float* workspace, long long workspace_floats, bm_stream_t stream);
long long bm_initial_linear_bwd_det_workspace(int B, int T, int O, int IL);
int bm_initial_linear_bwd_det(const float* dv, int ld_dv, const float* u, int ld_u, const float* il_w, int B, int T, int O,
                              int IL, int ld_du, float* du, float* d_il_w, float* d_il_b, float* workspace,
                              long long workspace_floats, bm_stream_t stream);
long long bm_sensor_chain_bwd_det_workspace(int B, int T, int O, int IL);
int bm_sensor_chain_bwd_det(const float* dx0, const float* meg, const float* il_w, const float* subj_w, const int* subject,
                            const float* u, const float* v, const int* subj_order, const int* subj_off, const int* rec_order,
                            const int* rec_off, int B, int C, int T, int O, int IL, int D, int ld_x0, int S, int R, float* dv,
                            float* du, float* d_subj_w, float* d_il_w, float* d_il_b, float* d_weights, float* workspace,
                            long long workspace_floats, bm_stream_t stream);
/* no workspace */
int bm_attention_weights_bwd_det(const float* dweights, const float* weights, const float* emb, int R, int C, int O, int P,
                                 float* dscores, float* dheads, bm_stream_t stream);
long long bm_head_bwd_params_det_workspace(int B, int T, int H, int F);
int bm_head_bwd_params_det(const float* dest, const float* x, const float* h1, const float* q, int B, int T, int H, int F,
                           float* dq, float* dw0, float* db0, float* dw2, float* db2, float* workspace,
                           long long workspace_floats, bm_stream_t stream);
long long bm_head_bwd_det_workspace(int B, int T, int H, int F);
int bm_head_bwd_det(const float* dest, const float* x, const float* w0, const float* w2, const float* h1, const float* q,
                    int B, int T, int H, int F, float* dq, float* dx, float* dw0, float* db0, float* dw2, float* db2,
                    float* workspace, long long workspace_floats, bm_stream_t stream);
/* CLIP: the candidate sums of squares one block per candidate; same scratch as the default forms (bm_clip_workspace) */
int bm_candidate_inv_norms_det(const float* cand, int Bc, long long KT, double* ss, float* inv_norm, bm_stream_t stream);
int bm_clip_scores_det(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given, float* inv_norm,
                       float* scores, float* probs, float* workspace, long long workspace_floats, int* status,
                       bm_stream_t stream);
int bm_clip_loss_fwd_det(const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset,
                         float* inv_norm, float* scores, float* probs, float* row_loss, float* loss, float* workspace,
                         long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_fwd_pooled_det(const float* est, const float* cand, int Bb, const float* arena, const int* slots, int Bn,
        int Bc, long long KT, int target_offset, float* inv_norm, float* scores, float* probs, float* row_loss, float* loss,
        float* workspace, long long workspace_floats, int* status, bm_stream_t stream);

/* ---- TF32 forms (PyTorch's TF32 matmul precision in the drop-in modules) -------------------------------------------
 * Every `_tf32` entry point takes its default form's arguments and computes its contraction in single-pass TF32 instead of
 * 3xTF32: each fp32 operand element is rounded once to tf32 (round to nearest, ties away from zero: cvt.rna.tf32.f32, the
 * hi piece of bm_tc_weight_split), the products are exact, and they are accumulated in fp32 exactly as in the default
 * form (a fresh register tile per 32-wide K block, added into the running sum with round-to-nearest adds), so the result is
 * within ~1e-5 relative of an fp64 contraction of the rounded operands however long K is.  Everything outside the
 * contraction is unchanged: epilogues, the CLIP candidate norms (fp64 sums of squares of the fp32 values), softmax and the
 * FP32-FMA kernels the default forms fall back to for shapes outside the tensor-core gates.  The forms that take
 * w_hi / w_lo read only w_hi and accept w_lo == NULL; w_hi may then hold the raw fp32 weights (bm_tc_weight_split with NULL
 * lo outputs), which they round.  bm_clip_scores_det_tf32 / bm_clip_loss_fwd_det_tf32 combine both forms: repeated calls
 * are bitwise identical, as with the `_det` forms.  The fp16-piece entry points (`*_f16`) have no TF32 form. */
int bm_tc_conv1d_tf32(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* addend,
                      int B, int T, int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                      float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream);
int bm_tc_conv1d_persistent_tf32(const float* x, const float* w_raw, const float* bias, int accumulate, int B, int T,
                                 int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                                 float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream);
int bm_tc_pointwise_sel_tf32(const float* x, const float* w_hi, const float* w_lo, const int* wsel, int n_sets, int B,
                             int T, int Cin, int Ntot, float* y, int* status, bm_stream_t stream);
int bm_tc_sensor_mix_bwd_data_tf32(const float* du, const float* w_hi, const float* w_lo, const int* wsel, int n_sets,
                                   const float* mask, int B, int T, int Op, int Cp, int C, float* dmeg, int* status,
                                   bm_stream_t stream);
int bm_tc_wgrad_tf32(const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                     float* workspace, float* dw, float* dbias, int* status, bm_stream_t stream);
int bm_tc_wgrad_conv_tf32(const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                          float* workspace, float* dw, int* status, bm_stream_t stream);
int bm_tc_wgrad_grouped_tf32(const float* dy, const float* x, const int* order, const int* seg_off, int G, int B, int T,
                             int M, int N, float* out, int* status, bm_stream_t stream);
int bm_clip_scores_tf32(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given,
                        float* inv_norm, float* scores, float* probs, float* workspace, long long workspace_floats,
                        int* status, bm_stream_t stream);
int bm_clip_scores_det_tf32(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given,
                            float* inv_norm, float* scores, float* probs, float* workspace, long long workspace_floats,
                            int* status, bm_stream_t stream);
int bm_clip_loss_fwd_tf32(const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset,
                          float* inv_norm, float* scores, float* probs, float* row_loss, float* loss, float* workspace,
                          long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_fwd_det_tf32(const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset,
                              float* inv_norm, float* scores, float* probs, float* row_loss, float* loss,
                              float* workspace, long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_bwd_tf32(const float* probs, const float* inv_norm, const float* cand, const float* gout, int Bn,
                          int Bc, long long KT, int target_offset, float* G, float* dest, int* status,
                          bm_stream_t stream);
int bm_clip_loss_bwd_cand_tf32(const float* probs, const float* scores, const float* inv_norm, const float* est,
                               const float* cand, const float* gout, int Bn, int Bc, long long KT, int target_offset,
                               float* G, float* coef, float* dcand, int* status, bm_stream_t stream);
int bm_clip_scores_bwd_tf32(const float* dscores, const float* scores, const float* inv_norm, const float* est,
                            const float* cand, int Bn, int Bc, long long KT, float* G, float* coef, float* dest,
                            float* dcand, int* status, bm_stream_t stream);
int bm_clip_loss_fwd_pooled_tf32(const float* est, const float* cand, int Bb, const float* arena, const int* slots, int Bn,
        int Bc, long long KT, int target_offset, float* inv_norm, float* scores, float* probs, float* row_loss, float* loss,
        float* workspace, long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_fwd_pooled_det_tf32(const float* est, const float* cand, int Bb, const float* arena, const int* slots, int Bn,
        int Bc, long long KT, int target_offset, float* inv_norm, float* scores, float* probs, float* row_loss, float* loss,
        float* workspace, long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_bwd_pooled_tf32(const float* probs, const float* inv_norm, const float* cand, int Bb, const float* arena,
        const int* slots, const float* gout, int Bn, int Bc, long long KT, int target_offset, float* G, float* dest,
        int* status, bm_stream_t stream);


/* ---- bf16 forms (torch.autocast(dtype=torch.bfloat16) in the drop-in modules) -----------------------------------------
 * Every `_bf16` entry point takes its default form's arguments and computes its contraction with bf16 operands and fp32
 * accumulation: each fp32 operand element is rounded once to bf16 (round to nearest even: cvt.rn.bf16x2.f32; a weight
 * that arrives as the two tf32 pieces of bm_tc_weight_split is rounded as hi + lo), the products of bf16 values are exact
 * in fp32, and they are accumulated in fp32 exactly as in the default form (a fresh register tile per 32-wide K block,
 * added into the running sum with round-to-nearest adds), so the result is within ~1e-5 relative of an fp64 contraction of
 * the rounded operands however long K is, and the fixed reduction order of the `_det` forms is kept.  Inputs, outputs and
 * workspaces stay fp32: no new storage format.  Everything outside the contraction is unchanged, as for the TF32 forms:
 * epilogues, the CLIP candidate norms, softmax and the FP32-FMA kernels of the shapes outside the tensor-core gates.  The
 * forms that take w_hi / w_lo accept w_lo == NULL (w_hi then holds the raw fp32 weights).  bm_clip_scores_det_bf16 /
 * bm_clip_loss_fwd_det_bf16 combine both forms: repeated calls are bitwise identical.  The fp16-piece entry points
 * (`*_f16`) have no bf16 form.
 * The drop-in modules take these forms exactly when torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda")
 * == torch.bfloat16 hold at the forward of the autograd node that issues the call; its backward uses the mode its forward
 * recorded.  An fp16 autocast or a nested autocast(enabled=False) leaves every call as without autocast, and bf16 takes
 * precedence over PyTorch's TF32 matmul flag. */
int bm_tc_conv1d_bf16(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* addend,
                      int B, int T, int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                      float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream);
int bm_tc_conv1d_persistent_bf16(const float* x, const float* w_raw, const float* bias, int accumulate, int B, int T,
                                 int Cin, int Ntot, int Kw, int dilation, int sign, int glu, int act, int out_tmajor,
                                 float* y, float* aux, float* glu_out, double* stats, int* status, bm_stream_t stream);
int bm_tc_pointwise_sel_bf16(const float* x, const float* w_hi, const float* w_lo, const int* wsel, int n_sets, int B,
                             int T, int Cin, int Ntot, float* y, int* status, bm_stream_t stream);
int bm_tc_sensor_mix_bwd_data_bf16(const float* du, const float* w_hi, const float* w_lo, const int* wsel, int n_sets,
                                   const float* mask, int B, int T, int Op, int Cp, int C, float* dmeg, int* status,
                                   bm_stream_t stream);
int bm_tc_wgrad_bf16(const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                     float* workspace, float* dw, float* dbias, int* status, bm_stream_t stream);
int bm_tc_wgrad_conv_bf16(const float* dy, const float* x, int B, int T, int M, int N, int Ntrue, int Kw, int dilation,
                          float* workspace, float* dw, int* status, bm_stream_t stream);
int bm_tc_wgrad_grouped_bf16(const float* dy, const float* x, const int* order, const int* seg_off, int G, int B, int T,
                             int M, int N, float* out, int* status, bm_stream_t stream);
int bm_clip_scores_bf16(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given,
                        float* inv_norm, float* scores, float* probs, float* workspace, long long workspace_floats,
                        int* status, bm_stream_t stream);
int bm_clip_scores_det_bf16(const float* est, const float* cand, int Bn, int Bc, long long KT, int norms_given,
                            float* inv_norm, float* scores, float* probs, float* workspace, long long workspace_floats,
                            int* status, bm_stream_t stream);
int bm_clip_loss_fwd_bf16(const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset,
                          float* inv_norm, float* scores, float* probs, float* row_loss, float* loss, float* workspace,
                          long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_fwd_det_bf16(const float* est, const float* cand, int Bn, int Bc, long long KT, int target_offset,
                              float* inv_norm, float* scores, float* probs, float* row_loss, float* loss,
                              float* workspace, long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_bwd_bf16(const float* probs, const float* inv_norm, const float* cand, const float* gout, int Bn,
                          int Bc, long long KT, int target_offset, float* G, float* dest, int* status,
                          bm_stream_t stream);
int bm_clip_loss_bwd_cand_bf16(const float* probs, const float* scores, const float* inv_norm, const float* est,
                               const float* cand, const float* gout, int Bn, int Bc, long long KT, int target_offset,
                               float* G, float* coef, float* dcand, int* status, bm_stream_t stream);
int bm_clip_scores_bwd_bf16(const float* dscores, const float* scores, const float* inv_norm, const float* est,
                            const float* cand, int Bn, int Bc, long long KT, float* G, float* coef, float* dest,
                            float* dcand, int* status, bm_stream_t stream);
int bm_clip_loss_fwd_pooled_bf16(const float* est, const float* cand, int Bb, const float* arena, const int* slots, int Bn,
        int Bc, long long KT, int target_offset, float* inv_norm, float* scores, float* probs, float* row_loss, float* loss,
        float* workspace, long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_fwd_pooled_det_bf16(const float* est, const float* cand, int Bb, const float* arena, const int* slots, int Bn,
        int Bc, long long KT, int target_offset, float* inv_norm, float* scores, float* probs, float* row_loss, float* loss,
        float* workspace, long long workspace_floats, int* status, bm_stream_t stream);
int bm_clip_loss_bwd_pooled_bf16(const float* probs, const float* inv_norm, const float* cand, int Bb, const float* arena,
        const int* slots, const float* gout, int Bn, int Bc, long long KT, int target_offset, float* G, float* dest,
        int* status, bm_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* BM_B200_H_ */
