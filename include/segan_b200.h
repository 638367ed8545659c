/*
 * segan_b200.h -- C ABI of libsegan_b200.so: the H100 (sm_90a) kernels underneath the
 * santi-pdp/segan_pytorch Python API (Generator / Discriminator / SEGAN train step).
 *
 * The reference has no FFI of its own (it is pure Python over torch ops; SURVEY.md 8b): every
 * entry point below names the reference call site (file:line in santi-pdp/segan_pytorch) whose
 * library dispatch it replaces.  Conventions:
 *   - plain pointers + sizes, no torch types; every pointer is a DEVICE pointer unless noted
 *   - the caller owns all memory (outputs and workspaces included); nothing is retained
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*); no hidden syncs
 *   - return 0 on success, <0 on error; sg_last_error() gives the thread-local message
 *   - no C++ exceptions cross the boundary
 *
 * HBM layout ("NLC rows"): an activation of a layer with C channels and L positions is stored
 * time-major, channels innermost: [B][H + R + H][Cr] 16-bit, where a "row" groups `g`
 * consecutive positions (g = 4 for the input of a stride-4 conv, else 1), R = L / g rows,
 * Cr = g*C, and H explicit halo rows on each side (H = 4 rows = 16 positions for reflect-padded
 * conv inputs, 0 otherwise).  [B][L][C] and [B][L/4][4C] are the same bytes, which is what turns
 * the K=31 / stride-4 (transposed) convolutions into stride-1, 9-tap "tap-GEMMs" (DESIGN.md).
 * Waveform ends (C = 1) are fp32 [B][L], identical to the reference's NCL tensors.
 *
 * Phase shifts: every entry point with a `roll` argument also takes `roll_dev` (device int32*, or NULL).
 * When non-NULL the kernel reads the shift from *roll_dev and ignores `roll`: the launch then has no
 * per-step scalar, so a whole train step can be captured once in a CUDA graph and replayed while
 * the host only rewrites the small shift table (discriminator.py:160-172 draws new shifts every pass).
 */
#ifndef SEGAN_B200_H
#define SEGAN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SG_ABI_VERSION 3

/* Per-channel statistic buffers (sg_bn_stats `stats`, sg_act_bwd_* `red`, sg_colsum `tmp`) hold
 * SG_STAT_SLICES interleaved partial copies: [SG_STAT_SLICES][n_stats][C] doubles, zeroed by the caller;
 * the value of a statistic is the sum over the slices (spreads same-address atomics). */
#define SG_STAT_SLICES 8

/* status codes */
#define SG_OK 0
#define SG_ERR_INVALID -1
#define SG_ERR_LAUNCH -2
#define SG_ERR_UNSUPPORTED -3

/* element types */
#define SG_F32 0
#define SG_F16 1
#define SG_BF16 2

/* activation kinds */
#define SG_ACT_NONE 0
#define SG_ACT_PRELU 1
#define SG_ACT_TANH 2

/* tap-GEMM back ends */
#define SG_BACKEND_FFMA 0    /* CUDA-core fp32 reference implementation (validation / fallback) */
#define SG_BACKEND_TCGEN05 1 /* TMA + mbarrier + wgmma tensor cores (the product path; name kept for the ABI) */

int sg_abi_version(void);
const char* sg_last_error(void);
/* 1 if the current device is compute capability 9.0 (H100) and the sm_90a kernels can run */
int sg_device_ok(void);
/* Forward-form tap-GEMM schedule selector (0 | 1 | 2), kept for ABI compatibility: the sm_90a library has one
 * forward-form kernel (128-row tiles, two consumer warpgroups) and runs it for every setting.
 * Returns the previous setting.  Environment default: SEGAN_B200_CTA_PAIR. */
int sg_set_cta_pair(int on);
/* Tuning knobs of the HBM-bound streaming kernels, one per kernel family (`kind`):
 *   SG_EW_ACT_FWD (sg_act_fwd), SG_EW_BN_STATS (sg_bn_stats), SG_EW_BWD_REDUCE (sg_act_bwd_reduce),
 *   SG_EW_BWD_APPLY (sg_act_bwd_apply).
 * vec: channels per thread (4 | 8); unroll: rows in flight per thread and input stream (2 | 4 | 8 with
 * vec*unroll <= 32); cap: CTAs per SM (persistent grid beyond that).  For the two backward kinds vec == 8
 * selects the tiled kernel (unroll 2 | 4), vec == 4 the generic one.
 * vec == 16 (the default for act_fwd and both backward kinds) selects the TMA-staged kernels (stream_ew.cu:
 * cp.async.bulk row tiles through an mbarrier ring, 8 channels per consumer thread) wherever the call qualifies --
 * contiguous 16-bit tensors (leading dimension == C), no bf16 twin outputs, L >= 2 * halo + 3 -- and otherwise falls
 * back to the register-staged kernel with (8, unroll, cap).  Every variant computes the same values (up to fp32
 * summation order).  Also read once from the environment: SEGAN_B200_EW="kind,vec,unroll,cap[;...]".
 * Returns SG_OK or SG_ERR_INVALID. */
#define SG_EW_ACT_FWD 1
#define SG_EW_BN_STATS 2
#define SG_EW_BWD_REDUCE 3
#define SG_EW_BWD_APPLY 4
int sg_set_ew_variant(int kind, int vec, int unroll, int cap);
/* 16-bit format of every GRADIENT tensor the library reads or writes (the `g_*` arguments below, the col2im input,
 * the D head's g_z1): SG_F16 (default) or SG_BF16.  Returns the previous setting.
 * fp16 gradients carry 11 significant bits (bf16: 8) and share the forward tensors' format, so the weight-gradient
 * tap-GEMM reads the forward activations directly (wgmma cannot mix f16 x bf16 operands: with bf16
 * gradients every forward activation needs a bf16 twin).  Their narrower range is covered by a loss scale: the
 * `grad_scale` argument of sg_fc_tail_bwd / sg_l1_loss_bwd multiplies the loss gradients at their source, every
 * parameter gradient then carries the factor and the optimiser's `grad_scale` divides it out; 16-bit stores
 * saturate at +-65504.  (autograd in model.py:299,306,320 keeps fp32 gradients: this is the precision contract
 * of north_star's "fp16/bf16 sample windows".) */
int sg_set_grad_dtype(int dtype);
/* Split-K over the last, partial wave of sg_tapgemm_f_run's tensor-core kernel (needs sg_tapgemm_f.sk_ws):
 * max_split = largest number of CTAs one leftover tile is split over (0 | 1 = off, default 16; < 0 keeps it);
 * atomic_steps = cost-model constant: the finisher's cost of adding one 256-wide partial tile, in k-steps (<= 0
 * keeps it; a value below 1e-3 also drops the model's fixed cost, i.e. forces the split -- sweeps and tests).
 * Returns the previous max_split.  Environment: SEGAN_B200_STREAMK, SEGAN_B200_SK_ATOMIC. */
int sg_set_stream_k(int max_split, float atomic_steps);

/* ------------------------------------------------------------------------------------------
 * Tap-GEMM, forward form ("F"):
 *     out[b, m, n] = bias[n % bias_mod] + sum_{d = d_lo..d_hi} sum_{kc valid for d}
 *                        A[b, m + d, kc] * Wp[d + 4][n][kc]          m in [m_lo, m_hi), n in [n_lo, n_hi)
 * A is the channel-concatenation of up to two NLC-row tensors (a0 | a1); rows outside
 * [-a_halo, a_rows + a_halo) read as zero.  Wp is the packed weight [9][nc][kc].
 * Replaces: nn.Conv1d on a reflect-padded input (segan/models/modules.py:92-99), its data
 * gradient, nn.ConvTranspose1d (modules.py:136) and its data gradient, torch.cat of the skip
 * connection (segan/models/generator.py:76,205), and nn.Linear fc.0 (discriminator.py:112).
 * ------------------------------------------------------------------------------------------ */
typedef struct sg_tapgemm_f {
  const void* a0;     /* [B][a_halo + a_rows + a_halo][a0_c] */
  const void* a1;     /* same geometry, a1_c channels, or NULL */
  int32_t a0_c, a1_c; /* kc = a0_c + a1_c */
  int32_t a_rows, a_halo;
  int32_t a_dtype;    /* SG_F16 | SG_BF16 */
  const void* w;      /* packed [slots][nc][kc], w_dtype; slot = (d + 4) - w_tap0 */
  int32_t w_dtype;
  int32_t w_tap0;     /* tap index stored in slot 0 (0 for the 9-slot conv packs, 4 for a Linear) */
  int32_t kc, nc;
  int32_t d_lo, d_hi; /* inclusive, within [-4, 4] */
  /* per tap (index d+4): valid K range [k_lo, k_hi) and valid N range [n_lo, n_hi) in channels
     (multiples of 64); blocks outside are structurally zero in Wp and are skipped */
  int32_t tap_k_lo[9], tap_k_hi[9], tap_n_lo[9], tap_n_hi[9];
  void* out;          /* [B][out_halo + out_rows + out_halo][out_ld]; column of channel n = n - n_lo + out_col0 */
  int32_t out_ld, out_col0;
  int32_t out_dtype;  /* SG_F16 | SG_BF16 | SG_F32 (F32: atomically accumulated, pre-zeroed by caller) */
  int32_t out_rows, out_halo;
  int32_t m_lo, m_hi; /* rows computed per batch element (may reach into the out halo) */
  int32_t n_lo, n_hi; /* channels computed */
  const float* bias;  /* or NULL */
  int32_t bias_mod;   /* bias index = n % bias_mod */
  int32_t batch;
  int32_t ksplit;     /* >1 only with out_dtype == SG_F32 */
  int32_t backend;    /* SG_BACKEND_* */
  int32_t tile_n;     /* N tile of the tensor-core kernel: 0 = widest of 256/128/64 dividing n_hi-n_lo; 64|128|256 =
                         narrower tiles for the tail of a launch split against wave quantisation (132 SMs) */
  double* bn_stats;   /* or NULL.  Fused nn.BatchNorm1d batch statistics (modules.py:11,100) of the output: per
                         column sum and sum of squares of the stored (rounded) values over all computed rows,
                         accumulated into [SG_STAT_SLICES][2][nc] doubles (same buffer sg_bn_stats fills; caller
                         zeroes).  Tensor-core backend, 16-bit out, ksplit 1, n_lo = 0, n_hi = nc. */
  void* out2;         /* or NULL.  Fused second output out2[b][out2_halo + m][n] = PReLU_slope[n % slope_mod](out value), same
                         dtype / row pitch / column mapping as `out`, own halo: the consumer-ready activation of a Generator
                         block whose contraction feeds PReLU directly (modules.py:99-101,139-141; no norm layer), stored
                         next to the raw pre-activation the skip connection needs (generator.py:185,191).  With
                         out2_halo > 0 (reflect padding of the next conv, modules.py:92-98) position m is also written to
                         its mirror row -m or 2(out_rows-1)-m when it lies within out2_halo of an end; needs m_lo = 0,
                         m_hi = out_rows, out_rows >= 2*out2_halo + 3.  Tensor-core backend, 16-bit out. */
  int32_t out2_halo;
  const float* slope; /* with out2 == NULL and slope != NULL the PReLU is applied to `out` itself (inference decoder) */
  int32_t slope_mod;
  void* sk_ws;        /* or NULL.  Zero-initialised workspace of sg_tapgemm_f_workspace_bytes() bytes that lets the
                         tensor-core kernel split the tiles of its last, partial wave along K over several CTAs (fp32
                         partial sums in per-CTA slots, summed in slot order by whoever finishes a tile: deterministic;
                         counters, which the kernel leaves zeroed).  One workspace per stream: launches that may run
                         concurrently must not share it. */
} sg_tapgemm_f;

int sg_tapgemm_f_run(const sg_tapgemm_f* p, void* stream);
/* size of sg_tapgemm_f.sk_ws (device memory, zero-filled once by the caller) */
int64_t sg_tapgemm_f_workspace_bytes(void);
/* Diagnostics (SEGAN_B200_DEBUG bit 20): per-CTA phase timeline of the last forward-form tap-GEMM launch, 32 globaltimer
 * words (ns) per CTA for up to 160 CTAs -- [0] start, then per tile piece: accumulator ready, epilogue done, (split
 * tiles, bit 63 set) finisher done; last non-zero word = exit.  Copies min(max_words, 5120) words to the HOST buffer
 * and returns the count (-1 on a CUDA error).  Not used by the product path. */
int sg_debug_timeline(unsigned long long* host_out, int max_words);

/* ------------------------------------------------------------------------------------------
 * Tap-GEMM, weight-gradient form ("W"):
 *     dWp[d + 4][n][kc] += sum_{b, m in [0, g_rows)} G[b, m, n] * A[b, m + d, kc]
 * G: [B][g_rows][nc] (exact, no halo); A as above.  dWp fp32 packed [9][nc][kc], accumulated
 * atomically (caller zeroes it).  Replaces the weight gradient of nn.Conv1d / nn.ConvTranspose1d /
 * nn.Linear computed by autograd for model.py:299,306,320.
 * ------------------------------------------------------------------------------------------ */
typedef struct sg_tapgemm_w {
  const void* g;
  int32_t g_rows, g_dtype;
  const void* a0;
  const void* a1;
  int32_t a0_c, a1_c;
  int32_t a_rows, a_halo, a_dtype;
  int32_t kc, nc;
  int32_t d_lo, d_hi;
  int32_t tap_k_lo[9], tap_k_hi[9], tap_n_lo[9], tap_n_hi[9];
  float* dw; /* [slots][nc][kc] fp32; slot = (d + 4) - dw_tap0 */
  int32_t dw_tap0;
  int32_t batch;
  int32_t ksplit; /* number of position-range splits (>=1) */
  int32_t backend;
  const float* out_scale; /* or NULL: device scalar multiplying the accumulated products (1/sigma of a spectrally
                             normalised layer: the gradient w.r.t. W / sigma lands as G / sigma, sg_snorm_sigma) */
} sg_tapgemm_w;

int sg_tapgemm_w_run(const sg_tapgemm_w* p, void* stream);

/* ------------------------------------------------------------------------------------------
 * Weight packing (fp32 master [reference layout] -> 16-bit tap-GEMM operands) and gradient
 * unpacking (fp32 packed dWp -> fp32 reference layout).  kind:
 *   0 = Conv1d  W[cout][cin][31]      (modules.py:79)   -> Wf [9][cout][4cin]  and Wdg [9][4cin][cout]
 *   1 = ConvTranspose1d W[cin][cout][31] (modules.py:116) -> Wt [9][4cout][cin] and Wtd [9][cin][4cout]
 *       alpha (or NULL): per-input-channel scale for channels >= alpha_from (GSkip, generator.py:68-69)
 *   2 = Linear W[nout][c*T + t] (discriminator.py:112) -> W1p [nout][t*C + c] and W1dg [t*C + c][nout]
 * ------------------------------------------------------------------------------------------ */
int sg_pack_weights(int kind, const float* w, int c_out, int c_in, int t_len,
                    const float* alpha, int alpha_from,
                    void* w_fwd, void* w_dgrad, int dtype_fwd, int dtype_dgrad, void* stream);
/* dw (reference layout) = unpack(dwp); for kind 1 with alpha: dw[ci>=alpha_from] = alpha*dWeff and
 * dalpha[c] = sum_{co,k} dWeff[ci,co,k] * w[ci,co,k].  accumulate: 0 = overwrite, 1 = add */
int sg_unpack_wgrad(int kind, const float* dwp, int c_out, int c_in, int t_len,
                    const float* w, const float* alpha, int alpha_from,
                    float* dw, float* dalpha, int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------
 * Waveform-end layers (Cin or Cout in {1,2}: HBM-bound, CUDA cores).
 * ------------------------------------------------------------------------------------------ */
/* First encoder layer (G: 1 ch, D: 2 ch = candidate | reference; model.py:173-175 cat is never
 * materialised).  x0/x1: fp32 [B][L]; roll: signed circular shift applied before the reflect
 * pad (discriminator.py:160-172; 0 for G).  a_out: [B][L/4][cout] fp16 raw pre-activation
 * (+bias).  If h_out != NULL also writes PReLU(a) into the padded consumer-ready buffer
 * [B][4 + L/16 + 4][4*cout] with the reflect halo (G path, modules.py:98-101). */
int sg_wave_conv_fwd(const float* x0, const float* x1, int cin, int batch, int L, int roll,
                     const float* w, const float* bias, int cout,
                     void* a_out, const float* prelu, void* h_out, void* stream);
/* dW[cout][cin][31], dbias[cout] (or NULL) += over batch; g_a: [B][L/4][cout] bf16 */
int sg_wave_conv_wgrad(const float* x0, const float* x1, int cin, int batch, int L, int roll,
                       const void* g_a, int cout, float* dw, float* dbias, void* stream);
/* data gradient w.r.t. channel 0 of the (rolled, padded) input, un-rolled and halo-folded:
 * gx0[b][l] (=|+=) sum ...   Used in the G step (model.py:315-320). */
int sg_wave_conv_dgrad(const void* g_a, int batch, int L, int roll, const float* w, int cin,
                       int cout, float* gx0, int accumulate, void* stream);
/* Last decoder layer: ConvTranspose1d(cin -> 1) + bias + tanh (modules.py:135-141 with
 * act='Tanh').  x0|x1: [B][Lin][c0|c1] fp16 (decoder act | skip pre-activation, alpha folded
 * into w_eff by the caller: w_eff[ci][31]).  y: fp32 [B][4*Lin]. */
int sg_wave_deconv_fwd(const void* x0, int c0, const void* x1, int c1, int batch, int Lin,
                       const float* w_eff, const float* bias, float* y, void* stream);
/* backward of the above given gy [B][4Lin] fp32 and y: gpre = gy*(1-y^2);
 * gx: [B][Lin][c0+c1] bf16 (w.r.t. cat(x0,x1) i.e. already alpha-scaled for the skip half),
 * dw_eff[ci][31], dbias[1] accumulated.  gpre_ws: fp32 workspace [B][4*Lin]. */
int sg_wave_deconv_bwd(const void* x0, int c0, const void* x1, int c1, int batch, int Lin,
                       const float* w_eff, const float* gy, const float* y, float* gpre_ws,
                       void* gx, float* dw_eff, float* dbias, void* stream);

/* Tensor-core route for the same waveform-end layers: a 64-channel im2col of the waveform(s)
 * (col[b][t][ci*32+k] = pad(v_ci)[4t+k-off], 16-bit, fp16 and/or bf16 copy) makes them single-tap
 * tap-GEMMs with K = 64; the transposed forms are a GEMM followed by a shift-add. */
int sg_wave_im2col(const float* v0, const float* v1, int cin, int batch, int L, int roll, const int32_t* roll_dev,
                   int reflect, int off, void* col_f16, void* col_bf16, void* stream);
/* y[b][4m+r] = tanh(bias + sum_d P[b][m+d][(d+4)*4+r]); P fp32 [B][Lin][64] (last decoder block) */
int sg_wave_shiftadd_tanh(const float* P, int batch, int Lin, const float* bias, float* y, void* stream);
/* gx[b][unroll(reflect(q))] += sum_{4t+k-14=q} P2[b][t][col0+k]; P2 bf16 [B][L/4][64] (D input gradient;
 * col0 = 32*ci selects the input channel) */
int sg_wave_col2im_fold(const void* P2, int col0, int batch, int L, int roll, const int32_t* roll_dev, float* gx,
                        void* stream);
/* gpre = gy*(1-y^2); dbias += sum(gpre) */
int sg_tanh_bwd(const float* gy, const float* y, int64_t n, float* gpre, float* dbias, void* stream);

/* ------------------------------------------------------------------------------------------
 * Elementwise / reduction glue (HBM-bound).
 * ------------------------------------------------------------------------------------------ */
/* per-channel sum / sum of squares of a [rows_total][C] 16-bit tensor into double
 * stats[SG_STAT_SLICES][2][C] (accumulated; caller zeroes).  BatchNorm1d batch statistics, modules.py:11,100. */
int sg_bn_stats(const void* a, int dtype, int64_t rows_total, int C, double* stats, void* stream);
/* stats -> scale/shift (fp32 [2][C]: scale = gamma*invstd, shift = beta - mean*scale), saved
 * mean/invstd (fp32 [2][C]) and running-stat update (momentum 0.1, unbiased var, eps 1e-5). */
int sg_bn_finalize(const double* stats, int64_t count, int C, const float* gamma, const float* beta,
                   float eps, float momentum, float* running_mean, float* running_var,
                   float* scale_shift, float* mean_invstd, void* stream);
/* h = act(a*scale + shift) written to [B][oh + Lout_rows + oh][g*C] with circular roll and
 * reflect halo (the consumer's view).  scale_shift may be NULL.  a: [B][L][C] exact.
 * out_halo_pos = halo in positions (0 or 16).  act: SG_ACT_NONE|SG_ACT_PRELU.
 * The bf16 twins feed the weight-gradient tap-GEMM, whose two operands must share one 16-bit
 * format (wgmma rejects f16 x bf16; gradients are bf16 for range). */
int sg_act_fwd(const void* a, int dtype, int batch, int L, int C, const float* scale_shift,
               const float* slope, int act, int roll, const int32_t* roll_dev, int out_halo_pos, void* h,
               void* h_bf16 /* optional bf16 twin of h (same geometry) */,
               void* a_bf16 /* optional bf16 copy of a (exact geometry) */, void* stream);
/* backward of sg_act_fwd (+ optional BatchNorm backward).  g_h: gradient w.r.t. the consumer
 * view (bf16, same geometry as h incl. halo & roll) ; g_add: optional extra gradient w.r.t. the
 * PRE-activation `a` in exact geometry (the Generator's skips carry pre-activations,
 * generator.py:185,191), added after the activation derivative; may be NULL.
 * pass 1 (sg_act_bwd_reduce): red[0][C] = sum g_y*[y<0]*y (d slope), red[1][C] = sum g_pre (d beta),
 *   red[2][C] = sum g_pre * ahat (d gamma), where y = a*scale+shift, g_pre = g_y*act'(y).
 *   Without BatchNorm g_a = g_pre is final and pass 1 writes it when g_a_out_or_null != NULL.
 * pass 2 (sg_act_bwd_apply): g_a (bf16 exact) = no BN: g_pre ;
 *   BN: scale * (g_pre - red1/N - ahat*red2/N).  `red` of pass 2 is the buffer pass 1 wrote
 *   ([SG_STAT_SLICES][3][C]; the kernel adds the slices up).
 * sg_stat_grads: g_s[c] += sum over slices of red[slice][s][c] for s < n_stats (g_s may be NULL):
 *   the PReLU-slope / bias (beta) / gamma gradients of model.py:299,306,320 from the pass-1 statistics. */
/* g_h_ld / g_add_ld: row pitch in elements of g_h / g_add (>= C; lets a consumer read one half of
 * a channel-concatenated gradient in place; the pointers are pre-offset by the caller) */
int sg_act_bwd_reduce(const void* g_h, int g_h_ld, int in_halo_pos, int roll, const int32_t* roll_dev,
                      const void* g_add, int g_add_ld, const void* a, int dtype, int batch, int L, int C,
                      const float* scale_shift, const float* mean_invstd, const float* slope,
                      int act, double* red, void* g_a_out_or_null, void* stream);
int sg_act_bwd_apply(const void* g_h, int g_h_ld, int in_halo_pos, int roll, const int32_t* roll_dev,
                     const void* g_add, int g_add_ld, const void* a, int dtype, int batch, int L, int C,
                     const float* scale_shift, const float* mean_invstd, const float* slope,
                     int act, const double* red, int use_bn, void* g_a, void* stream);
int sg_stat_grads(const double* red, int C, int n_stats, float* g0, float* g1, float* g2, void* stream);
/* out[r][col0 + c] = (16-bit) ws[r][col0 + c], c < ncols: ws (fp32) and out share the geometry [rows][ld].  Final
 * step of a split-K tail launch of sg_tapgemm_f_run (fp32 partial sums accumulated with ksplit > 1). */
int sg_convert_f32_rows(const float* ws, void* out, int dtype, int64_t rows, int ld, int col0, int ncols,
                        void* stream);
/* fp32 NCL [B][C][L] <-> 16-bit NLC [B][L][C] (z input, generator.py:195-205; ret_hid outputs) */
int sg_ncl_to_nlc(const float* src, int batch, int C, int L, void* dst, int dtype, void* stream);
int sg_nlc_to_ncl(const void* src, int dtype, int batch, int C, int L, float* dst, void* stream);
/* per-channel column sums of a 16-bit [rows][C] tensor into fp32 out[C % mod] (bias gradients) */
int sg_colsum(const void* a, int dtype, int64_t rows, int C, int mod, float* out, int accumulate,
              double* tmp /* [C] workspace */, void* stream);

/* D head after fc.0 (discriminator.py:111-117): z1 = fc0_acc + b0 ; h1 = PReLU(z1) ; z2 = W2 h1 + b2 ;
 * h2 = PReLU(z2) ; logit = W4 h2 + b4.  Saves z1,z2 (fp32) for backward. */
int sg_fc_tail_fwd(const float* fc0_acc, const float* b0, const float* s1, const float* w2,
                   const float* b2, const float* s3, const float* w4, const float* b4, int batch,
                   float* z1, float* z2, float* logit, void* stream);
/* loss = mean((logit-target)^2)*weight ; g_logit = 2(logit-target)/B*weight ; backward through the
 * head: g_z1 (bf16 [B][256] for the fc.0 tap-GEMMs) and (if grads != NULL) parameter gradients
 * accumulated into: g_b0[256], g_s1[256], g_w2[128*256], g_b2[128], g_s3[128], g_w4[128], g_b4[1]. */
int sg_fc_tail_bwd(const float* z1, const float* z2, const float* logit,
                   const float* g_logit_in /* or NULL: use the fused MSE gradient below */, float target, float weight,
                   const float* s1, const float* w2, const float* s3, const float* w4, int batch,
                   float* loss_out, void* g_z1_bf16, float* ws /* fp32 [B*(1+128+256+256)] */,
                   float* g_b0, float* g_s1, float* g_w2, float* g_b2, float* g_s3, float* g_w4,
                   float* g_b4, float grad_scale /* loss scale: multiplies g_logit (not loss_out) */, void* stream);
/* G regression loss (model.py:318): loss = w * mean|y - clean| ; gy (+)= grad_scale*w*sign(y-clean)/(B*L) */
int sg_l1_loss_bwd(const float* y, const float* clean, int64_t n, float weight, float* loss_out,
                   float* gy, int accumulate, float grad_scale /* multiplies gy only */, void* stream);
/* --reg_loss mse_loss (model.py:79,318): loss = w * mean (y - clean)^2 ; gy (+)= grad_scale*2w*(y-clean)/(B*L).
 * Both losses add to *loss_out (may be NULL), summed in a fixed order (the same bits run to run); launches of the
 * two must not overlap each other on one device (per-device partial sums). */
int sg_mse_loss_bwd(const float* y, const float* clean, int64_t n, float weight, float* loss_out,
                    float* gy, int accumulate, float grad_scale /* multiplies gy only */, void* stream);

/* ------------------------------------------------------------------------------------------
 * WSEGAN's spectral term (model.py:638-653): pow_weight * mean| 10 log10(|STFT(G)|^2 + 1e-19) - 10 log10(|STFT(clean)|^2
 * + 1e-19) |, torch.stft(n_fft 2048, hop 160, win_length 320 rectangular, centre-padded, center=True, normalized).
 * Only 320 of a frame's 2048 samples are non-zero, so the STFT of a batch is ONE dense GEMM -- frames [B*(1 + L/160)][320]
 * x DFT [320][re | im of the 1025 bins] -- run by sg_tapgemm_f_run with a single tap; these are the kernels around it:
 *   sg_stft_frames      frames[b][t][n] = x[b][reflect(160 t + n - 160)]                       (16-bit A operand)
 *                       split != 0: rows of 960 = hi | lo | hi with x = hi + lo (two 16-bit halves, ~22 bits): against
 *                       the DFT operand [Dhi ; Dhi ; Dlo] one K = 960 GEMM gives the fp32-grade spectrum
 *   sg_logpow_l1        X_gen, X_clean fp32 [rows][ld] (re of bin f at column f, im at column half + f):
 *                       loss_out += weight * mean|...| ; g_x (16-bit, may be NULL) = grad_scale * d loss / d X_gen
 *   sg_stft_frames_fold g_wave[b][reflect(160 t + n - 160)] += scale * g_frames[b][t][n]        (overlap-add)
 * ------------------------------------------------------------------------------------------ */
int sg_stft_frames(const float* x, int batch, int L, void* frames, int dtype, int split, void* stream);
int sg_logpow_l1(const float* x_gen, const float* x_clean, int64_t rows, int bins, int half, int ld, float weight,
                 float* loss_out, void* g_x, int g_dtype, float grad_scale, void* stream);
int sg_stft_frames_fold(const float* g_frames, int batch, int L, float scale, float* g_wave, void* stream);

/* ------------------------------------------------------------------------------------------
 * Optimisers on flat fp32 buffers (torch.optim.RMSprop / Adam as used at model.py:221-225).
 * grad_scale multiplies the gradient first (1/world_size after an all-reduce SUM).
 * clear_grad != 0 zeroes `grad` as it is read (the next backward pass accumulates from zero: no separate fill).
 * ------------------------------------------------------------------------------------------ */
int sg_rmsprop_step(float* param, float* grad, float* square_avg, int64_t n, float lr,
                    float alpha, float eps, float grad_scale, int clear_grad, void* stream);
int sg_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                 float lr, float beta1, float beta2, float eps, int step, float grad_scale, int clear_grad,
                 void* stream);

/* ------------------------------------------------------------------------------------------
 * Packed-master path (training): master weights, optimiser state and gradients of a tap-GEMM layer stay in the
 * layout of its forward operand, M[n_taps][nc][kc] fp32 -- what sg_tapgemm_w_run produces and what the elementwise
 * optimisers above do not care about -- so a step needs no reference-layout round trip:
 *   sg_emit_operands : F[t][n][k] = M[t][n][k]*a(k) (forward operand), Dg[t][k][n] = M[T-1-t][n][k]*a(k) (data-
 *                      gradient operand), a(k) = alpha[k - alpha_from] for k >= alpha_from (GSkip, generator.py:68-69)
 *                      else 1; either destination may be NULL; dtypes SG_F16 | SG_BF16 | SG_F32.
 *   sg_alpha_grad    : in place dWp[t][n][k] *= alpha(k) for k >= alpha_from (the tap-GEMM differentiated w.r.t. the
 *                      alpha-scaled weights) and dalpha[k - alpha_from] += sum_{t,n} dWp*M (before the scaling).
 *   sg_pack_weights(kind, w, ..., w_fwd = M, w_dgrad = NULL, SG_F32, ...) imports a reference-layout tensor and
 *   sg_unpack_wgrad(kind, M, ..., alpha = NULL, ..., accumulate = 0) exports one (state_dict, checkpoints).
 * sg_wave_wgrad_fold / sg_last_deconv_wgrad_fold: the waveform-end layers' weight gradients out of their single-tap
 * GEMM results (dwq, see engine.py), accumulated atomically into reference-layout gradients. */
int sg_emit_operands(const float* master, int n_taps, int nc, int kc, const float* alpha, int alpha_from,
                     void* w_fwd, void* w_dgrad, int dtype_fwd, int dtype_dgrad,
                     const float* scale_dev /* or NULL: device scalar multiplying every element (1/sigma of a
                                               spectrally normalised layer, sg_snorm_sigma) */, void* stream);
int sg_alpha_grad(float* dwp, const float* master, int n_taps, int nc, int kc, const float* alpha, int alpha_from,
                  float* dalpha, void* stream);
/* Spectral normalisation (norm_type='snorm': modules.py:12-14, discriminator.py:118-121 -> torch.nn.utils.spectral_norm)
 * on a packed master M[n_taps][nc][kc] holding weight_orig:
 *   sg_snorm_sigma: training != 0: one power iteration v = normalize(W^T u), u = normalize(W v) in place (u [nc], v
 *     [n_taps*kc] in packed slots), scal[2] = sigma = u^T W v, scal[3] = 1/sigma; training == 0: sigma from the
 *     stored vectors.  scal: 4 device floats; work: nc device floats.  The operands are then emitted with
 *     sg_emit_operands(..., scale_dev = scal + 3).
 *   sg_snorm_grad: gradient w.r.t. the normalised weight (packed, what sg_tapgemm_w_run produced) -> gradient
 *     w.r.t. weight_orig in place: dW = G / sigma - <G, W> / sigma^2 * u v^T  (u, v constants, as torch
 *     differentiates sigma).  dot_ws: one device float. */
int sg_snorm_sigma(const float* master, int n_taps, int nc, int kc, float* u, float* v, float* scal, float* work,
                   int training, void* stream);
int sg_snorm_grad(float* dwp, const float* master, int n_taps, int nc, int kc, const float* u, const float* v,
                  const float* scal, float* dot_ws, void* stream);
/* The same correction for the big layers whose gradients of several passes (D real / fake / ... each with its own
 * power-iteration state) accumulate in one bucket: the weight-gradient GEMM scales by 1/sigma_p itself
 * (sg_tapgemm_w.out_scale); the sigma term's scalar of pass p is  coef_p = <dL/dW~, W~> / sigma_p  and, the layer
 * output being linear in W~,  <dL/dW~, W~> = <g_pre, x - bias>  comes from the activation-backward statistics
 * (sg_act_bwd_reduce's red: [1] = sum g_pre, [2] = sum g_pre * x) -- sg_snorm_coef; one sweep then subtracts
 * sum_p coef_p * u_p v_p^T -- sg_snorm_rank1 (u [n_pass][nc], v [n_pass][n_taps*kc], coef [n_pass]). */
int sg_snorm_coef(const double* red, const float* bias, int C, const float* scal, float* coef_out, void* stream);
int sg_snorm_rank1(float* dwp, int n_taps, int nc, int kc, int n_pass, const float* u, const float* v,
                   const float* coef, void* stream);
int sg_wave_wgrad_fold(float* dwq /* the blocks read are cleared */, int cin, float* dw, void* stream);
int sg_last_deconv_wgrad_fold(float* dwq /* the blocks read are cleared */, int half, const float* w, const float* alpha, float* dw,
                              float* dalpha, void* stream);
/* the same fold for a Generator without skips (skip=False): dwq[2][64][2][cin] (s, k-slot, s', c) -> dW[cin][1][31]
 * += dwq[0][k][0][c] + dwq[1][k][1][c]; no alpha */
int sg_last_deconv_wgrad_fold_1src(float* dwq /* the blocks read are cleared */, int cin, float* dw, void* stream);

/* ------------------------------------------------------------------------------------------
 * Convolutional skip connection (GSkip skip_type='conv', generator.py:43-49): nn.Conv1d(C, C, K, stride 1,
 * padding K//2) on the encoder's [B][L][C] pre-activation.  In the grouped view [B][L/4][4C] it is a forward-form
 * tap-GEMM with kc = nc = 4C over the taps d = -D..D, D = (K/2 + 3) / 4 (w_tap0 = 4 - D, a_halo = 0: the zero
 * padding is the tap-GEMM's out-of-range rows):
 *     W'[d + D][(po, co)][(pi, ci)] = W[co][ci][4d + pi - po + K/2]   (0 where that tap is outside [0, K))
 * K must be odd and at most 33, C a multiple of 64; anything else returns SG_ERR_INVALID.
 *   sg_skipconv_emit       W fp32 [C][C][K] (reference layout) -> w_fwd [2D+1][4C][4C] (dtype_fwd) and/or w_dgrad,
 *                          the data-gradient operand: per-tap transpose of W' with tap d <-> -d (dtype_dgrad).
 *                          Either destination may be NULL; dtypes SG_F16 | SG_BF16 | SG_F32.
 *   sg_skipconv_wgrad_fold dwq fp32 [2D+1][4C][4C], the weight-gradient tap-GEMM's result over the grouped rows ->
 *                          dw [C][C][K] += the sum of the four copies of every tap.  Leaves all of dwq zeroed
 *                          (the copies and the structurally zero blocks the GEMM computed alike), so it needs no
 *                          fill before the next accumulation.
 * ------------------------------------------------------------------------------------------ */
int sg_skipconv_emit(const float* w, int C, int K, void* w_fwd, void* w_dgrad, int dtype_fwd, int dtype_dgrad,
                     void* stream);
int sg_skipconv_wgrad_fold(float* dwq, int C, int K, float* dw, void* stream);

/* ------------------------------------------------------------------------------------------
 * Pooled Discriminator heads (pool_type 'conv' / 'gmax' / 'gavg' / 'mlp', discriminator.py:122-146,175-192) on the last
 * tower activation h: fp16 NLC [B][Lq][C] (no halo, no roll), C a multiple of 64, Lq <= 4096.
 *   SG_DHEAD_CONV  a[b][t] = pool_w . h[b][t] + pool_b[0]  (pool_conv = Conv1d(C, 1, 1))   logit = fc_w[Lq] . a + fc_b
 *   SG_DHEAD_GMAX  p[b][c] = max_t h[b][t][c]  (AdaptiveMaxPool1d(1))                      logit = fc_w[C] . p + fc_b
 *   SG_DHEAD_GAVG  p[b][c] = mean_t h[b][t][c] (AdaptiveAvgPool1d(1))                      logit = fc_w[C] . p + fc_b
 *   SG_DHEAD_MLP   logit[b][t] = pool_w . h[b][t] + pool_b[0]  (mlp.2 = Conv1d(C, 1, 1); h is the mlp's PReLU output):
 *                  B * Lq logits, no fc (fc_w, fc_b, pooled, g_fc_* unused), loss and d loss / d logit over all of them
 * sg_dhead_fwd: logit fp32 [B] ([B][Lq] for mlp); pooled fp32 = a [B][Lq] (conv, int_act['avg_conv_h']) or p [B][C]; argmax int32
 *   [B][C] (gmax only, else may be NULL): the first t holding the maximum, where a NaN replaces the running maximum
 *   (torch's rule: the gradient goes there).  Deterministic: no atomics.
 * sg_dhead_bwd: the backward of  weight * mean((logit - target)^2)  fused with the loss (loss_out += it; may be
 *   NULL), or of a given d loss / d logit (g_logit_in fp32 [B] / [B][Lq], or NULL), both multiplied by grad_scale (the loss
 *   scale, as sg_fc_tail_bwd).  Writes every element of g_h [B][Lq][C] in the gradient dtype (sg_set_grad_dtype;
 *   gmax: zero except at the argmax).  Parameter gradients (each may be NULL: the G step) are ADDED atomically:
 *   g_pool_w [C], g_pool_b [1] (conv, mlp), g_fc_w [Lq | C], g_fc_b [1].
 * ------------------------------------------------------------------------------------------ */
#define SG_DHEAD_CONV 1
#define SG_DHEAD_GMAX 2
#define SG_DHEAD_GAVG 3
#define SG_DHEAD_MLP 4
int sg_dhead_fwd(int pool_type, const void* h, int batch, int Lq, int C, const float* pool_w, const float* pool_b,
                 const float* fc_w, const float* fc_b, float* pooled, int32_t* argmax, float* logit, void* stream);
int sg_dhead_bwd(int pool_type, const void* h, int batch, int Lq, int C, const float* pool_w, const float* fc_w,
                 const float* pooled, const int32_t* argmax, const float* logit, const float* g_logit_in,
                 float target, float weight, float* loss_out, void* g_h, float* g_pool_w, float* g_pool_b,
                 float* g_fc_w, float* g_fc_b, float grad_scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * Inference tail (clean.py:72 -> model.py:156 -> se_dataset.py:119-126): de-emphasis
 * x[n] = coef*x[n-1] + y[n] per utterance as a parallel scan; and the inverse used on input.
 * ------------------------------------------------------------------------------------------ */
int sg_deemphasis(const float* y, int64_t n, float coef, float* x, void* stream);
/* n_seg independent utterances inside one buffer: segment b = [seg[2b], seg[2b] + seg[2b+1]) (element offset, length;
 * device int64 pairs), each filtered from a zero state by its own thread block (clean.py across files). */
int sg_deemphasis_segments(const float* y, const int64_t* seg, int n_seg, float coef, float* x, void* stream);
int sg_preemphasis(const float* x, int64_t n, float coef, float* y, void* stream);
/* Input contract on the device (se_dataset.py:108-117,191-199,355-368): int16 PCM windows [n_windows][L] ->
 * normalize_wave_minmax -> pre_emphasize(coef) -> fp32 [n_windows][L] (coef <= 0: no pre-emphasis).  The reference
 * pre-emphasises the whole file before slicing: prev[w] (int32, or NULL) is the PCM sample that precedes window w in
 * its file, SG_PCM_NO_PREV when the window starts the file (y[0] = x[0]).  Lets the loader ship 2 bytes per sample
 * over PCIe and drops the host-side preprocessing. */
#define SG_PCM_NO_PREV 0x7fffffff
int sg_pcm16_to_wave(const int16_t* pcm, const int32_t* prev, int64_t n_windows, int L, float coef, float* out,
                     const int32_t* valid_len /* or NULL: per window, samples >= valid_len[w] are written as 0 (the zero
                                                 padding of an utterance's last window, model.py:122-131) */,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEGAN_B200_H */
