/* b200audio -- C ABI of the H100-native speech-inference hot path.
 *
 * The reference (Blaizzy/mlx-audio) is pure Python on Apple MLX: it has no FFI for this path.
 * Each entry point below replaces the MLX primitive call sites listed beside it (paths relative
 * to /root/reference/mlx_audio); INTEGRATION.md shows the ctypes binding a maintainer would add.
 *
 * Conventions (SURVEY.md section 8b "C-ABI layer"):
 *   - every function returns 0 on success or a negative B2A_E_* code; b2a_last_error() gives a
 *     thread-local message; nothing is ever allocated -- the caller owns every buffer, including
 *     the workspaces, whose sizes the *_ws_bytes helpers report;
 *   - all pointers are DEVICE pointers unless the name ends in _host; activations are float32,
 *     channels-last [B, L, C] with explicit batch / row strides in ELEMENTS;
 *   - `stream` is a cudaStream_t passed as void*; kernels are asynchronous on it.
 */
#ifndef B200AUDIO_H
#define B200AUDIO_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2A_OK 0
#define B2A_E_INVALID (-1)   /* bad argument (ValueError on the Python side) */
#define B2A_E_CUDA (-2)      /* CUDA runtime error (RuntimeError) */
#define B2A_E_UNSUPPORTED (-3)

/* activation codes used by prologues / epilogues */
enum {
  B2A_ACT_NONE = 0,
  B2A_ACT_LRELU = 1,      /* p0 = negative slope                (istftnet.py:721, nn.LeakyReLU) */
  B2A_ACT_SNAKE = 2,      /* x + b[c]*sin(a[c]*x)^2             (istftnet.py:382, snac/layers.py:124, speech_tokenizer.py:123) */
  B2A_ACT_ELU = 3,        /* alpha = 1                          (mimi/modules/seanet.py:102) */
  B2A_ACT_GELU = 4,       /* exact erf                          (whisper.py:415, modules.py:536) */
  B2A_ACT_GELU_TANH = 5,  /* tanh approximation                 (mimi/modules/transformer.py:141) */
  B2A_ACT_TANH = 6,
  B2A_ACT_SIGMOID = 7,
  B2A_ACT_SILU = 8,
  B2A_ACT_CLIP1 = 9       /* clip to [-1, 1]                    (speech_tokenizer.py:880) */
};

const char* b2a_last_error(void);
int32_t b2a_version(void);
int32_t b2a_device_sm_count(void);

/* ---- 1-D convolution family --------------------------------------------------------------
 * Replaces mx.conv1d / mx.conv_transpose1d / nn.Linear call sites:
 *   tts/models/kokoro/istftnet.py:128-166,811,915; codec/models/mimi/modules/conv.py:41-48,103-109;
 *   codec/models/snac/layers.py:58,111-118; stt/models/whisper/whisper.py:430-431; every nn.Linear
 *   (a Linear is the K=1 case with L = rows).
 * y[b,l,co] = epilogue( bias[co] + sum_{k,ci} W[k][ci][co] * pre(x[b, l*stride - pad_left + k*dilation, ci]) )
 *   pre(v)   = act_pre( v*pre_scale[b,ci] + pre_shift[b,ci] ), and 0 outside [0,L) (pad_mode 0) or
 *              the clamped edge sample (pad_mode 1)
 *   epilogue(v) = ( act_post(v) * post_cscale[b?,co] + res[b, l/res_div, co] ) * out_scale   (+= y if accumulate)
 * Transposed form (scatter rule of mx.conv_transpose1d, no kernel flip), with q = l + pad_left:
 *   y[b,l,co] = epilogue( bias[co] + sum_{ci} sum_{k: (q-k)%stride==0} W[k][ci][co] * pre(x[b,(q-k)/stride,ci]) )
 * Weights are pre-packed by the host as float32 [K][Cin/groups][Cout] (bf16-exact values).
 * groups must be 1 (dense) or == Cin == Cout (depthwise, W is [K][C]).
 */
typedef struct {
  const float* x; int64_t x_bs; int64_t x_ld;
  int32_t B, L, Cin;
  const float* w; const float* bias;
  float* y; int64_t y_bs; int64_t y_ld;
  int32_t Lout, Cout;
  int32_t K, stride, dilation, pad_left, groups, pad_mode;
  const float* pre_scale; const float* pre_shift;      /* [B,Cin] or NULL */
  int32_t pre_act; float pre_p0; const float* pre_a; const float* pre_b;   /* per-Cin snake params */
  int32_t post_act; float post_p0;
  const float* post_cscale; int64_t post_cscale_bs;    /* [Cout] (bs 0) or [B,Cout] or NULL */
  const float* res; int64_t res_bs; int64_t res_ld; int32_t res_div;
  float out_scale; int32_t accumulate;
  /* optional: emit the NEXT tensor-core layer's operand instead of y -- act_emit(value) split into bf16 planes hi / lo
   * [B, Lout, emit_ld] (what b2a_prep_bf16 would produce from y); depthwise stride-1 layers with Cout % 64 == 0 only
   * (snac/layers.py:208-231: Snake -> depthwise conv -> Snake -> 1x1 conv).  y may be NULL then. */
  void* emit_hi; void* emit_lo; int64_t emit_ld;
  int32_t emit_act; float emit_p0; const float* emit_a; const float* emit_b;
} b2a_conv1d_t;

int32_t b2a_conv1d_cl(const b2a_conv1d_t* p, void* stream);
int32_t b2a_convtr1d_cl(const b2a_conv1d_t* p, void* stream);

/* kernel of the calling host thread's last successful b2a_conv1d_cl / b2a_convtr1d_cl launch: out[0] = B2A_CONV_PATH_*, out[1..3] its
 * variant -- narrow: (prologue ACT it was compiled for, -1 = generic, 0, vector staging); dense: (BN, CI, 0); dw_tiled4: (CW, KT,
 * SNAKE); dw_tiled: (KT, 0, 0); convtr_dense: (BN = 64, CI, 0); the others (0, 0, 0).  All zero before the first launch.  Host-side
 * record only. */
enum {
  B2A_CONV_PATH_LINEAR_ROWS = 1,
  B2A_CONV_PATH_NARROW = 2,
  B2A_CONV_PATH_DENSE = 3,
  B2A_CONV_PATH_DW_TILED4 = 4,
  B2A_CONV_PATH_DW_TILED = 5,
  B2A_CONV_PATH_DW = 6,
  B2A_CONV_PATH_CONVTR_DENSE = 7,
  B2A_CONV_PATH_CONVTR_DW = 8
};
int32_t b2a_conv1d_cl_last_path(int32_t* out4);

/* Kokoro's harmonic-source convs (istftnet.py noise_convs) on har [B, L, 22] (contiguous): (K, stride) = (12, 6) or (1, 1), Cout a
 * multiple of 128, weights packed [K][22][Cout] as for b2a_conv1d_cl, zero padding, bias then y [B, Lout, Cout] (contiguous).
 * Bit-identical to b2a_conv1d_cl on the same layer (x 8-byte, w and y 16-byte aligned). */
int32_t b2a_kokoro_source_conv(const float* x, int32_t B, int32_t L, const float* w, const float* bias, float* y, int32_t Lout,
                               int32_t Cout, int32_t K, int32_t stride, int32_t pad_left, void* stream);

/* ---- tensor-core path for dense stride-1 convs / Linears (csrc/gemm_tc.cu) --------------------------------
 * b2a_prep_bf16: the conv prologue (pre_scale/shift + activation, as in b2a_conv1d_t) evaluated once per element and
 * stored as two bf16 planes hi = bf16(v), lo = bf16(v - hi), each [B, L, cpad] (cpad multiple of 64, pad channels zero);
 * lo == NULL stores hi only.
 * b2a_conv1d_tc: Y[b,l,n] = epilogue( sum_tap sum_ci (hi+lo)[b, l + shifts[tap], ci] * W[tap][n][ci] ), rows outside
 * [0,L) read as zero (TMA out-of-bounds fill == the conv's zero padding).  W is bf16 [taps][Cout][cin_pad]; Cout % 32 == 0.
 * wgmma (bf16 x bf16 -> fp32 in registers), operands staged by TMA; epilogue fields as in b2a_conv1d_t.
 * f16 != 0: planes and weights are IEEE fp16 instead of bf16 (fp16 checkpoints such as Whisper's: weights stay exact).
 * up_stride > 0: TRANSPOSED conv with K = taps * up_stride in polyphase form -- Cout = up_stride * C, W[tap j][r*C + co][ci] =
 * w[k = r + j*up_stride][ci][co], shifts[j] = -j; GEMM row m / column (r, co) lands on output row m*up_stride + r - up_crop
 * (rows outside [0, Lout) dropped), i.e. the GEMM output IS the up-sampled signal, no col2im pass. */
int32_t b2a_prep_bf16(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, int32_t cpad,
                      const float* scale, const float* shift, int32_t act, float p0, const float* a, const float* b,
                      void* hi, void* lo, int32_t f16, void* stream);
int32_t b2a_conv1d_tc(const void* a_hi, const void* a_lo, int32_t f16, int32_t B, int32_t L, int32_t cin_pad, const void* w_bf16,
                      const void* w_lo, /* NULL, or the low plane bf16(w - w_hi) of an fp32 checkpoint's weights */
                      int32_t taps, const int32_t* shifts_host, int32_t Cout, int32_t Lout, const float* bias,
                      int32_t post_act, float post_p0, const float* cscale, int64_t cscale_bs, const float* res,
                      int64_t res_bs, int64_t res_ld, int32_t res_div, float out_scale, int32_t accumulate, float* y,
                      int64_t y_bs, int64_t y_ld, int32_t up_stride, int32_t up_crop, void* emit_hi, void* emit_lo,
                      int64_t emit_ld, void* attn_ws, int32_t attn_heads, float attn_scale, void* stream);
/* b2a_conv1d_tc also writes its consumer's A operand from the epilogue (up_stride == 0 only; at most one of the two):
 *   emit_hi != NULL: bf16 planes bf16(y), bf16(y - hi) [B, Lout, emit_ld] (lo == NULL: hi only) -- what b2a_prep_bf16 makes of y;
 *   attn_ws != NULL: y is a fused [q | k | v] projection (Cout = 3 * 64 * attn_heads) and the epilogue fills b2a_attention_tc's
 *   workspace attn_ws (Tq = Tk = Lout, scale attn_scale) as its prologue would; then call it with operands_ready = 1.
 * The N tile is the widest divisor of Cout up to 128 unless that grid covers under half the SMs; then the widest whose grid still
 * covers them all (or 32).  Launched with programmatic dependent launch: weight tiles are fetched before the dependency wait. */

/* ---- Kokoro's ALBERT encoder layers in one persistent launch (csrc/albert.cu) -------------------------------
 * num_hidden_layers passes of the shared AlbertLayer (modules.py:497-560: qkv projection, attention, attn_out + residual, LayerNorm,
 * ffn + GELU, ffn_out + residual, LayerNorm) over h [T, hidden] fp32, in place, B = 1, 64 <= T <= 512, hidden = 64 * heads.  Inputs:
 * h and its bf16 planes h_hi / h_lo [T, hidden] (what b2a_layernorm / b2a_conv1d_tc emit; h_lo NULL when planes == 1); both are
 * overwritten.  Weights as for b2a_conv1d_tc: bf16 [N][K] in the order qkv [3 hidden][hidden], attn_out [hidden][hidden],
 * ffn [inter][hidden], ffn_out [hidden][inter]; ln_* = (attention LayerNorm, full-layer LayerNorm); scale = the softmax scale.
 * Every element is computed as b2a_conv1d_tc(planes / attention-operand epilogue), b2a_attention_tc(operands_ready) and
 * b2a_layernorm(planes) compute it, so the result equals that launch sequence bit for bit. */
typedef struct {
  int32_t T, layers, heads, hidden, inter, planes;
  const void* w[4];
  const float* bias[4];
  const float* ln_w[2];
  const float* ln_b[2];
  float eps, scale;
  float* h; void* h_hi; void* h_lo;
} b2a_albert_t;
/* bytes of the workspace b2a_albert_encoder needs (256-byte aligned; its first word is the launch's grid barrier, reset by a memset
 * in front of the kernel) */
int64_t b2a_albert_ws_bytes(int32_t T, int32_t heads, int32_t hidden, int32_t inter);
/* One cooperative launch of one CTA per SM.  err: a device word that a grid barrier which sees no progress for 10 s sets to 1 (the
 * output is then invalid); it is never cleared here.  timeline: NULL, or int64 [layers * 7][SM count][2] that a timeline build of the
 * kernel fills with globaltimer (ns) at the start and end of every stage of every CTA (profiling). */
int32_t b2a_albert_encoder(const b2a_albert_t* a, void* ws, uint32_t* err, int64_t* timeline, void* stream);

/* profiling aid: CTA (0,0,0) of subsequent b2a_conv1d_tc launches stamps clock64() at its phase boundaries into dbg8[0..6]
 * (entry, setup done, first operands landed, last operands landed, accumulator ready, epilogue done, exit); NULL disables. */
int32_t b2a_conv1d_tc_debug(void* dbg8);

/* tiling of the calling host thread's last successful b2a_conv1d_tc launch: out[0..4] = N tile (BN), grid x (row tiles), grid y
 * (Cout / BN), grid z (batch), operand stages; all zero before the first launch.  Host-side record only. */
int32_t b2a_conv1d_tc_last_config(int32_t* out5);

/* strided 2-D copy (concat without torch.cat): dst[r, c] = src[r, c] */
int32_t b2a_copy2d(const float* src, int64_t src_ld, float* dst, int64_t dst_ld, int64_t rows, int32_t cols, void* stream);
/* dst[r, :] = src[idx[r], :] (+ add[r % add_period, :] if add != NULL) -- the alignment expansion `x @ pred_aln_trg` of
 * kokoro.py:148-170, nn.Embedding, and token + positional embedding (whisper.py:483-486) */
int32_t b2a_gather_rows(const float* src, int64_t src_ld, const int64_t* idx, float* dst, int64_t dst_ld,
                        int64_t rows, int32_t cols, int64_t n_src_rows, const float* add, int64_t add_ld, int64_t add_period,
                        void* stream);
/* Duration head + alignment (kokoro.py:140-164): if dur_f != NULL, pred_dur[t] = clip(round_half_even(dur_f[t] / speed), 1, 100)
 * with nan->1, +inf->100, -inf->1 (mx.nan_to_num / mx.round / mx.clip); else pred_dur = dur_i.  Then idx_out[f] = token of
 * frame f (device prefix sum, frames beyond max_frames dropped) and *total_dev = sum(pred_dur). */
int32_t b2a_durations_to_index(const float* dur_f, const int64_t* dur_i, int32_t T, float speed, int64_t* pred_dur_out,
                               int64_t* idx_out, int64_t max_frames, int64_t* total_dev, void* stream);

/* ---- normalisation -----------------------------------------------------------------------
 * InstanceNorm statistics folded with the AdaIN affine (istftnet.py:216-268,327-338):
 *   scale[b,c] = (1+gamma[b,c]) * rstd[b,c],  shift[b,c] = beta[b,c] - scale[b,c]*mean[b,c]
 * with gb = [B, 2C] (gamma | beta) or NULL for plain InstanceNorm; biased variance, eps inside sqrt.
 * ws: float64 workspace of b2a_adain_ws_bytes(B,L,C) bytes. */
int64_t b2a_adain_ws_bytes(int32_t B, int32_t L, int32_t C);
int32_t b2a_adain_coeffs(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C,
                         const float* gb, float eps, float* scale, float* shift, void* ws, void* stream);
/* (sum, sumsq) over L of every channel of x [B, L, C], ADDED to n_dst (1..4) binned accumulators laid out [B][.][2][4] int64; dst[i] points
 * at the first channel's bins, dst_bs[i] int64 elements separate batches.  This is the statistics format b2a_conv1d_fused consumes (pre_mode 2)
 * and produces (stats_out); the stand-alone kernel covers tensors no fused conv produced (LSTM outputs, concatenated side channels). */
int32_t b2a_channel_stats(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, int64_t* const* dst,
                          const int64_t* dst_bs, int32_t n_dst, void* stream);
/* AdaIN (scale, shift) [B, C] from binned statistics [B, C, 2, 4] (for consumers outside the fused conv: depthwise layers). */
int32_t b2a_coeffs_from_stats(const int64_t* stats, int32_t B, int32_t L, int32_t C, const float* gb, float eps, float* scale, float* shift,
                              void* stream);
/* y[r,:] = LN(x[r,:] + res[r,:]) * w + b, or (1+ada[c])*LN + ada[C+c] when ada != NULL
 * (nn.LayerNorm, modules.py:71-90 AdaLayerNorm). rms != 0 -> RMSNorm (no mean, talker.py:267). */
int32_t b2a_layernorm(const float* x, int64_t x_ld, const float* res, int64_t res_ld, float* y, int64_t y_ld,
                      int64_t rows, int32_t C, const float* w, const float* b, const float* ada, float eps,
                      int32_t rms, int32_t post_act, float post_p0, void* emit_hi, void* emit_lo, int64_t emit_ld, void* stream);
/* emit_hi != NULL: also the bf16 planes bf16(y), bf16(y - hi) of every row, [rows, emit_ld] (lo may be NULL) -- the next GEMM's
 * A operand, as b2a_prep_bf16 would make it.  Needs C % 8 == 0, C <= 1024 and 16-byte aligned rows. */

/* ---- attention -----------------------------------------------------------------------------
 * softmax(scale * q k^T + mask) v with fp32 softmax; replaces mx.fast.scaled_dot_product_attention
 * (mimi/modules/transformer.py:109, talker.py:307) and the unfused form (whisper.py:371-385, modules.py:497-505).
 * q [B,Tq,H,D], k/v [B,Tk,Hkv,D] with token strides *_ld and batch strides *_bs (elements); head h at +h*D.
 * causal != 0: key j visible to query i iff j <= i + q_offset; window > 0 (only with causal != 0, else an invalid argument): also
 * i + q_offset - j < window.  q, k, v, o 16-byte aligned, all strides multiples of 4. */
typedef struct {
  const float* q; const float* k; const float* v; float* o;
  int64_t q_bs, q_ld, k_bs, k_ld, v_bs, v_ld, o_bs, o_ld;
  int32_t B, Tq, Tk, H, Hkv, D;
  float scale; int32_t causal, q_offset, window;
  const int32_t* k_len;     /* [B] valid key count or NULL */
  /* b2a_attention_tc only: */
  void* emit_hi; void* emit_lo; int64_t emit_ld;   /* optional bf16 planes bf16(o), bf16(o - hi) [B, Tq, emit_ld] for the next GEMM */
  int32_t operands_ready;   /* != 0: ws already holds the q / k / v planes (b2a_conv1d_tc's attention-operand epilogue); q, k, v unused */
} b2a_attn_t;
int32_t b2a_attention(const b2a_attn_t* p, void* stream);
/* Same contract on the tensor cores (wgmma) for D == 64, H == Hkv, k_len == NULL: S = QK^T and PV as fp16 hi/lo-plane MMAs
 * (fp32-grade products), online softmax with one thread per query row.  ws: device scratch of b2a_attention_tc_ws_bytes bytes
 * (fp16 planes of q * scale * log2(e), k and the transposed v, keys zero-padded to a multiple of 8).  Launched with programmatic
 * dependent launch.
 * Operand envelope: the result is fp32-grade (within 2e-5 of float64) while the operands stay above ~2^-10 in magnitude and
 * q * scale * log2(e), k and v stay below fp16's 65504.  fp16's subnormal floor (2^-24) limits the lo planes, which matters for v
 * (it scales the output): v of rms 2^-6 .. 2^8 measured within 2e-6 on an H100 80GB HBM3 (700 W); v of rms 2^-10 is emulated at
 * 1.4e-5; v of rms 1e-4 measured 1.4e-4, as a float64 emulation of the split predicts.  Small q or k only shrink the scores.
 * tests/test_attention_norm_matrix_gpu.py pins these numbers. */
int64_t b2a_attention_tc_ws_bytes(int32_t B, int32_t H, int32_t Tq, int32_t Tk);
int32_t b2a_attention_tc(const b2a_attn_t* p, void* ws, void* stream);
/* in-place rotary embedding on x [B,T,H,D] (token stride ld): traditional != 0 rotates pairs (2i,2i+1)
 * (nn.RoPE(traditional=True), mimi/modules/transformer.py:75-77), else (i, i+D/2) (talker.py:14-18). */
int32_t b2a_rope(float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t H, int32_t D,
                 int32_t offset, float base, int32_t traditional, void* stream);

/* ---- bidirectional LSTM recurrence (modules.py:93-285) ------------------------------------
 * xproj [B,T,2,4H] = x @ Wx^T + b_ih + b_hh for (forward|backward), gate order i,f,g,o;
 * wh [2,4H,H]; out [B,T,2H] (forward | backward).  H must be 256 (Kokoro) -- one 8-CTA cluster
 * per (direction, batch) keeps Wh in registers; each warp runs its 4 hidden units' step on its own and
 * pushes their new h into every CTA's shared memory (distributed shared memory, one mbarrier per step). */
int32_t b2a_lstm_bidir(const float* xproj, const float* wh, float* out, int64_t out_ld, int32_t B, int32_t T, int32_t H, void* stream);

/* ---- DSP ------------------------------------------------------------------------------------
 * b2a_stft: dsp.py:385-433 on a batch of 1-D signals. out_re/out_im [B, frames, n_fft/2+1].
 * pad_mode: 0 none (center=False), 1 reflect, 2 constant.  window [n_fft] (already zero-padded). */
int32_t b2a_stft(const float* x, int64_t x_bs, int32_t B, int64_t n, const float* window, int32_t n_fft, int32_t hop,
                 int32_t pad_mode, int64_t frames, float* out_re, float* out_im, void* stream);
/* Whisper log-mel (stt/models/whisper/audio.py:41-82): frames-major [B, frames, n_mels]; `frames` excludes the
 * dropped last STFT frame; n = samples per signal (right zero padding of `padding` samples is virtual).
 * gmax [B] scratch for the per-utterance max. */
int32_t b2a_whisper_logmel(const float* x, int64_t x_bs, int32_t B, int64_t n, int64_t padding, const float* window,
                           const float* filters, int32_t n_mels, int64_t frames, float* out, float* gmax, void* stream);
/* dsp.py:436-513 / 663-738: inverse rFFT per frame, synthesis window, overlap-add, divide by sum(w^2) (norm_sq) or
 * sum(w), clamp denominators as the reference does (mode 0: where(wsum>1e-10); mode 1: max(wsum,1e-10)).
 * re/im [B, n_freq, T]; out [B, out_len] starting at sample `trim` of the OLA buffer. ws: B*T*n_fft floats. */
int32_t b2a_istft(const float* re, const float* im, int32_t B, int32_t n_fft, int32_t T, int32_t hop, const float* window,
                  int32_t norm_sq, int32_t clamp_mode, int64_t trim, int64_t out_len, float* out, float* ws, void* stream);

/* Polyphase resampling, the arithmetic of scipy.signal.resample_poly(x, up, down, window=h, padtype="edge") that the reference
 * calls on the host (resample.py:29-47): x [B, n_in] float32, h float64 FIR ALREADY multiplied by `up`, n_pre_pad / n_pre_remove
 * as SciPy derives them (host side: mlx_audio_b200/resample.py), out [B, n_out] float32, float64 accumulation. */
int32_t b2a_resample_poly(const float* x, int64_t x_bs, int32_t B, int64_t n_in, const double* h, int32_t n_h, int32_t up,
                          int32_t down, int64_t n_pre_pad, int64_t n_pre_remove, float* out, int64_t n_out, void* stream);

/* ---- Kokoro hn-NSF source + iSTFT head (istftnet.py:548-709, 453-545, 826-835) ------------
 * f0 [B, n_frames] (the F0 curve, one value per 300 samples); noise [B, n_frames*300, 9] injected N(0,1) (or NULL);
 * lin_w [9], lin_b [1] = m_source.l_linear.  har [B, n_frames*60+1, 22] = (|STFT| , angle) of the tanh-merged source,
 * n_fft 20 hop 5 periodic Hann, reflect-centred.  n_down = ceil(float(300*n_frames) * float(1/300)) is the length of the
 * reference's down-sampled phase track (interpolate.py:43-50; n_frames or n_frames+1 by floating-point rounding -- a parity
 * quirk the host evaluates exactly as the reference does).  src_ws: float [B, n_frames*300]; ph_ws: double [B, n_down, 9]. */
int32_t b2a_kokoro_source(const float* f0, int32_t B, int32_t n_frames, int32_t n_down, const float* noise, const float* lin_w,
                          const float* lin_b, float* har, float* src_ws, double* ph_ws, void* stream);
/* x [B, T, 22] = conv_post output -> audio [B, (T-1)*5] : exp / sin heads, cos/sin, 20-point inverse rFFT, periodic Hann,
 * overlap-add, / sum(w^2), trim 10 samples each side (phase in [-1,1] so mlx_unwrap is the identity). */
int32_t b2a_kokoro_istft_head(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, float* audio, void* stream);

/* ---- fused dense conv1d / nn.Linear / polyphase ConvTranspose1d on wgmma (csrc/conv_fused.cu) ------------------------------
 * One launch = [InstanceNorm / AdaIN coefficients from the producer's (sum, sumsq)] + input activation + bf16/fp16 hi(+lo) split +
 * sum over taps of row-shifted GEMMs + bias / activation / channel scale / residual / scale / accumulate (+ polyphase scatter) +
 * (sum, sumsq) of the output for the NEXT layer's InstanceNorm.  Replaces, per layer, the call sites of mx.conv1d / conv_transpose1d /
 * nn.Linear TOGETHER WITH the elementwise chain in front of them: AdaIN1d + Snake / LeakyReLU in AdaINResBlock1 and AdainResBlk1d
 * (tts/models/kokoro/istftnet.py:216-396, 853-933), the generator's ups / conv_post (:725-835), ALBERT's Linear layers
 * (tts/models/kokoro/modules.py:434-645).  Up to B2A_CONVF_MAX_PROBLEMS independent problems share one persistent grid (the three
 * parallel resblocks of a generator stage).  x: fp32 [B, L, Cin] (16-byte aligned, row stride % 4 == 0); optional x1 / x2 (same
 * strides) are added to x first (the resblock average of the previous stage), then * in_scale.  Weights as for b2a_conv1d_tc:
 * 16-bit [taps][N][cin_pad] (+ optional lo plane).  y: fp32 [B, Lout, C].  pre_mode 0: no affine; 1: x*scale[b,c]+shift[b,c];
 * 2: scale/shift derived in-kernel from pre_stats [B, Cin, 2, 4] = (sum, sumsq) over L (biased variance, eps) and gamma|beta rows
 * pre_gb [B, 2 Cin] (NULL: plain InstanceNorm).  stats_out [B, C, 2, 4] is ADDED to (zero it before the launch).  A statistic is four
 * int64 bins counting multiples of 2^(-100 + 40 k): integer atomics make the accumulation order-independent, so results are
 * bit-reproducible across runs and between eager launches and graph replays (csrc/common.cuh: repro_add / repro_value).
 * ws: zero-initialised scratch (>= 16 MiB recommended) for split-K partial tiles; NULL disables K splitting. */
#define B2A_CONVF_MAX_PROBLEMS 4
typedef struct {
  const float* x; const float* x1; const float* x2; int64_t x_bs, x_ld; float in_scale;
  int32_t B, L, Cin;
  int32_t pre_mode; const float* pre_scale; const float* pre_shift; const int64_t* pre_stats; const float* pre_gb; int64_t pre_gb_bs; float pre_eps;
  int32_t pre_act; float pre_p0; const float* pre_a; const float* pre_b;
  const void* w_hi; const void* w_lo; int32_t cin_pad, taps, N; int32_t shifts[32];
  int32_t Lout; const float* bias; int32_t post_act; float post_p0; const float* cscale; int64_t cscale_bs;
  const float* res; int64_t res_bs, res_ld; int32_t res_div; float out_scale; int32_t accumulate;
  float* y; int64_t y_bs, y_ld;
  int32_t up_stride, up_crop;
  int64_t* stats_out;
} b2a_convf_t;
int32_t b2a_conv1d_fused_debug(void* stamps /* device uint64 [grid][16] or NULL: phase time stamps of the next launches */);
int32_t b2a_conv1d_fused(const b2a_convf_t* problems, int32_t n_problems, int32_t planes, int32_t f16, void* ws, int64_t ws_bytes, void* stream);
/* 1 when a launch of one problem with taps spanning `span` rows (0..64), N GEMM columns over C output channels (N = up_stride * C in
 * polyphase mode, else N = C), wplanes weight planes (2: w_lo set) and `planes` activation planes finds room for two weight stages in
 * shared memory, else 0 (b2a_conv1d_fused would return B2A_E_UNSUPPORTED).  Host-side only. */
int32_t b2a_conv1d_fused_fits(int32_t span, int32_t N, int32_t C, int32_t wplanes, int32_t planes);
/* tiling of the calling host thread's last successful b2a_conv1d_fused launch: out[0] = problems, out[1] = grid (CTAs),
 * out[2 + 2 i], out[3 + 2 i] = N tile and K split of problem i in the caller's order (i < 4, unused slots zero).  Host-side only. */
int32_t b2a_conv1d_fused_last_config(int32_t* out10);

/* out[i] ~ N(0,1), i < n: Philox4x32-10 keyed by `seed`, counter `offset + i/4`, Box-Muller.  The production replacement for
 * mx.random.normal in SineGen / NoiseBlock (istftnet.py:649, snac/layers.py:263); parity tests inject the noise instead. */
int32_t b2a_randn(float* out, int64_t n, uint64_t seed, uint64_t offset, void* stream);
/* Same draws with {seed, offset} read from DEVICE memory (state[0], state[1]); a second one-thread launch then advances state[1] by the
 * (n + 3) / 4 counters used, so a captured CUDA graph draws fresh noise on every replay the way mx.random's global state advances. */
int32_t b2a_randn_dev(float* out, int64_t n, uint64_t* state, void* stream);

/* ---- Whisper decode step (stt/models/whisper/decoding.py:307-325,349-442) -----------------------------------
 * One launch = SuppressBlank + SuppressTokens + ApplyTimestampRules + GreedyDecoder.update(temperature 0) for every row:
 * next_out[b] = argmax of the filtered logits (eot once a row has ended), sum_logprobs[b] += its log-probability while the row
 * is live, *not_done += 1 per row whose next token is not eot.  tokens [B, >= cur_len] is the device-resident history
 * (no per-step tolist()); suppress_mask / blank_mask are additive 0/-inf vectors [V] (NULL = none); max_initial_ts < 0 = off.
 * temperature > 0 (the fallback temperatures of whisper.py:957-995): the next token is a categorical draw from softmax(filtered / temperature)
 * -- inverse CDF in index order driven by u[b] in [0,1) -- and the log-probability bookkeeping uses the un-tempered logits, as
 * GreedyDecoder.update does (decoding.py:307-325). */
int32_t b2a_whisper_greedy_step(const float* logits, int64_t logits_bs, const int64_t* tokens, int64_t tokens_bs,
                                int32_t B, int32_t cur_len, int32_t sample_begin, int32_t V, const float* suppress_mask,
                                const float* blank_mask, int32_t eot, int32_t no_timestamps, int32_t timestamp_begin,
                                int32_t max_initial_ts, int32_t without_timestamps, int64_t* next_out,
                                float* sum_logprobs, int32_t* not_done, float temperature, const float* u, void* stream);

/* Fused LM sampler (tts/models/qwen3_tts/qwen3_tts.py:805-860 over lm/sample_utils.py:131-239,279): additive suppress mask ->
 * sign-aware repetition penalty on the `seen` set -> temperature (<= 0: argmax) -> top-k -> top-p -> min-p -> categorical draw
 * by inverse CDF in index order with the caller's uniform u[b] (MLX's PRNG is not reproducible; tests inject u).  V <= 4096.
 * out[b * out_stride] receives the token; mark_seen != 0 also sets seen[b][token] (generated_token_ids.append, :1402).
 * finished (optional, uint8 [B], in/out) implements the batch loop's bookkeeping (:1880-1887,1923-1929): a finished row emits eos
 * and is not marked; a row that samples eos becomes finished.
 * filtered_out (optional) receives the filtered, temperature-scaled logits the draw is made from. */
int32_t b2a_sample_token(const float* logits, int64_t logits_bs, int32_t B, int32_t V, const float* suppress_mask,
                         uint8_t* seen, int64_t seen_bs, int32_t mark_seen, float repetition_penalty, float temperature,
                         int32_t top_k, float top_p, float min_p, const float* u, int64_t* out, int64_t out_stride,
                         float* filtered_out, uint8_t* finished, int32_t eos, void* stream);

/* ---- autoregressive LM step (Qwen3-TTS talker / code predictor, tts/models/qwen3_tts/talker.py) -----------------------
 * All position-dependent scalars may come from device memory (base_dev, tidx) so that one captured CUDA graph replays
 * every frame of Model.generate's loop (qwen3_tts.py:1323-1404) without host round trips.
 *
 * b2a_gemv_bf16: y[m, n] = sum_k W[n,k] xn[m,k] (+ bias[n]) (+ res[m,n]) for M <= 8 activation rows -- nn.Linear at decode
 * time (talker.py:284-286,314,335).  W bf16 row-major [N, w_ld].  norm_w != NULL fuses the preceding nn.RMSNorm
 * (talker.py:388,395; x * rsqrt(mean(x^2) + eps) * norm_w).  mode 1 fuses SwiGLU (talker.py:319-321): W rows interleaved
 * (gate_0, up_0, gate_1, ...), y[m, n/2] = silu(gate) * up, y has N/2 columns.  prefetch (optional): the NEXT projection's
 * weights, prefetch_bytes of them are pulled into L2 (prefetch.global.L2) while this kernel runs, so the dependent launch that
 * follows finds them on chip. */
int32_t b2a_gemv_bf16(const float* x, int64_t x_ld, int32_t M, int32_t K, const void* w_bf16, int64_t w_ld, int32_t N,
                      const float* bias, const float* norm_w, float norm_eps, int32_t mode, const float* res, int64_t res_ld,
                      float* y, int64_t y_ld, const void* prefetch, int64_t prefetch_bytes, void* stream);
/* TalkerAttention / CodePredictorAttention / DecoderAttention up to the cache update (talker.py:288-307,558-572;
 * speech_tokenizer.py:291-296): qkv [B,S,(Hq+2Hkv) D] -> per-head RMSNorm of q and k (weights [D], NULL = none), rotary
 * embedding in the rotate_half convention, q_out [B,S,Hq,D], k/v appended to the caches [B,Smax,Hkv,D] at row base + s,
 * base = *base_dev (or base_host when base_dev is NULL).  Rotary position of frequency slot i: pos3[axis,b,s] with the
 * interleaved-MRoPE axis rule of talker.py:139-184 (axis 1 if i%3==1 && i<3*sec_h, axis 2 if i%3==2 && i<3*sec_w, else 0);
 * pos3 NULL = base + s on every axis (sec_h = sec_w = 0 gives the standard RoPE of talker.py:68-113), minus pos_shift[b] (clamped at
 * 0) when pos_shift != NULL: the cumsum(attention_mask) - 1 positions of left-padded batches (talker.py:452-457).
 * Per-row cache positions (continuous batching, replacing the KVCache.merge / BatchKVCache.extract of continuous_batching.py:140,178,
 * 309-324, and the attention_mask of :280-302): base_rows [B] != NULL takes the place of the scalar base, so row b, query s goes to cache
 * row and rotary position base_rows[b] + s; a negative value is a left-padding row and writes nothing.  slot [B] != NULL is the cache
 * batch index row b reads and writes (NULL = b).  Both NULL: unchanged behaviour. */
int32_t b2a_qknorm_rope_cache(const float* qkv, int64_t qkv_bs, int64_t qkv_ss, int32_t B, int32_t S, int32_t Hq, int32_t Hkv,
                              int32_t D, const float* q_norm_w, const float* k_norm_w, float eps, const int32_t* pos3,
                              const int32_t* base_dev, int32_t base_host, int32_t sec_h, int32_t sec_w, float theta,
                              float* q_out, int64_t qo_bs, int64_t qo_ss, float* k_cache, float* v_cache, int64_t c_bs,
                              int64_t c_ss, int32_t smax, const int32_t* pos_shift, const int32_t* base_rows, const int32_t* slot,
                              void* stream);
/* mx.fast.scaled_dot_product_attention against the KV cache with GQA (talker.py:309-312): query s attends cache rows
 * [kv_start[b], base + s] (causal inside the new block; kv_start NULL = 0, else the left-padding count of
 * qwen3_tts.py:486-604's batches).  out [B,S,Hq*D].  max_k bounds base + S (shared-memory sizing).  base_rows / slot as in
 * b2a_qknorm_rope_cache: query s of row b sees cache rows [kv_start[b], base_rows[b] + s] of cache batch slot[b]; a query whose
 * position is negative (left padding) has a zero output. */
int32_t b2a_attn_decode(const float* q, int64_t q_bs, int64_t q_ss, const float* k_cache, const float* v_cache, int64_t c_bs,
                        int64_t c_ss, float* out, int64_t o_bs, int64_t o_ss, int32_t B, int32_t S, int32_t Hq, int32_t Hkv,
                        int32_t D, float scale, const int32_t* base_dev, int32_t base_host, const int32_t* kv_start,
                        int32_t max_k, const int32_t* base_rows, const int32_t* slot, void* stream);
/* The same contract as b2a_attn_decode for long prefills (talker.py:288-312 over a prompt of >= 64 rows: the in-context voice-cloning
 * prompt) on the tensor cores: head_dim 128, Hq = 2 Hkv.  One CTA per (64 query rows, kv head, batch row); both query heads of the GQA
 * pair share each K / V tile, which is read once from the fp32 cache and split into fp16 hi / lo planes (3-product scores and P V,
 * fp32 accumulate).  Keys are taken in a fixed order: bit-reproducible.  Query row s sees cache rows [kv_start[b], min(base + s,
 * max_k - 1)].  Rows 16-byte aligned (q, caches); out rows 8-byte aligned.  base_rows / slot as in b2a_attn_decode; key tiles
 * outside a CTA's ragged key range (including tiles whose query rows are all left padding) are skipped, not masked. */
int32_t b2a_attn_prefill(const float* q, int64_t q_bs, int64_t q_ss, const float* k_cache, const float* v_cache, int64_t c_bs,
                         int64_t c_ss, float* out, int64_t o_bs, int64_t o_ss, int32_t B, int32_t S, int32_t Hq, int32_t Hkv,
                         int32_t D, float scale, const int32_t* base_dev, int32_t base_host, const int32_t* kv_start,
                         int32_t max_k, const int32_t* base_rows, const int32_t* slot, void* stream);
/* y[r, i] = silu(gate) * up (talker.py:319-321, speech_tokenizer.py:321-322) for the batched (prefill) path: x [rows, 2I] holds
 * (gate | up) halves, or interleaved (gate_0, up_0, gate_1, ...) pairs -- the row order b2a_gemv_bf16 mode 1 uses. */
int32_t b2a_swiglu(const float* x, int64_t x_ld, int64_t rows, int32_t I, int32_t interleaved, float* y, int64_t y_ld, void* stream);
/* Next talker input (qwen3_tts.py:1383-1398): out[b] = text(b) + sum_g tables[g][codes[b,g]].  tables_dev / bins_dev are DEVICE
 * arrays of G table pointers / table sizes; an out-of-range code sets *err_flag_dev.  text(b) follows the batch rule of
 * _next_batch_input_embeds(pad_when_index_clamped=True) (qwen3_tts.py:993-1015): text row min(tidx[b], n_text-1), replaced by pad
 * (tts_pad_embed) when that is >= n_text-1; afterwards tidx[b] += 1 for rows that are not finished.  text and tidx are given
 * together or not at all; without them text(b) = pad (NULL = 0). */
int32_t b2a_embed_sum(const int64_t* codes, int64_t codes_bs, int32_t B, int32_t G, int32_t dim, const float* const* tables_dev,
                      const int32_t* bins_dev, const float* text, int64_t text_bs, int64_t text_ss, int32_t n_text,
                      const float* pad, float* out, int64_t out_bs,
                      int32_t* err_flag_dev, int32_t* tidx, const uint8_t* finished, void* stream);
/* *p += v on the stream (KVCache.offset bookkeeping, lm/models/cache.py:112-155, kept on the device). */
int32_t b2a_incr_i32(int32_t* p, int32_t v, void* stream);
/* End of a continuous-batching frame over B slots (the per-request bookkeeping of _advance_active, continuous_batching.py:201-216):
 * for every slot whose finished[b] is 0 after the frame's sample (the sampler sets it on EOS; empty slots are kept at 1),
 * out[b, frames[b], :] = codes[b, :G] (out row stride out_bs), frames[b] += 1, lengths[b] += 1, finished[b] = 1 once
 * frames[b] >= cap[b] (the max_tokens test of :210-213), else u[g, b] = u_tab[b, frames[b], g] (row stride u_bs) for the next
 * frame.  Finished and empty slots are unchanged, so a CUDA graph of the frame needs no host scalar. */
int32_t b2a_slot_advance(int32_t* lengths, int32_t* frames, uint8_t* finished, const int32_t* cap, const int64_t* codes, int32_t G,
                         int64_t* out, int64_t out_bs, const float* u_tab, int64_t u_bs, float* u, int32_t B, void* stream);

/* ---- codec (RVQ decode) ---------------------------------------------------------------------
 * out[b,t,:] (+)= sum_q codebooks[q][codes[b,q,t]][:]   (mimi/modules/quantization.py:47-49,103-108;
 * speech_tokenizer.py:431-490).  codes int64 [B, nq, T]; codebooks [nq, bins, dim]. Returns B2A_E_INVALID if any code
 * is out of range (checked on device, reported via *err_flag_dev != 0). */
int32_t b2a_rvq_decode(const int64_t* codes, int64_t codes_bs, int64_t codes_qs, int32_t B, int32_t nq, int64_t T,
                       const float* codebooks, int32_t bins, int32_t dim, float* out, int64_t out_ld, int32_t* err_flag_dev, void* stream);
/* Residual-VQ ENCODE: codes[row, q] = nearest entry of codebooks[q] to the row's residual, q = 0 .. nq-1, the residual shrinking by the
 * chosen entry after every level (mimi/modules/quantization.py:37-45, 90-101; speech_tokenizer.py:957-1058 uses the same quantizer).
 * x [rows, dim] fp32 (row stride x_ld); codebooks [nq, bins, dim]; c2 [nq, bins] float64: mode 0 (Euclidean) |e|^2 / 2, score = c2 - x.e;
 * mode 1 (SNAC, snac/vq.py:56-73: one level, L2-normalised rows -- codebooks must hold the NORMALISED table) |en|^2, score = |xn|^2 - 2 xn.en
 * + c2.  Scores accumulate in float64; ties -> lowest index.  codes int64, element (row, q) at row * codes_row_stride + q * codes_level_stride. */
int32_t b2a_rvq_encode(const float* x, int64_t x_ld, int64_t rows, int32_t dim, const float* codebooks, const double* c2, int32_t bins,
                       int32_t nq, int32_t mode, int64_t* codes, int64_t codes_row_stride, int64_t codes_level_stride, void* stream);
/* SNAC from_codes (snac/vq.py:111-131): z[b,t,:] = sum_l ( W_l @ E_l[codes_l[b, t / stride_l]] + bias_l ),
 * codes_l int64 [B, T/stride_l]; E_l [bins, cd]; W_l [cd][dim] (packed, K=1); out [B,T,dim]. */
int32_t b2a_snac_from_codes(const int64_t* const* codes_host_ptrs, const int32_t* strides_host, int32_t n_levels,
                            const float* const* emb_host_ptrs, const float* const* w_host_ptrs, const float* const* bias_host_ptrs,
                            int32_t B, int64_t T, int32_t bins, int32_t cd, int32_t dim, float* out, int32_t* err_flag_dev, void* stream);

/* ---- Descript Audio Codec quantiser (dac.cu; codec/models/descript/nn/quantize.py) ------------------------------------------
 * One level of the factorised residual quantiser, all pointers to DEVICE memory; the table of levels itself lives in device memory.
 * w_in [dim][cd] and w_out [cd][dim] are the weight-norm-folded 1x1 projections in packed (K = 1) conv layout, cb the code book
 * [bins][cd], cbn its rows L2-normalised (x / max(|x|, 1e-12), rounded to fp32), c2[i] = |cbn[i]|^2 in float64.  lat_off = the level's
 * first channel in the concatenated latents (sum of the previous levels' cd).  Decode reads cb, w_out, b_out, cd, lat_off only. */
typedef struct {
  const float* w_in; const float* b_in;
  const float* cbn; const double* c2;
  const float* cb;
  const float* w_out; const float* b_out;
  int32_t cd; int32_t lat_off;
} b2a_dac_level_t;
/* ResidualVectorQuantize.__call__ (quantize.py:87-120 over VectorQuantize.__call__ / decode_latents :25-63) in one launch, for
 * n_levels <= the model's code books: per level z_e = w_in r + b_in, idx = argmin_i |z_e/|z_e||^2 - 2 z_e/|z_e| . cbn_i + |cbn_i|^2 (float64
 * scores, lowest index on ties), z_q_l = w_out cb[idx] + b_out, r -= z_q_l.  z [B*T, dim] fp32 rows (row stride z_ld, channels-last);
 * outputs codes int64 [B, n_levels, T], latents [B, latent_channels, T] (the un-normalised z_e of every level), z_q [B, T, dim] and
 * loss_part float64 [ceil(B*T / 8)]: its sum is the reference's commitment loss (= its codebook loss in the forward pass), the per-level
 * mean of (z_e - cb[idx])^2 summed over levels.  z == NULL runs from_latents (quantize.py:133-151) instead: z_e is READ from latents.
 * A CTA holds 8 frames' residual and z_q in b2a_dac_rvq_encode_smem_bytes of dynamic shared memory. */
int64_t b2a_dac_rvq_encode_smem_bytes(int32_t dim);
int32_t b2a_dac_rvq_encode(const float* z, int64_t z_ld, int32_t B, int64_t T, int32_t dim, const b2a_dac_level_t* levels_dev, int32_t n_levels,
                           int32_t bins, int32_t latent_channels, int64_t* codes, float* latents, float* z_q, double* loss_part, void* stream);
/* ResidualVectorQuantize.from_codes (quantize.py:122-131) for the first n_levels code books: out[b,t,:] = sum_l ( w_out_l cb_l[codes[b,l,t]]
 * + b_out_l ), and z_p [B, latent_channels, T] = the gathered rows (NULL: not wanted).  codes int64, element (b, l, t) at b * codes_bs +
 * l * codes_qs + t.  A code outside [0, bins) sets *err_flag_dev (and decodes as 0). */
int32_t b2a_dac_from_codes(const int64_t* codes, int64_t codes_bs, int64_t codes_qs, int32_t B, int32_t n_levels, int64_t T,
                           const b2a_dac_level_t* levels_dev, int32_t bins, int32_t latent_channels, int32_t dim, float* out, float* z_p,
                           int32_t* err_flag_dev, void* stream);

/* ---- BigVGAN anti-aliased activation (bigvgan.cu; codec/models/bigvgan/resample.py, activation.py) ---------------------------
 * Activation1d(SnakeBeta) (resample.py:157-177, activation.py:42-51) in one pass: x [B, L, C] fp32 (element (b, t, c) at b * x_bs +
 * t * x_ld + c) -> [B, L, C].  UpSample1d (resample.py:122-136): edge pad 5 rows, MLX conv_transpose1d scatter y[2i + k] += x[i] f_up[k]
 * (no kernel flip) per channel, times 2, crop 15 rows each side; SnakeBeta v = u + inv_beta[c] sin(alpha[c] u)^2 with the Snake sine of
 * common.cuh; alpha = exp(alpha) and inv_beta = 1 / (exp(beta) + 1e-9) precomputed per channel for snake_logscale; DownSample1d
 * (resample.py:79-98): edge pad 5 | 6 rows of v, 12-tap f_down at stride 2.  f_up / f_down: the 12 taps as the checkpoint holds them.
 * Output either fp32 y (row stride y_ld, batch stride y_bs) or the next tensor-core conv's bf16 planes hi / lo (lo may be NULL)
 * [B, L, cpad] contiguous, pad channels zeroed, split as b2a_prep_bf16 splits them; exactly one of y / hi.  ratio 2 and 12 taps
 * only (all BigVGAN uses): anything else is B2A_E_UNSUPPORTED.  Fixed tap order: bit-reproducible, independent of B. */
int32_t b2a_aa_snakebeta(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, const float* alpha, const float* inv_beta,
                         const float* f_up, const float* f_down, int32_t ratio, int32_t taps, float* y, int64_t y_bs, int64_t y_ld, void* hi,
                         void* lo, int32_t cpad, void* stream);

/* ---- streaming decoder state (stream.cu) ------------------------------------------------------
 * One entry of a grouped row-range launch on fp32 [B, rows, C] views: dst[b, r, c] = src[b, r, c] (COPY) or += (ADD), element
 * (b, r, c) at b * bs + r * ld + c.  The incremental Qwen3-TTS speech-tokenizer decoder keeps its state with it:
 *   COPY: the last (K-1)*dilation input rows of a causal conv become the history head of the next call's input buffer -- replaces
 *         CausalConv1d.step (speech_tokenizer.py:71-83), ConvNeXtBlock.step's depthwise conv (:151-159), DecoderInitialConv.step
 *         (:719-728) and DecoderOutputConv.step (:771-780); also the KV-cache growth of the decoder transformer (:610-617);
 *   ADD:  the r-row overflow of a decoder block's transposed conv (bias included) is added into the head rows of the next call's
 *         output -- DecoderBlockUpsample.step (:645-656). */
#define B2A_ROWOP_COPY 0
#define B2A_ROWOP_ADD 1
#define B2A_ROWOPS_MAX 32
typedef struct {
  const float* src; int64_t src_bs, src_ld;
  float* dst; int64_t dst_bs, dst_ld;
  int32_t B, rows, C, op;
} b2a_rowop_t;
/* All n <= B2A_ROWOPS_MAX entries in one launch.  Entries run concurrently: an entry's destination may not overlap its own source or
 * any range another entry reads or writes (B2A_E_INVALID otherwise).  Empty entries are skipped. */
int32_t b2a_stream_rows(const b2a_rowop_t* ops, int32_t n, void* stream);

/* ---- incremental Mimi codec (mimi_stream.cu): Mimi.decode_step / encode_step (codec/models/mimi/mimi.py:164-176) ----------------
 * b2a_conv1d_stream: StreamableConv1d.step (mimi/modules/conv.py:245-273) -- a causal conv over the virtual input [history | new rows],
 * history = the H input rows the previous call did not consume.  p->x holds the L new rows (x may be NULL when L == 0), p->Lout must be
 * the number of complete windows, (H + L - keff) / stride + 1 or 0, keff = (K-1)*dilation + 1, and output row l reads virtual rows
 * l*stride + k*dilation (p->pad_left is ignored).  Prologue (pre_act, pre_p0), bias, post_act, post_cscale, res / res_div, out_scale as
 * in b2a_conv1d_t; dense only (groups 1); no pre_scale / shift, Snake, emit or accumulate.  The same launch writes the new history,
 * virtual rows [Lout*stride, H + L), into the other slot of hist: float [2][B][keff-1][Cin] with batch stride hist_bs (>= (keff-1)*Cin),
 * slot (*step_dev & 1) being read -- so the caller flips the parity once per step (b2a_stream_advance) and never concatenates.
 * fresh != 0: the first call of a stream, the history rows are the causal left padding instead -- zeros (pad_mode 0) or the first new
 * row (pad_mode 1, replicate); a fresh call with L == 0 writes nothing.  The padding is a row of the activated input, so a prologue with
 * act(0) != 0 (sigmoid) needs pad_mode 1; stride <= keff (B2A_E_INVALID otherwise). */
int32_t b2a_conv1d_stream(const b2a_conv1d_t* p, float* hist, int64_t hist_bs, int32_t H, const int32_t* step_dev, int32_t fresh,
                          void* stream);
/* b2a_convtr1d_stream: StreamableConvTranspose1d.step (conv.py:315-331) -- y [B, L*stride, Cout] = bias + the transposed conv of the L new
 * rows (scatter rule of b2a_convtr1d_cl, no crop) + tail on the first K - stride rows; tail [B, K - stride, Cout] (batch stride tail_bs,
 * row stride Cout, zero at the start of a stream) is then replaced by output rows [L*stride, L*stride + K - stride) WITHOUT the bias (the
 * reference subtracts it).  Dense or depthwise (groups == Cin == Cout); prologue activation, bias and out_scale only; K - stride <= L*stride.
 * With K == stride there is no tail and tail may be NULL. */
int32_t b2a_convtr1d_stream(const b2a_conv1d_t* p, float* tail, int64_t tail_bs, void* stream);
/* Windowed attention over a ring KV cache (transformer.py:79-112 with the growing KVCache and the context mask), position counter on the
 * device so that a captured step replays without host scalars:
 * b2a_ring_rope_kv: qkv [B, T, 3 H D] ([q | k | v], head h at +h*D, token stride qkv_ld): interleaved-pair RoPE (nn.RoPE traditional, base)
 *   of q (in place) and k at absolute positions *pos_dev + t; rotated k and v stored at ring row (*pos_dev + t) % cap of k_ring / v_ring
 *   [B, cap, H D] (batch stride ring_bs).
 * b2a_ring_attn: out[b, t, h] = softmax(scale q k^T) v over the ring positions [max(0, p - window + 1), p], p = *pos_dev + t (keys in
 *   ascending position order, fixed reduction trees: bit-reproducible); q [B, T, H D] rows (the rotated q of b2a_ring_rope_kv).  D == 64,
 *   window <= 1024, cap >= window + T - 1 (a new row never overwrites a key some query of the call still sees), 16-byte aligned ring rows.
 *   Neither advances the counter. */
int32_t b2a_ring_rope_kv(float* qkv, int64_t qkv_bs, int64_t qkv_ld, int32_t B, int32_t T, int32_t H, int32_t D, float base,
                         float* k_ring, float* v_ring, int64_t ring_bs, int32_t cap, const int32_t* pos_dev, void* stream);
int32_t b2a_ring_attn(const float* q, int64_t q_bs, int64_t q_ld, const float* k_ring, const float* v_ring, int64_t ring_bs, int32_t cap,
                      float* out, int64_t o_bs, int64_t o_ld, int32_t B, int32_t T, int32_t H, int32_t D, float scale, int32_t window,
                      const int32_t* pos_dev, void* stream);
/* End of a streaming step: ctr[0] (ring position) += dpos, ctr[1] (history slot parity counter) += 1. */
int32_t b2a_stream_advance(int32_t* ctr, int32_t dpos, void* stream);

/* ---- Qwen3-TTS speaker encoder (ECAPA-TDNN, tts/models/qwen3_tts/speaker_encoder.py) and its log-mel front end -------------- */
/* qwen3_tts.py:64-121 (mel_spectrogram): reflect pad of (1024-256)/2 samples (no repeated edge), STFT (n_fft 1024, hop 256,
 * center=False, periodic Hann `window`), sqrt(|X|^2 + 1e-9) @ filters^T (Slaney mel, [n_mels, 513]), log(max(., 1e-5)).
 * x [B, n] (row stride x_bs), n > 384; out [B, frames, n_mels] contiguous with frames = 1 + (n + 768 - 1024) / 256. */
int32_t b2a_spk_logmel(const float* x, int64_t x_bs, int32_t B, int64_t n, const float* window, const float* filters, int32_t n_mels,
                       int64_t frames, float* out, void* stream);
/* speaker_encoder.py:11-26 (reflect_pad_1d) as the operand of the following conv, which then runs unpadded: x [B, T, C] ->
 * rows reflect(r - pad) for r in [0, T + 2 pad), either fp32 out_f32 [B, T+2pad, C] contiguous, or the tensor-core conv's bf16
 * planes hi / lo (lo may be NULL) [B, T+2pad, cpad] with zeroed pad channels.  Exactly one of out_f32 / hi; pad < T. */
int32_t b2a_spk_reflect_pad(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, int32_t pad, float* out_f32,
                            void* hi, void* lo, int32_t cpad, void* stream);
/* speaker_encoder.py:60-101 (Res2NetBlock, with the TimeDelayNetBlocks of :29-57): y [B, T, scale*C] -> z [B, T, scale*C]; chunk 0
 * copied, chunk i = relu(conv(reflect_pad(chunk_i + chunk_{i-1}' ))) for i >= 1 (chunk 1 without the add) -- the whole dependent chain
 * in one launch, one CTA per (item, `tile` rows), halo recomputed.  w [scale-1][K][C_in][C_out] fp32, bias [scale-1][C];
 * (K-1)*dilation even, pad = (K-1)*dilation/2 < T.  Shared memory per CTA: b2a_spk_res2net_smem_bytes (B2A_E_UNSUPPORTED > 227 KB). */
int64_t b2a_spk_res2net_smem_bytes(int32_t C, int32_t scale, int32_t K, int32_t pad, int32_t tile);
int32_t b2a_spk_res2net(const float* y, int64_t y_bs, int64_t y_ld, float* z, int64_t z_bs, int64_t z_ld, const float* w, const float* bias,
                        int32_t B, int32_t T, int32_t C, int32_t scale, int32_t K, int32_t dilation, int32_t tile, void* stream);
/* Per-channel mean over T (speaker_encoder.py:127, :191) and, with_std, sqrt(var + eps) (:192, biased var) of x [B, T, C]:
 * out[b*o_bs + c] = mean, out[b*o_bs + C + c] = std.  Fixed summation order (bit-reproducible). */
int32_t b2a_spk_channel_stats(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, int32_t with_std, float eps,
                              float* out, int64_t o_bs, void* stream);
/* speaker_encoder.py:124-133 after the mean: gate[b] = sigmoid(w2 relu(w1 mean[b] + b1) + b2); w1 [S, C], w2 [C, S]; gate [B, C]. */
int32_t b2a_spk_se_gate(const float* mean, int64_t m_bs, int32_t B, int32_t C, int32_t S, const float* w1, const float* b1, const float* w2,
                        const float* b2, float* gate, void* stream);
/* speaker_encoder.py:133,168: out = y * gate[b, c] + res (out may be a channel slice of the MFA concatenation, :293-295). */
int32_t b2a_spk_se_apply(const float* y, int64_t y_bs, int64_t y_ld, const float* gate, const float* res, int64_t r_bs, int64_t r_ld,
                         float* out, int64_t o_bs, int64_t o_ld, int32_t B, int32_t T, int32_t C, void* stream);
/* One row per item: y[b*y_bs + j] = act(bias[j] + w[j*w_ld : +K] . x[b*x_bs : +K]) (act: B2A_ACT_*; LRELU means ReLU).  The statistics
 * half of the pooling TDNN (:177,202) and the final 1x1 projection (:269-303). */
int32_t b2a_spk_gemv(const float* x, int64_t x_bs, int32_t B, int32_t K, const float* w, int64_t w_ld, int32_t N, const float* bias,
                     int32_t act, float* y, int64_t y_bs, void* stream);
/* speaker_encoder.py:202-203 with the TDNN split as W_x.x + (W_m.mean + W_s.std + b): h = tanh(relu(h + cb[b])) in place, h [B, T, A],
 * cb [B, A] contiguous. */
int32_t b2a_spk_asp_act(float* h, int64_t h_bs, int64_t h_ld, const float* cb, int32_t B, int32_t T, int32_t A, void* stream);
/* speaker_encoder.py:208-216: softmax over TIME of logits [B, T, C] per channel (max-subtracted), weighted mean of x [B, T, C] and
 * sqrt(max(weighted var, eps)) -> pooled[b*p_bs + c] = mean, pooled[b*p_bs + C + c] = std.  Fixed summation order. */
int32_t b2a_spk_asp_pool(const float* logits, int64_t l_bs, int64_t l_ld, const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T,
                         int32_t C, float eps, float* pooled, int64_t p_bs, void* stream);

/* ---- Vocos (vocos.cu; codec/models/vocos/vocos.py, mel.py, dsp.py:385-513) ---------------------------------------------------
 * ConvNeXtBlock's dwconv + norm (vocos.py:183-187), or with K == 0 VocosBackbone's norm / final_layer_norm (:263-274), in one pass:
 * x [B, L, C] fp32 (element (b, t, c) at b * x_bs + t * x_ld + c).  dw_w [K, C] + dw_b [C] (or NULL): a depthwise conv with zero "same"
 * padding K / 2, taps summed in ascending order; K odd <= 15, or 0 for no conv.  LayerNorm over C (eps from the caller, fp32 statistics
 * in a fixed order), then either w (or NULL) and b (or NULL: final_layer_norm with bias=False), or, when ada != NULL, AdaLayerNorm's
 * per-row scale v + shift (vocos.py:209-214) from ada[b * ada_bs + c] (scale) and ada[b * ada_bs + C + c] (shift).  Output fp32 y (row
 * stride y_ld, batch stride y_bs; may be NULL), and / or the next GEMM's bf16 planes hi / lo (lo may be NULL) [B, L, C] contiguous,
 * C % 64 == 0.  C % 4 == 0, C <= 1024, 16-byte aligned rows.  A batch row's result does not depend on B. */
int32_t b2a_vocos_dwnorm(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t C, const float* dw_w, const float* dw_b,
                         int32_t K, const float* w, const float* b, const float* ada, int64_t ada_bs, float eps, float* y, int64_t y_bs,
                         int64_t y_ld, void* hi, void* lo, void* stream);
/* ISTFTHead after its linear (vocos.py:126-140 with dsp.py:436-513): h [B, T, h_ld], h_ld >= n_fft + 2 (the linear's padded row), holds
 * log-magnitudes in columns [0, n_fft/2 + 1) and phases in the next n_fft/2 + 1.  S = min(exp(mag), 100) (cos p + i sin p); irfft per
 * frame (imaginary parts of the DC and Nyquist bins ignored), times the symmetric Hann `window` [n_fft], overlap-add at `hop`, divided by
 * the summed window where that sum is > 1e-10, n_fft / 2 trimmed at each end: out [B, (T - 1) hop] (batch stride out_bs).  Gathered per
 * output sample -- no workspace, no scatter; frames and bins summed in ascending order.  Even n_fft <= 2048 (1280 included), else
 * B2A_E_UNSUPPORTED. */
int32_t b2a_vocos_istft_head(const float* h, int64_t h_bs, int64_t h_ld, int32_t B, int32_t T, int32_t n_fft, int32_t hop, const float* window,
                             float* out, int64_t out_bs, void* stream);
/* mel.py:8-33 (log_mel_spectrogram) at n_fft 1024 / hop 256 on b2a_spk_logmel's kernel: reflect pad n_fft / 2 = 512 (no repeated edge),
 * symmetric Hann `window` [1024], |X| (no epsilon) @ filters^T (HTK, norm None, [n_mels, 513]), log(max(., 1e-5)); the stft's last frame
 * is dropped and never computed.  x [B, n] (row stride x_bs), n > 512; out [B, frames, n_mels] contiguous with frames = n / 256. */
int32_t b2a_vocos_logmel(const float* x, int64_t x_bs, int32_t B, int64_t n, const float* window, const float* filters, int32_t n_mels,
                         int64_t frames, float* out, void* stream);

/* ---- EnCodec (encodec.cu; codec/models/encodec/encodec.py) --------------------------------------------------------------------
 * One unidirectional LSTM layer (encodec.py:89-169) over xproj [R, T, 4H] contiguous (x Wx^T + bias, gates i, f, g, o), W_h [4H, H]
 * fp32; h0 = c0 = 0.  out [R, T, H] contiguous = h, plus skip [R, T, H] (or NULL) -- EncodecLSTM's residual on its last layer.  One
 * cluster of H / 32 CTAs per 4 rows (1 for R == 1); a row's result does not depend on R.  H in {128, 256, 512}, else B2A_E_UNSUPPORTED,
 * as is a device that cannot schedule the cluster.  `err` (uint32, zeroed by the caller) is set to 1 when a step waited more than 10 s
 * (that call's output is then invalid). */
int32_t b2a_encodec_lstm(const float* xproj, const float* wh, const float* skip, float* out, int32_t R, int32_t T, int32_t H, uint32_t* err,
                         void* stream);
/* The input side of EncodecConv1d (encodec.py:212-245): y [B, pad_left + T + pad_right, C] from x [B, T, C] (strides x_bs, x_ld; y_bs,
 * y_ld) with reflect (no repeated edge; pad_left, pad_right < T, else B2A_E_INVALID) or zero padding.  Each source value first gets
 * v * scale[b, C] + shift[b, C] (both or neither NULL: a GroupNorm applied from b2a_encodec_gn_coeffs) and then ELU when `elu`; zero
 * padding stays 0.  res (or NULL; strides res_bs, res_ld) is added afterwards and requires pad_left == pad_right == 0. */
int32_t b2a_encodec_pad(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, int32_t pad_left, int32_t pad_right,
                        int32_t reflect, const float* scale, const float* shift, int32_t elu, const float* res, int64_t res_bs, int64_t res_ld,
                        float* y, int64_t y_bs, int64_t y_ld, void* stream);
/* GroupNorm(1, C) (MLX, pytorch_compatible) of x [B, T, C]: mean and biased variance over T x C per row in float64 with a fixed order
 * (independent of B), folded with gamma / beta [C] (NULL: 1 / 0) into scale[b, c] = gamma rstd, shift[b, c] = beta - mean gamma rstd
 * ([B, C] contiguous).  ws: b2a_encodec_gn_ws_bytes(B) bytes of device memory.  Two launches. */
int64_t b2a_encodec_gn_ws_bytes(int32_t B);
int32_t b2a_encodec_gn_coeffs(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t T, int32_t C, const float* gamma,
                              const float* beta, float eps, float* scale, float* shift, void* ws, void* stream);
/* Encodec._encode_frame's normalisation (encodec.py:574-579) per chunk row r of x [R, L, C]: v = x * mask[r, t] (mask uint8 with row
 * stride mask_bs, or NULL), scale[r] = sqrt(mean_t(mean_c v)^2) + 1e-8 (float64 sums), y [R, L, C] contiguous = v / scale[r]. */
int32_t b2a_encodec_normalize(const float* x, int64_t x_bs, int64_t x_ld, int32_t R, int32_t L, int32_t C, const uint8_t* mask,
                              int64_t mask_bs, float* y, float* scale, void* stream);
/* Encodec._linear_overlap_add (encodec.py:654-677) of N chunk decodes frames [N, B, L, C] contiguous, each first multiplied by
 * scale[n * B + b] (or NULL), at `stride` <= L, with the triangular weight 0.5 - |(j + 1) / (L + 1) - 0.5|, divided by the summed
 * weights and truncated: out [B, Tout, C] contiguous, Tout <= stride (N - 1) + L.  Chunks summed in ascending order. */
int32_t b2a_encodec_ola(const float* frames, int32_t N, int32_t B, int32_t L, int32_t C, const float* scale, int32_t stride, int32_t Tout,
                        float* out, void* stream);

/* ---- Soprano TTS (soprano.cu; tts/models/soprano/soprano.py, decoder.py) ------------------------------------------------------
 * mlx-lm's make_sampler(temperature, top_p) (lm/sample_utils.py:11-70) as soprano.py:336-346 applies it, to RAW logits [B, V] (row
 * stride logits_bs), one CTA per row:
 *   temperature == 0: argmax, the first index on ties (soprano.py:343-344);
 *   0 < top_p < 1: apply_top_p (sample_utils.py:206-238) on the raw logits: a token is kept iff the inclusive cumulative sum of
 *     exp(logit) in ascending order (ties: lower index first) exceeds 1 - top_p.  exp is fp32 (an overflow to inf keeps every token from
 *     that rank up), the sums are float64 in a fixed order.  When nothing is kept (every logit -inf) the token is 0, MLX's categorical
 *     of an all -inf row;
 *   then categorical_sampling (:279): logits * float32(1 / temperature), drawn by the inverse CDF in index order of their softmax with
 *     u[b * u_bs + step] in [0, 1), step = *step_dev (0 when NULL).
 * Writes out[b] and hist[b * hist_bs + step] (hist may be NULL); a row whose token is stop0 or stop1 gets finished[b] = 1, and a row
 * with finished[b] set writes nothing (finished may be NULL).  A row's result does not depend on B.  Any V >= 1; rows of at most
 * 36 864 logits are staged in shared memory, longer ones are read from global memory on each of the 8 radix passes. */
int32_t b2a_lm_sample_mlx(const float* logits, int64_t logits_bs, int32_t B, int32_t V, float temperature, double top_p, const float* u,
                          int64_t u_bs, const int32_t* step_dev, int64_t* out, int64_t* hist, int64_t hist_bs, uint8_t* finished,
                          int32_t stop0, int32_t stop1, void* stream);
/* SopranoDecoder's up-sampling (decoder.py:102-112 with interpolate.py:61-117, mode "linear", align_corners=True): x [B, L, H] (strides
 * x_bs, x_ld) -> Lo = up (L - 1) + 1 rows, row i = x[lo] (1 - f) + x[hi] f in fp32 with pos = float(i) * float((L - 1) / (Lo - 1)),
 * lo = floor(pos), hi = min(lo + 1, L - 1), f = pos - lo (for up = 4: 0, .25, .5, .75); L = 1 broadcasts the row.  Output fp32 y (strides
 * y_bs, y_ld) or the bf16 hi / lo planes [B, Lo, cpad] of the next tensor-core conv (lo may be NULL; channels >= H are 0). */
int32_t b2a_soprano_upsample(const float* x, int64_t x_bs, int64_t x_ld, int32_t B, int32_t L, int32_t H, int32_t up, float* y, int64_t y_bs,
                             int64_t y_ld, void* hi, void* lo, int32_t cpad, void* stream);
/* dst[b * dst_bs + r * dst_ld + c] = src[b * src_bs + c] for c < H with r = *idx_dev + add: one hidden row per batch row stored at a
 * device-resident step index (rows outside [0, cap) are skipped). */
int32_t b2a_soprano_store_rows(const float* src, int64_t src_bs, int32_t B, int32_t H, float* dst, int64_t dst_bs, int64_t dst_ld,
                               const int32_t* idx_dev, int32_t add, int32_t cap, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200AUDIO_H */
