/* styletts2_b200 -- C ABI of the H100 (sm_90a) StyleTTS 2 inference hot path.
 *
 * The reference (yl4579/StyleTTS2) is pure Python/PyTorch and has no FFI: the calls this
 * library replaces are the ATen operator calls inside the reference's nn.Module.forward
 * methods.  Each entry point below cites the reference call site(s) it stands in for.
 * The Python host side (styletts2_b200/*.py) binds these with ctypes and keeps the
 * reference's module names, forward signatures and state-dict keys (INTEGRATION.md).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer to fp32 (or int32/int64 where said), owned by the
 *    caller; nothing is allocated or freed here; no hidden synchronisation;
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it;
 *  - activations are [B, C, L] with L contiguous ("conv layout") or row-major
 *    [rows, features] ("row layout"); batch strides are in ELEMENTS;
 *  - return value: 0 on success, else a cudaError_t value; st2_last_error() describes it.
 *  - there is NO CPU fallback: without a CUDA device every compute call fails.
 */
#ifndef STYLETTS2_B200_H
#define STYLETTS2_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define ST2_ABI_VERSION 2

/* activation codes (prologue / epilogue selectors) */
#define ST2_ACT_NONE 0
#define ST2_ACT_LRELU 1 /* F.leaky_relu(x, slope) */
#define ST2_ACT_SNAKE 2 /* x + sin(alpha x)^2 / alpha, alpha per channel */
#define ST2_ACT_TANH 3
#define ST2_ACT_GELU 4 /* exact erf GELU (nn.GELU default) */
#define ST2_ACT_GELU_TANH 5 /* "gelu_new" tanh approximation (transformers AlbertConfig.hidden_act, PL-BERT) */

const char* st2_last_error(void);
int st2_abi_version(void);
/* number of kernels launched by this library since load (bench.py "gpu_launches") */
long long st2_launch_count(void);

/* ------------------------------------------------------------------ weight preparation
 * torch.nn.utils.weight_norm (dim=0): w[r,:] = v[r,:] * g[r] / ||v[r,:]||_2
 * (re-evaluated every forward by the reference: Modules/istftnet.py:30-46, models.py:293;
 * here folded once at load). */
int st2_weight_norm_fold(const float* v, const float* g, float* w, int rows, int cols, void* stream);
/* out[r] = ||v[r,:]||_2 with the fold kernel's own reduction: a folded weight w re-imported as (weight_v = w,
 * weight_g = st2_row_norm(w)) folds back to exactly w (checkpoint export of folded weights, styletts2_b200/checkpoint.py) */
int st2_row_norm(const float* v, float* out, int rows, int cols, void* stream);
/* Conv1d weight [Cout,Cin,K] -> kernel layout [Cin][K][Cout] */
int st2_conv_weight_layout(const float* w, float* wt, int Cout, int Cin, int K, void* stream);
/* ConvTranspose1d weight [Cin,Cout,K] (stride S, padding P) -> polyphase layout
 * [S][Cin][J][Cout], J = ceil(K/S): phase r is a J-tap stride-1 conv (see st2_conv_transpose1d). */
int st2_convT_weight_layout(const float* w, float* wp, int Cin, int Cout, int K, int S, int P, void* stream);

/* ------------------------------------------------------------------ fused Conv1d
 * y[b,co,oidx(q)] = epi( bias[co] + sum_{ci,k} W[co,ci,k] * pre(x[b,ci, q*stride + k*dil - pad]) )
 *   pre(v) = act_pre(a[b,ci]*v + b[b,ci])  (AdaIN affine, then LeakyReLU / Snake); zero outside [0,Lin)
 *   epi(v) = act_out( accum( (v + res[b,co, oidx >> res_shift]) / out_div ) )
 * and optionally per-(b,co) partial statistics (count, mean, M2) of the stored values for the
 * NEXT InstanceNorm (fixed-order, deterministic; merged by st2_adain_coef).
 * Replaces: F.conv1d call sites of Modules/istftnet.py:70,73,361,377,445-448,511-517,
 * Modules/hifigan.py:69-72,330,344, models.py:293,390-395,506-510 together with the
 * AdaIN1d / Snake / LeakyReLU / residual / MRF-mean elementwise ops around them. */
typedef struct st2_conv_args {
  const float* x;         /* [B, Cin, Lin] */
  long long x_bstride;    /* elements between utterances */
  int Cin, Lin;
  const float* w;         /* [Cin][K][Cout] (st2_conv_weight_layout) */
  const float* bias;      /* [Cout] or NULL */
  float* y;               /* rows of length y_len */
  long long y_bstride;
  int Cout;
  int Lq;                 /* number of output positions q computed */
  int y_len;              /* row length of y */
  int y_tstride, y_toffset; /* oidx = q*y_tstride + y_toffset */
  int B, K, stride, dil, pad;
  const float* pre_a;     /* [B,Cin] or NULL (no affine) */
  const float* pre_b;
  int pre_act;            /* ST2_ACT_NONE / LRELU / SNAKE */
  float pre_slope;
  const float* pre_alpha; /* [Cin] for SNAKE */
  const float* res;       /* residual rows of length res_len, or NULL */
  long long res_bstride;
  int res_len, res_shift;
  float out_div;          /* 1.0 if unused; (res+sc)/sqrt(2) of AdainResBlk1d (models.py:415) */
  int accum_mode;         /* 0: y=v   1: y+=v   2: y=(y+v)/accum_div  (MRF mean, istftnet.py:369-375) */
  float accum_div;
  int out_act;            /* ST2_ACT_NONE / ST2_ACT_TANH */
  float* stats;           /* [B,Cout,stats_nparts,3] or NULL */
  int stats_nparts, stats_part_offset;
  int dup_q0_to;          /* >=0: the q==0 value is also stored at that index (reflection pad, istftnet.py:366) */
} st2_conv_args;
int st2_conv1d(const st2_conv_args* a, void* stream);
/* number of stats partials st2_conv1d writes for Lq outputs */
int st2_conv_stats_parts(int Lq);

/* Tensor-core path of the same fused Conv1d (stride 1): wgmma implicit GEMM with register accumulators,
 * operands split into planes so that 16-bit / 8-bit tensor-core products reproduce the fp32 convolution (fp32
 * accumulate), weights streamed by 1-D TMA bulk copies.  `mode` selects the precision recipe (csrc/conv_tc.cu):
 *   ST2_TC_FAST      fp16 high planes + ONE e4m3 K=32 MMA carrying both correction terms: 2 MMA-times per product,
 *                    error ~2^-16 per product (vocoder / decoder convolutions; waveform bar 1e-3);
 *   ST2_TC_ACCURATE  two fp16 planes per operand, 3 MMAs, separate accumulator for the correction terms: error at
 *                    the fp32-SIMT level (F0 / N predictor: F0 is integrated into a phase of 1e4..1e6 rad downstream);
 *   ST2_TC_F16X3     the accurate planes in a single accumulator (A/B testing).
 * `wtc` is the st2_conv_tc_weight_layout buffer (st2_conv_tc_weight_bytes bytes) built from the folded fp32 weight
 * [Cout,Cin,K] FOR THE SAME mode.  a->w is ignored; every other field means what it means for st2_conv1d,
 * except that the output positions must be contiguous (y_tstride == 1, y_toffset == 0), there is no reflection
 * duplicate (dup_q0_to < 0), and it writes ONE statistics partial per 64-column tile (stats_nparts >= offset + ceil(Lq/64)).
 * x must live in an allocation whose first byte is 16-byte aligned (cudaMalloc / the PyTorch caching allocator):
 * rows are fetched as 16-byte copies of their aligned superset window.  Operand range: |z| < 1000 after the
 * prologue, |w| < 16 (fp16 planes of 64 z and 4096 w); larger values give inf/NaN loudly.
 * max_ctas > 0 caps the persistent grid (testing).  Same call sites as st2_conv1d. */
#define ST2_TC_FAST 0
#define ST2_TC_ACCURATE 1
#define ST2_TC_F16X3 2
/* Flag OR-ed into `mode` (FAST recipe, Cout <= 128): TIME-MAJOR weight layout and kernel -- frames on the MMA's M axis
 * (each of the two consumer warpgroups takes 64 frames of a 128-frame tile), output channels on N = Cout rounded up to 32
 * (16 for Cout <= 16): no tensor-pipe time or weight traffic for absent channels.  One fp16 and one e4m3 accumulator per
 * warpgroup; the epilogue computes the output values through a shared-memory slot, group by group, and reduces the
 * InstanceNorm partials over the warpgroup's four warps in shared memory.  Layout and launch must use the same mode value.
 * (Cout = 256 as two channel blocks was measured: no gain over the channel-major kernel and 3-16 % slower narrow layers
 * from the extra tile decode -- not kept.) */
#define ST2_TC_TMAJOR 16
long long st2_conv_tc_weight_bytes(int Cout, int Cin, int K);
int st2_conv_tc_weight_layout(const float* w, void* out, int Cout, int Cin, int K, int mode, void* stream);
int st2_conv_tc_supported(int Cin, int Cout, int K, int stride, int dil);
int st2_conv1d_tc(const st2_conv_args* a, const void* wtc, int mode, int max_ctas, void* stream);
/* Timing experiments only (tools/conv_tc_shapes.py --ablate), tensor-core convs: 4 stagers skip the conversion,
 * 16 no weight copies, 32 no raw activation copies.  Results are wrong while any bit is set; 0 restores. */
int st2_debug_set_flags(int flags);
/* Polyphase ConvTranspose1d on the same tensor-core kernels (one launch per phase); wtc from
 * st2_convT_tc_weight_layout (st2_convT_tc_weight_bytes bytes, an upper bound for every mode).  Arguments as
 * st2_conv_transpose1d, with y rows contiguous (a->y_len = Lin*S (+1)): the S phase convolutions store contiguous rows
 * into `tmp` (S*B*Cout*Lin floats, caller-owned), then one memory-bound kernel interleaves the phases into y, adds the
 * residual (a->res), applies the reflection duplicate and writes ONE statistics record per (b, co) (a->stats
 * [B,Cout,1,3], stats_nparts == 1). */
long long st2_convT_tc_weight_bytes(int Cin, int Cout, int K, int S);
int st2_convT_tc_weight_layout(const float* w, void* out, int Cin, int Cout, int K, int S, int P, int mode, void* stream);
int st2_conv_transpose1d_tc2(const st2_conv_args* a, const void* wtc, int mode, int K, int S, int P, int reflect_left1, float* tmp,
                             void* stream);

/* ConvTranspose1d (stride S, K taps, padding P; output length Lin*S) as S polyphase
 * stride-1 convolutions through the same fused kernel; `a` describes the x / y / prologue /
 * epilogue exactly as for st2_conv1d with K,stride,dil,pad,Lq,y_tstride,y_toffset,w ignored;
 * wp is the st2_convT_weight_layout buffer.  reflect_left1 != 0 implements
 * ReflectionPad1d((1,0)) on the output (istftnet.py:365-366): y has Lin*S+1 columns.
 * stats needs room for S*st2_conv_stats_parts(Lin) partials.
 * Replaces: Generator.ups[i] (istftnet.py:364, hifigan.py:333). */
int st2_conv_transpose1d(const st2_conv_args* a, const float* wp, int K, int S, int P, int reflect_left1, void* stream);

/* ------------------------------------------------------------------ InstanceNorm / AdaIN
 * per-(b,c) (count, mean, M2) over L for a tensor not produced by st2_conv1d. */
int st2_instance_stats(const float* x, long long bstride, int B, int C, int L, float* stats, void* stream);
/* AdaIN1d coefficients (Modules/istftnet.py:15-25, models.py:349-359): merges the partials
 * (Chan, fp64), biased variance, eps; a=(1+gamma)*rstd, b=beta-mean*a with gamma=gb[b, c],
 * beta=gb[b, C+c] (gb row stride gb_stride). */
int st2_adain_coef(const float* stats, int nparts, const float* gb, long long gb_stride, int B, int C,
                   float eps, float* a, float* b, void* stream);
/* residual path of an upsampling AdainResBlk1d (models.py:404-407): y[b,c,:2L] =
 * depthwise ConvTranspose1d(k3,s2,p1,op1)(lrelu_0.2(a*x+b)) with weight pw[C,3], bias pb[C]. */
int st2_adain_lrelu_pool(const float* x, long long x_bstride, const float* a, const float* b, const float* pw,
                         const float* pb, float slope, int B, int C, int L, float* y, long long y_bstride, void* stream);
/* TextEncoder block tail (models.py:270-282,295-296,310): LayerNorm over CHANNELS of a
 * [B,C,L] tensor, LeakyReLU(slope), zero where t >= lengths[b] (lengths may be NULL). in place ok. */
int st2_channel_layernorm_lrelu(const float* x, float* y, const float* gamma, const float* beta, float eps,
                                float slope, const int* lengths, int B, int C, int L, void* stream);

/* ------------------------------------------------------------------ row-layout ops (denoiser, duration encoder)
 * For each row r=(b,n), width C:
 *   h = (h_in ? h_in[r,:] : [xs * x[b,0:Cx] | emb[r,0:C-Cx]]) + (add ? add[b,:] : 0);  h_out[r,:] = h (if h_out)
 *   z = LayerNorm(h) (eps);  out1 = z*(g1 (+1 if ada)) + b1;  out2 likewise (if out2)
 *   g/b are [C] vectors (gb_bstride==0) or per-utterance rows (gb_bstride = row stride).
 * Replaces: modules.py:392-397 (x cat/expand, x+mapping), 556-557 (norm, norm_context),
 * 18-38 (AdaLayerNorm), models.py:418-438. */
typedef struct st2_rows_args {
  const float* h_in; long long h_in_ld;
  const float* x; int Cx; float xs; const float* emb; long long emb_ld;
  const float* add;       /* [B,C] or NULL */
  float* h_out; long long h_out_ld;
  const float* g1; const float* b1; const float* g2; const float* b2; long long gb_bstride; int ada;
  float* out1; long long out1_ld; float* out2; long long out2_ld;
  int B, N, C; float eps;
  const int* lengths;     /* rows n >= lengths[b] are written as zeros (masked_fill), may be NULL */
} st2_rows_args;
int st2_rows_ln(const st2_rows_args* a, void* stream);
/* The same per-row work over M packed token rows (only the valid rows of every utterance, concatenated): the utterance of
 * row r is row_utt[r] (int32 [M]), which selects x, add and the per-utterance g/b rows; a->N and a->lengths are unused. */
int st2_rows_ln_packed(const st2_rows_args* a, const int* row_utt, int M, void* stream);
/* dst[(b,n), col0 + j] = (n < lengths[b]) ? src[b, j] : 0   (style concat, models.py:539-541,551-552) */
int st2_bcast_cols(float* dst, long long ld, int col0, const float* src, int B, int N, int W, const int* lengths, void* stream);
/* out[b,:] = mean_n h[(b,n),:]  (modules.py:399) */
int st2_mean_rows(const float* h, long long ld, int B, int N, int C, float* out, void* stream);
/* out[b,:] = mean of rows offsets[b] .. offsets[b+1]-1 of h (packed rows, offsets int32 [B+1], every segment non-empty);
 * the summation order of st2_mean_rows, so equal segments give identical bits. */
int st2_mean_segments(const float* h, long long ld, const int* offsets, int B, int C, float* out, void* stream);

/* C[M,Nf] = act(A W^T + bias) + R.  A element (m,k): A + (m / a_L)*a_bs + (m % a_L)*a_ls + k*a_ks
 * (row layout: a_L=M, a_ls=K, a_ks=1; conv layout [B,K,L]: a_L=L, a_bs=K*L, a_ls=1, a_ks=L).
 * W is [Nf,K] row-major (torch Linear / conv1x1 weight).  Replaces every nn.Linear on the path
 * (modules.py:256-261,484-490,521,333-338; models.py:674,451; LSTM input projections). */
int st2_linear(const float* A, long long a_bs, long long a_ls, long long a_ks, int a_L, const float* W,
               const float* bias, const float* R, long long ldr, float* C, long long ldc, int M, int Nf, int K,
               int act, void* stream);

/* Tensor-core path of st2_linear for row-layout inputs (A element (m,k) at A + m*lda + k): wgmma GEMM with register
 * accumulators at fp32 accuracy -- operands split into three bf16 planes, six MMAs per product (the integer duration
 * boundary is downstream of the denoiser).  wtc from st2_linear_tc_weight_layout (st2_linear_tc_weight_bytes bytes),
 * built from the fp32 weight [Nf,K].  Same call sites as st2_linear. */
long long st2_linear_tc_weight_bytes(int Nf, int K);
int st2_linear_tc_weight_layout(const float* w, void* out, int Nf, int K, void* stream);
int st2_linear_tc(const float* A, long long lda, const void* wtc, const float* bias, const float* R, long long ldr, float* C,
                  long long ldc, int M, int Nf, int K, int act, void* stream);
/* Same GEMM with the activation operand pre-split ONCE into fp16 (high, low*2^11) operand stages by st2_linear_tc_split
 * (st2_linear_tc_split_bytes bytes): both operands then reach shared memory by 1-D TMA bulk copies and no warp spends
 * issue slots on conversion (the on-the-fly path re-splits the same rows once per 128-feature output block).
 * planes == NULL falls back to on-the-fly splitting of A. */
/* Range guard of the fp16-plane GEMM, attention and tensor-core convs: *flag_out = 1 if any operand split since the last
 * call left fp16's range or was NaN -- GEMM activations / weights and attention q / k / v with |x| >= 65504, conv operands
 * after their power-of-two scales (|z| >= 65504 / 64 after the prologue, |w| >= 65504 / 4096) -- the result of that GEMM /
 * attention / conv is then inf/NaN, not silently wrong; all flags are cleared.  Synchronises with the device (call it
 * after a pass, outside CUDA-graph capture). */
int st2_range_flag_fetch(int* flag_out);
long long st2_linear_tc_split_bytes(int M, int K);
int st2_linear_tc_split(const float* A, long long lda, int M, int K, void* planes, void* stream);
int st2_linear_tc_pre(const float* A, long long lda, const void* planes, const void* wtc, const float* bias, const float* R,
                      long long ldr, float* C, long long ldc, int M, int Nf, int K, int act, void* stream);

/* Multi-head attention without mask (modules.py:523-535): q [B*N, H*D], kv [B*N, 2*H*D]
 * (k | v), out [B*N, H*D]; softmax(q k^T * scale) v per (b,h). D must be 64. */
int st2_attention(const float* q, const float* kv, float* out, int B, int N, int H, int D, float scale, void* stream);
/* General form: q rows at q + m*q_ld, k / v rows at k|v + m*kv_ld, out rows at out + m*out_ld (head h in columns
 * h*D..); lengths (int32 [B]) or NULL = key-padding mask (keys n >= lengths[b] excluded), as the additive -inf
 * attention mask of transformers.AlbertModel (PL-BERT, Utils/PLBERT/util.py:6-12). */
int st2_attention_ex(const float* q, long long q_ld, const float* k, const float* v, long long kv_ld, float* out, long long out_ld,
                     const int* lengths, int B, int N, int H, int D, float scale, void* stream);
/* The same contraction on the tensor cores (wgmma, register accumulators for S and O, fp16 two-plane split with separate
 * correction accumulators = fp32 accuracy; csrc/attention_tc.cu): one CTA per (64 query rows, head, utterance), keys in
 * blocks of 128.  Needs D == 64, row strides that are multiples of 4 floats and 16-byte aligned pointers
 * (st2_attention_tc_supported); arguments as st2_attention_ex.  Every length must be >= 1: a row with no valid key has
 * a zero softmax sum and a non-finite output, here and in st2_attention_ex.  q / k / v values that reach the fp16 planes
 * (valid keys, query rows < N) raise the range flag of st2_range_flag_fetch when |x| >= 65504 or NaN. */
int st2_attention_tc_supported(long long q_ld, long long kv_ld, long long out_ld, int D);
int st2_attention_tc(const float* q, long long q_ld, const float* k, const float* v, long long kv_ld, float* out, long long out_ld,
                     const int* lengths, int B, int N, int H, int D, float scale, void* stream);
/* The same kernel on packed rows: utterance b owns rows offsets[b] .. offsets[b+1]-1 of q, k, v and out (offsets int32
 * [B+1], every n_b = offsets[b+1] - offsets[b] >= 1, max_len >= every n_b).  Attention stays inside each utterance's rows;
 * rows of other utterances are neither read as keys nor written.  Grid (ceil(max_len/64), H, B).  With offsets[b] = b*N it
 * computes the bits of st2_attention_tc(lengths = NULL).  The range flag sees valid rows and keys only. */
int st2_attention_tc_packed(const float* q, long long q_ld, const float* k, const float* v, long long kv_ld, float* out,
                            long long out_ld, const int* offsets, int B, int max_len, int H, int D, float scale, void* stream);
/* ALBERT embeddings: out[(b,n), :] = word[tokens[b,n]] + pos[n] + type0   (E columns) */
int st2_embedding_sum_rows(const long long* tokens, const float* word, const float* pos, const float* type0, int B, int N, int E,
                           float* out, void* stream);

/* Bidirectional single-layer LSTM recurrence (models.py:300,450,453,523; gate order i,f,g,o).
 * gx [B*L, 8H] = x W_ih^T + b_ih + b_hh for (fwd | bwd); whh [2][4H][H]; out element
 * (b,t,dir*H+j) at out + b*o_bs + t*o_ts + (dir*H+j)*o_cs.  lengths (int32 [B]) or NULL gives
 * pack_padded_sequence semantics (backward pass starts at lengths[b]-1; padded steps = 0).
 * work: >= 6*B*H + 64 floats of scratch.
 * H == 256 (every LSTM of the reference configs) runs on 8-CTA clusters with DSMEM exchange; st2_debug_lstm_cluster(0)
 * forces the cooperative-launch kernel used for other sizes (testing). */
int st2_debug_lstm_cluster(int enable);
/* Profiling aid: device buffer of 8 int64 <- per-phase cycle sums of CTA 0 / thread 0 of the
 * cluster LSTM kernel {wait, fma, reduce, gates, push, steps}; NULL disables. */
int st2_debug_lstm_trace(void* buf);
int st2_lstm_bidir(const float* gx, const float* whh, float* out, long long o_bs, long long o_ts, long long o_cs,
                   const int* lengths, int B, int L, int H, float* work, void* stream);

/* ------------------------------------------------------------------ sampler (sampler.py:193-208,497-510)
 * d = (x_eval - (c_skip*x_eval + c_out*x_pred)) / sigma_eval;  out = x_base + d*dt (+ eps*sigma_up).
 * If x_pred_masked != NULL: x_pred := masked + (x_pred - masked)*cfg_scale first (modules.py:420-423). */
int st2_kdiff_step(const float* x_eval, const float* x_pred, const float* x_pred_masked, float cfg_scale,
                   float c_skip, float c_out, float sigma_eval, const float* x_base, float dt, const float* eps,
                   float sigma_up, float* out, int n, void* stream);
/* out = a*x (c_in scaling, sampler.py:205) */
int st2_scale(const float* x, float a, float* out, int n, void* stream);
/* LearnedPositionalEmbedding (modules.py:657-671): out[b,:] = [t, sin(2 pi w t), cos(2 pi w t)], w [half] */
int st2_time_embedding(const float* t /* [B] */, const float* w, int half, int B, float* out, long long ld, void* stream);
/* out = a*x + b*y (style blending alpha/beta, Inference_LibriTTS.ipynb#cell16) */
int st2_axpby(const float* x, float a, const float* y, float b, float* out, int n, void* stream);

/* ------------------------------------------------------------------ text / duration glue
 * out[b,c,n] = (n < lengths[b]) ? table[tokens[b,n], c] : 0   (models.py:303-306) */
int st2_embedding_cl(const long long* tokens, const float* table, const int* lengths, int B, int N, int C, float* out, void* stream);
/* pred_dur[b,n] = max(1, rint(sum_j sigmoid(logits[b,n,j]))) (+last_plus on the last REAL token n==lengths[b]-1)
 * -- integer boundary (Inference_LJSpeech.ipynb#cell17: `pred_dur[-1] += 5`; cell 29 / LibriTTS cell 16: no increment).
 * lengths [B] int32 or NULL (= N): padded tokens n >= lengths[b] get duration 0 (they emit no frames, as when the
 * reference runs the utterance alone).  dur_f (optional) receives the pre-rounding sums. */
int st2_durations(const float* logits, int B, int N, int J, int last_plus, const int* lengths, int* pred_dur, float* dur_f,
                  void* stream);
/* frame -> token map from durations: tok[b,t] for t < T (T = row length), exclusive scan per utterance;
 * frames beyond sum(dur[b]) map to the last token.  total[b] = sum(dur[b]). */
int st2_frame_tokens(const int* dur, int B, int N, int T, int shift_right, int* tok, int* total, void* stream);
/* Polyphase view of a conv input for STRIDED convolutions (noise_convs of the generators, istftnet.py:334-343 /
 * hifigan.py:298-302: kernel 2*stride, stride S): xp[b, c*S + r, q] = x[b, c, q*S + r - pad], q < Lp (zero outside).
 * conv1d(x, w, stride=S, padding=pad) with K = J*S taps == conv1d(xp[..., :Lout + J - 1], wp, stride=1, padding=0) with
 * wp[co, c*S + r, j] = w[co, c, j*S + r]: the strided conv then runs on the tensor-core kernel. */
int st2_polyphase_gather(const float* x, long long x_bstride, int B, int C, int L, int S, int pad, int Lp, float* xp, void* stream);
/* alignment expansion (d^T @ aln, t_en @ aln; #cell17) as a gather:
 *  rows: out[(b,t), c] = src[(b,tok[b,t]), c]      src row layout [B*N, C] (ld)
 *  cl  : out[b,c,t]    = src[b,c,tok[b,t]]         src conv layout [B,C,N] */
int st2_expand_rows(const float* src, long long src_ld, const int* tok, int B, int N, int T, int C, float* out, long long out_ld, void* stream);
int st2_expand_cl(const float* src, const int* tok, int B, int C, int N, int T, float* out, long long out_bstride, void* stream);

/* ------------------------------------------------------------------ harmonic source + (i)STFT
 * SineGen + SourceModuleHnNSF (istftnet.py:146-247,283-297 == hifigan.py:117-218,254-268):
 * f0 [B,F] (F = 2T frames), nearest-upsampled by `scale`; 9 harmonics; fp64 phase accumulation as
 * torch.cumsum on CPU; linear interpolation with PyTorch's align_corners=False rule;
 * uv = f0 > 10; noise [B, F*scale, 9] = the randn_like draw (istftnet.py:242) injected (parity mode), or NULL:
 * the kernel draws it in place with Philox4x32-10 + Box-Muller from (seed, offset) (throughput mode);
 * lin_w [9], lin_b [1] = m_source.l_linear; out [B, F*scale] = tanh(linear(.)). */
int st2_sine_source(const float* f0, int B, int F, int scale, const float* noise, const float* lin_w,
                    const float* lin_b, float* out, float* phase_work /* B*9*F floats */, unsigned long long seed,
                    unsigned long long offset, const unsigned long long* epoch /* device, nullable */, void* stream);
/* out[0..n) ~ N(0,1): Philox4x32-10 counter RNG + Box-Muller, stream (seed, offset) -- stands in for torch.randn_like on
 * the path (sampler.py:509) in throughput mode. */
int st2_randn(float* out, long long n, unsigned long long seed, unsigned long long offset,
              const unsigned long long* epoch /* device, nullable */, void* stream);
/* *epoch += 1 on the stream: the draw counter's upper words live in device memory so that a captured CUDA graph
 * produces fresh noise at every replay. */
int st2_rng_advance(unsigned long long* epoch, void* stream);
/* TorchSTFT.transform (istftnet.py:91-97): n_fft 20, hop 5, hann, center/reflect.
 * x [B,L] -> har [B,22,L/5+1] = [|X| ; angle X]. */
int st2_stft20(const float* x, int B, int L, float* har, void* stream);
/* conv_post tail + TorchSTFT.inverse (istftnet.py:378-380,99-104): x [B,22,Fr] ->
 * spec=exp(x[:11]), phase=sin(x[11:]) -> istft (n_fft 20, hop 5) -> wav [B, 5*(Fr-1)]. */
int st2_istft20_expsin(const float* x, int B, int Fr, float* wav, void* stream);
/* Wire format after the path (SURVEY section 8 f4; the notebooks hand the fp32 array to IPython.display.Audio /
 * soundfile): out[i] = saturate_int16(rint(wav[i] * 32767 * gain)), round half to even. */
int st2_pcm16(const float* wav, long long n, float gain, short* out, void* stream);

/* ------------------------------------------------------------------ reference-style path (SURVEY section 8 row f2)
 * compute_style (Demo/Inference_LibriTTS.ipynb cell 5): wave -> log-mel -> StyleEncoder x2 (models.py:139-164).
 *
 * spectral_norm(nn.Conv2d) in eval mode (models.py:36-38,109-114,142,152): sigma = u . (W_mat v) with the stored
 * power-iteration vectors; wt[(ci*KH*KW + k) * Cout + co] = weight_orig[co][ci][k] / sigma  (n = Cin/groups*KH*KW).
 * sigma_work: 1 float of device scratch (receives sigma). */
int st2_spectral_norm_fold(const float* weight_orig, const float* u, const float* v, int Cout, int n, float* wt,
                           float* sigma_work, void* stream);
/* Dense stride-1 Conv2d with the ResBlk elementwise ops fused (models.py:116-137):
 * out = (conv2d(pre(x)) + bias [+ res]) * out_scale, pre = LeakyReLU(slope) when pre_act != 0.
 * x [B,Cin,H,W]; wt from st2_spectral_norm_fold ([Cin*KH*KW][Cout]); out/res [B,Cout,Ho,Wo] with
 * Ho = H + 2*pad - KH + 1.  KHxKW in {1x1, 3x3, 5x5}. */
typedef struct st2_conv2d_args {
  const float* x;
  const float* wt;
  const float* bias;   /* [Cout] or NULL (conv1x1 has none, models.py:114) */
  const float* res;    /* or NULL */
  float* out;
  int B, Cin, H, W, Cout, KH, KW, pad;
  int pre_act;
  float slope;
  float out_scale;     /* 1/sqrt(2) for the ResBlk merge (models.py:137), else 1 */
} st2_conv2d_args;
int st2_conv2d(const st2_conv2d_args* a, void* stream);
/* LearnedDownSample('half') (models.py:37-38): depthwise 3x3, stride 2, padding 1; w = st2_spectral_norm_fold output
 * for weight_orig [C,1,3,3] (layout [9][C]); out [B,C,(H-1)/2+1,(W-1)/2+1]. */
int st2_dwconv3x3_s2(const float* x, const float* w, const float* bias, float* out, int B, int C, int H, int W, void* stream);
/* DownSample('half') (models.py:73-78): x [BC,H,W] -> [BC, H/2, (W+1)/2]; an odd W repeats its last column first. */
int st2_avgpool_half(const float* x, float* out, int BC, int H, int W, void* stream);
/* AdaptiveAvgPool2d(1) + LeakyReLU (models.py:153-154): x [rows, hw] -> out [rows]. */
int st2_mean_hw_lrelu(const float* x, float* out, int rows, int hw, float slope, void* stream);
/* torchaudio MelSpectrogram(n_fft 2048, win 1200, hop 300) framing: frames[(b*F+f), m] = wave[b, reflect(f*hop - win/2 + m)] * window[m],
 * F = 1 + L/hop (center=True, reflect padding, window centred in the n_fft frame).  The DFT and the HTK filterbank are two
 * st2_linear GEMMs; st2_mel_power squares the [re | im] halves in between; st2_logmel finishes with
 * out[b,m,f] = (log(eps + mel) - mean) / std  (preprocess(), notebook cell 5). */
int st2_mel_frames(const float* wave, const float* window, int B, int L, int win, int hop, int n_fft, float* frames, void* stream);
int st2_mel_power(const float* y /* [rows, 2*nf] */, int rows, int nf, float* p /* [rows, nf] */, void* stream);
int st2_logmel(const float* mel /* [B*F, M] */, int B, int F, int M, float eps, float mean, float stdv, float* out /* [B,M,F] */,
               void* stream);

#ifdef __cplusplus
}
#endif
#endif
