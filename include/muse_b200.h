/* muse_b200.h - C ABI of libmuse_b200.so: the H100 (sm_90a) hot path of huggingface/open-muse.
 *
 * The reference (pure PyTorch, no FFI of its own) reaches the device through torch ops; each
 * entry point below replaces the torch call(s) cited next to it (paths relative to the reference
 * repo).  All functions:
 *   - take raw device pointers + sizes + a cudaStream_t (passed as void*), never torch types;
 *   - enqueue work on that stream and return immediately (asynchronous, like the torch ops);
 *   - allocate nothing: scratch and outputs are caller-provided;
 *   - return 0 (MUSE_OK) or a non-zero status; muse_last_error() gives the message (thread-local).
 * Dtype codes: 0 = float32, 1 = bfloat16.  "bf16" pointers are 16-bit bfloat16 arrays.
 */
#ifndef MUSE_B200_H_
#define MUSE_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define MUSE_OK 0
#define MUSE_ERR_INVALID 1
#define MUSE_ERR_CUDA 2
#define MUSE_ERR_UNSUPPORTED 3

#define MUSE_B200_ABI_VERSION 3

/* library / device plumbing */
int muse_abi_version(void);
const char* muse_last_error(void);
int muse_set_device(int device);            /* cudaSetDevice for this library's runtime instance */
int muse_device_info(int* sm_major, int* sm_minor, int* num_sms);

/* Data-parallel training: leave `n` SMs free for the collective (NCCL) kernels that run concurrently with backward.  The
 * persistent GEMM kernels then launch (SM count - n) CTAs, so a CTA never has to wait for an SM an all-reduce CTA is
 * holding (with a static tile assignment such a late CTA would delay the whole GEMM by its full duration).  n = 0 restores
 * the full grid.  Process-wide, set once after init (the reference reaches this path through accelerate / DDP,
 * training/train_maskgit_imagenet.py:305). */
int muse_reserve_sms(int n);

/* Programmatic dependent launch.  The reference's step is a chain of several hundred short torch kernels on one stream
 * (muse/modeling_transformer.py:875-904 per layer, :1397-1454 per decode step); here every kernel of the library opens
 * with griddepcontrol.launch_dependents / griddepcontrol.wait, and with this switch on each launch carries
 * cudaLaunchAttributeProgrammaticStreamSerialization, so a kernel's CTAs are scheduled and run their prologue while the
 * tail of the previous grid drains (memory effects stay in stream order: the wait precedes every global access).
 * Applies to eager launches and, through stream capture, to the CUDA graphs of the train step and the decode loop.
 * Process-wide; set it before capturing graphs.  Initial value: environment variable MUSE_B200_PDL if set, else the
 * build default MUSE_B200_PDL_DEFAULT. */
#define MUSE_B200_PDL_DEFAULT 0
int muse_set_pdl(int enabled);
int muse_get_pdl(void);

/* GEMM epilogues */
#define MUSE_EPI_BF16 0        /* C bf16 = acc                                   */
#define MUSE_EPI_F32 1         /* C fp32 = acc                                   */
#define MUSE_EPI_ATOMIC_F32 2  /* C fp32 += acc (split-K; weight gradients)      */
#define MUSE_EPI_RESADD_F32 3  /* C fp32 = res fp32 + bf16(acc) (residual add)   */
#define MUSE_EPI_SPLITK_F32 4  /* C fp32 = acc, deterministic split-K (muse_gemm_bf16_splitk only) */

/* C[M,N] = opA(A) * opB(B)^T, bf16 inputs, fp32 accumulation.
 *   a_mn == 0: A is row-major [M,K] (pitch lda); a_mn == 1: A is row-major [K,M].
 *   b_mn == 0: B is row-major [N,K] (pitch ldb); b_mn == 1: B is row-major [K,N].
 * Replaces every nn.Linear forward (muse/modeling_transformer.py:198-200,218,789-798,980,984) and,
 * through the a_mn/b_mn views, their autograd dgrad / wgrad matmuls. */
int muse_gemm_bf16(const void* A, const void* B, void* C, const float* res, int M, int N, int K, int lda, int ldb,
                   int ldc, int a_mn, int b_mn, int epilogue, void* stream);

/* Weight-gradient GEMM with a run-to-run reproducible result: C fp32 [M,N] = opA(A) * opB(B)^T split over K (= tokens) so
 * that the few output tiles fill the SMs; every split stores its partial tile into `ws` and a second kernel sums the
 * partials in split order and stores C (no zero fill of C needed, no atomics on C).  One ws per stream.  Replaces the autograd weight-gradient matmuls of every nn.Linear (muse/modeling_transformer.py:198-200,218,
 * 789-798,980,984), which the reference's bf16 step computes reproducibly. */
long long muse_gemm_splitk_workspace_bytes(int M, int N, int K);
int muse_gemm_bf16_splitk(const void* A, const void* B, float* C, int M, int N, int K, int lda, int ldb, int ldc,
                          int a_mn, int b_mn, void* ws, long long ws_bytes, void* stream);

/* fp32 -> bf16 weight packing: table_dev is a device array of n_entries
 * {const float* src; bf16* dst; int64 numel; int64 first_block} with 1024 elements per block.
 * Replaces autocast's per-Linear weight casts (torch.autocast, training/train_maskgit_imagenet.py:152). */
int muse_pack_bf16(const void* table_dev, int n_entries, long long total_blocks, void* stream);
int muse_cast_bf16(const float* src, void* dst_bf16, long long n, void* stream);

/* One pass over all parameters: AdamW (training/train_maskgit_imagenet.py:242-261,438 -- torch.optim.AdamW / apex FusedAdam,
 * decoupled weight decay, bias-corrected) + EMAModel.step of the UPDATED weights (muse/modeling_ema.py:89-126, same decay
 * schedule incl. warm-up / update_after_step / update_every) + the bf16 copy into the packed GEMM operand cache.
 * entries_host: HOST array of n_entries {float* p; const float* g; float* m; float* v; float* ema (nullable);
 * bf16* packed (nullable); int64 numel (multiple of 4); int64 reserved}: the table is passed to the kernels as launch
 * arguments in chunks of 48 tensors (no device copy of it exists, so the call can be captured even when buffers moved).
 * step_dev (int64, steps taken so far) is incremented on the device and scal_dev (8 floats) receives the per-step scalars, so
 * the call is CUDA-graph capturable; lr_dev (nullable device float) overrides lr_host. */
int muse_adamw_ema_step(const void* entries_host, int n_entries, float* scal_dev, long long* step_dev,
                        const float* lr_dev, float lr_host, float beta1, float beta2, float eps, float weight_decay,
                        int ema_enabled, float ema_decay, float ema_min_decay, int ema_update_after_step,
                        int ema_update_every, int ema_use_warmup, float ema_inv_gamma, float ema_power, void* stream);

/* Embed.forward (muse/modeling_transformer.py:942-957): out[b,s,:] = word[ids[b,s],:] + pos[s,:] (fp32). */
int muse_embed_fwd(const long long* ids, const float* word, const float* pos, float* out, int B, int S, int H,
                   int vocab, void* stream);
/* its backward: dword[ids] += dx (atomic: dword must be initialised, order-dependent), dpos[s] = sum_b dx[b,s] (stored). */
int muse_embed_bwd(const long long* ids, const float* dx, float* dword, float* dpos, int B, int S, int H, int vocab,
                   void* stream);

/* Reproducible variant (the reference's index_add backward is deterministic on its bf16 CPU path): `order` = stable
 * argsort of the flattened ids, `bounds[v]` = first sorted position holding id v (vocab + 1 entries, bounds[vocab] = B*S).
 * dword[v] (all vocab rows, STORED) = sum of dx[t] over ids[t] == v in ascending t; dpos as above.  ws:
 * muse_embed_bwd_sorted_workspace_bytes(B*S, H, vocab) bytes, 16-byte aligned. */
long long muse_embed_bwd_sorted_workspace_bytes(int tokens, int H, int vocab);
int muse_embed_bwd_sorted(const long long* order, const long long* bounds, const float* dx, float* dword, float* dpos,
                          void* ws, int B, int S, int H, int vocab, void* stream);

/* LayerNorm (weight only, :124-137) / RMSNorm (:79-100) over the last dim of [rows,H].
 *   y = (res ? res : 0) + norm(v) * w ; mean/rstd [rows] are saved for backward.  v = x (act 0), gelu(x) (act 1: the
 *   exact-erf GELU of MlmLayer :980-983) or, with act 2, x is [rows, 2H] = [a | b] and v = bf16(gelu(a)) * b: the
 *   FeedForward GLU product (:789-792) feeding mid_mlp_layer_norm (:795-796) without materialising it.
 *   rms = 1 selects RMSNorm. */
int muse_norm_fwd(const void* x, int x_dtype, const float* w, const float* res, void* y, int y_dtype, float* mean,
                  float* rstd, int rows, int H, float eps, int act, int rms, void* stream);
/* dx = norm_bwd(dy) (* gelu'(x) if act 1) (+ dres if given).  Weight gradient dw[H] = sum_rows dy * xhat (nullable):
 *   dx_bf16_copy (nullable; fp32 dx, H <= 1024, no GLU): a bf16 copy of dx written in the same pass (the residual-stream
 *   gradient is the next GEMM operand).
 *   dw_ws given (muse_norm_bwd_workspace_floats(rows, H, act) floats): dw is STORED, reduced in a fixed order -> run-to-run
 *   bit-identical, no zero fill needed; dw_ws null: dw += ... with atomics (caller zero-fills; order-dependent).
 * act 2: dx is [rows, 2H] = d[a | b] (LayerNorm backward and GLU backward in one pass; v is recomputed from x).
 * y_fwd (nullable, act 2 with bf16 tensors only): the forward output bf16 [rows, H]; when given, the row reductions of
 * the first pass come from (dy, y_fwd) alone instead of re-evaluating the GELU over [a | b]. */
int muse_norm_bwd(const void* dy, int dy_dtype, const void* x, int x_dtype, const float* w, const float* mean,
                  const float* rstd, const float* dres, const void* y_fwd, void* dx, int dx_dtype, void* dx_bf16_copy,
                  float* dw, float* dw_ws, int rows, int H, int act, int rms, void* stream);
long long muse_norm_bwd_workspace_floats(int rows, int H, int act);

/* Two chained norms of a normformer layer in one pass (muse/modeling_transformer.py:882-884 then :787):
 *   x2 fp32 = res fp32 + norm1(a bf16) * w1   (post_attn_layer_norm + residual add)
 *   h2 bf16 = norm2(x2) * w2                  (FeedForward.pre_mlp_layer_norm, always LayerNorm: rms2 = 0)
 * and their joint backward: dx2 = norm2_bwd(d_h2) + dres, d_a = norm1_bwd(dx2); dw2 / dw1 are STORED (fixed-order
 * reduction; ws = 2 * muse_norm_bwd_workspace_floats(rows, H, 0) floats).  H % 8 == 0, H <= 1024. */
int muse_norm2_fwd(const void* a, const float* res, const float* w1, const float* w2, float* x2, void* h2, float* mean1,
                   float* rstd1, float* mean2, float* rstd2, int rows, int H, float eps, int rms1, int rms2, void* stream);
int muse_norm2_bwd(const void* d_h2, const float* x2, const float* w2, const float* mean2, const float* rstd2,
                   const float* dres, const void* a, const float* w1, const float* mean1, const float* rstd1, float* dx2,
                   void* d_a, float* dw2, float* dw1, float* ws, int rows, int H, int rms1, int rms2, void* stream);

/* GLU of FeedForward (:789-792): ab bf16 [rows, 2I] = [wi_0(x) | wi_1(x)], out bf16 [rows, I] = gelu(a) * b. */
int muse_glu_fwd(const void* ab, void* out, long long rows, int I, void* stream);
int muse_glu_bwd(const void* ab, const void* dout, void* dab, long long rows, int I, void* stream);

/* Attention.attention (:221-241) fused: O = softmax(Q K^T * scale) V per (batch, head), head_dim 64 or 48
 * (configs/imagenet.yaml: hidden 768 / 16 heads).  Q/K/V/O are bf16 with row strides (elements) q_rs/k_rs/v_rs/o_rs, head h at
 * column offset h*head_dim,
 * batch b at row offset b*Sq (Q,O) or b*Skv (K,V).  lse fp32 [B,nh,Sq] is saved for backward. */
int muse_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int B, int nh, int Sq, int Skv,
                  int head_dim, int q_rs, int k_rs, int v_rs, int o_rs, float scale, void* stream);
/* dvec: fp32 scratch [B,nh,Sq]. */
int muse_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                  float* dvec, void* dq, void* dk, void* dv, int B, int nh, int Sq, int Skv, int head_dim, int q_rs,
                  int k_rs, int v_rs, int o_rs, int do_rs, int dq_rs, int dk_rs, int dv_rs, float scale,
                  void* stream);

/* F.cross_entropy(logits.view(-1,V), labels.view(-1), ignore_index=-100, label_smoothing) (:1276-1280).
 * logits bf16 [rows, ld] (ld >= V, multiple of 8). lse/row_loss: fp32 [rows] scratch (lse kept for bwd).
 * loss_out[0] = mean loss, loss_out[1] = number of non-ignored rows. */
int muse_ce_fwd(const void* logits, const long long* labels, float* lse, float* row_loss, float* loss_out, int rows,
                int V, int ld, float label_smoothing, void* stream);
/* dlogits bf16 [rows, ld] = dloss[0]/N * (softmax - (1-ls) onehot - ls/V); zero for ignored rows / pad cols. */
int muse_ce_bwd(const void* logits, const long long* labels, const float* lse, const float* dloss,
                const float* loss_out, const float* row_scale, void* dlogits, int rows, int V, int ld,
                float label_smoothing, void* stream);  /* row_scale (nullable) fp32 [rows]: per-row weight w_r / sum w
                                                          replacing the 1 / #valid of the mean (loss_weight of v2 :305-317) */

/* ---- MaskGiTUViT_v2 forward (muse/modeling_transformer_v2.py); dtype codes as muse_norm_fwd (0 = fp32, 1 = bf16) ----
 * Prenorm-residual norm (unfused_rms_norm / unfused_layer_norm, :673-738) fused with the adaLN modulation that follows it
 * in TransformerLayer / GLUFeedForward (:757-792, :926-951, AdaLNModulation :1025-1037):
 *   r_out = a + r (r NULL: r_out = a; r_out NULL: not stored);  y = norm(r_out) * w  [* (1 + scale_b) + shift_b].
 * scale_shift (nullable) fp32: scale of sample b at [b*ss_stride, +H), shift at [b*ss_stride + H, +H); a row belongs to
 * sample row / rows_per_sample.  H <= 1024, H % 8 == 0. */
int muse_add_norm_mod_fwd(const void* a, int a_dtype, const float* r, const float* w, const float* scale_shift,
                          long long ss_stride, int rows_per_sample, float* r_out, void* y, int y_dtype, int rows, int H,
                          float eps, int rms, void* stream);
/* ResBlock head (:604-612): depthwise 3x3 'same' conv (groups = C, no bias; output rounded to bf16 like the autocast conv)
 * + Norm2D over channels.  x fp32 [B,h,w,C] token-major, wk fp32 [9, C] (tap-major), norm_w fp32 [C] or NULL -> y bf16. */
int muse_dwconv3x3_norm_fwd(const float* x, const float* wk, const float* norm_w, void* y, void* conv_out, int B, int h,
                            int w, int C, float eps, int rms, void* stream);  /* conv_out (nullable) bf16: saved for bwd */
/* nn.GELU + GlobalResponseNorm (:741-751) on x bf16 [B, HW, C]: g = gelu(x), Gx = ||g||_2 over the HW tokens,
 * Nx = Gx / (mean_c Gx + 1e-6), out = gamma * (g * Nx) + beta + g (bf16).  sumsq_ws (Gx^2) and nx_ws: fp32 [B, C],
 * left filled for muse_grn_bwd. */
int muse_grn_fwd(const void* x, const float* gamma, const float* beta, void* out, float* sumsq_ws, float* nx_ws, int B,
                 int HW, int C, void* stream);
/* AdaLNModulation at the end of a ResBlock (:617): x fp32 [B*rows_per_sample, C] *= (1 + scale_b), += shift_b, in place. */
int muse_adaln_apply(float* x, const float* scale_shift, long long ss_stride, int B, int rows_per_sample, int C,
                     void* stream);
/* F.silu feeding the adaLN / kv mappers (:812, :1031): y bf16 = silu(x), n % 8 == 0. */
int muse_silu_bf16(const void* x, int x_dtype, void* y, long long n, void* stream);
/* Backward of the five ops above (training of MaskGiTUViT_v2).  Reductions accumulate (+=) into zero-initialised buffers.
 * add_norm_mod: dy = grad of y, dr_out = grad of the prenorm-residual output (nullable), x = the saved r_out;
 *   g = norm_bwd(dy * (1 + scale)) + dr_out is written to da (grad of a) and dr (grad of r, nullable); dw[H] +=,
 *   dscale_shift[b] += (sum_rows dy * n | sum_rows dy) with the layout of scale_shift. */
int muse_add_norm_mod_bwd(const void* dy, int dy_dtype, const float* dr_out, const float* x, const float* w,
                          const float* scale_shift, long long ss_stride, int rows_per_sample, void* da, int da_dtype,
                          float* dr, float* dw, float* dscale_shift, int rows, int H, float eps, int rms, void* stream);
/* dy bf16 = grad of the normalised output, conv = conv_out saved by the forward, x = the forward input; dc_ws fp32
 * [B*h*w, C] scratch; dx fp32 = dres (nullable) + transposed depthwise conv of d_conv; dwk [9,C], dnorm_w [C] +=. */
int muse_dwconv3x3_norm_bwd(const void* dy, const void* conv, const float* x, const float* wk, const float* norm_w,
                            const float* dres, float* dc_ws, float* dx, float* dwk, float* dnorm_w, int B, int h, int w,
                            int C, float eps, int rms, void* stream);
/* x = forward input (bf16), dout bf16, nx / sumsq from the forward, s1_ws fp32 [B,C] scratch -> dx bf16; dgamma, dbeta +=. */
int muse_grn_bwd(const void* x, const void* dout, const float* nx, const float* sumsq, const float* gamma, float* s1_ws,
                 void* dx, float* dgamma, float* dbeta, int B, int HW, int C, void* stream);
/* y = x * (1 + scale_b) + shift_b: dx = dy * (1 + scale_b); dscale_shift[b] += (sum dy * x | sum dy). */
int muse_adaln_bwd(const float* dy, const float* x, const float* scale_shift, long long ss_stride, float* dx,
                   float* dscale_shift, int B, int rows_per_sample, int C, void* stream);
/* dx (+)= dy * silu'(x); dy bf16, x / dx dtype codes (bf16/bf16, bf16/fp32, fp32/fp32). */
int muse_silu_bwd(const void* dy, const void* x, int x_dtype, void* dx, int dx_dtype, long long n, int accumulate,
                  void* stream);

/* VectorQuantizer.get_code (muse/modeling_maskgit_vqgan.py:303-316,342-348): ids[r] = argmin_c
 * fl(fl(|z_r|^2 + |e_c|^2) - 2 z_r.e_c), first minimum. z fp32 [n,D] (NHWC-flattened), codebook fp32
 * [ncodes,D], enorm_ws fp32 [ncodes] scratch, dmin (optional) fp32 [n]. Bit-exact vs oracle/vq_oracle.c. */
int muse_vq_argmin(const float* z, const float* codebook, float* enorm_ws, long long* ids, float* dmin, int n,
                   int ncodes, int D, void* stream);
/* VectorQuantizer.get_soft_code (muse/modeling_maskgit_vqgan.py:327-340): soft fp32 [n,ncodes] = softmax_c(-d[r,c]/temp)
 * with d exactly as muse_vq_argmin; ids = argmin d (expo_noise NULL, stochastic=False) or multinomial(soft,1) realised
 * as argmax_c soft/q with q = expo_noise fp32 [n,ncodes] ~ Exp(1) drawn by the caller (stochastic=True). */
int muse_vq_soft_code(const float* z, const float* codebook, float* enorm_ws, float* soft, long long* ids,
                      const float* expo_noise, float temp, int n, int ncodes, int D, void* stream);
/* VectorQuantizer.get_codebook_entry (:318-324): out fp32 [B, D, P] (NCHW) = codebook[ids[B,P]]. */
int muse_vq_lookup_nchw(const long long* ids, const float* codebook, float* out, int B, int P, int D, int ncodes,
                        void* stream);

/* One generate2 decoding step (muse/modeling_transformer.py:1424-1454 + muse/sampling.py:9-35) as a token-parallel pass over
 * the logits and noise plus a per-row re-mask:
 * categorical sample (argmax softmax/q_exp == torch.multinomial(p,1) given the same Exp(1) draws), confidence
 * = log p_sel + temperature * gumbel(u), per-row (k+1)-th smallest cut-off, re-mask.  logits bf16 with
 * row_stride / batch_stride in elements (first K columns used); logits_unc (nullable) + guidance fuse CFG (:1410-1414).
 * input_ids/sampled/next_ids int64 [B,L]; q_exp fp32 [B,L,K]; u fp32 [B,L]; conf_out fp32 [B,L] (required: it carries the
 * confidences from the first kernel to the second). */
int muse_sample_step(const void* logits, const void* logits_unc, long long row_stride, long long batch_stride,
                     float guidance, const long long* input_ids, const float* q_exp, const float* u,
                     long long* sampled, long long* next_ids, float* conf_out, int B, int L, int K,
                     long long mask_id, int mask_len, float temperature, void* stream);

/* MaskGitVQGAN encoder/decoder blocks, fp32 NHWC (muse/modeling_maskgit_vqgan.py).
 * conv2d: Conv2dSame (:33-45) stride 1, ksize 1|3, x [B,Hi,Wi,Cin] (upsample2x = 2: stride 2, pad (0,1,0,1), Hi = 2H;
 * Hi=H/2 if upsample2x == 1: nearest x2 of :146 folded
 * into the gather), wk [ksize*ksize*Cin, Cout] packed (tap-major, then input channel), optional bias [Cout] and
 * residual [B,H,W,Cout] (ResnetBlock :82-85) -> y [B,H,W,Cout]. */
int muse_conv2d_nhwc(const float* x, const float* wk, const float* bias, const float* res, float* y, int B, int H,
                     int W, int Cin, int Cout, int ksize, int upsample2x, void* stream);
/* nn.GroupNorm(groups, C, eps) + F.silu (:61-79), deterministic (no atomics). Scratch: partials_ws float
 * [muse_groupnorm_workspace_floats(B,HW,C)] (-1 if the shape is unsupported), scale_shift_ws float [B*C*2].
 * Output either y (fp32) or the pair y_hi / y_lo (bf16 planes with y = hi + lo, the operand form of
 * muse_conv2d_nhwc_tc); the unused form is NULL.  precomputed_tiles > 0: partials_ws already holds the {sum, sumsq}
 * per [image][tile][C] written by muse_conv2d_nhwc_tc(stats=...) for x and the statistics pass is skipped. */
long long muse_groupnorm_workspace_floats(int B, int HW, int C);
int muse_groupnorm_silu_nhwc(const float* x, const float* gamma, const float* beta, float* y, void* y_hi, void* y_lo,
                             float* partials_ws, float* scale_shift_ws, int B, int HW, int C, int groups, float eps,
                             int precomputed_tiles, int apply_silu, void* stream);  /* apply_silu 0: plain GroupNorm
                             (AttnBlock.norm of the taming VQGAN, modeling_taming_vqgan.py:137-150) */
/* Conv2dSame (:33-45) on the Hopper (wgmma) tensor cores with fp32-level accuracy (3 bf16 products hi*hi + lo*hi + hi*lo,
 * fp32 accumulation): x_hi/x_lo bf16 [B,H,W,Cin], w_hi/w_lo bf16 [Cout, ksize*ksize*Cin] (tap-major, then input
 * channel), optional bias [Cout] and residual [B,H,W,Cout] -> y fp32 [B,H,W,Cout].
 * muse_conv2d_tc_supported says whether the geometry is handled (Cin % 64 == 0, W a multiple or a divisor of 128 ...);
 * other shapes use muse_conv2d_nhwc.  stats (nullable, Cout > 16): fp32 [B][tiles][Cout][2] receives {sum, sumsq} of y
 * per pixel tile, tiles = muse_conv2d_tc_tiles_per_image(...) -- the GroupNorm statistics of the next layer for free.
 * upsample2x (UpsamplingBlock :141-149, ksize 3): H, W are the output dims, x_hi/x_lo the LOW-resolution input
 * [B,H/2,W/2,Cin] and w_hi/w_lo the four 2x2 parity matrices stacked as [4*Cout, 4*Cin] (row = parity*Cout + co with
 * parity = 2*(y&1) + (x&1); column = (a*2+b)*Cin + ci for window offset (a,b); entries are sums of the 3x3 taps that
 * land on the same low-resolution pixel); tiles_per_image returns 0 when the upsample form is unsupported. */
int muse_conv2d_tc_supported(int H, int W, int Cin, int Cout, int ksize);
int muse_conv2d_tc_tiles_per_image(int H, int W, int Cin, int Cout, int ksize, int upsample2x);
int muse_conv2d_nhwc_tc(const void* x_hi, const void* x_lo, const void* w_hi, const void* w_lo, const float* bias,
                        const float* res, float* y, float* stats, int B, int H, int W, int Cin, int Cout, int ksize,
                        int mode, void* stream);
/* mode & 3: 0 plain, 1 upsample2x (above), 2 = ksize 2 with taps at offsets (0,0),(0,1),(1,0),(1,1) and zeros beyond the
 * right / bottom edge: the stride-2 3x3 convolution with pad (0,1,0,1) of the taming Downsample
 * (modeling_taming_vqgan.py:47-62) after muse_split_s2d_bf16_nhwc, weights [Cout, 4 taps * 4 Cin].  mode & 4: per-image
 * weights [B][Cout][K] -- the attention products of AttnBlock (:160-170) run as 1x1 convolutions whose weights are the
 * image's own keys / values.  */
/* space-to-depth + split: x fp32 [B,2Ho,2Wo,C] -> bf16 planes [B,Ho,Wo,4C], channel = (row parity*2 + col parity)*C + c. */
int muse_split_s2d_bf16_nhwc(const float* x, void* hi, void* lo, int B, int Ho, int Wo, int C, void* stream);
/* softmax(scale * x) over rows of n fp32 values (AttnBlock attention weights :162-163), written as bf16 hi/lo planes, or
 * as plain fp32 when out_f32 is given (hi / lo then unused). */
int muse_softmax_split_rows(const float* x, void* hi, void* lo, float* out_f32, long long rows, int n, float scale,
                            void* stream);
/* fp32 [B,H/(1+up),W/(1+up),C] -> bf16 planes hi = bf16(x), lo = bf16(x - hi), [B,H,W,C]; upsample2x folds the nearest
 * x2 of UpsamplingBlock (:146) into the gather. */
int muse_split_bf16_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int C, int upsample2x, void* stream);
/* Stem convolutions with ksize*ksize*Cin <= 64 (3 -> 128 conv_in): im2col of the taps into 64-wide bf16 hi/lo rows
 * [B,H,W,64] (tap-major, zero padded), consumed by muse_conv2d_nhwc_tc as a 1x1 convolution with Cin = 64. */
int muse_im2col_split_nhwc(const float* x, void* hi, void* lo, int B, int H, int W, int Cin, int ksize, void* stream);
/* F.avg_pool2d(2,2) (:112): x [B,2Ho,2Wo,C] -> y [B,Ho,Wo,C]. */
int muse_avgpool2_nhwc(const float* x, float* y, int B, int Ho, int Wo, int C, void* stream);
/* Decoder output (fp32, any layout; the caller passes the NHWC tensor) -> display bytes with the reference's recipe
 * (muse/pipeline_muse.py:245-252): byte = (uint8)(255 * ((clip(2x - 1, -1, 1) + 1) / 2)), same fp32 operation order. */
int muse_image_to_uint8(const float* x, unsigned char* y, long long n, void* stream);

/* [B, rows, cols] -> [B, cols, rows] (NCHW <-> NHWC at the model boundary). */
int muse_transpose_batched(const float* in, float* out, int B, int rows, int cols, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MUSE_B200_H_ */
