/* vitron_b200 — C ABI of the H100 (sm_90a) kernels behind Vitron's multimodal forward path.
 *
 * The reference (SkyworkAI/Vitron) has no FFI of its own: its "operator interface" for this path
 * is a set of torch nn.Module forwards (SURVEY.md §8b).  Every entry point below replaces the
 * arithmetic of the reference call cited next to it; the Python drop-in modules in vitron_b200/
 * keep the reference's class names / signatures and call these through ctypes.
 *
 * Conventions (all entry points):
 *   - plain pointers + sizes, device pointers unless stated; bf16 = 2-byte bfloat16 storage;
 *   - no allocation, no implicit synchronisation, work is enqueued on `stream`;
 *   - returns 0 (VB_OK) or a negative VB_ERR_* code, never throws;
 *   - re-entrant provided distinct (stream, workspace) pairs.
 */
#ifndef VITRON_B200_H_
#define VITRON_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

#define VB_ACT_NONE 0
#define VB_ACT_GELU 1       /* exact erf GELU  (nn.GELU(), CLIP "gelu")            */
#define VB_ACT_QUICK_GELU 2 /* x*sigmoid(1.702x) (CLIP "quick_gelu")                */
#define VB_ACT_RELU 3
#define VB_ACT_SILU 4

#define VB_GLU_NONE 0
#define VB_GLU_SWIGLU 1 /* silu(a) * b   — LlamaMLP: a = gate_proj, b = up_proj     */
#define VB_GLU_GEGLU 2  /* a * gelu(b)   — GEGLU: x, gate = proj(x).chunk(2)       */

/* Fused GEMM / conv epilogue:  v = rowscale[row] * acc + bias[col] + rowbias[row / rowbias_rows][col];
 *   (rowscale = 1/rms(x_row) turns a GEMM on un-normalised rows against RMSNorm-weight-folded weights
 *    into LlamaRMSNorm -> Linear; M <= 16: rms_eps > 0 makes the kernel compute it from A itself)
 *   GLU: columns are packed in blocks of 32 = [16 x a | 16 x b] -> 16 outputs; else v = act(v);
 *   out = residual ? residual[row, col] + alpha * v : alpha * v;   stored as bf16 (or fp32). */
typedef struct vb_epilogue {
  const void* bias;     /* bf16 [N] or NULL */
  const void* rowbias;  /* bf16 [groups, N] or NULL */
  int64_t rowbias_rows; /* rows per rowbias group */
  const void* residual; /* bf16 [M, ldr] or NULL (may alias `out`) */
  int64_t ldr;
  float alpha;
  int32_t act;
  int32_t glu;
  int32_t out_fp32;
  const float* rowscale; /* fp32 [M] or NULL */
  float rms_eps;         /* > 0 (M <= 16 only, rowscale NULL): rowscale = rsqrt(mean(A_row^2) + rms_eps) */
} vb_epilogue;

/* ---- library ---------------------------------------------------------------------------- */
const char* vb200_version(void);
const char* vb200_last_error(void); /* text of the last CUDA error seen by this library */
int vb200_device_ok(void);          /* 1 iff the current device is sm_90 (H100) */
/* Programmatic Dependent Launch for the decode-step kernels (gemv, decode attention, splice, rope table,
 * arg-max): when on, each of them is launched with programmaticStreamSerialization and overlaps its
 * prologue / weight prefetch with the tail of its predecessor. Returns the previous setting.
 * Contract while it is on: the weight operand W of an M <= 16 vb200_gemm_bf16 call (the weight-streaming kernel requests its
 * first weight groups BEFORE the dependency wait) must be a constant, i.e. not written by kernels still in flight on the
 * stream; activations used as W (attention-style products) belong on the M > 16 paths or in a PDL-off region. */
int vb200_set_pdl(int enable);
/* Attention kernel selection for vb200_attention: 0 = automatic (wgmma kernel for head_dim 40..160
 * with >= 96 query rows, mma.sync otherwise), 1 = mma.sync only, 2 = wgmma whenever supported.
 * Both kernels compute the same function; the switch exists so the parity tests can pin each of them. */
int vb200_set_attention_impl(int impl);
/* Diagnostics for the wgmma attention kernel: every mbarrier wait in it is bounded (~0.5 s); if one expires
 * the CTA drains instead of hanging the GPU and records where. out3 = {site id (0 = never fired), packed block
 * index, thread}; reading clears the record. Synchronises the device. */
int vb200_attention_watchdog(uint32_t* out3);
/* Resident CTAs per SM (registers / shared memory) of the wgmma attention kernel for head_dim 64 or 128. */
int vb200_attention_tc_occupancy(int head_dim);

/* ---- GEMM: out[M,N] = epi(A[M,K] @ W[N,K]^T), wgmma + TMA (gemm.cu, gemm_v2.cuh) -------
 * Replaces every nn.Linear on the path: HF LlamaAttention/LlamaMLP/lm_head (transformers 4.31,
 * call sites vitron/model/language_model/llava_llama.py:91-102), CLIPAttention/CLIPMLP
 * (languagebind/image/modeling_image.py:136-151), mm_projector (multimodal_projector/
 * builder.py:33-51), region MLP (region_extractor/layer.py:17-20), UNet/SEEM/GLIGEN linears.
 * M <= 16 runs the weight-streaming kernel (gemv.cu: HBM-bound, no workspace). 16 < M <= 64 with a large weight runs swap-AB + split-K (weights stream through the 128-row tile slot; a reduce
 * kernel sums the partials in split order and applies the epilogue) and needs the workspace reported by
 * vb200_gemm_bf16_workspace_size; so do the split-K shapes of M > 64 (else the call runs unsplit). lda/ldw/ldo in elements, multiples of 8. */
size_t vb200_gemm_bf16_workspace_size(int64_t M, int64_t N, int64_t K);
int vb200_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out, int64_t ldo,
                    int64_t M, int64_t N, int64_t K, const vb_epilogue* epi, void* workspace,
                    size_t workspace_bytes, cudaStream_t stream);

/* ---- NF4 weights (gemv_nf4.cu; format stated in vitron_b200/nf4.py) --------------------------
 * The reference's `load_pretrained_model(..., load_4bit=True)` (vitron/model/builder.py:36-46) loads the LLM through
 * bitsandbytes as NF4 with double-quantised block scales. Here a weight W_eff[N, K] (K % 64 == 0) is
 *   codes:  uint8 [N, ceil(K/128) * 64], 4-bit codes into bitsandbytes' nf4 table, in the kernel's byte order (nf4.py
 *           pack_codes); the row stride is implied by K;
 *   scales: fp16 [N, K / 64], one scale per (row, 64-column block): W_eff[n, k] = nf4[code] * float(scale[n, k / 64]).
 * vb200_gemm_nf4: out = epi(rowscale ⊙ (A · diag(kscale) · W_effᵀ)) with every vb_epilogue feature of vb200_gemm_bf16
 * (rms_eps computes the row scale from the raw A), for M <= 32 (else VB_ERR_UNSUPPORTED); kscale is an optional fp32
 * [K] column scale (16-byte aligned) applied to A in fp32 and rounded to bf16 before the products, which is how the
 * RMSNorm gain reaches a weight that was quantised unfolded. One launch, no workspace. lda multiple of 8.
 * vb200_nf4_dequant: out[N, K] bf16 (contiguous, 16-byte aligned) = bf16_rn((nf4[code] * scale) * kscale[k]), fp32
 * products in that order (kscale NULL = 1), bit-identical to nf4.py; larger M runs it into a workspace and then
 * vb200_gemm_bf16. Both follow the PDL rule of vb200_gemm_bf16's weight operand: codes, scales and kscale are
 * requested before the dependency wait and must be constants. */
int vb200_gemm_nf4(const void* A, int64_t lda, const void* codes, const void* scales, const float* kscale, void* out,
                   int64_t ldo, int64_t M, int64_t N, int64_t K, const vb_epilogue* epi, cudaStream_t stream);
int vb200_nf4_dequant(const void* codes, const void* scales, const float* kscale, void* out, int64_t N, int64_t K,
                      cudaStream_t stream);



/* ---- implicit-GEMM convolution on NHWC activations, im2col-free (gemm.cu) ----------------
 * X [nb,h,w,cin]; Wt [cout, kh*kw, ceil64(cin)] (zero padded); out [nb,ho,wo,cout].
 * Replaces nn.Conv2d 3x3/1x1 (i2vgen util.py:651,677; Upsample/Downsample util.py:579-607,
 * 732-756), Conv3d (3,1,1) as kh=3,kw=1 over [b, f, h*w, c] (util.py:1360-1375), SEEM FPN convs
 * (transformer_encoder_fpn.py:54-107). stride in {1,2}. Convolutions whose output-pixel tiles cannot fill the SMs
 * (the 1280-channel UNet levels) run split-K over (tap, channel-chunk) steps: fp32 partials in the
 * workspace reported by vb200_conv_nhwc_workspace_size (0 for every other shape); with workspace == NULL the call
 * runs unsplit. */
size_t vb200_conv_nhwc_workspace_size(int64_t nb, int64_t h, int64_t w, int64_t cin, int64_t cout, int kh, int kw,
                                      int stride, int pad_h, int pad_w);
int vb200_conv_nhwc_bf16(const void* X, const void* Wt, void* out, int64_t nb, int64_t h,
                         int64_t w, int64_t cin, int64_t cout, int kh, int kw, int stride,
                         int pad_h, int pad_w, const vb_epilogue* epi, void* workspace,
                         size_t workspace_bytes, cudaStream_t stream);
/* 0 = epilogue variants specialised by feature set (default), 1 = only the variants that resolve every epilogue
 * feature at run time. Returns the previous setting. For A/B measurements and parity tests. */
int vb200_set_gemm_impl(int impl);
/* Variant switches / measurement aids of the v2 kernel. `resident_b` is a bit set (default 1): bit 0 = the "weight slab stays
 * in shared memory" variant for K <= 320, bit 1 = also for K <= 640, other bits are ignored. `dbg`: bit 0 makes the
 * epilogue store nothing (wrong results: timing of the main loop alone). -1 keeps a setting.
 * Returns the previous (resident_b | dbg << 8). */
int vb200_set_gemm_debug(int resident_b, int dbg);

/* direct (SIMT) convolution for the two odd-shaped layers (cin < 8-aligned or tiny cout) */
int vb200_conv_nhwc_direct(const void* X, const void* Wt, const void* bias, void* out, int64_t nb,
                           int64_t h, int64_t w, int64_t cin, int64_t cout, int kh, int kw,
                           int stride, int pad_h, int pad_w, cudaStream_t stream);

/* ---- normalisation (norm.cu) ----------------------------------------------------------------
 * rmsnorm: HF LlamaRMSNorm (fp32 statistics). layernorm: nn.LayerNorm. groupnorm: nn.GroupNorm
 * over NHWC [n, spatial, c] (+ optional SiLU / ReLU), i2vgen util.py:640-655,1358-1375. */
int vb200_rmsnorm(const void* x, int64_t ldx, const void* weight, void* out, int64_t ldo,
                  int64_t rows, int64_t d, float eps, cudaStream_t stream);
/* out[row] = rsqrt(mean(x_row^2) + eps), fp32: the rowscale of the RMSNorm-folded GEMMs (prefill) */
int vb200_row_rstd(const void* x, int64_t ldx, float* out, int64_t rows, int64_t d, float eps,
                   cudaStream_t stream);
int vb200_layernorm(const void* x, int64_t ldx, const void* weight, const void* bias, void* out,
                    int64_t ldo, int64_t rows, int64_t d, float eps, cudaStream_t stream);
/* workspace: zero-filled ONCE by the caller before first use; the kernels leave its counters zeroed (no per-call memset) */
size_t vb200_groupnorm_workspace_size(int64_t n, int64_t groups, int64_t c);
int vb200_groupnorm_nhwc(const void* x, const void* weight, const void* bias, void* out, int64_t n,
                         int64_t spatial, int64_t c, int64_t groups, float eps, int act,
                         void* workspace, size_t workspace_bytes, cudaStream_t stream);

/* ---- attention (attention.cu) ---------------------------------------------------------------
 * Flash-style softmax(QK^T*scale + mask)V with generic element strides (batch, seq, head); the
 * head dim is contiguous. kv_len: int32 [B] valid keys per batch or NULL. causal: key j visible
 * to query i iff j <= i + (Skv - Sq) and j < kv_len[b]. mask: uint8, non-zero = masked out, element strides
 * (mb, mh, mq) with keys contiguous, or NULL. Rows with every key masked produce zeros.
 * The wgmma kernel loads whole 64-key blocks: V in [kv_len[b], Skv) and V under masked keys enter P·V with weight 0,
 * so they must be finite (0 · NaN is NaN).
 * Replaces HF LlamaAttention / CLIPAttention eager bmm+softmax, xformers
 * memory_efficient_attention (i2vgen util.py:253-258; GLIGEN attention.py:176,247) and SEEM
 * multi_head_attention_forward (utils/attn.py:296-316). head_dim in {40,64,80,128,160}. */
int vb200_attention(const void* q, const void* k, const void* v, void* out, int64_t B, int64_t H,
                    int64_t Sq, int64_t Skv, int64_t head_dim, int64_t q_sb, int64_t q_ss,
                    int64_t q_sh, int64_t k_sb, int64_t k_ss, int64_t k_sh, int64_t v_sb,
                    int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss, int64_t o_sh,
                    float scale, int causal, const int32_t* kv_len, const uint8_t* mask,
                    int64_t m_sb, int64_t m_sh, int64_t m_sq, cudaStream_t stream);
/* Same with a workspace: few-query attention over long memories (SEEM: 101 queries x 8 heads over up to 16384 keys is 8
 * CTAs) is split over the keys — every CTA writes its un-normalised partial O and (max, sum) to the workspace and a merge
 * kernel combines them. vb200_attention_workspace_size reports the bytes (0 when the shape is not split); no zero-fill
 * needed. With workspace == NULL the call runs unsplit (= vb200_attention). */
size_t vb200_attention_workspace_size(int64_t B, int64_t H, int64_t Sq, int64_t Skv, int64_t head_dim, int causal);
int vb200_attention_ws(const void* q, const void* k, const void* v, void* out, int64_t B, int64_t H,
                       int64_t Sq, int64_t Skv, int64_t head_dim, int64_t q_sb, int64_t q_ss,
                       int64_t q_sh, int64_t k_sb, int64_t k_ss, int64_t k_sh, int64_t v_sb,
                       int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss, int64_t o_sh,
                       float scale, int causal, const int32_t* kv_len, const uint8_t* mask,
                       int64_t m_sb, int64_t m_sh, int64_t m_sq, void* workspace, size_t workspace_bytes,
                       cudaStream_t stream);
/* Paged prefill attention (attention_tc.cu): a chunk of new queries over keys that sit in the paged KV cache
 * (k_pages / v_pages [num_pages, H, page_size, head_dim] bf16, block_table int32 [B, max_pages], as in the decode path
 * below). q [B, Sq, H, head_dim] with element strides (q_sb, q_ss, q_sh), e.g. the q third of the fused qkv rows after
 * vb200_rope_kv_append has rotated them and written the chunk's K / V to its pages. Row b holds q_len[b] <= Sq queries
 * (int32 device arrays q_start / q_len [B]) at cache positions q_start[b] + i: key j is visible to query i iff
 * j <= q_start[b] + i; keys come from page block_table[b, j / page_size]. Query rows i >= q_len[b] are written as zeros.
 * q_start[b] + q_len[b] <= max_kv_len <= max_pages * page_size; keys at or past max_kv_len are never attended and
 * block-table entries past ceil(max_kv_len / page_size) are never read. Pages are loaded whole: the V values of every slot
 * in a page a row reads must be finite, including slots past its visible keys (they enter P·V with weight 0, and 0 · NaN
 * is NaN); a zero-initialised cache, as PagedKVCache keeps, satisfies this. block_table rows are max_pages apart.
 * Stands in for HF LlamaAttention with past_key_values (transformers 4.31: torch.cat of the cache, causal mask offset by
 * the past length). head_dim 128 and page_size 64 only (else VB_ERR_UNSUPPORTED). Strides multiples of 8, q / out /
 * pages 16-byte aligned. A grid of fewer (128-query tile, head, row) CTAs than SMs is split over the keys through the
 * workspace reported by vb200_attention_paged_workspace_size (0 = unsplit; with workspace == NULL the call runs
 * unsplit); the partials are merged in a fixed order, so repeated calls are bit-identical. */
size_t vb200_attention_paged_workspace_size(int64_t B, int64_t H, int64_t Sq, int64_t head_dim, int64_t max_kv_len);
int vb200_attention_paged(const void* q, int64_t q_sb, int64_t q_ss, int64_t q_sh, const void* k_pages,
                          const void* v_pages, int64_t num_pages, const int32_t* block_table, int64_t max_pages,
                          const int32_t* q_start, const int32_t* q_len, void* out, int64_t o_sb, int64_t o_ss,
                          int64_t o_sh, int64_t B, int64_t H, int64_t Sq, int64_t head_dim, int64_t page_size,
                          int64_t max_kv_len, float scale, void* workspace, size_t workspace_bytes,
                          cudaStream_t stream);
/* tiny sequences (S <= 32, head_dim 64): temporal attention of the video tower
 * (modeling_video.py:105-127) and of TemporalTransformer (util.py:1061-1066). */
int vb200_attention_short(const void* q, const void* k, const void* v, void* out, int64_t nseq,
                          int64_t H, int64_t S, int64_t head_dim, int64_t q_sb, int64_t q_ss,
                          int64_t q_sh, int64_t k_sb, int64_t k_ss, int64_t k_sh, int64_t v_sb,
                          int64_t v_ss, int64_t v_sh, int64_t o_sb, int64_t o_ss, int64_t o_sh,
                          int64_t inner, int64_t q_so, int64_t k_so, int64_t v_so, int64_t o_so,
                          float scale, cudaStream_t stream);
/* (sequence index s = outer*inner + in lives at outer*x_so + in*x_sb; inner <= 0: single level) */

/* ---- LLaMA decode path (llm.cu) -------------------------------------------------------------
 * Paged KV cache per layer: k_pages / v_pages [num_pages, n_heads, page_size, head_dim] bf16,
 * block_table int32 [B, max_pages]. (The reference grows KV with torch.cat.) */
int vb200_rope_kv_append(void* qkv, int64_t ld_qkv, const int32_t* positions,
                         const int32_t* batch_of_token, const int32_t* slot_of_token, void* k_pages,
                         void* v_pages, const int32_t* block_table, int64_t max_pages,
                         int64_t tokens, int64_t n_heads, int64_t head_dim, int64_t page_size,
                         float rope_theta, cudaStream_t stream);
/* split-KV decode attention workspace: [16 KB of arrival counters (B * n_heads <= 4096) | per-split partials]; zero-filled
 * ONCE by the caller. The counter prefix has a fixed size so that ONE buffer sized for the largest batch can serve calls
 * (and captured graphs) of every smaller batch size in any order. */
size_t vb200_attn_decode_workspace_size(int64_t B, int64_t n_heads, int64_t head_dim,
                                        int64_t max_splits);
int vb200_attn_decode_paged(const void* q, int64_t ld_q, const void* k_pages, const void* v_pages,
                            const int32_t* block_table, int64_t max_pages, const int32_t* kv_len,
                            void* out, int64_t ld_o, int64_t B, int64_t n_heads, int64_t head_dim,
                            int64_t page_size, int64_t max_kv_len, float scale, void* workspace,
                            size_t workspace_bytes, cudaStream_t stream);
/* rope_table[b] = [cos(pos_b f_i) | sin(pos_b f_i)] fp32, i < head_dim/2: once per decode step */
int vb200_rope_table(const int32_t* positions, float* table, int64_t B, int64_t head_dim, float rope_theta,
                     cudaStream_t stream);
/* decode step with RoPE + KV append fused in: qkv rows [B, 3*H*hd] hold the UN-rotated q | k | v of the
 * new token (slot kv_len[b]-1): q and k are rotated on the fly with rope_table, k/v are written to their
 * page, then attention runs over kv_len[b] keys. Replaces rope_kv_append + attn_decode_paged. */
int vb200_attn_decode_rope(const void* qkv, int64_t ld_qkv, const float* rope_table, void* k_pages,
                           void* v_pages, const int32_t* block_table, int64_t max_pages,
                           const int32_t* kv_len, void* out, int64_t ld_o, int64_t B, int64_t n_heads,
                           int64_t head_dim, int64_t page_size, int64_t max_kv_len, float scale,
                           void* workspace, size_t workspace_bytes, cudaStream_t stream);
/* beam-indirect decode step (vb200_attn_decode_rope for beam search): row b reads key j >= gen_start[b] from the pages
 * of row beam_src[b * src_ld + j], through that row's block table; keys below gen_start (the shared prompt) through its
 * own. Every row still appends its new token's K / V to its own pages. Requires src_ld >= max_kv_len. */
int vb200_attn_decode_rope_beam(const void* qkv, int64_t ld_qkv, const float* rope_table, void* k_pages,
                                void* v_pages, const int32_t* block_table, int64_t max_pages, const int32_t* kv_len,
                                const int32_t* beam_src, int64_t src_ld, const int32_t* gen_start, void* out,
                                int64_t ld_o, int64_t B, int64_t n_heads, int64_t head_dim, int64_t page_size,
                                int64_t max_kv_len, float scale, void* workspace, size_t workspace_bytes,
                                cudaStream_t stream);
/* inputs_embeds[b, s] = srcmap >= 0 ? embed[srcmap] : feats[-srcmap-1] : the device half of
 * prepare_inputs_labels_for_multimodal (vitron/model/llava_arch.py:478-521); pad rows (srcmap ==
 * INT32_MIN) are zero-filled. */
int vb200_splice_multimodal(const void* embed, int64_t vocab, const void* feats,
                            int64_t n_feat_rows, const int32_t* srcmap, void* out, int64_t rows,
                            int64_t d, cudaStream_t stream);
int vb200_argmax_rows(const void* logits, int is_fp32, int64_t ld, int64_t rows, int64_t n,
                      int64_t* out_idx, cudaStream_t stream);

/* greedy step: out_idx[b] = argmax(logits[b]); next_src[b] = idx (int32, feeds the next
 * splice/embedding gather); token_log[b, kv_len[b]-prompt_len[b]] = idx; positions[b]++, kv_len[b]++.
 * Stands in for HF GenerationMixin.greedy_search's per-token host round trip. */
int vb200_argmax_advance(const float* logits, int64_t ld, int64_t rows, int64_t n, int64_t* out_idx,
                         int32_t* next_src, int32_t* positions, int32_t* kv_len, int64_t* token_log,
                         int64_t log_stride, const int32_t* prompt_len, cudaStream_t stream);

/* Sampling parameters, read by the kernel from DEVICE memory (one captured decode graph serves every setting). */
typedef struct vb_sample_params {
  float temperature; /* > 0; callers clamp with max(T, 1e-6) */
  int32_t top_k;     /* 0 = off; k >= number of non-NaN logits is off too */
  float top_p;       /* >= 1 = off */
  uint32_t reserved;
  uint64_t seed;     /* Philox key: (low 32 bits, high 32 bits) */
} vb_sample_params;

/* sampled step: the same bookkeeping as vb200_argmax_advance (out_idx optional) with the token drawn per row b from
 *   1. z_i = logit_i / T; NaN logits are never drawn; a row with no number gives token 0;
 *   2. top-k: keep i iff z_i >= the k-th largest z (ties at the threshold are kept);
 *   3. p_i = exp(z_i - max z) over the kept set;
 *   4. top-p: keep i iff (kept mass of p_j > p_i) / (kept total) < top_p (value-based: ties stay together, the
 *      maximum always stays; HF TopPLogitsWarper with min_tokens_to_keep = 1);
 *   5. x = Philox4x32-10(counter (t, b, 0, 0), key (seed_lo, seed_hi)), t = kv_len[b] - prompt_len[b] (0 without
 *      kv_len / prompt_len: the token of the prefill logits); u = (x[0] >> 8) * 2^-24; the token is the first kept
 *      index, in vocabulary order, whose inclusive prefix sum of kept p exceeds u * (sum of kept p).
 * Masses are fixed point (2^-40 units): the result does not depend on the order of the device's sums. One CTA per
 * row, the row staged in shared memory: n <= 49152 (else VB_ERR_UNSUPPORTED). Stands in for HF
 * GenerationMixin.sample's logits warpers + torch.multinomial and its per-token host round trip. */
int vb200_sample_advance(const float* logits, int64_t ld, int64_t rows, int64_t n, const vb_sample_params* params,
                         int64_t* out_idx, int32_t* next_src, int32_t* positions, int32_t* kv_len,
                         int64_t* token_log, int64_t log_stride, const int32_t* prompt_len, cudaStream_t stream);

/* Beam-search parameters, read by the kernel from DEVICE memory (one captured decode graph serves every setting). */
typedef struct vb_beam_params {
  double length_penalty;   /* a double, as the Python float transformers uses */
  int32_t early_stopping;  /* 0: False, 1: True, 2: "never" (HF 4.31) */
  int32_t pad_token_id;
  int32_t input_len;       /* input_ids.shape[1]: a hypothesis of t generated tokens has length input_len + t */
  int32_t max_length;      /* input_len + max_new_tokens ("never" with length_penalty > 0) */
  int32_t n_eos;           /* 0..8 */
  int32_t eos[8];
} vb_beam_params;          /* 64 bytes: 4 bytes of tail padding */

/* workspace of vb200_beam_advance and vb200_beam_sample_advance: [16 KB of arrival counters (B <= 4096) | candidates];
 * zero-filled ONCE by the caller */
size_t vb200_beam_workspace_size(int64_t rows);
/* beam step of HF 4.31 beam_search for B requests x k beams (row r = b * k + j, 1 <= k <= 16, 2 <= n <= 49152, else
 * VB_ERR_UNSUPPORTED), stated in float64 in vitron_b200/beam.py:
 *   score[r, i] = log_softmax(logits[r])[i] + beam_score[r] (fp32; NaN counts as -inf);
 *   the request's top 2k of the flat [k * n] scores, ties to the lower flat index j * n + i;
 *   walked in rank order: an EOS (any of params->eos) at rank < k becomes a hypothesis (score / L^length_penalty, L =
 *   input_len + t, t = kv_len - prompt_len), at rank >= k it is skipped; other candidates fill the k next beams;
 *   per request at most k hypotheses (hyp_score f64 / hyp_len / hyp_seq [B * k] indexed b * k + slot, hyp_count [B],
 *   generated ids hyp_ids [B * k, hyp_ld]); the lowest score, earliest added among equals, is evicted;
 *   done[b] follows BeamHypotheses.is_done (early_stopping True / False / "never"); a done request's beams get
 *   pad_token_id, score 0 and themselves as parent. If fewer than k non-EOS candidates are left, the missing beams
 *   continue their own row with pad_token_id and score -1e9 (4.31 raises there).
 * Bookkeeping of child row c: beam_score, parent (parent row), next_src = token, token_log[c, t] = token,
 * positions++, kv_len++. beam_src [B * k, src_ld]: entry (c, P + j), P = prompt_len, names the row that logged token j
 * of c's history and holds its K / V: children copy their parent's entries [P, P + t), then entry P + t = c.
 * Deterministic: the same inputs give bit-identical outputs whatever the order in which the rows' CTAs finish. */
int vb200_beam_advance(const float* logits, int64_t ld, int64_t B, int64_t k, int64_t n, const vb_beam_params* params,
                       float* beam_score, int32_t* parent, int32_t* done, int32_t* beam_src, int64_t src_ld,
                       double* hyp_score, int32_t* hyp_len, int32_t* hyp_seq, int32_t* hyp_count, int64_t* hyp_ids,
                       int64_t hyp_ld, int32_t* next_src, int32_t* positions, int32_t* kv_len, int64_t* token_log,
                       int64_t log_stride, const int32_t* prompt_len, void* workspace, size_t workspace_bytes,
                       cudaStream_t stream);
/* beam-sampling step of HF 4.31 beam_sample (do_sample with num_beams = k) for B searches x k beams, stated in float64
 * in vitron_b200/beam.py: vb200_beam_advance's arguments, limits and bookkeeping, plus sampling parameters in DEVICE
 * memory (temperature, top_k, top_p, seed of vb_sample_params). Per search b, step t = kv_len - prompt_len of row b * k:
 *   w[r, i] = (log_softmax(logits[r])[i] + beam_score[r]) / T (fp32; NaN counts as -inf), the warpers applied AFTER
 *   adding the running beam scores, as 4.31 does (its beam_sample starts every beam at score 0). Temperature compounds
 *   into the carried scores: at T < 1 a long search's w leaves the fp32 range and becomes -inf, where 4.31 raises;
 *   a search with no entry above -inf has no draws, and its beams continue their own rows with pad and score -1e9;
 *   per row, the kept set of vb200_sample_advance's top-k and top-p over w (within a row, w is the sampler's logit / T
 *   plus a constant: the kernel cuts on (logit - max logit) / T), with top-k at least 2 when on and top-p keeping every
 *   entry with fewer than 2 strictly larger kept ones (min_tokens_to_keep = 2);
 *   draws: key = w - log(-log U) over the kept entries with w > -inf, U = (2 * (x >> 9) + 1) * 2^-24 in (0, 1), x =
 *   word f % 4 of Philox4x32-10(counter (t, b, f / 4, 1), key (seed_lo, seed_hi)), f = j * n + i the flat index; the
 *   2k largest keys (ties to the lower flat index) are the draws without replacement (torch.multinomial as an
 *   exponential race); entries whose probability underflows to 0 rank after every positive one and are drawn in key
 *   order where 4.31 raises; fewer than 2k keyed entries give fewer draws;
 *   the draws are ranked by w (descending, ties to the lower flat index) and run through vb200_beam_advance's scorer
 *   with w as the candidate score: new beam scores and hypothesis scores are warped scores.
 * Deterministic: bit-identical outputs whatever the order in which the rows' CTAs finish. */
int vb200_beam_sample_advance(const float* logits, int64_t ld, int64_t B, int64_t k, int64_t n,
                              const vb_beam_params* params, float* beam_score, int32_t* parent, int32_t* done,
                              int32_t* beam_src, int64_t src_ld, double* hyp_score, int32_t* hyp_len, int32_t* hyp_seq,
                              int32_t* hyp_count, int64_t* hyp_ids, int64_t hyp_ld, int32_t* next_src,
                              int32_t* positions, int32_t* kv_len, int64_t* token_log, int64_t log_stride,
                              const int32_t* prompt_len, void* workspace, size_t workspace_bytes,
                              const vb_sample_params* sample_params, cudaStream_t stream);

/* ---- vision / diffusion glue (vision.cu) ----------------------------------------------------
 * patchify: NCHW pixels -> [nb*gh*gw, kpad] rows ordered (c, py, px) for the patch-embed GEMM
 * (HF CLIPVisionEmbeddings Conv2d(3,1024,14,14,bias=False)); vit_embed adds cls + position and
 * applies pre_layrnorm (modeling_image.py:651-655). */
int vb200_patchify(const void* pixels, int in_is_fp32, void* out, int64_t nb, int64_t c, int64_t h,
                   int64_t w, int64_t patch, int64_t kpad, cudaStream_t stream);
int vb200_vit_embed_ln(const void* patch_out, const void* cls, const void* pos, const void* ln_w,
                       const void* ln_b, void* out, int64_t nb, int64_t npatch, int64_t d,
                       float eps, cudaStream_t stream);
/* nearest x2 upsample NHWC (util.py:579-607) */
int vb200_upsample2x_nhwc(const void* x, void* out, int64_t nb, int64_t h, int64_t w, int64_t c,
                          cudaStream_t stream);
/* out = a + b (bf16, n elements), with optional broadcast period for b */
int vb200_add_bf16(const void* a, const void* b, void* out, int64_t n, int64_t b_period,
                   cudaStream_t stream);
/* out[row] = x[row] + table[(row / group_rows) % period] — LanguageBind temporal_embedding add on
 * '(b t) n d' rows (modeling_video.py:110-113) */
int vb200_add_rowgroup(const void* x, const void* table, void* out, int64_t rows, int64_t d,
                       int64_t group_rows, int64_t period, cudaStream_t stream);
/* classifier-free guidance combine u + s (y - u) in fp32 (diffusion_ddim.py:156-158) */
int vb200_cfg_combine(const void* y, const void* u, void* out, float scale, int64_t n,
                      cudaStream_t stream);
/* region mask pooling: feats [B, g*g, C] bf16, boxes fp32 [B,4] on a image_size canvas ->
 * pooled [B, C] (region_extractor/layer.py:27-43,77-112 incl. the x-indexes-rows quirk) */
int vb200_region_mask_pool(const void* feats, const float* boxes, void* out, int64_t B,
                           int64_t grid, int64_t c, int64_t image_size, cudaStream_t stream);
/* SEEM mask head: mask logits [Q, H, W] fp32 -> next-layer bool attention mask [Q, h2*w2]
 * = bilinear(align_corners=False) resize, sigmoid < 0.5; rows that end up fully masked are
 * cleared (seem.py:569-574, attention_data_struct.py:187). */
int vb200_seem_attn_mask(const float* mask_logits, uint8_t* out_mask, int64_t Q, int64_t H,
                         int64_t W, int64_t h2, int64_t w2, cudaStream_t stream);
/* F.interpolate(mode="bilinear", align_corners=False) of NHWC bf16 images [nb, H, W, C] -> [nb, h2, w2, C] (C % 8 == 0).
 * SEEM inference path without aux outputs: mask_features resized once per feature level so that the attention-mask logits
 * of seem.py:569-574 (bilinear of einsum('bqc,bchw->bqhw')) become one small GEMM per layer (bilinear is linear). */
int vb200_resize_bilinear_nhwc(const void* x, void* out, int64_t nb, int64_t H, int64_t W, int64_t C,
                               int64_t h2, int64_t w2, cudaStream_t stream);

/* out = softmax over the last dim of fp32 x [rows, n] (row stride ldx) -> bf16 [rows, n] (row stride ldo): the
 * single-head c-channel attention of the first-stage VAE's AttnBlock (i2vgen-xl tools/modules/autoencoder.py:418-442),
 * whose QK^T and PV are vb200_gemm_bf16 calls. */
int vb200_softmax_rows(const float* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int64_t n,
                       cudaStream_t stream);

/* ---- input pre-processing (preprocess.cu) — SURVEY.md §8(f3) ------------------------------------
 * LanguageBind image transform ToTensor -> Resize(224, BICUBIC) -> CenterCrop(224) -> Normalize
 * (languagebind/image/processing_image.py:15-25) and video transform /255 -> NormalizeVideo -> ShortSideScale(224)
 * -> CenterCropVideo(224) -> horizontal flip (video/processing_video.py:26-70), fused: uint8 HWC frames
 * [n, h, w, 3] -> normalised planar output, dst element offset = frame*dst_n + channel*dst_c + y*ow + x
 * (image batch [n,3,oh,ow]: dst_n = 3*oh*ow, dst_c = oh*ow; video clip [3,n,oh,ow]: dst_n = oh*ow, dst_c = n*oh*ow).
 * (rh, rw) = size of the virtual resized frame, (top, left) = crop offset inside it. mode: 0 bilinear,
 * 1 bicubic (A = -0.75, torchvision 0.15 tensor path = the version the reference pins), 2 antialiased bicubic
 * (torchvision >= 0.17 default). mean3 / std3 are HOST pointers to 3 floats. */
int vb200_preprocess_frames(const uint8_t* src, void* dst, int64_t n, int64_t h, int64_t w, int64_t rh,
                            int64_t rw, int64_t top, int64_t left, int64_t oh, int64_t ow, int64_t dst_n,
                            int64_t dst_c, const float* mean3, const float* std3, int mode, int flip,
                            int out_bf16, cudaStream_t stream);

/* ---- FocalNet backbone glue (focal.cu) — SEEM backbone, SURVEY.md §8(f1) -------------------------
 * reference: modules/SEEM/demo_code/xdecoder/backbone/focal.py */
#define VB_FOCAL_MAX_LEVELS 6
/* stem PatchEmbed Conv2d(c, C, k, stride, pad) as im2col rows for vb200_gemm_bf16 (focal.py:311-338): NCHW
 * pixels (fp32 or bf16) -> [nb*ho*wo, kpad] bf16, columns ordered (c, ky, kx) like weight.reshape(C, -1), zero
 * beyond c*k*k and outside the image (this also realises the pad-to-multiple-of-patch of :325-328). */
int vb200_im2col_nchw(const void* pixels, int in_is_fp32, void* out, int64_t nb, int64_t c, int64_t h,
                      int64_t w, int64_t k, int64_t stride, int64_t pad, int64_t ho, int64_t wo,
                      int64_t kpad, cudaStream_t stream);
/* depthwise Conv2d(c, c, k, padding=k/2, groups=c, bias=False) [+ GELU] on NHWC bf16 (focal.py:80-89,105).
 * x: [nb, h, w, ld_in] view (first c channels of every pixel row), wt: [k*k, c] tap-major, out: [nb, h, w, c].
 * k in {3, 5, 7, 9, 11}; act = VB_ACT_NONE | VB_ACT_GELU. */
/* kernel selection for vb200_dwconv_nhwc: 0 = automatic (default), 1 = 8-channel-per-thread kernel, 2 / 3 = channel-pair
 * kernel with 16 / 32-pixel strips. All compute the same function (the switch lets the parity tests and the bench pin
 * each one). Returns the previous setting. */
int vb200_set_dwconv_impl(int impl);
int vb200_dwconv_nhwc(const void* x, int64_t ld_in, const void* wt, void* out, int64_t nb, int64_t h,
                      int64_t w, int64_t c, int64_t k, int act, cudaStream_t stream);
/* out[b, ch] = act(mean over the t rows of x[b]) in fp32, x [nb, t, c] bf16 (ctx.mean(2).mean(3) + GELU,
 * focal.py:107); deterministic two-stage reduction through the workspace. */
size_t vb200_colmean_workspace_size(int64_t nb, int64_t t, int64_t c);
int vb200_colmean(const void* x, float* out, int64_t nb, int64_t t, int64_t c, int act, void* workspace,
                  size_t workspace_bytes, cudaStream_t stream);
/* ctx_all = scale * (sum_l ctx_l * gates[:, l] + glob * gates[:, nlev]) (focal.py:103-111): ctx_levels = nlev
 * device pointers to [nb*t, c] bf16, gates = bf16 view with row stride ld_g, glob fp32 [nb, c]. */
int vb200_focal_modulate(const void* const* ctx_levels, int64_t nlev, const void* gates, int64_t ld_g,
                         const float* glob, void* out, int64_t nb, int64_t t, int64_t c, float scale,
                         cudaStream_t stream);
/* out[rows, c] = a (row stride ld_a) * b (row stride ld_b): x_out = q * h(ctx_all) (focal.py:113) */
int vb200_mul_rows(const void* a, int64_t ld_a, const void* b, int64_t ld_b, void* out, int64_t rows,
                   int64_t c, cudaStream_t stream);
/* out = residual + LayerNorm(x) * weight + bias (residual / bias may be NULL), d <= 2048: the post-LN +
 * layerscale residual of FocalModulationBlock (focal.py:190-199; gamma folded into weight / bias by the host) */
int vb200_layernorm_add(const void* x, int64_t ldx, const void* weight, const void* bias, const void* residual,
                        int64_t ldr, void* out, int64_t ldo, int64_t rows, int64_t d, float eps,
                        cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* VITRON_B200_H_ */
