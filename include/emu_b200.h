/* emu_b200 — C ABI of the H100-native engine for baaivision/Emu's multimodal generate path.
 *
 * The reference has no FFI: the path sits behind Python methods (SURVEY.md §8b).  These entry points are what a
 * reference-side binding (ctypes, see INTEGRATION.md) calls in place of the library calls the reference makes:
 *
 *   emu_vit_forward      <-  self.visual(image) + pooling            Emu2/emu/emu.py:77-90, eva_vit.py:402-431
 *                            (Emu1: visual.forward_features + ln_visual   Emu1/models/modeling_emu.py:125)
 *   emu_llm_prefill      <-  self.decoder.lm.model(inputs_embeds=..., attention_mask=...)   Emu2/emu/emu.py:133-138
 *                            and step 0 of self.decoder.lm.generate(inputs_embeds=...)       Emu2/emu/emu.py:213-229
 *   emu_llm_decode       <-  steps 1..T of lm.generate (HF LlamaModel.forward with KV cache + lm_head), and the
 *                            cache-equivalent single-position regression steps of generate_image (emu.py:109-147)
 *   emu_llm_embed        <-  self.decoder.lm.model.embed_tokens(input_ids)                   Emu2/emu/emu.py:119,193
 *   emu_project          <-  project_up / project_down / stu_regress_head                    Emu2/emu/emu.py:53-55
 *   emu_cformer_forward  <-  self.cformer(image_features)                 Emu1/models/causal_former.py:43-62
 *   emu_unet_forward     <-  self.unet(latents, t, encoder_hidden_states, added_cond_kwargs) Emu2/emu/diffusion.py:136-141
 *   emu_denoise_step     <-  one iteration of the denoising loop (cat, scale_model_input, unet, CFG, Euler step)
 *                                                                                            Emu2/emu/diffusion.py:130-149
 *   emu_vae_decode       <-  self.vae.decode(latents / scaling_factor)                       Emu2/emu/diffusion.py:214-219
 *
 * Conventions: every pointer is a CUDA device pointer unless named host_*; all activations are bf16
 * (uint16_t storage) unless stated; the caller owns activation buffers, the engine owns packed weights, the KV
 * cache and workspaces; every call enqueues on the caller's cudaStream_t and returns without synchronising;
 * return value 0 = ok, negative = error (see EMU_ERR_*), message via emu_last_error(); nothing throws or aborts.
 * There is no CPU fallback: without a CUDA device every compute entry point returns EMU_ERR_CUDA.
 */
#ifndef EMU_B200_H
#define EMU_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EMU_OK 0
#define EMU_ERR_INVALID (-1)
#define EMU_ERR_CUDA (-2)
#define EMU_ERR_NOMEM (-3)
#define EMU_ERR_STATE (-4)
#define EMU_ERR_UNSUPPORTED (-5)
#define EMU_ERR_NCCL (-6)

#define EMU_DTYPE_F32 0
#define EMU_DTYPE_BF16 1
#define EMU_DTYPE_F16 2

typedef struct EmuEngine EmuEngine;
typedef void* emu_stream_t; /* cudaStream_t */

typedef struct EmuConfig {
  /* --- LLaMA decoder (Emu2/emu/conf/llama_config/config.json; Emu1/models/llama_config) --- */
  int llm_hidden, llm_layers, llm_heads, llm_head_dim, llm_ffn, llm_vocab;
  float llm_rms_eps, llm_rope_theta;
  int llm_max_batch; /* sequences x beams held in the KV cache, <= 32 (more than 8 rows decode on the GEMM path) */
  int llm_max_seq;   /* KV slots per sequence */
  /* --- EVA-CLIP ViT (Emu2/emu/conf/emu_conf.py:7-33; Emu1/models/Emu-14B.json) --- */
  int vit_image, vit_patch, vit_width, vit_layers, vit_heads, vit_mlp;
  float vit_ln_eps;
  int vit_postnorm;   /* Emu2: x + LN(f(x)); Emu1: x + f(LN(x)) */
  int vit_final_ln;   /* Emu1 ln_visual applied after the last block */
  int vit_max_batch;
  /* --- Causal-Former (Emu1/models/causal_former.py) : 0 layers = absent --- */
  int cf_layers, cf_dim, cf_heads, cf_ffn, cf_queries, cf_enc_width, cf_out_dim, cf_buckets, cf_max_distance;
  /* --- UNet / VAE presence flags; their topology comes from emu_unet_configure() --- */
  int reserved[8];
} EmuConfig;

/* ---- engine life cycle ---- */
int emu_engine_create(const EmuConfig* cfg, int tp_rank, int tp_size, const void* nccl_unique_id /*128 B or NULL*/,
                      EmuEngine** out);
void emu_engine_destroy(EmuEngine* e);
const char* emu_last_error(EmuEngine* e);
/* which real attention heads tensor-parallel rank `tp_rank` owns (heads need not divide tp_size: Emu2 has 52) */
int emu_tp_head_range(int n_heads, int tp_size, int tp_rank, int* start, int* count);
/* 128-byte ncclUniqueId for rank 0 to broadcast to the other ranks before emu_engine_create */
int emu_nccl_unique_id(void* out128);

/* Hand one reference state-dict tensor to the engine (reference key names, SURVEY.md §8b "weight contract").
 * The engine converts to bf16, repacks (fused QKV with RoPE-pair interleave, interleaved gate/up, padded patch
 * kernel), shards for tensor parallelism, and keeps its own copy; the caller may free src afterwards. */
int emu_engine_load_tensor(EmuEngine* e, const char* state_dict_key, const void* src, int dtype, const int64_t* shape,
                           int ndim, emu_stream_t stream);

/* ---- EVA ViT ---- */
/* image [B,3,S,S] bf16 NCHW -> pooled tokens [B,n_query,width] (pool=1, Emu2 encode_image) or raw tokens
 * [B,1+G*G,width] after the optional final LayerNorm (pool=0, Emu1) */
int emu_vit_forward(EmuEngine* e, const void* image_nchw, int B, void* out, int n_query, int pool, emu_stream_t s);

/* ---- LLaMA decoder ---- */
int emu_llm_reset(EmuEngine* e, emu_stream_t s); /* forget the KV cache */
int emu_llm_embed(EmuEngine* e, const int32_t* ids, int n, void* out_embeds, emu_stream_t s);
/* inputs_embeds [B,N,H]; attention_mask [B,N] int32, LEFT padded (Emu2/emu/emu.py:58); appends N positions.
 * hf_positions=1: rope position = index - n_pad (HF generate); 0: arange incl. pads (lm.model without position_ids).
 * last_hidden [B,N,H] = post-final-RMSNorm hidden states (hidden_states[-1], emu.py:144) or NULL;
 * logits_last [B,V] fp32 = lm_head(last position) or NULL. */
int emu_llm_prefill(EmuEngine* e, const void* inputs_embeds, const int32_t* attention_mask, int B, int N,
                    int hf_positions, void* last_hidden, float* logits_last, emu_stream_t s);
/* One autoregressive step for B cached sequences. Exactly one of token_ids [B] (device) / embeds [B,H] is given.
 * beam_src_idx [B] (device) reorders the KV cache first (HF _reorder_cache) or NULL.
 * logits [B,V] fp32 and/or hidden [B,H] (post-final-norm) may be NULL.
 * next_ids [B] (device, may be NULL): argmax(logits) with token `ban_id` excluded (min_length EOS suppression, -1 = none). */
int emu_llm_decode(EmuEngine* e, const int32_t* token_ids, const void* embeds, const int32_t* beam_src_idx, int B,
                   float* logits, void* hidden, int32_t* next_ids, int ban_id, emu_stream_t s);
int emu_llm_cur_len(EmuEngine* e);
/* Re-map the cached sequences: row b of the new cache (new_B rows) = row src_idx[b] (device int32) of the current one.  Beam
 * search prefills each prompt ONCE and then expands its cache row to num_beams rows (HF expands the inputs and prefills
 * num_beams identical copies — same result, num_beams x the prompt work).  new_B <= llm_max_batch. */
int emu_llm_expand(EmuEngine* e, const int32_t* src_idx, int new_B, emu_stream_t s);
/* y[M,out] = x[M,in] W^T for the small projections: which = 0 project_up, 1 project_down, 2 stu_regress_head */
int emu_project(EmuEngine* e, int which, const void* x, int M, void* y, emu_stream_t s);

/* ---- Emu1 Causal-Former ---- */
int emu_cformer_forward(EmuEngine* e, const void* vit_tokens /*[B,Nv,enc_width]*/, int B, int Nv,
                        void* out /*[B,queries,out_dim]*/, emu_stream_t s);

/* ---- diffusion (Emu2-Gen / Emu1 pipeline) ---- */
typedef struct EmuUNetConfig {
  int in_channels, out_channels;
  int n_blocks;                    /* len(block_out_channels) */
  int block_out_channels[4];
  int layers_per_block;
  int transformer_layers[4];       /* per down block; 0 = no attention in that block */
  int head_dim;                    /* attention head width (SDXL: 64); 0 = use num_heads instead */
  int cross_attention_dim;
  int use_linear_projection;
  int addition_time_embed_dim;     /* 0 = no text_time conditioning (SD-1.5 class) */
  int projection_class_embeddings_input_dim;
  int norm_groups;
  float norm_eps;
  int mid_transformer_layers;      /* transformer layers of the mid block; 0 = as many as the last down block (SDXL).  SD-1.5 has
                                      a plain last down block but one cross-attention layer in the mid block */
  int num_heads;                   /* used when head_dim == 0: the same head COUNT at every level (SD-1.5: 8 heads, i.e. head
                                      widths 40 / 80 / 160 — the Emu1 pipeline, Emu1/models/pipeline.py:37-39) */
} EmuUNetConfig;
int emu_unet_configure(EmuEngine* e, const EmuUNetConfig* cfg);
int emu_unet_forward(EmuEngine* e, const void* latents_nchw /*[B2,C,h,w] bf16*/, float timestep,
                     const void* ctx /*[B2,L,Cc]*/, int L, const void* text_embeds /*[B2,Cc] or NULL*/,
                     const int32_t* time_ids /*[B2,6] or NULL*/, int B2, int h, int w, void* noise_pred /*[B2,C,h,w]*/,
                     emu_stream_t s);
/* fused cat -> scale_model_input -> UNet -> CFG combine -> Euler step; latents [B,4,h,w] updated in place (fp32) */
int emu_denoise_step(EmuEngine* e, float* latents_inout, float sigma, float sigma_next, float timestep, float guidance,
                     const void* ctx, int L, const void* text_embeds, const int32_t* time_ids, int B, int h, int w,
                     emu_stream_t s);
/* The same fused iteration with a linear multistep scheduler instead of Euler — PNDM / PLMS as the Emu1 pipeline runs it
 * (Emu1/models/pipeline.py:112-127: scale_model_input = identity, unet, CFG, PNDMScheduler.step with skip_prk_steps):
 *   e = CFG(eps);  m = wc*e + w0*h0 + w1*h1 + w2*h2;  x_prev = a * x + b * m
 * host_coef8 (HOST, 8 floats) = {a, b, wc, w0, w1, w2, unused, flags}; flags bit 0: push e into the eps history, bit 1: x is the
 * sample saved earlier (PLMS repeats its first timestep), bit 2: save the incoming latent.  state: DEVICE fp32 [4][B*C*h*w]
 * (three history planes, newest first, + the saved sample), zero-initialised by the caller.  ctx = [cond; uncond] [2B, L, Cc]
 * when guidance > 1.  The scalars are computed by emu_b200/emu1/scheduler.py from the scheduler config. */
int emu_denoise_step_multistep(EmuEngine* e, float* latents_inout, float* state, const float* host_coef8, float timestep,
                               float guidance, const void* ctx, int L, int B, int h, int w, emu_stream_t s);
typedef struct EmuVAEConfig {
  int latent_channels, out_channels, n_blocks;
  int block_out_channels[4];
  int layers_per_block, norm_groups;
} EmuVAEConfig;
int emu_vae_configure(EmuEngine* e, const EmuVAEConfig* cfg);
int emu_vae_decode(EmuEngine* e, const void* latents_nchw /*bf16, already / scaling_factor*/, int B, int h, int w,
                   float* image_nhwc_01, emu_stream_t s);

/* ---- stand-alone operators (parity tests and micro-benchmarks; same kernels the engine launches) ---- */
int emu_op_gemm(const void* A, int lda, const void* W, int ldw, int M, int N, int K, const void* bias,
                const void* residual, int ldr, int epi_mode, void* C, int ldc, int out_fp32, int force_bn,
                emu_stream_t s);
/* C[B, N] = epilogue(X[B, K] . W[N, K]^T) for B <= 32 activation rows: the projection kernel of the decode step with more than
   8 cache rows (num_beams x batch of `lm.generate`, Emu2/emu/emu.py:213-229).  epi_mode EPI_NONE (+ residual) or EPI_SWIGLU.
   EMU_ERR_UNSUPPORTED for shapes / epilogues it does not take (use emu_op_gemm). */
int emu_op_gemm_skinny(const void* X, int ldx, const void* W, int ldw, int B, int N, int K, const void* residual, int ldr,
                       int epi_mode, void* C, int ldc, int out_fp32, emu_stream_t s);
int emu_op_conv3x3(const void* x_nhwc, int NB, int H, int W, int Cin, const void* w_k /*[Cout, 9*Cin]*/, int Cout,
                   const void* bias, const void* residual, void* y_nhwc, emu_stream_t s);
int emu_op_gemv(const void* W, int N, int K, const void* x, int ldx, int B, const void* norm_w, float eps,
                int mode, const void* bias, const void* residual, int ldr, void* y, int ldy, int out_fp32, int pdl,
                emu_stream_t s);
int emu_op_gemv_rope_qkv(const void* W, int n_heads, int head_dim, int K, const void* x, int ldx, int B,
                         const void* norm_w, float eps, const void* rope_cos, const void* rope_sin, const int32_t* pos,
                         const int32_t* pos_off, void* q_out, void* k_cache, void* v_cache, int t_max, emu_stream_t s);
int emu_op_attn_prefill(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk, int D,
                        const int64_t* strides12 /*q,k,v,o x (batch,token,head)*/, float scale, int causal,
                        const int32_t* kv_start, const float* bias, emu_stream_t s);
int emu_op_attn_decode(const void* q, const void* k_cache, const void* v_cache, int B, int H, int D, int t_max,
                       const int32_t* pos, const int32_t* start, float scale, void* out, int max_len, emu_stream_t s);
int emu_op_rmsnorm(const void* x, const void* w, void* y, int rows, int cols, float eps, emu_stream_t s);
int emu_op_layernorm(const void* x, const void* w, const void* b, const void* residual, void* y, int rows, int cols,
                     float eps, emu_stream_t s);

/* Image pre-processing (SURVEY.md §8f-2): TF.Resize((out_h, out_w), BICUBIC) -> ToTensor -> Normalize(mean, std) as in
 * Emu2/emu/chat.py:35-39, Emu2/emu/diffusion.py:59-63, Emu1/models/pipeline.py:59-63, bit-exact with torchvision + Pillow
 * (Pillow ImagingResample: two-pass fixed-point bicubic on uint8).  rgb_hwc: DEVICE pointer to [H, W, 3] uint8;
 * mean3 / std3: HOST pointers to 3 floats; out_chw: device [3, out_h, out_w] of out_dtype (EMU_DTYPE_F32 / _BF16). */
int emu_preprocess_image(const uint8_t* rgb_hwc, int H, int W, int out_h, int out_w, const float* mean3, const float* std3,
                         void* out_chw, int out_dtype, emu_stream_t s);

/* numpy_to_pil's `(images * 255).round().astype("uint8")` (Emu2/emu/diffusion.py:231-234) on the device: image01 = the fp32
 * [0, 1] image emu_vae_decode wrote; round-half-to-even; n elements. */
int emu_image_to_uint8(const float* image01, uint8_t* out, int64_t n, emu_stream_t s);

/* Device-side beam-search step (SURVEY.md §8f-1).  Replaces, inside HF GenerationMixin._beam_search as driven by
 * Emu2/emu/emu.py:213-229 (num_beams=5, length_penalty=-1) and Emu1/models/modeling_emu.py:162-179, the vocabulary-wide
 * work of one step:
 *   log_softmax(logits) -> RepetitionPenaltyLogitsProcessor -> NoRepeatNGramLogitsProcessor -> MinLength EOS ban ->
 *   PrefixConstrainedLogitsProcessor -> + running beam score -> topk(2*beams) over the flattened [beams*vocab] scores of
 *   every batch row.
 * logits [batch*beams, vocab] fp32 is processed IN PLACE: on return it holds the processed log-probabilities + the row's running
 * score (HF's accumulated_log_probs) — the sampling strategies rely on that (beam-sample draws its candidates from them,
 * `_sample` with processors feeds them to emu_sample_tokens); keep <= 32.  running_scores [batch*beams] may be NULL;
 * prev_tokens: DEVICE int32 rows of the tokens generated so far, row r at prev_tokens + r*prev_stride, prev_len valid (may be
 * NULL); penalty_on_logits = 1 applies the repetition penalty to the raw logits (HF greedy / sampling) instead of the
 * log-probabilities (HF beam search); no_repeat_ngram = n-gram size (0 = off); allowed [batch*beams, vocab] bytes, 0 = banned
 * (the mask prefix_allowed_tokens_fn produces, Emu1/mm_eval/models/emu.py:97-109) or NULL; ban_id < 0 disables the EOS ban.
 * Outputs out_lp / out_idx [batch, keep]: scores (largest first) and flat indices beam*vocab + token. */
int emu_beam_topk(float* logits, const float* running_scores, int batch, int beams, int vocab, int keep, int ban_id,
                  const int32_t* prev_tokens, int prev_len, int prev_stride, float repetition_penalty, int penalty_on_logits,
                  int no_repeat_ngram, const uint8_t* allowed, float* out_lp, int* out_idx, emu_stream_t s);

/* The hypothesis bookkeeping of the same HF step (running beams, finished beams, early-stopping heuristic) on the device, so
 * that a beam-search step never synchronises with the host: consumes emu_beam_topk's outputs, updates the state arrays in
 * place and writes the next step's inputs for emu_llm_decode (next_tokens -> token_ids, beam_src -> beam_src_idx).
 * State (all DEVICE, caller-allocated): running_seq / sequences [2][batch, beams, max_length] int32 (two planes, the live one
 * is plane cur_len & 1 before the call and (cur_len + 1) & 1 after), running_scores / beam_scores [batch, beams] fp32,
 * is_finished / fin_len [batch, beams] int32, unsat [batch] int32 (initially 1), done [1] int32 (initially 0; once set every
 * later call is a no-op).  fin_div = (cur_len + 1) ** length_penalty, best_div = best_len ** length_penalty (host scalars);
 * early_stopping: 0 False, 1 True, 2 "never".  batch <= 8, beams <= 16. */
int emu_beam_step(const float* topk_lp, const int32_t* topk_idx, int batch, int beams, int vocab, int cur_len, int max_length,
                  int eos_id, float fin_div, float best_div, int early_stopping, int32_t* running_seq, float* running_scores,
                  int32_t* sequences, float* beam_scores, int32_t* is_finished, int32_t* fin_len, int32_t* unsat,
                  int32_t* done, int32_t* next_tokens, int32_t* beam_src, emu_stream_t s);

/* Device-side sampling step (SURVEY.md §8f-1): HF warper order temperature -> top-k (0 = off) -> top-p (1 = off) and one
 * multinomial draw per row, as GenerationMixin does for do_sample=True (Emu2/emu/chat.py:46-57 forwards the knobs).
 * logits [rows, vocab] fp32 (not modified); ban_id < 0 disables the min-length EOS ban; the draw is a counter-based
 * hash of (seed, offset, row) — statistically equivalent to torch.multinomial, not bit-identical to its Philox stream. */
int emu_sample_tokens(const float* logits, int rows, int vocab, float temperature, int top_k, float top_p, int ban_id,
                      uint64_t seed, uint64_t offset, int32_t* out_ids, emu_stream_t s);

/* Diagnostics: emu_op_gemm (bf16 output) with per-CTA phase time stamps.  stamps: DEVICE [number of SMs][8] uint64, per CTA
 * {globaltimer ns at entry, then SM clock64 at: entry, set-up done, first TMA issued, first stage landed, last MMA retired,
 * epilogue started, epilogue done} of the CTA's first tile.  tools/gemm_phases.py turns them into a phase table. */
int emu_debug_gemm_phases(const void* A, int lda, const void* W, int ldw, int M, int N, int K, const void* bias,
                          const void* residual, int ldr, int epi_mode, void* C, int ldc, int force_bn,
                          unsigned long long* stamps, emu_stream_t s);

/* Diagnostics: emu_op_gemv (bf16 output) with per-CTA phase time stamps.  stamps: DEVICE [number of SMs][8] uint64, per CTA {globaltimer
 * ns at entry, then SM clock64 at: entry, barriers ready, dependency resolved (griddepcontrol.wait), x staged, first weight
 * chunk landed, own chunks consumed and rows flushed, exit}.  tools/gemv_phases.py prints the table. */
int emu_debug_gemv_phases(const void* W, int N, int K, const void* x, int ldx, int B, const void* norm_w, float eps, int mode,
                          const void* residual, int ldr, void* y, int ldy, int pdl, unsigned long long* stamps,
                          emu_stream_t s);

/* number of kernels this library has launched since load (bench.py's gpu_launches) */
uint64_t emu_launch_count(void);
const char* emu_version(void);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_H */
