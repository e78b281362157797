/* emu_b200 — C ABI of the built-in NSFW safety checker, the last stage of both image pipelines.
 *
 * Replaces, on the device, what the reference runs on every generated image (Emu2/emu/diffusion.py:154-166, 236-249;
 * Emu1/models/pipeline.py:132-141, 203-215):
 *   CLIPImageProcessor(preprocessor_config.json)  ->  StableDiffusionSafetyChecker(images, clip_input)
 * i.e. the CLIP ViT-L/14 vision tower (transformers CLIPVisionModel), visual_projection, the cosine scores against the
 * 3 special-care + 17 concept embeddings with their thresholds, and the black-out of flagged images.
 * Conventions as in emu_b200.h (device pointers, caller's stream, no synchronisation, EMU_* return codes).
 */
#ifndef EMU_B200_SAFETY_H
#define EMU_B200_SAFETY_H

#include "emu_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct EmuSafetyConfig {
  /* vision tower: safety_checker/config.json "vision_config" (ViT-L/14: 224, 14, 1024, 24, 16, 4096) + projection_dim */
  int image_size, patch_size, width, layers, heads, mlp, proj_dim;
  int n_special, n_concepts; /* rows of special_care_embeds / concept_embeds (3 / 17), at most 64 together */
  float ln_eps;
  /* feature extractor: feature_extractor/preprocessor_config.json (shortest_edge 224, crop 224 = image_size) */
  int resize_shortest_edge, crop_size;
  float image_mean[3], image_std[3];
} EmuSafetyConfig;

/* Set the checker's topology; afterwards emu_engine_load_tensor takes the `safety_checker.*` keys.  Replaces an earlier
 * configuration and its weights. */
int emu_safety_configure(EmuEngine* e, const EmuSafetyConfig* cfg);

/* The whole check on a batch of generated images, in place and without a host synchronisation:
 * images_bhwc: DEVICE uint8 [B, H, W, 3] (numpy_to_pil's pixels); flagged images are set to zero (black).
 * flags: DEVICE int32 [B], 1 = NSFW concept detected.  scores: DEVICE fp32 [B, n_special + n_concepts] or NULL — the
 * reference's special_scores then concept_scores before rounding (cos - threshold + adjustment).
 * EMU_ERR_STATE names the part that is not configured or not loaded. */
int emu_safety_check(EmuEngine* e, uint8_t* images_bhwc, int B, int H, int W, int32_t* flags, float* scores, emu_stream_t s);

/* The tower alone: pixel_values [B, 3, image_size, image_size] bf16 (CLIP-normalised) -> image_embeds [B, proj_dim] bf16
 * = visual_projection(post_layernorm(CLS token)). */
int emu_safety_embed(EmuEngine* e, const void* pixel_values, int B, void* image_embeds, emu_stream_t s);

/* CLIPImageProcessor on the device, bit-exact with transformers' CLIPImageProcessorPil: resize so the shortest edge is
 * `size` (PIL bicubic on uint8), centre crop crop x crop, /255, (x - mean) / std in fp32.  images_bhwc: DEVICE uint8
 * [B, H, W, 3]; mean3 / std3: HOST 3 floats; out: DEVICE [B, 3, crop, crop] of out_dtype (EMU_DTYPE_F32 / _BF16). */
int emu_preprocess_clip(const uint8_t* images_bhwc, int B, int H, int W, int size, int crop, const float* mean3,
                        const float* std3, void* out_bchw, int out_dtype, emu_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* EMU_B200_SAFETY_H */
