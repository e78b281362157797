"""emu_b200 — H100-native (sm_90a) engine for baaivision/Emu's multimodal generate path.

Python host code mirrors the reference's public API — emu2.emu.EmuModel (generate / generate_image / encode_image),
emu2.chat.EmuChatGeneration, emu2.diffusion.EmuVisualGeneration, emu1.modeling_emu.Emu, emu1.pipeline.EmuGenerationPipeline —
and calls hand-written CUDA through the C ABI declared in include/emu_b200.h (libemu_b200.so).  There is no CPU fallback.

Around them: generation.generate (the decoding strategies of `lm.generate`), checkpoint (streaming ingestion of the reference's
checkpoint formats), serve (the demo back end's HTTP contract over a request-batching scheduler), emu1.inference /
emu1.image_inference (the reference's example entry points).
"""
__version__ = "0.1.0"
