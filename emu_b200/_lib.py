"""ctypes binding of libemu_b200.so (the C ABI in include/emu_b200.h).

There is no CPU fallback: importing this module only loads the library; every compute entry point needs a
CUDA device and raises :class:`EmuError` otherwise.  If the shared library is missing the import fails loudly.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libemu_b200.so")

EMU_OK = 0
ERRORS = {-1: "EMU_ERR_INVALID", -2: "EMU_ERR_CUDA", -3: "EMU_ERR_NOMEM", -4: "EMU_ERR_STATE",
          -5: "EMU_ERR_UNSUPPORTED", -6: "EMU_ERR_NCCL"}
DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2
EPI_NONE, EPI_GELU, EPI_SWIGLU, EPI_GEGLU, EPI_RELU = 0, 1, 2, 3, 4


class EmuError(RuntimeError):
    pass


class EmuConfig(C.Structure):
    _fields_ = [
        ("llm_hidden", C.c_int), ("llm_layers", C.c_int), ("llm_heads", C.c_int), ("llm_head_dim", C.c_int),
        ("llm_ffn", C.c_int), ("llm_vocab", C.c_int),
        ("llm_rms_eps", C.c_float), ("llm_rope_theta", C.c_float),
        ("llm_max_batch", C.c_int), ("llm_max_seq", C.c_int),
        ("vit_image", C.c_int), ("vit_patch", C.c_int), ("vit_width", C.c_int), ("vit_layers", C.c_int),
        ("vit_heads", C.c_int), ("vit_mlp", C.c_int),
        ("vit_ln_eps", C.c_float), ("vit_postnorm", C.c_int), ("vit_final_ln", C.c_int), ("vit_max_batch", C.c_int),
        ("cf_layers", C.c_int), ("cf_dim", C.c_int), ("cf_heads", C.c_int), ("cf_ffn", C.c_int),
        ("cf_queries", C.c_int), ("cf_enc_width", C.c_int), ("cf_out_dim", C.c_int), ("cf_buckets", C.c_int),
        ("cf_max_distance", C.c_int),
        ("reserved", C.c_int * 8),
    ]


class EmuUNetConfig(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("out_channels", C.c_int), ("n_blocks", C.c_int),
        ("block_out_channels", C.c_int * 4), ("layers_per_block", C.c_int), ("transformer_layers", C.c_int * 4),
        ("head_dim", C.c_int), ("cross_attention_dim", C.c_int), ("use_linear_projection", C.c_int),
        ("addition_time_embed_dim", C.c_int), ("projection_class_embeddings_input_dim", C.c_int),
        ("norm_groups", C.c_int), ("norm_eps", C.c_float), ("mid_transformer_layers", C.c_int), ("num_heads", C.c_int),
    ]


class EmuVAEConfig(C.Structure):
    _fields_ = [
        ("latent_channels", C.c_int), ("out_channels", C.c_int), ("n_blocks", C.c_int),
        ("block_out_channels", C.c_int * 4), ("layers_per_block", C.c_int), ("norm_groups", C.c_int),
    ]


# every symbol declared in include/emu_b200.h (tests/test_abi.py checks the header against this list)
SYMBOLS = [
    "emu_beam_topk", "emu_beam_step", "emu_sample_tokens", "emu_image_to_uint8", "emu_preprocess_image", "emu_engine_create", "emu_engine_destroy", "emu_last_error", "emu_nccl_unique_id", "emu_tp_head_range", "emu_engine_load_tensor",
    "emu_vit_forward", "emu_llm_reset", "emu_llm_embed", "emu_llm_prefill", "emu_llm_decode", "emu_llm_cur_len", "emu_llm_expand",
    "emu_project", "emu_cformer_forward", "emu_unet_configure", "emu_unet_forward", "emu_denoise_step",
    "emu_denoise_step_multistep", "emu_vae_configure", "emu_vae_decode", "emu_op_gemm", "emu_op_gemm_skinny", "emu_op_conv3x3", "emu_op_gemv", "emu_op_gemv_rope_qkv",
    "emu_op_attn_prefill", "emu_op_attn_decode", "emu_op_rmsnorm", "emu_op_layernorm", "emu_launch_count",
    "emu_debug_gemm_phases", "emu_debug_gemv_phases",
    "emu_version",
]

_lib = None


def load():
    """Load libemu_b200.so; raise if it has not been built (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EmuError("libemu_b200.so not found at %s — run `python -m emu_b200.build` (needs nvcc)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    lib.emu_last_error.restype = C.c_char_p
    lib.emu_last_error.argtypes = [C.c_void_p]
    lib.emu_version.restype = C.c_char_p
    lib.emu_launch_count.restype = C.c_uint64
    lib.emu_engine_destroy.restype = None
    lib.emu_engine_destroy.argtypes = [C.c_void_p]
    lib.emu_engine_create.argtypes = [C.POINTER(EmuConfig), C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
    _lib = lib
    return lib


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, int):
        return C.c_void_p(t)
    assert t.is_cuda, "engine arguments must be CUDA tensors"
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(rc, engine=None):
    if rc == EMU_OK:
        return
    msg = ERRORS.get(rc, str(rc))
    if engine is not None:
        detail = load().emu_last_error(engine)
        if detail:
            msg += ": " + detail.decode()
    raise EmuError(msg)


def require_cuda():
    if not torch.cuda.is_available():
        raise EmuError("emu_b200 needs a CUDA device (H100 / sm_90a); there is no CPU fallback")


_DT = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16, torch.float16: DTYPE_F16}


class Engine:
    """Thin RAII wrapper over EmuEngine*; methods map 1:1 to the C ABI."""

    def __init__(self, cfg: EmuConfig, tp_rank=0, tp_size=1, nccl_uid: bytes = None):
        require_cuda()
        self.lib = load()
        self.cfg = cfg
        self.h = C.c_void_p()
        uid = C.create_string_buffer(nccl_uid, 128) if nccl_uid is not None else None
        rc = self.lib.emu_engine_create(C.byref(cfg), tp_rank, tp_size, uid, C.byref(self.h))
        check(rc)
        self.tp_rank, self.tp_size = tp_rank, tp_size

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self.lib.emu_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights ----
    def load_tensor(self, key: str, t: torch.Tensor):
        t = t.detach()
        if not t.is_contiguous():
            t = t.contiguous()
        if t.dtype not in _DT:
            t = t.float()
        shape = (C.c_int64 * max(t.dim(), 1))(*([int(s) for s in t.shape] or [1]))
        src = C.c_void_p(t.data_ptr())
        rc = self.lib.emu_engine_load_tensor(self.h, key.encode(), src, _DT[t.dtype], shape, max(t.dim(), 1), _stream())
        check(rc, self.h)

    def load_state_dict(self, sd, prefix=""):
        for k, v in sd.items():
            if k.endswith("rotary_emb.inv_freq"):
                continue
            self.load_tensor(prefix + k, v)

    # ---- ViT ----
    def vit_forward(self, image: torch.Tensor, n_query: int, pool=True):
        c = self.cfg
        B = image.shape[0]
        image = image.to(torch.bfloat16).contiguous()
        G = c.vit_image // c.vit_patch
        if pool:
            out = torch.empty(B, n_query, c.vit_width, dtype=torch.bfloat16, device=image.device)
        else:
            out = torch.empty(B, G * G + 1, c.vit_width, dtype=torch.bfloat16, device=image.device)
        check(self.lib.emu_vit_forward(self.h, _ptr(image), B, _ptr(out), n_query, 1 if pool else 0, _stream()), self.h)
        return out

    # ---- LLM ----
    def llm_reset(self):
        check(self.lib.emu_llm_reset(self.h, _stream()), self.h)

    def llm_embed(self, ids: torch.Tensor):
        ids32 = ids.to(torch.int32).contiguous()
        out = torch.empty(*ids.shape, self.cfg.llm_hidden, dtype=torch.bfloat16, device=ids.device)
        check(self.lib.emu_llm_embed(self.h, _ptr(ids32), ids32.numel(), _ptr(out), _stream()), self.h)
        return out

    def llm_prefill(self, embeds, attention_mask=None, hf_positions=True, want_hidden=False, want_logits=True):
        B, N, H = embeds.shape
        embeds = embeds.to(torch.bfloat16).contiguous()
        mask = attention_mask.to(torch.int32).contiguous() if attention_mask is not None else None
        hidden = torch.empty(B, N, H, dtype=torch.bfloat16, device=embeds.device) if want_hidden else None
        logits = torch.empty(B, self.cfg.llm_vocab, dtype=torch.float32, device=embeds.device) if want_logits else None
        check(self.lib.emu_llm_prefill(self.h, _ptr(embeds), _ptr(mask), B, N, 1 if hf_positions else 0, _ptr(hidden),
                                       _ptr(logits), _stream()), self.h)
        return hidden, logits

    def llm_decode(self, token_ids=None, embeds=None, beam_src=None, logits=None, hidden=None, next_ids=None,
                   ban_id=-1, B=None):
        if B is None:
            B = token_ids.shape[0] if token_ids is not None else embeds.shape[0]
        # the C entry point takes bare pointers: a short buffer would be written past its end
        c = self.cfg
        for name, t, need, dt in (("logits", logits, B * c.llm_vocab, torch.float32), ("hidden", hidden, B * c.llm_hidden, torch.bfloat16),
                                  ("next_ids", next_ids, B, torch.int32), ("token_ids", token_ids, B, torch.int32),
                                  ("beam_src", beam_src, B, torch.int32), ("embeds", embeds, B * c.llm_hidden, torch.bfloat16)):
            if t is not None and (t.dtype != dt or t.numel() < need or not t.is_contiguous()):
                raise ValueError(f"llm_decode: {name} must be a contiguous {dt} tensor of at least {need} elements, got "
                                 f"{tuple(t.shape)} {t.dtype}")
        check(self.lib.emu_llm_decode(self.h, _ptr(token_ids), _ptr(embeds), _ptr(beam_src), B, _ptr(logits),
                                      _ptr(hidden), _ptr(next_ids), ban_id, _stream()), self.h)

    def cur_len(self):
        return self.lib.emu_llm_cur_len(self.h)

    def llm_expand(self, src_idx, new_B):
        """cache row b <- row src_idx[b] for b < new_B (beam search: one prefill per prompt, then num_beams cache rows)"""
        src = src_idx.to(torch.int32).contiguous()
        check(self.lib.emu_llm_expand(self.h, _ptr(src), int(new_B), _stream()), self.h)

    def sample_tokens(self, logits, temperature=1.0, top_k=0, top_p=1.0, ban_id=-1, seed=0, offset=0):
        return op_sample_tokens(logits, temperature, top_k, top_p, -1 if ban_id is None else ban_id, seed, offset)

    def beam_topk(self, logits, running_scores, batch, beams, keep, ban_id=-1, prev_tokens=None, prev_len=0,
                  repetition_penalty=1.0, penalty_on_logits=False, no_repeat_ngram=0, allowed=None):
        if ban_id is None:
            ban_id = -1
        lg = logits if (logits.dtype == torch.float32 and logits.is_contiguous()) else logits.float().contiguous()
        return op_beam_topk(lg, running_scores, batch, beams, keep, ban_id=int(ban_id), prev_tokens=prev_tokens,
                            prev_len=prev_len, repetition_penalty=float(repetition_penalty),
                            penalty_on_logits=penalty_on_logits, no_repeat_ngram=int(no_repeat_ngram or 0), allowed=allowed)

    def beam_state(self, batch, beams, max_length, pad_token_id, device):
        return BeamState(batch, beams, max_length, pad_token_id, device)

    def beam_step(self, st, topk_lp, topk_idx, cur_len, eos_token_id, length_penalty, early_stopping):
        """emu_beam_step: hypothesis bookkeeping of one HF beam-search step on the device (no host synchronisation)."""
        best_len = st.max_length if (early_stopping == "never" and length_penalty > 0.0) else cur_len + 1
        es = 1 if early_stopping is True else (2 if early_stopping == "never" else 0)
        check(self.lib.emu_beam_step(_ptr(topk_lp), _ptr(topk_idx), st.batch, st.beams, self.cfg.llm_vocab, cur_len,
                                     st.max_length, int(eos_token_id), C.c_float(float((cur_len + 1) ** length_penalty)),
                                     C.c_float(float(best_len ** length_penalty)), es, _ptr(st.running_seq),
                                     _ptr(st.running_scores), _ptr(st.sequences), _ptr(st.beam_scores), _ptr(st.is_finished),
                                     _ptr(st.fin_len), _ptr(st.unsat), _ptr(st.done), _ptr(st.next_tokens), _ptr(st.beam_src),
                                     _stream()), self.h)
        st.done_calls.add_(st.done)   # device-side count of the calls that ended with `done` set (see BeamState.result)

    # ---- Emu1 Causal-Former ----
    def cformer_forward(self, vit_tokens, n_queries, out_dim):
        B, Nv, _ = vit_tokens.shape
        vit_tokens = vit_tokens.to(torch.bfloat16).contiguous()
        out = torch.empty(B, n_queries, out_dim, dtype=torch.bfloat16, device=vit_tokens.device)
        check(self.lib.emu_cformer_forward(self.h, _ptr(vit_tokens), B, Nv, _ptr(out), _stream()), self.h)
        return out

    def vae_configure(self, vcfg: "EmuVAEConfig"):
        self.vcfg = vcfg
        check(self.lib.emu_vae_configure(self.h, C.byref(vcfg)), self.h)

    def vae_decode(self, latents):
        """latents [B,4,h,w] bf16 (already divided by the scaling factor) -> images [B, 8h, 8w, 3] fp32 in [0,1]"""
        B, _, h, w = latents.shape
        latents = latents.to(torch.bfloat16).contiguous()
        f = 2 ** (self.vcfg.n_blocks - 1)
        out = torch.empty(B, h * f, w * f, self.vcfg.out_channels, dtype=torch.float32, device=latents.device)
        check(self.lib.emu_vae_decode(self.h, _ptr(latents), B, h, w, _ptr(out), _stream()), self.h)
        return out

    # ---- diffusion ----
    def unet_configure(self, ucfg: "EmuUNetConfig"):
        self.ucfg = ucfg
        check(self.lib.emu_unet_configure(self.h, C.byref(ucfg)), self.h)

    def unet_forward(self, latents, timestep, ctx, text_embeds=None, time_ids=None):
        """latents [B2,C,h,w] bf16 NCHW, ctx [B2,L,Cc], text_embeds [B2,Cc], time_ids [B2,6] int32 -> noise [B2,C,h,w]"""
        B2, Cc, h, w = latents.shape
        latents = latents.to(torch.bfloat16).contiguous()
        ctx = ctx.to(torch.bfloat16).contiguous()
        te = text_embeds.to(torch.bfloat16).contiguous() if text_embeds is not None else None
        ti = time_ids.to(torch.int32).contiguous() if time_ids is not None else None
        out = torch.empty(B2, self.ucfg.out_channels, h, w, dtype=torch.bfloat16, device=latents.device)
        check(self.lib.emu_unet_forward(self.h, _ptr(latents), C.c_float(float(timestep)), _ptr(ctx), ctx.shape[1],
                                        _ptr(te), _ptr(ti), B2, h, w, _ptr(out), _stream()), self.h)
        return out

    def denoise_step(self, latents_f32, sigma, sigma_next, timestep, guidance, ctx, text_embeds, time_ids):
        """One iteration of the denoise loop, latents [B,4,h,w] fp32 updated in place. ctx = [cond; uncond]."""
        B, _, h, w = latents_f32.shape
        assert latents_f32.dtype == torch.float32 and latents_f32.is_contiguous()
        check(self.lib.emu_denoise_step(self.h, _ptr(latents_f32), C.c_float(float(sigma)), C.c_float(float(sigma_next)),
                                        C.c_float(float(timestep)), C.c_float(float(guidance)), _ptr(ctx), ctx.shape[1],
                                        _ptr(text_embeds), _ptr(time_ids), B, h, w, _stream()), self.h)

    def denoise_step_multistep(self, latents_f32, state_f32, coef8, timestep, guidance, ctx):
        """One PNDM / PLMS iteration (emu_denoise_step_multistep): latents [B,4,h,w] fp32 in place, state [4,B,4,h,w] fp32."""
        B, _, h, w = latents_f32.shape
        assert latents_f32.dtype == torch.float32 and latents_f32.is_contiguous()
        assert state_f32.dtype == torch.float32 and state_f32.is_contiguous() and state_f32.numel() == 4 * latents_f32.numel()
        coef = (C.c_float * 8)(*[float(v) for v in coef8])
        check(self.lib.emu_denoise_step_multistep(self.h, _ptr(latents_f32), _ptr(state_f32), coef, C.c_float(float(timestep)),
                                                  C.c_float(float(guidance)), _ptr(ctx), ctx.shape[1], B, h, w, _stream()),
              self.h)

    def project(self, which: int, x: torch.Tensor, out_dim: int):
        x2 = x.reshape(-1, x.shape[-1]).to(torch.bfloat16).contiguous()
        y = torch.empty(x2.shape[0], out_dim, dtype=torch.bfloat16, device=x.device)
        check(self.lib.emu_project(self.h, which, _ptr(x2), x2.shape[0], _ptr(y), _stream()), self.h)
        return y.reshape(*x.shape[:-1], out_dim)


# ---- stand-alone operators (used by tests and micro-benchmarks) ----
def op_gemm(A, W, bias=None, residual=None, epi=EPI_NONE, out_fp32=False, force_bn=0):
    require_cuda()
    lib = load()
    M, K = A.shape
    N = W.shape[0]
    n_out = N // 2 if epi in (EPI_SWIGLU, EPI_GEGLU) else N
    Cm = torch.empty(M, n_out, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=A.device)
    rc = lib.emu_op_gemm(_ptr(A), A.stride(0), _ptr(W), W.stride(0), M, N, K, _ptr(bias), _ptr(residual),
                         residual.stride(0) if residual is not None else 0, epi, _ptr(Cm), n_out,
                         1 if out_fp32 else 0, force_bn, _stream())
    check(rc)
    return Cm


def op_gemm_skinny(X, W, residual=None, epi=EPI_NONE, out_fp32=False):
    """X [B <= 32, K] . W [N, K]^T through the wide-decode projection kernel (gemm_skinny.cu)"""
    require_cuda()
    lib = load()
    B, K = X.shape
    N = W.shape[0]
    n_out = N // 2 if epi == EPI_SWIGLU else N
    Cm = torch.empty(B, n_out, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=X.device)
    check(lib.emu_op_gemm_skinny(_ptr(X), X.stride(0), _ptr(W), W.stride(0), B, N, K, _ptr(residual),
                                 residual.stride(0) if residual is not None else 0, epi, _ptr(Cm), n_out, 1 if out_fp32 else 0,
                                 _stream()))
    return Cm


def debug_gemm_phases(A, W, bias=None, residual=None, epi=EPI_NONE, force_bn=0):
    """emu_op_gemm + per-CTA phase stamps -> (C, stamps [148, 8] int64 on the host)"""
    require_cuda()
    lib = load()
    M, K = A.shape
    N = W.shape[0]
    n_out = N // 2 if epi in (EPI_SWIGLU, EPI_GEGLU) else N
    Cm = torch.empty(M, n_out, dtype=torch.bfloat16, device=A.device)
    stamps = torch.zeros(148, 8, dtype=torch.int64, device=A.device)
    check(lib.emu_debug_gemm_phases(_ptr(A), A.stride(0), _ptr(W), W.stride(0), M, N, K, _ptr(bias), _ptr(residual),
                                    residual.stride(0) if residual is not None else 0, epi, _ptr(Cm), n_out, force_bn,
                                    _ptr(stamps), _stream()))
    return Cm, stamps.cpu()


def op_conv3x3(x_nhwc, w_k, bias=None, residual=None):
    require_cuda()
    lib = load()
    NB, H, W_, Cin = x_nhwc.shape
    Cout = w_k.shape[0]
    y = torch.empty(NB, H, W_, Cout, dtype=torch.bfloat16, device=x_nhwc.device)
    check(lib.emu_op_conv3x3(_ptr(x_nhwc), NB, H, W_, Cin, _ptr(w_k), Cout, _ptr(bias), _ptr(residual), _ptr(y),
                             _stream()))
    return y


def op_gemv(W, x, norm_w=None, eps=1e-6, mode=EPI_NONE, bias=None, residual=None, out_fp32=False, pdl=False):
    require_cuda()
    lib = load()
    N, K = W.shape
    B = x.shape[0]
    n_out = N // 2 if mode == EPI_SWIGLU else N
    y = torch.empty(B, n_out, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=x.device)
    rc = lib.emu_op_gemv(_ptr(W), N, K, _ptr(x), x.stride(0), B, _ptr(norm_w), C.c_float(eps), mode, _ptr(bias),
                         _ptr(residual), residual.stride(0) if residual is not None else 0, _ptr(y), n_out,
                         1 if out_fp32 else 0, 1 if pdl else 0, _stream())
    check(rc)
    return y


def op_gemv_rope_qkv(W, n_heads, head_dim, x, norm_w, eps, rope_cos, rope_sin, pos, pos_off, k_cache, v_cache, t_max):
    require_cuda()
    lib = load()
    B = x.shape[0]
    q = torch.empty(B, n_heads * head_dim, dtype=torch.bfloat16, device=x.device)
    rc = lib.emu_op_gemv_rope_qkv(_ptr(W), n_heads, head_dim, W.shape[1], _ptr(x), x.stride(0), B, _ptr(norm_w),
                                  C.c_float(eps), _ptr(rope_cos), _ptr(rope_sin), _ptr(pos), _ptr(pos_off), _ptr(q),
                                  _ptr(k_cache), _ptr(v_cache), t_max, _stream())
    check(rc)
    return q


def op_attn_prefill(q, k, v, scale, causal=False, kv_start=None, bias=None):
    """q [B,Nq,H,D], k/v [B,Nk,H,D] (any strides with contiguous D) -> [B,Nq,H,D]"""
    require_cuda()
    lib = load()
    B, Nq, H, D = q.shape
    Nk = k.shape[1]
    out = torch.empty(B, Nq, H, D, dtype=torch.bfloat16, device=q.device)
    st = []
    for t in (q, k, v, out):
        assert t.stride(3) == 1
        st += [t.stride(0), t.stride(1), t.stride(2)]
    st12 = (C.c_int64 * 12)(*st)
    rc = lib.emu_op_attn_prefill(_ptr(q), _ptr(k), _ptr(v), _ptr(out), B, H, Nq, Nk, D, st12, C.c_float(scale),
                                 1 if causal else 0, _ptr(kv_start), _ptr(bias), _stream())
    check(rc)
    return out


def op_preprocess_image(img_u8_hwc, out_h, out_w, mean, std, dtype=torch.float32):
    """[H, W, 3] uint8 CUDA tensor -> [3, out_h, out_w] fp32/bf16: Resize(BICUBIC) + ToTensor + Normalize, bit-exact with the
    reference's torchvision + Pillow transform."""
    require_cuda()
    lib = load()
    assert img_u8_hwc.dtype == torch.uint8 and img_u8_hwc.dim() == 3 and img_u8_hwc.shape[2] == 3 and img_u8_hwc.is_cuda
    img = img_u8_hwc.contiguous()
    H, W, _ = img.shape
    out = torch.empty(3, out_h, out_w, dtype=dtype, device=img.device)
    m3 = (C.c_float * 3)(*[float(v) for v in mean])
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    code = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16}[dtype]
    check(lib.emu_preprocess_image(_ptr(img), H, W, out_h, out_w, m3, s3, _ptr(out), code, _stream()))
    return out


def op_image_to_uint8(image01):
    """fp32 [0,1] CUDA tensor -> uint8 (x * 255, round half to even) — numpy_to_pil's conversion on the device."""
    require_cuda()
    x = image01.contiguous()
    assert x.dtype == torch.float32 and x.is_cuda
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    check(load().emu_image_to_uint8(_ptr(x), _ptr(out), C.c_int64(x.numel()), _stream()))
    return out


def op_sample_tokens(logits, temperature=1.0, top_k=0, top_p=1.0, ban_id=-1, seed=0, offset=0):
    """logits [R, V] fp32 CUDA -> int32 [R]: temperature -> top-k -> top-p -> multinomial on the device."""
    require_cuda()
    lg = logits if (logits.dtype == torch.float32 and logits.is_contiguous()) else logits.float().contiguous()
    out = torch.empty(lg.shape[0], dtype=torch.int32, device=lg.device)
    check(load().emu_sample_tokens(_ptr(lg), lg.shape[0], lg.shape[1], C.c_float(temperature or 1.0), int(top_k or 0),
                                   C.c_float(1.0 if top_p is None else top_p), int(ban_id), C.c_uint64(seed & (2 ** 64 - 1)),
                                   C.c_uint64(offset), _ptr(out), _stream()))
    return out


class BeamState:
    """Device-resident state of one beam search (layout documented at emu_beam_step in include/emu_b200.h)."""

    def __init__(self, batch, beams, max_length, pad_token_id, device):
        self.batch, self.beams, self.max_length = batch, beams, max_length
        i32 = dict(dtype=torch.int32, device=device)
        self.running_seq = torch.full((2, batch, beams, max_length), pad_token_id, **i32)
        self.sequences = torch.full((2, batch, beams, max_length), pad_token_id, **i32)
        self.running_scores = torch.zeros(batch, beams, dtype=torch.float32, device=device)
        self.running_scores[:, 1:] = -1e9
        self.beam_scores = torch.full((batch, beams), -1e9, dtype=torch.float32, device=device)
        self.is_finished = torch.zeros(batch, beams, **i32)
        self.fin_len = torch.zeros(batch, beams, **i32)
        self.unsat = torch.ones(batch, **i32)
        self.done = torch.zeros(1, **i32)
        self.done_calls = torch.zeros(1, **i32)
        self.next_tokens = torch.zeros(batch * beams, **i32)
        self.beam_src = torch.zeros(batch * beams, **i32)

    def live(self, cur_len):
        """the plane holding the sequences after `cur_len` tokens"""
        return cur_len & 1

    def is_done(self):
        return bool(self.done.item())   # the only device->host synchronisation of the loop

    def final_len(self, cur_len):
        """The step count at which the search finished.  The host polls `done` only every few steps and the steps launched
        in between are no-ops on this state — they do not flip the sequence planes either — so the plane that holds the
        final hypotheses is the one of the step that SET `done`, not of the step at which the host noticed:
        calls made = cur_len, of which done_calls ended with `done` set  =>  finished after cur_len + 1 - done_calls steps."""
        late = int(self.done_calls.item())
        return cur_len + 1 - late if late > 0 else cur_len

    def result(self, cur_len, n=1):
        """the n best finished hypotheses of every batch row, best first: [batch * n, longest of them] (HF
        num_return_sequences; the reference's default and Emu1's num_captions=1 take n = 1)"""
        cur_len = self.final_len(cur_len)
        best = self.sequences[self.live(cur_len), :, :n, :].reshape(self.batch * n, self.max_length)
        gen_len = int(self.fin_len[:, :n].max())
        return best[:, :gen_len].to(torch.int64)


def op_beam_topk(logits, running_scores, batch, beams, keep, ban_id=-1, prev_tokens=None, prev_len=0, repetition_penalty=1.0,
                 penalty_on_logits=False, no_repeat_ngram=0, allowed=None):
    """logits [batch*beams, V] fp32 (overwritten), running_scores [batch, beams] fp32 -> (scores [batch, keep] fp32,
    flat indices [batch, keep] int32 = beam*V + token), HF _beam_search step semantics.  prev_tokens: int32 [batch*beams, L]
    (any row stride), prev_len valid tokens per row."""
    require_cuda()
    lib = load()
    V = logits.shape[-1]
    assert logits.dtype == torch.float32 and logits.is_contiguous()
    rs = running_scores.to(torch.float32).contiguous().view(-1) if running_scores is not None else None
    stride = 0
    if prev_tokens is not None and prev_len > 0:
        assert prev_tokens.dtype == torch.int32 and prev_tokens.stride(-1) == 1
        prev_tokens = prev_tokens.reshape(batch * beams, -1) if prev_tokens.dim() != 2 else prev_tokens
        stride = prev_tokens.stride(0)
    else:
        prev_tokens, prev_len = None, 0
    if allowed is not None:
        allowed = allowed.to(torch.uint8).contiguous()
    out_lp = torch.empty(batch, keep, dtype=torch.float32, device=logits.device)
    out_idx = torch.empty(batch, keep, dtype=torch.int32, device=logits.device)
    check(lib.emu_beam_topk(_ptr(logits), _ptr(rs), batch, beams, V, keep, ban_id, _ptr(prev_tokens), int(prev_len), int(stride),
                            C.c_float(repetition_penalty), 1 if penalty_on_logits else 0, int(no_repeat_ngram), _ptr(allowed),
                            _ptr(out_lp), _ptr(out_idx), _stream()))
    return out_lp, out_idx


def op_attn_decode(q, k_cache, v_cache, pos, start, scale, max_len):
    """q [B,H*D]; caches [B,H,T,D]; pos/start int32 [B] -> [B,H*D]"""
    require_cuda()
    lib = load()
    B, H, T, D = k_cache.shape
    out = torch.empty(B, H * D, dtype=torch.bfloat16, device=q.device)
    rc = lib.emu_op_attn_decode(_ptr(q), _ptr(k_cache), _ptr(v_cache), B, H, D, T, _ptr(pos), _ptr(start),
                                C.c_float(scale), _ptr(out), max_len, _stream())
    check(rc)
    return out


def op_rmsnorm(x, w, eps):
    require_cuda()
    y = torch.empty_like(x)
    check(load().emu_op_rmsnorm(_ptr(x), _ptr(w), _ptr(y), x.shape[0], x.shape[1], C.c_float(eps), _stream()))
    return y


def op_layernorm(x, w, b, eps, residual=None):
    require_cuda()
    y = torch.empty_like(x)
    check(load().emu_op_layernorm(_ptr(x), _ptr(w), _ptr(b), _ptr(residual), _ptr(y), x.shape[0], x.shape[1],
                                  C.c_float(eps), _stream()))
    return y


def launch_count():
    return int(load().emu_launch_count())
