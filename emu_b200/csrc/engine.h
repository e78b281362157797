// emu_b200 — engine state (packed weights, KV cache, workspaces, CUDA graphs) behind the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/emu_b200.h"
#include "ops.h"

namespace emu {

extern unsigned long long g_launches;  // kernels launched by this library (graph replays included)
inline void count_launch(int n = 1) { g_launches += n; }

struct LlmLayer {
  bf16 *wqkv = nullptr, *wo = nullptr, *wgu = nullptr, *wdown = nullptr, *ln1 = nullptr, *ln2 = nullptr;
  // which reference tensors have arrived: q k v o gate up down ln1 ln2 (fused buffers are allocated by the first of their
  // parts, so a pointer check alone cannot tell a complete layer from one that is missing k_proj or up_proj)
  unsigned loaded = 0;
  static constexpr unsigned kAll = 0x1ff;
};
struct VitBlock {
  bf16 *wqkv = nullptr, *bqkv = nullptr, *wproj = nullptr, *bproj = nullptr;
  bf16 *wfc1 = nullptr, *bfc1 = nullptr, *wfc2 = nullptr, *bfc2 = nullptr;
  bf16 *ln1w = nullptr, *ln1b = nullptr, *ln2w = nullptr, *ln2b = nullptr;
  unsigned bias_loaded = 0;  // bit 0 q_bias, bit 1 v_bias (they share the fused qkv bias buffer)
};

constexpr int kLlmMaxRows = 32;  // sequences x beams held in the KV cache

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
};

// slot mode: the host mirror of one slot.  Live at length len, or free and keeping the first `kept` positions of its own row
// (prefix caching; 0 = nothing).  own = how many leading positions of a live slot's table row are its own physical row: its
// whole length while it was never re-parented (grows), the join length of a beam group's first slot, 0 for a forked slot.
struct Slot {
  int len = 0;     // host mirror of d_pos (0 = free)
  int group = -1;  // first slot of its beam group, -1 = free
  int kept = 0, own = 0;
  bool grows = false;
  bool regress = false;  // a regression slot (include/emu_b200_regress.h): joined through emu_llm_regress_join
  bool live() const { return group >= 0; }
  void set_live(int self, int L) { *this = Slot{L, self, 0, L, true}; }
  void set_kept(int K) { *this = Slot{0, -1, K, 0, false}; }
  void set_free() { set_kept(0); }
  void set_fork(const Slot& src) { *this = Slot{src.len, src.group, 0, 0, false}; }  // its table row points into src's
  void advance() {  // a decode step
    if (!live()) return;
    len += 1;
    if (grows) own += 1;
  }
};

struct UNetModel;  // unet.cu
struct VaeModel;   // vae.cu
struct CFormerModel;  // cformer.cu
struct SafetyModel;   // safety.cu

}  // namespace emu

struct EmuEngine {
  EmuConfig cfg{};
  int tp_rank = 0, tp_size = 1;
  void* nccl_comm = nullptr;
  // NVLink peer-memory exchange for the decode loop (tp_exchange.cu); tp_peer[r] = rank r's exchange buffer mapped here
  bool tp_p2p = false;
  bool tp_ll = false;  // row-parallel GEMVs push {value, flag} words to the peers from their epilogue
  bool tp_fold = false;  // ... and the first CTAs of the same GEMV finish the exchange (poll + reduce + residual add) in their tail
  float* tp_comm = nullptr;
  float* tp_peer[8] = {};
  float* dec_part = nullptr;  // this rank's fp32 partial of a row-parallel projection [Bmax, hidden]
  std::string err;
  std::vector<void*> owned;  // every cudaMalloc the engine made

  // ---- LLaMA ----
  int Hl = 0, Fl = 0, Vl = 0;  // local head slots / ffn columns / vocab rows
  int head_start = 0, head_count = 0;  // real heads owned by this rank (head_count <= Hl)
  std::vector<emu::LlmLayer> layers;
  emu::bf16 *embed = nullptr, *final_norm = nullptr, *lm_head = nullptr;
  emu::bf16 *rope_cos = nullptr, *rope_sin = nullptr;
  emu::bf16* kv = nullptr;  // [L][2][Bmax][Hl][T][D]
  int cur_len = 0;
  int cache_B = 0;
  int *d_pos = nullptr, *d_start = nullptr, *d_posoff = nullptr;
  emu::bf16 *proj_up = nullptr, *proj_down = nullptr, *stu_head = nullptr;
  int proj_up_in = 0, proj_up_out = 0, proj_down_in = 0, proj_down_out = 0, stu_in = 0, stu_out = 0;
  // decode workspaces
  emu::bf16 *dec_h = nullptr, *dec_q = nullptr, *dec_attn = nullptr, *dec_act = nullptr, *dec_tmp = nullptr;
  emu::bf16 *dec_xn = nullptr, *dec_qkv = nullptr;  // wide decode (> 8 cache rows) only
  float* dec_attn_ws = nullptr;
  float* sk_ws = nullptr;      // gemm_skinny K-split partial sums (wide decode)
  int* sk_counters = nullptr;
  bool wide_skinny = true;     // EMU_WIDE_SKINNY=0: wide decode projections on gemm_tc instead
  int* kv_indir = nullptr;     // [llm_max_batch][llm_max_seq]: cache row holding token t of sequence b (beam re-parenting)
  bool kv_indir_dirty = false;  // table differs from identity
  bool kv_copy = false;         // EMU_KV_COPY=1: move the cache on a re-parent (HF `_reorder_cache`) instead
  int* dec_counters = nullptr;
  float* dec_logits_local = nullptr;
  float *dec_logits_shard = nullptr, *dec_logits_gather = nullptr;
  // prefill workspaces (grown on demand)
  emu::DevBuf pf_h, pf_xn, pf_qkv, pf_attn, pf_act, pf_tmp, pf_last;
  emu::DevBuf step_idx, step_logits;  // slot-mode prefill: its segment lists and logits rows, and the logits of those rows
  // slot mode (continuous batching, include/emu_b200_slots.h): every cache row is a slot holding its own sequence
  int n_slots = 0;               // > 0: slot mode with this many slots
  std::vector<emu::Slot> slots;  // [n_slots]
  int* d_active = nullptr;       // [kLlmMaxRows] 1 = live slot: the decode step advances its position
  // [kLlmMaxRows] left-pad starts / position offsets of the segments being prefilled (join, extend, mixed step)
  int *d_join_start = nullptr, *d_join_posoff = nullptr;
  int *d_kept_start = nullptr, *d_kept_posoff = nullptr;  // [kLlmMaxRows] a kept slot's real left-pad start / position offset
  // regression slots (include/emu_b200_regress.h), allocated by the first regression join: per slot its feedback
  // [kLlmMaxRows, width] and next output row [kLlmMaxRows]; the projected rows [kLlmMaxRows, width], and the step's decoder
  // inputs / final-normed hidden rows [kLlmMaxRows, hidden]
  emu::bf16 *rg_fb = nullptr, *rg_r = nullptr, *rg_x = nullptr, *rg_h = nullptr;
  int* rg_k = nullptr;
  // speculative decoding (include/emu_b200_spec.h), allocated by the first verify: the verify rows' q|k|v [8, 3 * Hl * D], the
  // verify attention's split workspace and per-head counters, and sp_idx[i] = i (i <= 8: the one segment's cache row 0 and
  // row count n for the packed RoPE / KV append).  spec_n = rows of the last verify at cache length spec_len (0: none).
  emu::bf16* sp_qkv = nullptr;
  float* sp_ws = nullptr;
  int *sp_counters = nullptr, *sp_idx = nullptr;
  int spec_n = 0, spec_len = 0;
  // decode graphs keyed by the baked-in arguments (the last int: 1 = slot mode, whose step advances live rows only;
  // 2 = a regression step, keyed by (B, embeds = its decoder inputs, hidden = out, ban_id = L); 16 + ban_rows = a verify)
  typedef std::tuple<int, const void*, const void*, const void*, const void*, const void*, const void*, int, int> GraphKey;
  std::map<GraphKey, cudaGraphExec_t> graphs;
  std::map<GraphKey, int> graph_nodes;
  bool use_graphs = true;
  cudaStream_t cap_stream = nullptr;

  // ---- ViT ----
  std::vector<emu::VitBlock> vit;
  emu::bf16 *vit_wpatch = nullptr, *vit_bpatch = nullptr, *vit_cls = nullptr, *vit_pos = nullptr;
  emu::bf16 *vit_lnf_w = nullptr, *vit_lnf_b = nullptr;
  int vit_kpad = 0;
  emu::DevBuf vit_x, vit_y, vit_qkv, vit_att, vit_mlp, vit_patches;

  // ---- optional sub-models ----
  emu::UNetModel* unet = nullptr;
  emu::VaeModel* vae = nullptr;
  emu::CFormerModel* cformer = nullptr;
  emu::SafetyModel* safety = nullptr;

  // helpers
  int fail(int code, const std::string& msg) {
    err = msg;
    return code;
  }
  void* dmalloc(size_t bytes);
  int ensure(emu::DevBuf& b, size_t bytes);
};

namespace emu {
// load-time helpers shared by the sub-model files
int to_bf16_device(EmuEngine* e, const void* src, int dtype, size_t n, bf16** out, bool* temp, cudaStream_t st);
int nccl_allreduce_bf16(EmuEngine* e, bf16* buf, size_t n, cudaStream_t st);
int tp_exchange_setup(EmuEngine* e, int (*allgather_bytes)(EmuEngine*, const void*, void*, size_t),
                      int (*allreduce_min_int)(EmuEngine*, int*));
void tp_exchange_teardown(EmuEngine* e);
int tp_reduce_add(EmuEngine* e, const float* part, bf16* h, long n_elem, int pdl, cudaStream_t st);
int tp_gather_logits(EmuEngine* e, const float* shard, float* logits, int B, int pdl, cudaStream_t st);
int tp_ll_prepare(EmuEngine* e, GemvArgs& g, int idx);
int tp_ll_reduce(EmuEngine* e, bf16* h, long n_elem, int idx, int pdl, cudaStream_t st);
unsigned* tp_step_counter(EmuEngine* e);

// preprocess.cu: CLIPImageProcessor (shortest-edge bicubic resize + centre crop) restricted to the crop window
struct ClipPlan {
  int H = 0, W = 0, rh = 0, rw = 0, top = 0, left = 0, crop = 0;
  bool need_h = false, need_v = false;
  int row0 = 0, rows = 0;  // input rows the horizontal pass produces
  int ksh = 0, ksv = 0;
  std::vector<int> tab;    // [bounds_h | coeffs_h | bounds_v | coeffs_v] of the window
  size_t off_kh = 0, off_bv = 0, off_kv = 0;
};
int clip_plan(int H, int W, int size, int crop, ClipPlan* p);
size_t clip_tmp_bytes(const ClipPlan& p, int B);
int clip_launch(const ClipPlan& p, const int* d_tab, const uint8_t* in, int B, uint8_t* tmp, void* out, const float* mean3,
                const float* std3, int out_bf16, cudaStream_t st);

// sub-model entry points
int unet_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim, cudaStream_t st);
int vae_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim, cudaStream_t st);
int cformer_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim, cudaStream_t st);
void unet_destroy(UNetModel*);
void vae_destroy(VaeModel*);
void cformer_destroy(CFormerModel*);
int safety_load_tensor(EmuEngine* e, const std::string& key, const bf16* src, const int64_t* shape, int ndim, cudaStream_t st);
void safety_destroy(SafetyModel*);
}  // namespace emu
