// emu_b200 — device-side generation control for beam search (SURVEY.md §8f-1): the vocabulary-wide part of one HF
// `_beam_search` step (transformers GenerationMixin, driven from Emu2/emu/emu.py:213-229 with num_beams=5,
// length_penalty=-1) — log_softmax, repetition penalty, min-length EOS ban, "+ running beam score" and the top-2·beams
// selection over beams x vocab — as three small kernels instead of full-vocabulary torch ops, and the [batch, 2·beams]
// hypothesis bookkeeping that follows (emu_beam_step) as one more, so that a beam-search step never leaves the device:
// the next tokens and the KV-cache reorder indices are chained device-to-device into the CUDA-graphed decode step and
// the host only reads the "finished" flag every few steps.
#include <cuda_runtime.h>

#include "common.cuh"
#include "engine.h"
#include "ops.h"

namespace emu {

// x[r, :] = log_softmax(x[r, :]) + add[r]     (one 1024-thread CTA per row, fp32, three passes over an L2-resident row)
__global__ void __launch_bounds__(1024) logsoftmax_add_kernel(float* __restrict__ x, const float* __restrict__ add, int V) {
  __shared__ float red[33];
  float* row = x + (long)blockIdx.x * V;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += blockDim.x) m = fmaxf(m, row[i]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = red[threadIdx.x];
    v = warp_max(v);
    if (threadIdx.x == 0) red[32] = v;
  }
  __syncthreads();
  m = red[32];
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x) s += expf(row[i] - m);
  s = block_sum(s, red);
  const float shift = m + logf(s) - (add ? add[blockIdx.x] : 0.f);
  for (int i = threadIdx.x; i < V; i += blockDim.x) row[i] -= shift;
}

// HF RepetitionPenaltyLogitsProcessor on scores that already carry `add[r]`: s < 0 ? s * p : s / p at every previously
// generated token (each distinct token once, like gather -> where -> scatter)
__global__ void rep_penalty_kernel(float* x, const float* __restrict__ add, const int* __restrict__ prev, int prev_len,
                                   int prev_stride, int V, float penalty) {
  const int r = blockIdx.x;
  const int* p = prev + (long)r * prev_stride;
  for (int j = threadIdx.x; j < prev_len; j += blockDim.x) {
    const int t = p[j];
    if (t < 0 || t >= V) continue;
    bool first = true;
    for (int k = 0; k < j; ++k) first = first && (p[k] != t);
    if (!first) continue;
    const float a = add ? add[r] : 0.f;
    float s = x[(long)r * V + t] - a;
    s = s < 0.f ? s * penalty : s / penalty;
    x[(long)r * V + t] = s + a;
  }
}

__global__ void ban_token_kernel(float* x, int V, int ban) {
  if (ban >= 0 && ban < V) x[(long)blockIdx.x * V + ban] = -INFINITY;
}

// HF NoRepeatNGramLogitsProcessor: ban every token that would complete an n-gram already present in the row's generated
// tokens (Emu1/models/modeling_emu.py:110-115 forwards no_repeat_ngram_size to generate)
__global__ void no_repeat_ngram_kernel(float* x, const int* __restrict__ prev, int prev_len, int prev_stride, int V, int n) {
  const int r = blockIdx.x;
  const int* p = prev + (long)r * prev_stride;
  if (prev_len + 1 < n) return;
  const int* tail = p + prev_len - (n - 1);  // the n-1 most recent tokens
  for (int i = threadIdx.x; i + n - 1 < prev_len; i += blockDim.x) {
    bool same = true;
    for (int k = 0; k < n - 1; ++k) same = same && (p[i + k] == tail[k]);
    const int t = p[i + n - 1];
    if (same && t >= 0 && t < V) x[(long)r * V + t] = -INFINITY;
  }
}

// HF PrefixConstrainedLogitsProcessor (Emu1/mm_eval/models/emu.py:97-109): allowed [rows, V] bytes, 0 = banned
__global__ void allowed_mask_kernel(float* x, const unsigned char* __restrict__ allowed, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    if (!allowed[i]) x[i] = -INFINITY;
}

// ----------------------------------------------------------------------------------------------
// One step of the hypothesis bookkeeping of HF's vectorised `_beam_search` (transformers >= 4.50: running beams, finished
// beams, early-stopping heuristic), for all batch rows, in ONE small CTA.  Every array is tiny ([batch, beams] or
// [batch, beams, max_length]); thread 0 of each row's warp makes the decisions in the exact order and fp32 arithmetic of
// the torch formulation (tests/test_generation_cpu.py pins that formulation against the reference's lm.generate), the
// whole CTA then moves the token rows.  Sequences are ping-ponged between two planes (parity of cur_len) so that the
// gathers never read what they write.  When *done is already set the step is a no-op (the host polls `done` only every
// few steps; the decode steps it launched in between are harmless).
// ----------------------------------------------------------------------------------------------
struct BeamStepArgs {
  const float* topk_lp;   // [batch, 2*beams]
  const int* topk_idx;    // [batch, 2*beams] flat beam*V + token
  int batch, beams, vocab, cur_len, max_length, eos_id;
  float fin_div;          // (cur_len + 1) ** length_penalty
  float best_div;         // best_len ** length_penalty
  int early_stopping;     // 0 = False, 1 = True, 2 = "never"
  int* running_seq;       // [2][batch, beams, max_length]
  float* running_scores;  // [batch, beams]
  int* sequences;         // [2][batch, beams, max_length]
  float* beam_scores;     // [batch, beams]
  int* is_finished;       // [batch, beams]
  int* fin_len;           // [batch, beams] length of each finished hypothesis
  int* unsat;             // [batch]  "next_token_hits_criteria / improvement still possible" flag of each row
  int* done;              // [1]
  int* next_tokens;       // [batch * beams] -> emu_llm_decode token_ids
  int* beam_src;          // [batch * beams] -> emu_llm_decode beam_src_idx
};
constexpr int kBeamMaxRows = 8;    // batch rows per call
constexpr int kBeamMaxBeams = 16;

__global__ void __launch_bounds__(256) beam_step_kernel(BeamStepArgs a) {
  __shared__ int s_run_src[kBeamMaxRows][kBeamMaxBeams];   // candidate index feeding each new running beam
  __shared__ int s_fin_src[kBeamMaxRows][kBeamMaxBeams];   // < nb: old finished slot, >= nb: candidate (index - nb)
  __shared__ int s_all_hits[kBeamMaxRows], s_all_fin[kBeamMaxRows], s_unsat[kBeamMaxRows];
  if (*a.done) return;
  const int nb = a.beams, keep = 2 * nb, L = a.max_length, V = a.vocab;
  const int b = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pin = a.cur_len & 1, pout = pin ^ 1;
  const long plane = (long)a.batch * nb * L;
  if (b < a.batch && lane == 0) {
    const float* lp = a.topk_lp + (long)b * keep;
    const int* ix = a.topk_idx + (long)b * keep;
    bool hits[2 * kBeamMaxBeams];
    float run_lp[2 * kBeamMaxBeams];
    bool all_hits = true;
    for (int c = 0; c < keep; ++c) {
      hits[c] = (ix[c] % V == a.eos_id) || (a.cur_len + 1 >= L);
      all_hits = all_hits && hits[c];
      run_lp[c] = lp[c] + (hits[c] ? 1.0f : 0.0f) * -1.0e9f;
    }
    // running beams of the next iteration: top-nb of run_lp (largest first, ties to the lower index)
    float new_run_sc[kBeamMaxBeams];
    {
      bool used[2 * kBeamMaxBeams];
      for (int c = 0; c < keep; ++c) used[c] = false;
      for (int k = 0; k < nb; ++k) {
        int best = -1;
        for (int c = 0; c < keep; ++c)
          if (!used[c] && (best < 0 || run_lp[c] > run_lp[best])) best = c;
        used[best] = true;
        s_run_src[b][k] = best;
        new_run_sc[k] = run_lp[best];
      }
    }
    // finished beams: merge the old ones with the candidates that just finished, keep the best nb
    bool full = true;
    for (int k = 0; k < nb; ++k) full = full && (a.is_finished[b * nb + k] != 0);
    const bool uns = a.unsat[b] != 0;
    float m_sc[3 * kBeamMaxBeams];
    int m_fin[3 * kBeamMaxBeams];
    for (int k = 0; k < nb; ++k) { m_sc[k] = a.beam_scores[b * nb + k]; m_fin[k] = a.is_finished[b * nb + k]; }
    for (int c = 0; c < keep; ++c) {
      const bool just = hits[c] && c < nb;
      float f = lp[c] / a.fin_div;
      f = f + ((full && a.early_stopping == 1) ? 1.0f : 0.0f) * -1.0e9f;
      f = f + (uns ? 0.0f : 1.0f) * -1.0e9f;
      f = f + (just ? 0.0f : 1.0f) * -1.0e9f;
      m_sc[nb + c] = f;
      m_fin[nb + c] = just ? 1 : 0;
    }
    float new_sc[kBeamMaxBeams];
    int new_fin[kBeamMaxBeams], new_len[kBeamMaxBeams];
    {
      bool used[3 * kBeamMaxBeams];
      for (int c = 0; c < 3 * nb; ++c) used[c] = false;
      for (int k = 0; k < nb; ++k) {
        int best = -1;
        for (int c = 0; c < 3 * nb; ++c)
          if (!used[c] && (best < 0 || m_sc[c] > m_sc[best])) best = c;
        used[best] = true;
        s_fin_src[b][k] = best;
        new_sc[k] = m_sc[best];
        new_fin[k] = m_fin[best];
        new_len[k] = best < nb ? a.fin_len[b * nb + best] : a.cur_len + 1;
      }
    }
    bool all_fin = true;
    float worst = 0.f;
    for (int k = 0; k < nb; ++k) {
      all_fin = all_fin && new_fin[k];
      worst = k == 0 ? new_sc[k] : fminf(worst, new_sc[k]);
    }
    const float best_running = new_run_sc[0] / a.best_div;
    bool any_better = false;
    for (int k = 0; k < nb; ++k) any_better = any_better || (best_running > (new_fin[k] ? worst : -1.0e9f));
    for (int k = 0; k < nb; ++k) {
      a.running_scores[b * nb + k] = new_run_sc[k];
      a.beam_scores[b * nb + k] = new_sc[k];
      a.is_finished[b * nb + k] = new_fin[k];
      a.fin_len[b * nb + k] = new_len[k];
      const int c = s_run_src[b][k];
      a.next_tokens[b * nb + k] = ix[c] % V;
      a.beam_src[b * nb + k] = ix[c] / V + b * nb;
    }
    a.unsat[b] = (uns && any_better) ? 1 : 0;
    s_unsat[b] = (uns && any_better) ? 1 : 0;
    s_all_hits[b] = all_hits ? 1 : 0;
    s_all_fin[b] = all_fin ? 1 : 0;
  }
  __syncthreads();
  // move the token rows (whole CTA): plane pin -> plane pout
  const int rows = a.batch * nb;
  for (int i = threadIdx.x; i < rows * L; i += blockDim.x) {
    const int t = i % L, k = (i / L) % nb, bb = i / (L * nb);
    const int* ix = a.topk_idx + (long)bb * keep;
    {  // running sequences
      const int c = s_run_src[bb][k];
      const int src_beam = ix[c] / V;
      a.running_seq[pout * plane + i] = t == a.cur_len ? ix[c] % V : a.running_seq[pin * plane + ((long)bb * nb + src_beam) * L + t];
    }
    {  // finished sequences
      const int m = s_fin_src[bb][k];
      int v;
      if (m < nb) v = a.sequences[pin * plane + ((long)bb * nb + m) * L + t];
      else {
        const int c = m - nb;
        v = t == a.cur_len ? ix[c] % V : a.running_seq[pin * plane + ((long)bb * nb + ix[c] / V) * L + t];
      }
      a.sequences[pout * plane + i] = v;
    }
  }
  if (threadIdx.x == 0) {
    bool improvement = false, all_fin = true, all_hits = true;
    for (int r = 0; r < a.batch; ++r) {
      improvement = improvement || s_unsat[r];
      all_fin = all_fin && s_all_fin[r];
      all_hits = all_hits && s_all_hits[r];
    }
    const bool open_beam = !(all_fin && a.early_stopping == 1);
    if (!(improvement && open_beam && !all_hits)) *a.done = 1;
  }
}

// top-`keep` of each group of n contiguous values (n = beams * V), largest first, ties to the lower index, NaN never
// selected, every index at most once (like torch.topk).  Two levels in ONE launch: the group is cut into slices, one CTA per
// slice keeps the slice in shared memory as order-preserving 64-bit items {key(value), ~index} and extracts its own top-keep
// by repeated block-max; the CTA that finishes a group last merges the per-slice candidates the same way.  (Round 1 walked
// the whole group `keep` times with one CTA: 10 dependent passes over 5 x 32k floats, ~0.4 ms of every beam step.)
constexpr int kTopkThreads = 256;
constexpr int kTopkMaxKeep = 32;
constexpr int kTopkMaxParts = 2 * kNumSMs;
constexpr int kTopkSlice = 4096;  // values per slice (shared-memory items: 32 KB)

__device__ __forceinline__ uint32_t topk_key(float x) {  // monotone map; 0 is reserved for "nothing" (NaN, taken, padding)
  if (x != x) return 0u;
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // -inf -> 0x007fffff > 0
}

// block-wide argmax over `items[0..cnt)`, `rounds` times; winner r goes to out[r] (0 when nothing is left) and is cleared
__device__ __forceinline__ void topk_rounds(unsigned long long* items, int cnt, int rounds, unsigned long long* out,
                                            unsigned long long* s_w /*[8]*/, bool local_index, unsigned base) {
  for (int r = 0; r < rounds; ++r) {
    unsigned long long best = 0ull;
    for (int i = threadIdx.x; i < cnt; i += kTopkThreads) {
      const unsigned long long v = items[i];
      best = v > best ? v : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ov = __shfl_xor_sync(0xffffffffu, best, o);
      best = ov > best ? ov : best;
    }
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = best;
    __syncthreads();
    best = s_w[0];
#pragma unroll
    for (int w = 1; w < kTopkThreads / 32; ++w) best = s_w[w] > best ? s_w[w] : best;
    if (threadIdx.x == 0) out[r] = best;
    if (best != 0ull) {
      // clear the winner: its slot is known from the index (slice level) or found by value (merge level: items are unique)
      if (local_index) {
        if (threadIdx.x == 0) items[(0xffffffffu - (unsigned)(best & 0xffffffffull)) - base] = 0ull;
      } else {
        for (int i = threadIdx.x; i < cnt; i += kTopkThreads)
          if (items[i] == best) items[i] = 0ull;
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kTopkThreads) topk_group_kernel(const float* __restrict__ x, long n, int keep, int parts,
                                                                  unsigned long long* cand /*[groups][parts][keep]*/,
                                                                  int* counters /*[groups]*/, float* out_val, int* out_idx) {
  __shared__ unsigned long long items[kTopkSlice];
  __shared__ unsigned long long s_w[kTopkThreads / 32];
  __shared__ unsigned long long s_out[kTopkMaxKeep];
  __shared__ int s_last;
  const int grp = blockIdx.y, part = blockIdx.x;
  const float* g = x + (long)grp * n;
  const long per = (n + parts - 1) / parts;
  const long lo = (long)part * per;
  const int cnt = (int)max(0L, min(per, n - lo));
  for (int i = threadIdx.x; i < cnt; i += kTopkThreads) {
    const uint32_t k = topk_key(__ldcg(g + lo + i));
    items[i] = k ? (((unsigned long long)k << 32) | (unsigned long long)(0xffffffffu - (unsigned)(lo + i))) : 0ull;
  }
  __syncthreads();
  topk_rounds(items, cnt, keep, s_out, s_w, true, (unsigned)lo);
  unsigned long long* mine = cand + ((long)grp * parts + part) * keep;
  if (threadIdx.x < keep) mine[threadIdx.x] = s_out[threadIdx.x];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(&counters[grp], 1);
    s_last = prev == parts - 1;
    if (s_last) counters[grp] = 0;  // self-reset for the next launch
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // merge: parts * keep candidates (<= 2048 by construction of `parts`)
  const int total = parts * keep;
  const unsigned long long* all = cand + (long)grp * parts * keep;
  for (int i = threadIdx.x; i < total; i += kTopkThreads) items[i] = __ldcg(all + i);
  __syncthreads();
  topk_rounds(items, total, keep, s_out, s_w, false, 0u);
  if (threadIdx.x < keep) {
    const unsigned long long w = s_out[threadIdx.x];
    const unsigned idx = w ? 0xffffffffu - (unsigned)(w & 0xffffffffull) : 0u;
    out_val[(long)grp * keep + threadIdx.x] = w ? __ldcg(g + idx) : -INFINITY;  // nothing left (NaN rows): -inf at index 0
    out_idx[(long)grp * keep + threadIdx.x] = (int)idx;
  }
}

// fallback for groups too large for the sliced kernel: one CTA walks the whole group `keep` times.
// DESTRUCTIVE: every selected entry is overwritten with -inf (the buffer is the decode step's scratch logits).
__global__ void __launch_bounds__(1024) topk_group_walk_kernel(float* x, long n, int keep, float* out_val, int* out_idx) {
  __shared__ float sv[32];
  __shared__ long si[32];
  float* g = x + (long)blockIdx.x * n;
  for (int k = 0; k < keep; ++k) {
    float best = -INFINITY;
    long bi = 0x7fffffffffffffffLL;
    for (long i = threadIdx.x; i < n; i += blockDim.x) {
      const float v = __ldcg(g + i);
      if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const long oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
      best = sv[threadIdx.x];
      bi = si[threadIdx.x];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const long oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (threadIdx.x == 0) {
        const bool any = bi != 0x7fffffffffffffffLL;  // all -inf / NaN rows: report index 0
        out_val[(long)blockIdx.x * keep + k] = best;
        out_idx[(long)blockIdx.x * keep + k] = any ? (int)bi : 0;
        if (any) g[bi] = -INFINITY;
        __threadfence_block();
      }
    }
    __syncthreads();
  }
}

static unsigned long long* g_topk_cand = nullptr;
static int* g_topk_counters = nullptr;
static int topk_groups(float* x, int groups, long n, int keep, float* out_val, int* out_idx, cudaStream_t st) {
  auto walk = [&]() {
    topk_group_walk_kernel<<<groups, 1024, 0, st>>>(x, n, keep, out_val, out_idx);
    return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
  };
  if (keep > kTopkMaxKeep || groups > 64 || n >= 0xffffffffL) return walk();
  if (!g_topk_cand) {  // first use (never under stream capture: the beam step is launched eagerly)
    if (cudaMalloc((void**)&g_topk_cand, (size_t)64 * kTopkSlice * sizeof(unsigned long long)) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMalloc((void**)&g_topk_counters, 64 * sizeof(int)) != cudaSuccess) return EMU_ERR_NOMEM;
    if (cudaMemset(g_topk_counters, 0, 64 * sizeof(int)) != cudaSuccess) return EMU_ERR_CUDA;
  }
  // slices of <= kTopkSlice values, as many as keep the merge inside one slice buffer and fill the SMs across the groups
  long parts = (n + kTopkSlice - 1) / kTopkSlice;
  const long want = (2 * kNumSMs + groups - 1) / groups;
  if (parts < want) parts = want;
  if (parts > kTopkSlice / keep) parts = kTopkSlice / keep;
  if (parts > kTopkMaxParts) parts = kTopkMaxParts;
  if ((n + parts - 1) / parts > kTopkSlice) return walk();  // group too large for this kernel's slice buffer
  topk_group_kernel<<<dim3((unsigned)parts, (unsigned)groups), kTopkThreads, 0, st>>>(x, n, keep, (int)parts, g_topk_cand,
                                                                                     g_topk_counters, out_val, out_idx);
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

// ----------------------------------------------------------------------------------------------
// sampling: HF warper order temperature -> top-k -> top-p, then one multinomial draw per row (Emu2/emu/chat.py:46-57 passes
// do_sample / top_k / top_p / temperature through to GenerationMixin).  Sort-free: both filters are thresholds found by a
// 32-step bitwise search over the order-preserving integer image of the scores, each step one pass over the L2-resident
// row; the draw is an inverse-CDF lookup in index order.  One 1024-thread CTA per row, logits are not modified.
//   top-k : keep x >= (k-th largest x)                         (ties with the k-th value are kept, as `scores < kth` does)
//   top-p : keep x_i iff mass{x > x_i} < top_p                  (== sorted-ascending cumsum <= 1 - top_p removed)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__global__ void __launch_bounds__(1024) sample_kernel(const float* __restrict__ logits, int V, float inv_temp, int top_k,
                                                      float top_p, int ban_id, unsigned long long seed,
                                                      unsigned long long offset, int* out_ids) {
  __shared__ float red[33];
  __shared__ float scan[32];
  __shared__ int s_pick;
  const float* row = logits + (long)blockIdx.x * V;
  const int tid = threadIdx.x;
  auto val = [&](int i) { return i == ban_id ? -INFINITY : row[i] * inv_temp; };
  // row maximum (softmax shift)
  float m = -INFINITY;
  for (int i = tid; i < V; i += 1024) m = fmaxf(m, val(i));
  m = warp_max(m);
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  if (tid < 32) {
    float v = warp_max(red[tid]);
    if (tid == 0) red[32] = v;
  }
  __syncthreads();
  m = red[32];
  __syncthreads();
  // ---- top-k threshold: largest t with count{key >= t} >= k ----
  uint32_t tk = 0;
  if (top_k > 0 && top_k < V) {
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = tk | (1u << bit);
      float cnt = 0.f;
      for (int i = tid; i < V; i += 1024) cnt += order_key(val(i)) >= cand ? 1.f : 0.f;
      cnt = block_sum(cnt, red);
      if (cnt >= (float)top_k) tk = cand;
    }
  }
  // ---- top-p threshold on the top-k-filtered distribution: smallest t with mass{key > t} < top_p * Z ----
  float z = 0.f;
  for (int i = tid; i < V; i += 1024) {
    const float x = val(i);
    z += order_key(x) >= tk ? __expf(x - m) : 0.f;
  }
  z = block_sum(z, red);
  uint32_t tp = 0;
  if (top_p < 1.0f) {
    const float target = top_p * z;
    tp = 0xFFFFFFFFu;
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = tp & ~(1u << bit);
      float mass = 0.f;
      for (int i = tid; i < V; i += 1024) {
        const float x = val(i);
        const uint32_t k = order_key(x);
        mass += (k > cand && k >= tk) ? __expf(x - m) : 0.f;
      }
      mass = block_sum(mass, red);
      if (mass < target) tp = cand;
    }
  }
  const uint32_t thr = tk > tp ? tk : tp;
  // ---- multinomial draw over the kept set, inverse CDF in index order (thread t owns a contiguous index chunk) ----
  const int chunk = (V + 1023) / 1024;
  const int i0 = tid * chunk, i1 = min(V, i0 + chunk);
  float local = 0.f;
  for (int i = i0; i < i1; ++i) {
    const float x = val(i);
    local += (order_key(x) >= thr && x > -INFINITY) ? __expf(x - m) : 0.f;
  }
  // block exclusive scan of `local`
  float incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, incl, o);
    if ((tid & 31) >= o) incl += n;
  }
  if ((tid & 31) == 31) scan[tid >> 5] = incl;
  if (tid == 0) s_pick = -1;
  __syncthreads();
  if (tid < 32) {
    float w = scan[tid], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float n = __shfl_up_sync(0xffffffffu, wi, o);
      if (tid >= o) wi += n;
    }
    scan[tid] = wi - w;  // exclusive prefix of the warp totals
    if (tid == 31) red[32] = wi;
  }
  __syncthreads();
  const float total = red[32];
  const float before = scan[tid >> 5] + incl - local;
  const uint64_t h = mix64(seed ^ mix64(offset * 0x100000001B3ull + blockIdx.x));
  const float u = (float)(h >> 40) * (1.0f / 16777216.0f) * total;  // 24 random bits -> [0, total)
  if (local > 0.f && u >= before && u < before + local) {
    float acc = before;
    int pick = -1;
    for (int i = i0; i < i1; ++i) {
      const float x = val(i);
      if (order_key(x) >= thr && x > -INFINITY) {
        acc += __expf(x - m);
        pick = i;
        if (u < acc) break;
      }
    }
    s_pick = pick;
  }
  __syncthreads();
  if (tid == 0) {
    int pick = s_pick;
    if (pick < 0) {  // rounding at the very end of the CDF: fall back to the arg-max (always kept)
      pick = 0;
    }
    out_ids[blockIdx.x] = pick;
  }
  // arg-max fallback needs the whole block: recompute only in the (rare) miss case
  if (s_pick < 0) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < V; i += 1024) {
      const float x = val(i);
      if (x > best || (x == best && i < bi)) { best = x; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    __shared__ float sv[32];
    __shared__ int si[32];
    if ((tid & 31) == 0) { sv[tid >> 5] = best; si[tid >> 5] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 32; ++w)
        if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
      out_ids[blockIdx.x] = bi;
    }
  }
}

}  // namespace emu

using namespace emu;

extern "C" int emu_sample_tokens(const float* logits, int rows, int vocab, float temperature, int top_k, float top_p,
                                 int ban_id, uint64_t seed, uint64_t offset, int32_t* out_ids, emu_stream_t stream) {
  if (!logits || !out_ids || rows < 1 || vocab < 1 || !(temperature > 0.f)) return EMU_ERR_INVALID;
  if (!(top_p > 0.f)) return EMU_ERR_INVALID;
  sample_kernel<<<rows, 1024, 0, (cudaStream_t)stream>>>(logits, vocab, 1.0f / temperature, top_k, top_p, ban_id,
                                                         (unsigned long long)seed, (unsigned long long)offset, out_ids);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}


extern "C" int emu_beam_topk(float* logits, const float* running_scores, int batch, int beams, int vocab, int keep, int ban_id,
                             const int32_t* prev_tokens, int prev_len, int prev_stride, float repetition_penalty,
                             int penalty_on_logits, int no_repeat_ngram, const uint8_t* allowed, float* out_lp,
                             int* out_idx, emu_stream_t stream) {
  if (!logits || !out_lp || !out_idx || batch < 1 || beams < 1 || vocab < 1 || keep < 1 || (long)keep > (long)beams * vocab)
    return EMU_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  const int rows = batch * beams;
  int nl = 2;
  const bool rep = prev_tokens && prev_len > 0 && repetition_penalty != 1.0f;
  // greedy / sampling apply the processors to the raw logits, beam search to the log-probabilities (HF _sample vs _beam_search)
  if (rep && penalty_on_logits) {
    rep_penalty_kernel<<<rows, 128, 0, st>>>(logits, nullptr, prev_tokens, prev_len, prev_stride, vocab, repetition_penalty);
    ++nl;
  }
  logsoftmax_add_kernel<<<rows, 1024, 0, st>>>(logits, running_scores, vocab);
  if (rep && !penalty_on_logits) {
    rep_penalty_kernel<<<rows, 128, 0, st>>>(logits, running_scores, prev_tokens, prev_len, prev_stride, vocab, repetition_penalty);
    ++nl;
  }
  if (prev_tokens && prev_len > 0 && no_repeat_ngram > 0) {
    no_repeat_ngram_kernel<<<rows, 128, 0, st>>>(logits, prev_tokens, prev_len, prev_stride, vocab, no_repeat_ngram);
    ++nl;
  }
  if (ban_id >= 0) {
    ban_token_kernel<<<rows, 1, 0, st>>>(logits, vocab, ban_id);
    ++nl;
  }
  if (allowed) {
    allowed_mask_kernel<<<2 * kNumSMs, 256, 0, st>>>(logits, allowed, (long)rows * vocab);
    ++nl;
  }
  const int rc = topk_groups(logits, batch, (long)beams * vocab, keep, out_lp, out_idx, st);
  count_launch(nl);
  if (rc != EMU_OK) return rc;
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

extern "C" int emu_beam_step(const float* topk_lp, const int32_t* topk_idx, int batch, int beams, int vocab, int cur_len,
                             int max_length, int eos_id, float fin_div, float best_div, int early_stopping,
                             int32_t* running_seq, float* running_scores, int32_t* sequences, float* beam_scores,
                             int32_t* is_finished, int32_t* fin_len, int32_t* unsat, int32_t* done, int32_t* next_tokens,
                             int32_t* beam_src, emu_stream_t stream) {
  if (!topk_lp || !topk_idx || !running_seq || !running_scores || !sequences || !beam_scores || !is_finished || !fin_len ||
      !unsat || !done || !next_tokens || !beam_src)
    return EMU_ERR_INVALID;
  if (batch < 1 || batch > kBeamMaxRows || beams < 1 || beams > kBeamMaxBeams || cur_len < 0 || cur_len >= max_length)
    return EMU_ERR_INVALID;
  BeamStepArgs a;
  a.topk_lp = topk_lp; a.topk_idx = topk_idx; a.batch = batch; a.beams = beams; a.vocab = vocab; a.cur_len = cur_len;
  a.max_length = max_length; a.eos_id = eos_id; a.fin_div = fin_div; a.best_div = best_div; a.early_stopping = early_stopping;
  a.running_seq = running_seq; a.running_scores = running_scores; a.sequences = sequences; a.beam_scores = beam_scores;
  a.is_finished = is_finished; a.fin_len = fin_len; a.unsat = unsat; a.done = done; a.next_tokens = next_tokens;
  a.beam_src = beam_src;
  beam_step_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(a);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}
