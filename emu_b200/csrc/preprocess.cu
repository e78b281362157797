// emu_b200 — image pre-processing on the GPU (SURVEY.md §8f-2): the step just before the ViT on every path,
//   TF.Resize((S, S), interpolation=BICUBIC) -> TF.ToTensor() -> TF.Normalize(mean, std)
// (Emu2/emu/chat.py:35-39, Emu2/emu/diffusion.py:59-63, Emu1/models/pipeline.py:59-63).  On a PIL image torchvision's
// Resize is Pillow's ImagingResample (libImaging/Resample.c): separable, fixed point on uint8, horizontal pass first,
// each pass rounded and clipped to uint8 — integer/byte work, restated here bit-exactly:
//   host : per-output-pixel windows and coefficients exactly as Pillow's precompute_coeffs + normalize_coeffs_8bpc
//          (double arithmetic, 22 fractional bits)
//   GPU  : pass 1  tmp[y, xx, c]  = clip8((2^21 + sum_x in[y, xmin+x, c] * k[xx, x]) >> 22)
//          pass 2  out[c, yy, xx] = ((clip8(...) / 255) - mean[c]) / std[c]      fp32 (IEEE divisions) or bf16 (RNE)
// Parity: tests/test_ops_gpu.py::test_preprocess_image — bit-exact against oracle/preprocess_oracle.py, which is itself
// pinned bit-exactly to the reference's own torchvision + Pillow transform (tests/test_oracle_cpu.py).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <vector>

#include "common.cuh"
#include "engine.h"

namespace emu {

constexpr int kPrecisionBits = 32 - 8 - 2;

static double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Pillow precompute_coeffs (in0 = 0, in1 = in_size) + normalize_coeffs_8bpc
static int precompute_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& kk) {
  const double scale = (double)in_size / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * filterscale;
  const int ksize = (int)std::ceil(support) * 2 + 1;
  bounds.assign((size_t)out_size * 2, 0);
  kk.assign((size_t)out_size * ksize, 0);
  std::vector<double> w(ksize);
  const double ss = 1.0 / filterscale;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = bicubic_filter((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    for (int x = 0; x < xmax; ++x) {
      const double v = ww != 0.0 ? w[x] / ww : w[x];
      kk[(size_t)xx * ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << kPrecisionBits)) : (int)(0.5 + v * (1 << kPrecisionBits));
    }
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
  }
  return ksize;
}

__device__ __forceinline__ int clip8(int v) {
  v >>= kPrecisionBits;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// horizontal pass: input rows [y0, y0 + H) of in [*, W, 3] -> out [H, outW, 3]; image blockIdx.y of a batch at in_bs / out_bs
// bytes.  The tables may cover a window of the resized width only (the CLIP centre crop): a pass is separable, so the
// columns it computes do not depend on the ones it skips.
__global__ void resample_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int H, int W, int outW,
                                  const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, int y0, long in_bs,
                                  long out_bs) {
  in += blockIdx.y * in_bs;
  out += blockIdx.y * out_bs;
  const long total = (long)H * outW;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int xx = (int)(idx % outW);
    const long y = idx / outW;
    const int x0 = bounds[2 * xx], n = bounds[2 * xx + 1];
    const int* k = kk + (long)xx * ksize;
    const uint8_t* p = in + ((y0 + y) * W + x0) * 3;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int x = 0; x < n; ++x) {
      const int kv = k[x];
      a0 += p[3 * x] * kv;
      a1 += p[3 * x + 1] * kv;
      a2 += p[3 * x + 2] * kv;
    }
    uint8_t* o = out + idx * 3;
    o[0] = (uint8_t)clip8(a0);
    o[1] = (uint8_t)clip8(a1);
    o[2] = (uint8_t)clip8(a2);
  }
}

// vertical pass + ToTensor + Normalize: columns [x0, x0 + outW) of in [*, in_w, 3] uint8 -> out [3, outH, outW] fp32 / bf16.
// has_v == 0: no resize, output row yy is input row y0 + yy.  Batch as in resample_h_kernel (out_bs in elements).
struct NormParams {
  float mean[3], stdv[3];
};
__global__ void resample_v_norm_kernel(const uint8_t* __restrict__ in, void* out, int H, int outH, int outW,
                                       const int* __restrict__ bounds, const int* __restrict__ kk, int ksize, int has_v,
                                       NormParams np, int out_bf16, int in_w, int x0, int y0, long in_bs, long out_bs) {
  in += blockIdx.y * in_bs + (long)x0 * 3;
  const long plane = (long)outH * outW;
  const long obase = blockIdx.y * out_bs;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < plane; idx += (long)gridDim.x * blockDim.x) {
    const int xx = (int)(idx % outW);
    const int yy = (int)(idx / outW);
    int u[3];
    if (has_v) {
      const int r0 = bounds[2 * yy], n = bounds[2 * yy + 1];
      const int* k = kk + (long)yy * ksize;
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int y = 0; y < n; ++y) {
        const uint8_t* p = in + ((long)(r0 + y) * in_w + xx) * 3;
        const int kv = k[y];
        a0 += p[0] * kv;
        a1 += p[1] * kv;
        a2 += p[2] * kv;
      }
      u[0] = clip8(a0); u[1] = clip8(a1); u[2] = clip8(a2);
    } else {
      const uint8_t* p = in + ((long)(y0 + yy) * in_w + xx) * 3;
      u[0] = p[0]; u[1] = p[1]; u[2] = p[2];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float f = __fdiv_rn(__fsub_rn(__fdiv_rn((float)u[c], 255.0f), np.mean[c]), np.stdv[c]);
      if (out_bf16) reinterpret_cast<bf16*>(out)[obase + c * plane + idx] = __float2bfloat16_rn(f);
      else reinterpret_cast<float*>(out)[obase + c * plane + idx] = f;
    }
  }
}

// image post-processing tail (Emu2/emu/diffusion.py:218-234): numpy_to_pil's (images * 255).round().astype("uint8") on the
// [0, 1] fp32 image the VAE decode produced — round-half-to-even, like numpy
__global__ void to_uint8_kernel(const float* __restrict__ x, uint8_t* __restrict__ y, long n) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float v = rintf(__fmul_rn(x[i], 255.0f));
    y[i] = (uint8_t)(v < 0.f ? 0.f : (v > 255.f ? 255.f : v));
  }
}

// ---- CLIPImageProcessor (the safety checker's feature extractor) ----
// resize so that the shortest edge is `size` (long edge int(size * long / short), transformers get_resize_output_image_size),
// PIL bicubic on uint8, then the centre crop top = (h' - crop) // 2, left = (w' - crop) // 2.  Only the crop window of the
// resized image is computed: the coefficient tables are sliced to it, and the horizontal pass runs only over the input rows
// the window's vertical taps reach.
int clip_plan(int H, int W, int size, int crop, ClipPlan* p) {
  if (H < 1 || W < 1 || size < 1 || crop < 1) return EMU_ERR_INVALID;
  const int sh = H <= W ? H : W, lo = H <= W ? W : H;
  const int rl = (int)((double)((long)size * lo) / sh);
  p->H = H; p->W = W; p->crop = crop;
  p->rh = H <= W ? size : rl;
  p->rw = H <= W ? rl : size;
  if (crop > p->rh || crop > p->rw) return EMU_ERR_INVALID;
  p->top = (p->rh - crop) / 2;
  p->left = (p->rw - crop) / 2;
  p->need_h = p->rw != W;
  p->need_v = p->rh != H;
  std::vector<int> bh, kh, bv, kv;
  p->ksh = p->need_h ? precompute_coeffs(W, p->rw, bh, kh) : 0;
  p->ksv = p->need_v ? precompute_coeffs(H, p->rh, bv, kv) : 0;
  // rows of the input the vertical window reads (all of the crop rows when there is no vertical resize)
  p->row0 = p->top;
  p->rows = crop;
  if (p->need_v) {
    int r0 = H, r1 = 0;
    for (int yy = p->top; yy < p->top + crop; ++yy) {
      r0 = bv[2 * yy] < r0 ? bv[2 * yy] : r0;
      r1 = bv[2 * yy] + bv[2 * yy + 1] > r1 ? bv[2 * yy] + bv[2 * yy + 1] : r1;
    }
    p->row0 = r0;
    p->rows = r1 - r0;
  }
  // table = [bounds_h | coeffs_h | bounds_v | coeffs_v] over the window; vertical starts relative to the first row the
  // horizontal pass produced (it writes rows [row0, row0 + rows) of the input as rows 0.. of its output)
  p->tab.clear();
  p->off_kh = p->off_bv = p->off_kv = 0;
  if (p->need_h) {
    for (int xx = p->left; xx < p->left + crop; ++xx) { p->tab.push_back(bh[2 * xx]); p->tab.push_back(bh[2 * xx + 1]); }
    p->off_kh = p->tab.size();
    p->tab.insert(p->tab.end(), kh.begin() + (size_t)p->left * p->ksh, kh.begin() + (size_t)(p->left + crop) * p->ksh);
  }
  p->off_bv = p->tab.size();
  if (p->need_v) {
    const int base = p->need_h ? p->row0 : 0;
    for (int yy = p->top; yy < p->top + crop; ++yy) { p->tab.push_back(bv[2 * yy] - base); p->tab.push_back(bv[2 * yy + 1]); }
    p->off_kv = p->tab.size();
    p->tab.insert(p->tab.end(), kv.begin() + (size_t)p->top * p->ksv, kv.begin() + (size_t)(p->top + crop) * p->ksv);
  }
  if (p->tab.empty()) p->tab.push_back(0);
  return EMU_OK;
}

size_t clip_tmp_bytes(const ClipPlan& p, int B) { return p.need_h ? (size_t)B * p.rows * p.crop * 3 : 0; }

int clip_launch(const ClipPlan& p, const int* d_tab, const uint8_t* in, int B, uint8_t* tmp, void* out, const float* mean3,
                const float* std3, int out_bf16, cudaStream_t st) {
  const long in_bs = (long)p.H * p.W * 3;
  const uint8_t* v_in = in;
  long v_bs = in_bs;
  int in_w = p.W, x0 = p.left, y0 = p.top;
  if (p.need_h) {
    const long total = (long)p.rows * p.crop;
    const int grid = (int)((total + 255) / 256 < 2 * kNumSMs ? (total + 255) / 256 : 2 * kNumSMs);
    resample_h_kernel<<<dim3(grid, B), 256, 0, st>>>(in, tmp, p.rows, p.W, p.crop, d_tab, d_tab + p.off_kh, p.ksh, p.row0,
                                                     in_bs, (long)p.rows * p.crop * 3);
    count_launch();
    v_in = tmp;
    v_bs = (long)p.rows * p.crop * 3;
    in_w = p.crop; x0 = 0; y0 = 0;  // the horizontal pass already cut the window (rows from row0 == top when no v-resize)
  }
  NormParams np;
  for (int c = 0; c < 3; ++c) { np.mean[c] = mean3[c]; np.stdv[c] = std3[c]; }
  const long plane = (long)p.crop * p.crop;
  const int grid = (int)((plane + 255) / 256 < 2 * kNumSMs ? (plane + 255) / 256 : 2 * kNumSMs);
  resample_v_norm_kernel<<<dim3(grid, B), 256, 0, st>>>(v_in, out, p.rows, p.crop, p.crop, d_tab + p.off_bv,
                                                        d_tab + p.off_kv, p.ksv, p.need_v ? 1 : 0, np, out_bf16, in_w, x0, y0,
                                                        v_bs, 3 * plane);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}

}  // namespace emu

using namespace emu;

extern "C" int emu_image_to_uint8(const float* image01, uint8_t* out, int64_t n, emu_stream_t stream) {
  if (!image01 || !out || n < 1) return EMU_ERR_INVALID;
  const int grid = (int)((n + 255) / 256 < 8 * kNumSMs ? (n + 255) / 256 : 8 * kNumSMs);
  to_uint8_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(image01, out, n);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? EMU_OK : EMU_ERR_CUDA;
}


extern "C" int emu_preprocess_image(const uint8_t* rgb_hwc, int H, int W, int out_h, int out_w, const float* mean3,
                                    const float* std3, void* out_chw, int out_dtype, emu_stream_t stream) {
  if (!rgb_hwc || !out_chw || !mean3 || !std3 || H < 1 || W < 1 || out_h < 1 || out_w < 1) return EMU_ERR_INVALID;
  if (out_dtype != EMU_DTYPE_F32 && out_dtype != EMU_DTYPE_BF16) return EMU_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  const bool need_h = out_w != W, need_v = out_h != H;
  std::vector<int> bh, kh, bv, kv;
  int ksh = 0, ksv = 0;
  if (need_h) ksh = precompute_coeffs(W, out_w, bh, kh);
  if (need_v) ksv = precompute_coeffs(H, out_h, bv, kv);
  // stream-ordered scratch: coefficient tables + the horizontally resampled image
  const size_t n_tab = bh.size() + kh.size() + bv.size() + kv.size();
  int* d_tab = nullptr;
  uint8_t* d_tmp = nullptr;
  if (n_tab && cudaMallocAsync((void**)&d_tab, n_tab * sizeof(int), st) != cudaSuccess) return EMU_ERR_NOMEM;
  int *d_bh = d_tab, *d_kh = d_bh + bh.size(), *d_bv = d_kh + kh.size(), *d_kv = d_bv + bv.size();
  int rc = EMU_OK;
  auto up = [&](int* dst, const std::vector<int>& src) {
    if (!src.empty() && cudaMemcpyAsync(dst, src.data(), src.size() * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = EMU_ERR_CUDA;
  };
  up(d_bh, bh); up(d_kh, kh); up(d_bv, bv); up(d_kv, kv);
  const uint8_t* v_in = rgb_hwc;
  if (!rc && need_h) {
    if (cudaMallocAsync((void**)&d_tmp, (size_t)H * out_w * 3, st) != cudaSuccess) rc = EMU_ERR_NOMEM;
    if (!rc) {
      const long total = (long)H * out_w;
      const int grid = (int)((total + 255) / 256 < 8 * kNumSMs ? (total + 255) / 256 : 8 * kNumSMs);
      resample_h_kernel<<<grid, 256, 0, st>>>(rgb_hwc, d_tmp, H, W, out_w, d_bh, d_kh, ksh, 0, 0, 0);
      v_in = d_tmp;
      count_launch();
    }
  }
  if (!rc) {
    NormParams np;
    for (int c = 0; c < 3; ++c) { np.mean[c] = mean3[c]; np.stdv[c] = std3[c]; }
    const long plane = (long)out_h * out_w;
    const int grid = (int)((plane + 255) / 256 < 8 * kNumSMs ? (plane + 255) / 256 : 8 * kNumSMs);
    resample_v_norm_kernel<<<grid, 256, 0, st>>>(v_in, out_chw, H, out_h, out_w, d_bv, d_kv, ksv, need_v ? 1 : 0, np,
                                                 out_dtype == EMU_DTYPE_BF16 ? 1 : 0, out_w, 0, 0, 0, 0);
    count_launch();
    if (cudaGetLastError() != cudaSuccess) rc = EMU_ERR_CUDA;
  }
  if (d_tmp) cudaFreeAsync(d_tmp, st);
  if (d_tab) cudaFreeAsync(d_tab, st);
  return rc;
}

extern "C" int emu_preprocess_clip(const uint8_t* images_bhwc, int B, int H, int W, int size, int crop, const float* mean3,
                                   const float* std3, void* out_bchw, int out_dtype, emu_stream_t stream) {
  if (!images_bhwc || !out_bchw || !mean3 || !std3 || B < 1 || H < 1 || W < 1 || size < 1 || crop < 1) return EMU_ERR_INVALID;
  if (out_dtype != EMU_DTYPE_F32 && out_dtype != EMU_DTYPE_BF16) return EMU_ERR_INVALID;
  ClipPlan p;
  if (clip_plan(H, W, size, crop, &p) != EMU_OK) return EMU_ERR_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int* d_tab = nullptr;
  uint8_t* d_tmp = nullptr;
  if (cudaMallocAsync((void**)&d_tab, p.tab.size() * sizeof(int), st) != cudaSuccess) return EMU_ERR_NOMEM;
  int rc = cudaMemcpyAsync(d_tab, p.tab.data(), p.tab.size() * sizeof(int), cudaMemcpyHostToDevice, st) == cudaSuccess
               ? EMU_OK : EMU_ERR_CUDA;
  const size_t tb = clip_tmp_bytes(p, B);
  if (!rc && tb && cudaMallocAsync((void**)&d_tmp, tb, st) != cudaSuccess) rc = EMU_ERR_NOMEM;
  if (!rc) rc = clip_launch(p, d_tab, images_bhwc, B, d_tmp, out_bchw, mean3, std3, out_dtype == EMU_DTYPE_BF16, st);
  if (d_tmp) cudaFreeAsync(d_tmp, st);
  cudaFreeAsync(d_tab, st);
  return rc;
}
