// Device-side pre / post-processing bookends of the hot path (SURVEY.md 8f-3):
//   resize      torchvision.transforms.functional.resize(antialias=True) as the reference calls it in resize_max_res
//               (marigold/util/image_util.py:90-120) and for the final prediction (marigold_depth_pipeline.py:306-312):
//               separable antialiased bilinear / bicubic (PIL-style triangle / Keys a = -0.5 filters whose support grows
//               with the down-scale factor) and nearest-exact; optional uint8 rounding and the [-1, 1] normalisation of
//               marigold_depth_pipeline.py:252-254 fused into the second pass.
//   colorize    colorize_depth_maps (image_util.py:38-76) + chw2hwc + uint8 cast (marigold_depth_pipeline.py:326-331):
//               a 256-entry colour table indexed with int(x * 256), written as HWC uint8.
// Both are HBM-bound streaming kernels; weights are recomputed per output element (a few dozen taps at most).
#include "common.cuh"
#include "kernels.h"
#include "launch.h"

namespace mgb {

__device__ __forceinline__ float aa_filter(float x, int bicubic) {
  x = fabsf(x);
  if (!bicubic) return x < 1.f ? 1.f - x : 0.f;
  const float a = -0.5f;
  if (x < 1.f) return ((a + 2.f) * x - (a + 3.f)) * x * x + 1.f;
  if (x < 2.f) return (((x - 5.f) * x + 8.f) * x - 4.f) * a;
  return 0.f;
}

// One pass along one axis. src element (n, y, x) at n * sn + y * sy + x * sx; the pass resamples the axis of length
// `in_len` (stride s_axis) to `out_len`; the other axis has length `other` (stride s_other). dst is dense
// [n][a][b] with the resampled axis in the position given by `axis_inner` (1: innermost).
template <typename T>
__global__ void __launch_bounds__(256)
    resize_pass_kernel(const T* __restrict__ src, float* __restrict__ dst, int N, int in_len, int out_len, int other,
                       long long sn, long long s_axis, long long s_other, int axis_inner, int mode, int post) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)N * out_len * other;
  const float scale = float(in_len) / float(out_len);
  const int interp = mode == 1 ? 4 : 2;
  const float support = scale >= 1.f ? (interp * 0.5f) * scale : interp * 0.5f;
  const float invscale = scale >= 1.f ? 1.f / scale : 1.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int o, q;
    long long r = i;
    if (axis_inner) { o = int(r % out_len); r /= out_len; q = int(r % other); r /= other; }
    else { q = int(r % other); r /= other; o = int(r % out_len); r /= out_len; }
    const int n = int(r);
    const T* base = src + n * sn + q * s_other;
    float v;
    if (mode == 2) {                                       // nearest-exact: floor((o + 0.5) * scale)
      const int sidx = min(int(floorf((o + 0.5f) * scale)), in_len - 1);
      v = float(base[sidx * s_axis]);
    } else {
      const float center = scale * (o + 0.5f);
      const int xmin = max(int(center - support + 0.5f), 0);
      const int xsize = min(int(center + support + 0.5f), in_len) - xmin;
      // weights normalised first, then accumulated in tap order (the order torch's antialias kernels use)
      float total_w = 0.f;
      for (int j = 0; j < xsize; ++j) total_w += aa_filter((j + xmin - center + 0.5f) * invscale, mode == 1);
      const float inv_total = total_w != 0.f ? 1.f / total_w : 0.f;
      float acc = 0.f;
      for (int j = 0; j < xsize; ++j) {
        const float w = aa_filter((j + xmin - center + 0.5f) * invscale, mode == 1) * inv_total;
        acc = fmaf(float(base[(xmin + j) * s_axis]), w, acc);
      }
      v = acc;
    }
    if (post >= 1) v = fminf(fmaxf(rintf(v), 0.f), 255.f);           // the resized image is uint8 in the reference
    if (post == 2) v = __fsub_rn(__fmul_rn(__fdiv_rn(v, 255.0f), 2.0f), 1.0f);   // rgb / 255.0 * 2.0 - 1.0 (depth_pipeline.py:252), un-fused
    dst[i] = v;
  }
}

// src [NC, H, W] (u8 or f32) -> dst f32 [NC, h, w]; tmp: NC * H * w floats. mode: 0 bilinear-aa, 1 bicubic-aa, 2 nearest-exact.
// post: 0 none, 1 round + clamp to [0, 255], 2 round + clamp, then x / 255 * 2 - 1.
int launch_resize(const void* src, int src_is_u8, int NC, int H, int W, float* dst, int h, int w, int mode, int post, float* tmp,
                  cudaStream_t stream) {
  if (NC < 1 || H < 1 || W < 1 || h < 1 || w < 1 || mode < 0 || mode > 2 || post < 0 || post > 2) {
    set_error("resize: bad argument");
    return MGB_ERR_INVALID;
  }
  // horizontal pass (W -> w), intermediate in float like torch's separable implementation (no rounding in between)
  const long long n1 = (long long)NC * H * w;
  if (src_is_u8)
    TRY(launch_pdl("resize", resize_pass_kernel<uint8_t>, grid_for(n1, 256), 256, 0, stream,
                   static_cast<const uint8_t*>(src), tmp, NC, W, w, H, (long long)H * W, 1LL, (long long)W, 1, mode, 0));
  else
    TRY(launch_pdl("resize", resize_pass_kernel<float>, grid_for(n1, 256), 256, 0, stream, static_cast<const float*>(src),
                   tmp, NC, W, w, H, (long long)H * W, 1LL, (long long)W, 1, mode, 0));
  // vertical pass (H -> h)
  const long long n2 = (long long)NC * h * w;
  return launch_pdl("resize", resize_pass_kernel<float>, grid_for(n2, 256), 256, 0, stream, (const float*)tmp, dst, NC, H,
                    h, w, (long long)H * w, (long long)w, 1LL, 0, mode, post);
}

// depth f32 [HW] -> uint8 [HW][3] (HWC); lut: uint8 [256][3] = (colormap LUT * 255) truncated, as the reference casts
__global__ void __launch_bounds__(256)
    colorize_kernel(const float* __restrict__ depth, long long HW, float dmin, float dmax, const uint8_t* __restrict__ lut,
                    uint8_t* __restrict__ out) {
  __shared__ uint8_t s_lut[768];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) s_lut[i] = lut[i];
  __syncthreads();
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    float d = (depth[p] - dmin) / (dmax - dmin);
    d = fminf(fmaxf(d, 0.f), 1.f);
    const int idx = min(int(d * 256.f), 255);               // matplotlib: int(x * N), x == 1 -> N - 1
    out[3 * p + 0] = s_lut[3 * idx + 0];
    out[3 * p + 1] = s_lut[3 * idx + 1];
    out[3 * p + 2] = s_lut[3 * idx + 2];
  }
}

int launch_colorize(const float* depth, long long HW, float dmin, float dmax, const uint8_t* lut, uint8_t* out,
                    cudaStream_t stream) {
  if (!depth || !lut || !out || HW < 1 || !(dmax > dmin)) { set_error("colorize: bad argument"); return MGB_ERR_INVALID; }
  return launch_plain("colorize", colorize_kernel, grid_for(HW, 256), 256, 0, stream, depth, HW, dmin, dmax, lut, out);
}

}  // namespace mgb
