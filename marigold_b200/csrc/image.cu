// Device-side pre / post-processing bookends of the hot path (SURVEY.md 8f-3):
//   resize      torchvision.transforms.functional.resize(antialias=True) as the reference calls it in resize_max_res
//               (marigold/util/image_util.py:90-120) and for the final prediction (marigold_depth_pipeline.py:306-312):
//               separable antialiased bilinear / bicubic (PIL-style triangle / Keys a = -0.5 filters whose support grows
//               with the down-scale factor) in the tap-window and weight arithmetic of torch's CPU kernel (the image,
//               resized on the host in the reference) or of torch's CUDA kernel (the prediction), bit for bit, and
//               nearest-exact;
//               optional uint8 rounding and the [-1, 1] normalisation of marigold_depth_pipeline.py:252-254 fused
//               into the second pass.
//   colorize    colorize_depth_maps (image_util.py:38-76) + chw2hwc + uint8 cast (marigold_depth_pipeline.py:326-331):
//               a 256-entry colour table indexed with int(x * 256), written as HWC uint8.
// Both are HBM-bound streaming kernels; weights are recomputed per output element (a few dozen taps at most).
#include "common.cuh"
#include "kernels.h"
#include "launch.h"

namespace mgb {

// The filters as torch's two kernels round them. torch CPU (aten/src/ATen/native/cpu/UpSampleKernel.cpp, compiled with
// FMA contraction in its AVX2 / AVX512 builds) evaluates cubic_convolution1 / 2 of ATen/native/UpSample.h and the
// triangle as float(1.0 - double(x)); torch CUDA (upsample_antialias in ATen/native/cuda/UpSample.cuh) evaluates its
// filter functors in float with nvcc's default contraction. Every rounding is spelled out so the build flags cannot move it.
__device__ __forceinline__ float aa_filter_cpu(float x, int bicubic) {
  x = fabsf(x);
  if (!bicubic) return x < 1.f ? __double2float_rn(1.0 - (double)x) : 0.f;
  if (x < 1.f) return __fmaf_rn(__fmul_rn(__fmaf_rn(1.5f, x, -2.5f), x), x, 1.f);         // ((A+2)x - (A+3)) x x + 1
  if (x < 2.f) return __fmaf_rn(__fmaf_rn(__fmaf_rn(-0.5f, x, 2.5f), x, -4.f), x, 2.f);    // ((Ax - 5A) x + 8A) x - 4A
  return 0.f;
}

__device__ __forceinline__ float aa_filter_cuda(float x, int bicubic) {
  x = fabsf(x);
  if (!bicubic) return x < 1.f ? __fsub_rn(1.f, x) : 0.f;
  if (x < 1.f) return __fmaf_rn(__fmul_rn(__fmaf_rn(1.5f, x, -2.5f), x), x, 1.f);         // ((a+2)x - (a+3)) x x + 1
  if (x < 2.f) return __fmul_rn(__fmaf_rn(__fmaf_rn(__fsub_rn(x, 5.f), x, 8.f), x, -4.f), -0.5f);  // (((x-5)x+8)x-4) a
  return 0.f;
}

// One output's tap window and the filter argument of its j-th tap, in the arithmetic of torch CPU (arith 0:
// _compute_indices_min_size_weights_aa, whose double literals promote the window bounds and the tap offset to double)
// or torch CUDA (arith 1: _compute_weights_span / _compute_weights as nvcc compiles them, all float, offset built as
// j + (xmin - center) with the centre contracted into an FMA). `center` holds the centre in CPU mode and o + 0.5f in
// CUDA mode.
struct AaAxis {
  float scale, support, invscale;
  int in_len, max_taps, arith;
  __device__ AaAxis(int in, int out, int interp, int arith_) : in_len(in), arith(arith_) {
    scale = __fdiv_rn(float(in), float(out));
    support = scale >= 1.f ? __fmul_rn(interp * 0.5f, scale) : interp * 0.5f;
    invscale = scale >= 1.f ? __double2float_rn(1.0 / (double)scale) : 1.f;
    max_taps = int(ceilf(support)) * 2 + 1;
  }
  __device__ __forceinline__ void window(int o, int& xmin, int& xsize, float& center) const {
    if (arith == 0) {
      center = __double2float_rn((double)scale * (o + 0.5));
      xmin = max(int((double)__fsub_rn(center, support) + 0.5), 0);
      xsize = min(int((double)__fadd_rn(center, support) + 0.5), in_len) - xmin;
      xsize = min(max(xsize, 0), max_taps);                        // torch CPU clips a window one tap too long
    } else {
      // nvcc contracts the centre scale * (o + 0.5f) into each of its uses, so it is never rounded on its own: the
      // window bounds are fma(t, scale, -/+support) and the offset base fma(-t, scale, xmin) (see weight())
      center = __fadd_rn(float(o), 0.5f);                        // t; the centre is scale * t, unrounded
      xmin = max(int(__fadd_rn(__fmaf_rn(center, scale, -support), 0.5f)), 0);
      xsize = min(int(__fadd_rn(__fmaf_rn(center, scale, support), 0.5f)), in_len) - xmin;
    }
  }
  __device__ __forceinline__ float weight(int j, int xmin, float center, int bicubic) const {
    if (arith == 0) {
      const float d = __fsub_rn(float(j + xmin), center);
      return aa_filter_cpu(__double2float_rn(((double)d + 0.5) * (double)invscale), bicubic);
    }
    const float d = __fadd_rn(__fadd_rn(float(j), __fmaf_rn(-center, scale, float(xmin))), 0.5f);
    return aa_filter_cuda(__fmul_rn(d, invscale), bicubic);
  }
};

// One pass along one axis. src element (n, y, x) at n * sn + y * sy + x * sx; the pass resamples the axis of length
// `in_len` (stride s_axis) to `out_len`; the other axis has length `other` (stride s_other). dst is dense
// [n][a][b] with the resampled axis in the position given by `axis_inner` (1: innermost).
template <typename T>
__global__ void __launch_bounds__(256)
    resize_pass_kernel(const T* __restrict__ src, float* __restrict__ dst, int N, int in_len, int out_len, int other,
                       long long sn, long long s_axis, long long s_other, int axis_inner, int mode, int arith, int post) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)N * out_len * other;
  const AaAxis ax(in_len, out_len, mode == 1 ? 4 : 2, arith);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int o, q;
    long long r = i;
    if (axis_inner) { o = int(r % out_len); r /= out_len; q = int(r % other); r /= other; }
    else { q = int(r % other); r /= other; o = int(r % out_len); r /= out_len; }
    const int n = int(r);
    const T* base = src + n * sn + q * s_other;
    float v;
    if (mode == 2) {                                       // nearest-exact: floor((o + 0.5) * scale)
      const int sidx = min(int(floorf((o + 0.5f) * ax.scale)), in_len - 1);
      v = float(base[sidx * s_axis]);
    } else {
      int xmin, xsize;
      float center;
      ax.window(o, xmin, xsize, center);
      // both torch kernels sum the raw weights in tap order, divide each by the sum, then accumulate t0 w0 + t1 w1 + ...
      // in tap order. torch CUDA fuses every later tap. torch CPU's compiler vectorises the products of taps 1 .. n - 1
      // four at a time and adds them in order, leaving the last (n - 1) % 4 taps to a scalar epilogue that fuses them.
      float total_w = 0.f;
      for (int j = 0; j < xsize; ++j) total_w = __fadd_rn(total_w, ax.weight(j, xmin, center, mode));
      const int first_fma = arith == 0 ? xsize - (xsize - 1) % 4 : 1;
      v = 0.f;
      for (int j = 0; j < xsize; ++j) {
        float w = ax.weight(j, xmin, center, mode);
        if (total_w != 0.f) w = __fdiv_rn(w, total_w);
        const float t = float(base[(xmin + j) * s_axis]);
        if (j == 0) v = __fmul_rn(t, w);
        else v = j >= first_fma ? __fmaf_rn(t, w, v) : __fadd_rn(v, __fmul_rn(t, w));
      }
    }
    if (post == 1 || post == 2) v = rintf(fminf(fmaxf(v, 0.f), 255.f));      // the resized image is uint8 in the reference
    if (post >= 2) v = __fsub_rn(__fmul_rn(__fdiv_rn(v, 255.0f), 2.0f), 1.0f);   // rgb / 255.0 * 2.0 - 1.0, un-fused
    dst[i] = v;
  }
}

// src [NC, H, W] (u8 or f32) -> dst f32 [NC, h, w]; tmp: NC * H * w floats. mode: 0 bilinear-aa, 1 bicubic-aa, 2 nearest-exact.
// arith: 0 torch CPU, 1 torch CUDA (antialiased modes only). post: 0 none, 1 clamp to [0, 255] + round half to even,
// 2 that, then x / 255 * 2 - 1, 3 x / 255 * 2 - 1 alone.
int launch_resize(const void* src, int src_is_u8, int NC, int H, int W, float* dst, int h, int w, int mode, int arith,
                  int post, float* tmp, cudaStream_t stream) {
  if (NC < 1 || H < 1 || W < 1 || h < 1 || w < 1 || mode < 0 || mode > 2 || arith < 0 || arith > 1 || post < 0 ||
      post > 3) {
    set_error("resize: bad argument");
    return MGB_ERR_INVALID;
  }
  // horizontal pass (W -> w) first, intermediate in float, as both torch kernels do
  const long long n1 = (long long)NC * H * w;
  if (src_is_u8)
    TRY(launch_pdl("resize", resize_pass_kernel<uint8_t>, grid_for(n1, 256), 256, 0, stream,
                   static_cast<const uint8_t*>(src), tmp, NC, W, w, H, (long long)H * W, 1LL, (long long)W, 1, mode, arith,
                   0));
  else
    TRY(launch_pdl("resize", resize_pass_kernel<float>, grid_for(n1, 256), 256, 0, stream, static_cast<const float*>(src),
                   tmp, NC, W, w, H, (long long)H * W, 1LL, (long long)W, 1, mode, arith, 0));
  // vertical pass (H -> h)
  const long long n2 = (long long)NC * h * w;
  return launch_pdl("resize", resize_pass_kernel<float>, grid_for(n2, 256), 256, 0, stream, (const float*)tmp, dst, NC, H,
                    h, w, (long long)H * w, (long long)w, 1LL, 0, mode, arith, post);
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
