// LPIPS of one intrinsic-image target (compute_iid_metric with metric_name "lpips", src/util/metric.py:263-288), as
// torchmetrics' LearnedPerceptualImagePatchSimilarity(net_type=..., normalize=True) scores one image pair. Each net is a
// table of steps (LpNet, built below from torchvision's module definitions) that one launch sequence runs:
//   prep    the maps compute_iid_metric hands the metric (iid_map.cuh: transform, up-to-scale s / k and clamp, invalid
//           elements set to 0), the [0, 1] check, 2 x - 1 and the scaling layer (x - shift) / scale, written as the bf16
//           operand of the first conv (pred, then gt):
//             alex     the pad-2, factor-4 space-to-depth blocks [2, ceil((H+4)/4), ceil((W+4)/4), 64]
//             vgg      NHWC [2, H, W, 64], channels 3..63 zero (as the VAE's conv_in pads its 3 channels)
//             squeeze  the four parity planes [2, 4, ceil(H/2), ceil(W/2), 64] of the stride-2 conv kind, channels 3..63 zero
//   convs   every conv through gemm_tc with a ReLU epilogue that writes the bf16 operand of the next step and, at a
//           tapped layer, the fp32 features the head reads:
//             alex     conv1 11 x 11 stride 4 pad 2 as a 3 x 3 unpadded conv over the blocks (kind 4); conv2 5 x 5 pad 2
//                      (kind 5); conv3..5 3 x 3 pad 1 (kind 0)
//             vgg      the thirteen 3 x 3 pad 1 convs (kind 0), conv1_1 over the 64-channel padded operand
//             squeeze  conv1 3 x 3 stride 2 unpadded: the stride-2 parity-plane kind 3 (input row 2 o + kh, kh = 0..2),
//                      whose output cropped to floor((H - 1) / 2) rows never reads past the image; each Fire module a
//                      1 x 1 squeeze (kind 1, its output padded to 64 channels by zero weight rows and bias), then the
//                      expand1x1 (kind 1) and expand3x3 (kind 0) GEMMs, which write the two halves of one NHWC output
//                      through its row pitch: the concat is never copied
//   pools   on the bf16 outputs (max commutes with rounding: exact): alex 3 x 3 stride 2 floor mode, vgg 2 x 2 stride 2
//           floor mode, squeeze 3 x 3 stride 2 ceil mode (the last window clipped to the input)
//   head    one launch over the L = 5 or 7 layers: per pixel sum_c w_c (f0_c / n0 - f1_c / n1)^2 with
//           n = sqrt(1e-8 + sum f^2) in double from the fp32 features, per-CTA double partials in a fixed order
//   final   the L spatial means, summed in float32 in layer order as Python's sum() adds the float32 means
// Only integer counts and order keys use atomics: equal inputs give equal bits.
#include <algorithm>

#include "common.cuh"
#include "iid_map.cuh"
#include "kernels.h"
#include "launch.h"
#include "ops.h"

namespace mgb {

constexpr int kPrepThreads = 256, kPoolThreads = 256, kHeadThreads = 256, kHeadPix = 64;
constexpr int kHeadMaxC = 512;
// flags: {elements outside [0, 1], max of ~key (the min) and max of key per map over non-NaN values, NaNs per map}
constexpr int kFlags = 7;

// torchmetrics ScalingLayer: shift and scale as float32 tensors
__constant__ float c_lp_shift[3] = {-0.030f, -0.088f, -0.188f};
__constant__ float c_lp_scale[3] = {0.458f, 0.448f, 0.450f};

__device__ __forceinline__ unsigned order_key(float v) {
  const unsigned u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float order_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

// Per-thread input checks of the two maps (torchmetrics' _valid_img and the range its message prints)
struct LpInputFlags {
  unsigned bad = 0, kmin[2] = {0u, 0u}, kmax[2] = {0u, 0u}, nan[2] = {0u, 0u};
};

// Element m of map i, channel c: recorded in f, then 2 m - 1 and the scaling layer in float32
__device__ __forceinline__ float lp_scaled_input(float m, int i, int c, LpInputFlags& f) {
  if (!(m >= 0.f && m <= 1.f)) ++f.bad;      // _valid_img: max <= 1 and min >= 0 (NaN fails)
  if (m != m) {
    ++f.nan[i];
  } else {
    f.kmin[i] = max(f.kmin[i], ~order_key(m));
    f.kmax[i] = max(f.kmax[i], order_key(m));
  }
  const float t = __fsub_rn(__fmul_rn(2.f, m), 1.f);     // normalize=True: 2 x - 1
  return __fdiv_rn(__fsub_rn(t, c_lp_shift[c]), c_lp_scale[c]);
}

__device__ __forceinline__ void lp_flush_flags(const LpInputFlags& f, unsigned* flags) {
  const unsigned bad = __reduce_add_sync(0xffffffffu, f.bad);
  unsigned r[6];
  for (int i = 0; i < 2; ++i) {
    r[2 * i] = __reduce_max_sync(0xffffffffu, f.kmin[i]);
    r[2 * i + 1] = __reduce_max_sync(0xffffffffu, f.kmax[i]);
    r[4 + i] = __reduce_add_sync(0xffffffffu, f.nan[i]);
  }
  if ((threadIdx.x & 31) == 0) {
    if (bad) atomicAdd(flags, bad);
    for (int j = 0; j < 4; ++j)
      if (r[j]) atomicMax(flags + 1 + j, r[j]);
    for (int i = 0; i < 2; ++i)
      if (r[4 + i]) atomicAdd(flags + 5 + i, r[4 + i]);
  }
}

// AlexNet. One thread per padded row rh of a 4 x 4 block, both maps: the 12 channels s2d_channel(rh, 0..3, 0..2), which
// are contiguous; the thread of row 3 also zeroes channels 48..63.
static_assert(s2d_channel(1, 0, 0) - s2d_channel(0, 0, 0) == 12 && s2d_channel(3, 3, 2) == 47,
              "lpips_prep_kernel writes the 12 channels of a block row as one run");
__global__ void __launch_bounds__(kPrepThreads)
    lpips_prep_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask, int H,
                      int W, int transform, const float* __restrict__ sk, int Hb, int Wb, bf16* __restrict__ out,
                      unsigned* __restrict__ flags) {
  const bool scaled = sk != nullptr;
  const float s = scaled ? sk[0] : 1.f, k = scaled ? sk[1] : 1.f;
  const long long HW = (long long)H * W, nb = (long long)Hb * Wb;
  LpInputFlags f;
  for (long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i4 < 4 * nb; i4 += (long long)gridDim.x * blockDim.x) {
    const long long b = i4 >> 2;
    const int rh = int(i4 & 3), bh = int(b / Wb), bw = int(b % Wb), y = 4 * bh + rh - 2;
    float v[2][12];
#pragma unroll
    for (int rw = 0; rw < 4; ++rw) {
      const int x = 4 * bw + rw - 2;
      const bool in = y >= 0 && y < H && x >= 0 && x < W;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float m[2] = {0.f, 0.f};
        if (in) iid_load_mapped(pred, gt, mask, c * HW + (long long)y * W + x, transform, scaled, s, k, &m[0], &m[1]);
#pragma unroll
        for (int i = 0; i < 2; ++i) v[i][s2d_channel(0, rw, c)] = in ? lp_scaled_input(m[i], i, c, f) : 0.f;  // 0: padding
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      bf16* row = out + ((size_t)i * nb + b) * kLpipsS2dC;
      uint2* o = reinterpret_cast<uint2*>(row + s2d_channel(rh, 0, 0));
#pragma unroll
      for (int q = 0; q < 3; ++q)
        o[q] = make_uint2(pack_bf16x2(v[i][4 * q], v[i][4 * q + 1]), pack_bf16x2(v[i][4 * q + 2], v[i][4 * q + 3]));
      if (rh == 3) {
        uint4* z = reinterpret_cast<uint4*>(row + 48);
        z[0] = z[1] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
  lp_flush_flags(f, flags);
}

// VGG16 and SqueezeNet. One thread per pixel of the operand, both maps: 64 channels, the three colours first. parity = 0:
// [2, H, W, 64] (Hs = H, Ws = W); parity = 1: the planes p = (y & 1) * 2 + (x & 1) [2, 4, Hs, Ws, 64] with Hs = ceil(H / 2),
// Ws = ceil(W / 2), zero where the pixel does not exist.
__global__ void __launch_bounds__(kPrepThreads)
    lpips_prep64_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                        int H, int W, int transform, const float* __restrict__ sk, int parity, int Hs, int Ws,
                        bf16* __restrict__ out, unsigned* __restrict__ flags) {
  const bool scaled = sk != nullptr;
  const float s = scaled ? sk[0] : 1.f, k = scaled ? sk[1] : 1.f;
  const long long HW = (long long)H * W, plane = (long long)Hs * Ws, n = parity ? 4 * plane : plane;
  LpInputFlags f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int y, x;
    if (parity) {
      const int p = int(i / plane);
      const long long r = i % plane;
      y = 2 * int(r / Ws) + (p >> 1);
      x = 2 * int(r % Ws) + (p & 1);
    } else {
      y = int(i / Ws);
      x = int(i % Ws);
    }
    const bool in = y < H && x < W;
    float v[2][3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float m[2] = {0.f, 0.f};
      if (in) iid_load_mapped(pred, gt, mask, c * HW + (long long)y * W + x, transform, scaled, s, k, &m[0], &m[1]);
#pragma unroll
      for (int j = 0; j < 2; ++j) v[j][c] = in ? lp_scaled_input(m[j], j, c, f) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      uint4* o = reinterpret_cast<uint4*>(out + ((size_t)j * n + i) * 64);
      o[0] = make_uint4(pack_bf16x2(v[j][0], v[j][1]), pack_bf16x2(v[j][2], 0.f), 0u, 0u);
#pragma unroll
      for (int q = 1; q < 8; ++q) o[q] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  lp_flush_flags(f, flags);
}

// K x K stride 2 max-pool without padding: bf16 NHWC [2, h, w, C] -> [2, ho, wo, C]; 8 channels per thread. A window that
// runs past the input (ceil mode's last one) is clipped to it: the clamped index repeats an element of the window, which
// leaves the max unchanged. In floor mode no index is clamped.
template <int K>
__global__ void __launch_bounds__(kPoolThreads)
    lpips_pool_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int h, int w, int C, int ho, int wo) {
  const int c8 = C / 8;
  const long long total = 2LL * ho * wo * c8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % c8) * 8;
    long long r = i / c8;
    const int ox = int(r % wo); r /= wo;
    const int oy = int(r % ho);
    const int n = int(r / ho);
    __nv_bfloat162 m[4];
#pragma unroll
    for (int dy = 0; dy < K; ++dy)
#pragma unroll
      for (int dx = 0; dx < K; ++dx) {
        const int yy = min(2 * oy + dy, h - 1), xx = min(2 * ox + dx, w - 1);
        const uint4 u = *reinterpret_cast<const uint4*>(x + (((size_t)n * h + yy) * w + xx) * C + c);
        const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) m[j] = (dy == 0 && dx == 0) ? p[j] : __hmax2(m[j], p[j]);
      }
    *reinterpret_cast<uint4*>(y + (((size_t)n * ho + oy) * wo + ox) * C + c) = *reinterpret_cast<const uint4*>(m);
  }
}

struct LpipsHead {
  const float* f[kLpMaxLayers];           // fp32 features [2, npix, C]: pred, then gt
  const float* lin;
  int L;
  int lin_off[kLpMaxLayers], npix[kLpMaxLayers], C[kLpMaxLayers], block0[kLpMaxLayers + 1];
};

__device__ __forceinline__ double warp_allsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;                               // the xor tree leaves the same bits in every lane
}

// One warp per pixel, a block per kHeadPix pixels of one layer. part[block] = sum over its pixels. Channels at or past C
// add exact zeros to the squared norms, so a layer's bits do not depend on kHeadMaxC.
__global__ void __launch_bounds__(kHeadThreads) lpips_head_kernel(const LpipsHead a, double* __restrict__ part) {
  int l = 0;
  while (l < a.L - 1 && int(blockIdx.x) >= a.block0[l + 1]) ++l;
  const int C = a.C[l], npix = a.npix[l];
  const float* f0 = a.f[l];
  const float* f1 = f0 + (size_t)npix * C;
  const float* lin = a.lin + a.lin_off[l];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p0 = (int(blockIdx.x) - a.block0[l]) * kHeadPix;
  double acc = 0.0;
  for (int i = warp; i < kHeadPix && p0 + i < npix; i += kHeadThreads / 32) {
    const size_t base = (size_t)(p0 + i) * C;
    float x[kHeadMaxC / 32], y[kHeadMaxC / 32];
    double s0 = 0.0, s1 = 0.0;
#pragma unroll
    for (int j = 0; j < kHeadMaxC / 32; ++j) {
      const int c = lane + 32 * j;
      x[j] = c < C ? f0[base + c] : 0.f;
      y[j] = c < C ? f1[base + c] : 0.f;
      s0 += double(x[j]) * x[j];
      s1 += double(y[j]) * y[j];
    }
    // torchmetrics _normalize_tensor: x / sqrt(eps + sum_c x^2), eps = 1e-8
    const double n0 = sqrt(1e-8 + warp_allsum(s0)), n1 = sqrt(1e-8 + warp_allsum(s1));
    double d = 0.0;
#pragma unroll
    for (int j = 0; j < kHeadMaxC / 32; ++j) {
      const int c = lane + 32 * j;
      if (c < C) {
        const double t = double(x[j]) / n0 - double(y[j]) / n1;
        d += double(lin[c]) * (t * t);
      }
    }
    acc += warp_allsum(d);
  }
  __shared__ double sh[kHeadThreads / 32];
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kHeadThreads / 32; ++w) t += sh[w];
    part[blockIdx.x] = t;
  }
}

// One warp. out = {lpips, elements outside [0, 1], min pred, max pred, min gt, max gt}
__global__ void lpips_final_kernel(const double* __restrict__ part, const LpipsHead a, const unsigned* __restrict__ flags,
                                   double* __restrict__ out) {
  float sum = 0.f;
  for (int l = 0; l < a.L; ++l) {
    double t = 0.0;
    for (int b = a.block0[l] + int(threadIdx.x); b < a.block0[l + 1]; b += 32) t += part[b];
    t = warp_allsum(t);
    sum = __fadd_rn(sum, float(t / double(a.npix[l])));   // the layer's float32 spatial mean, added in layer order
  }
  if (threadIdx.x != 0) return;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  out[0] = sum;
  out[1] = flags[0];
  for (int i = 0; i < 2; ++i) {                           // torch's min / max: NaN when the map holds a NaN
    const bool has_nan = flags[5 + i] != 0, any = flags[2 + 2 * i] != 0;
    out[2 + 2 * i] = has_nan || !any ? qnan : double(order_value(~flags[1 + 2 * i]));
    out[3 + 2 * i] = has_nan || !any ? qnan : double(order_value(flags[2 + 2 * i]));
  }
}

// ---- the nets: torchvision's features modules and the taps of torchmetrics' vendored lpips pretrained_networks ----
namespace {

struct NetBuilder {
  LpNet n{};
  // conv of torchvision shape [cout, cin, k, k] reading step `in`; n_cols: GEMM columns (cout unless padded); buf / col /
  // ldo: where it writes (default: its own buffer of n_cols columns)
  int conv(int in, int cout, int cin, int k, int kind, int tap, int n_cols = 0, int buf = -1, int col = 0, int ldo = 0) {
    const int c = n.nconv++, s = n.nsteps++;
    n.conv[c] = LpConv{cout, cin, k, n_cols ? n_cols : cout, (cin + 63) / 64 * 64};
    n.step[s] = LpStep{LP_CONV, in, buf < 0 ? s : buf, col, ldo ? ldo : n.conv[c].n, c, kind, tap, true};
    if (tap >= 0) n.C[tap] = n.step[s].ldo;
    return s;
  }
  int pool(int in, int op) {
    const int s = n.nsteps++;
    n.step[s] = LpStep{op, in, s, 0, n.step[in].ldo, -1, -1, -1, true};
    return s;
  }
  // torchvision Fire: squeeze 1 x 1 + ReLU (padded to 64 output channels), then [expand1x1 | expand3x3] + ReLU
  int fire(int in, int cin, int sq, int e, int tap) {
    const int s = conv(in, sq, cin, 1, 1, -1, 64);
    const int e1 = conv(s, e, sq, 1, 1, tap, 0, -1, 0, 2 * e);
    conv(s, e, sq, 3, 0, tap, 0, e1, e, 2 * e);
    return e1;
  }
};

// Extent along one image dimension of every step's output for an input of e pixels
void lp_extents(const LpNet& n, int e, int* out) {
  for (int s = 0; s < n.nsteps; ++s) {
    const LpStep& st = n.step[s];
    const int x = st.in < 0 ? e : out[st.in];
    int o = x;
    if (st.op == LP_CONV && st.kind == 4) {
      o = x + 4 < 11 ? 0 : (x + 4 - 11) / 4 + 1;          // 11 x 11, stride 4, pad 2
    } else if (st.op == LP_CONV && st.kind == 3) {
      o = x < 3 ? 0 : (x - 3) / 2 + 1;                    // 3 x 3, stride 2, unpadded
    } else if (st.op == LP_POOL2) {
      o = x / 2;
    } else if (st.op == LP_POOL3) {
      o = x < 3 ? 0 : (x - 3) / 2 + 1;
    } else if (st.op == LP_POOL3_CEIL) {                  // torch: ceil((x - 3) / 2) + 1, the last window starting inside
      o = x < 2 ? 0 : (x - 2) / 2 + 1;
      if (o > 0 && (o - 1) * 2 >= x) --o;
    }
    out[s] = o;
  }
}

LpNet finish(NetBuilder& b, const char* name, int prep) {
  LpNet& n = b.n;
  n.name = name;
  n.prep = prep;
  for (int s = 0; s < n.nsteps; ++s) {
    n.L = std::max(n.L, n.step[s].tap + 1);
    bool read = false;
    for (int t = s + 1; t < n.nsteps; ++t) read = read || n.step[t].in == n.step[s].buf;
    n.step[s].bf16_out = read;
  }
  int ext[kLpMaxSteps];
  for (n.min_size = 1;; ++n.min_size) {
    lp_extents(n, n.min_size, ext);
    bool ok = true;
    for (int s = 0; s < n.nsteps; ++s) ok = ok && ext[s] > 0;
    if (ok) break;
  }
  return n;
}

LpNet make_alex() {
  NetBuilder b;
  int x = b.conv(-1, 64, 3, 11, 4, 0);
  x = b.pool(x, LP_POOL3);
  x = b.conv(x, 192, 64, 5, 5, 1);
  x = b.pool(x, LP_POOL3);
  x = b.conv(x, 384, 192, 3, 0, 2);
  x = b.conv(x, 256, 384, 3, 0, 3);
  b.conv(x, 256, 256, 3, 0, 4);
  return finish(b, "AlexNet", LP_PREP_S2D4);
}

LpNet make_vgg() {
  NetBuilder b;
  const int level[5][3] = {{64, 64, 0}, {128, 128, 0}, {256, 256, 256}, {512, 512, 512}, {512, 512, 512}};
  int x = -1, cin = 3;
  for (int l = 0; l < 5; ++l) {
    if (l) x = b.pool(x, LP_POOL2);
    const int convs = level[l][2] ? 3 : 2;
    for (int j = 0; j < convs; ++j) {
      x = b.conv(x, level[l][j], cin, 3, 0, j == convs - 1 ? l : -1);
      cin = level[l][j];
    }
  }
  return finish(b, "VGG16", LP_PREP_PLAIN);
}

LpNet make_squeeze() {
  NetBuilder b;
  int x = b.conv(-1, 64, 3, 3, 3, 0);
  x = b.pool(x, LP_POOL3_CEIL);
  x = b.fire(x, 64, 16, 64, -1);
  x = b.fire(x, 128, 16, 64, 1);
  x = b.pool(x, LP_POOL3_CEIL);
  x = b.fire(x, 128, 32, 128, -1);
  x = b.fire(x, 256, 32, 128, 2);
  x = b.pool(x, LP_POOL3_CEIL);
  x = b.fire(x, 256, 48, 192, 3);
  x = b.fire(x, 384, 48, 192, 4);
  x = b.fire(x, 384, 64, 256, 5);
  b.fire(x, 512, 64, 256, 6);
  return finish(b, "SqueezeNet 1.1", LP_PREP_PARITY);
}

}  // namespace

const LpNet* lpips_net(int net) {
  static const LpNet nets[3] = {make_alex(), make_vgg(), make_squeeze()};
  return net >= MGB_LPIPS_ALEX && net <= MGB_LPIPS_SQUEEZE ? &nets[net] : nullptr;
}

// ---- geometry and workspace ----
struct LpipsPlan {
  int ph, pw;                                 // the prep operand's extent (blocks, pixels or plane pixels)
  int h[kLpMaxSteps], w[kLpMaxSteps];         // step outputs
  int bn[kLpMaxSteps], splits[kLpMaxSteps], stages[kLpMaxSteps];
  size_t pre, f[kLpMaxSteps], act[kLpMaxSteps], splitk, part, flags, out, total;
  LpipsHead head;                             // pointers relative to the workspace (filled by launch_lpips)
  int tap_step[kLpMaxLayers];                 // the step that owns each tapped layer's buffer
};

static size_t up256(size_t x) { return (x + 255) & ~size_t(255); }

static int conv_taps(int kind) { return kind == 5 ? 25 : kind == 1 ? 1 : 9; }

static LpipsPlan lpips_plan(const LpNet& n, int H, int W) {
  LpipsPlan p{};
  if (n.prep == LP_PREP_S2D4) {
    p.ph = (H + 4 + 3) / 4; p.pw = (W + 4 + 3) / 4;
  } else if (n.prep == LP_PREP_PARITY) {
    p.ph = (H + 1) / 2; p.pw = (W + 1) / 2;
  } else {
    p.ph = H; p.pw = W;
  }
  lp_extents(n, H, p.h);
  lp_extents(n, W, p.w);
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o = up256(o + bytes); return at; };
  p.pre = take(size_t(2) * (n.prep == LP_PREP_PARITY ? 4 : 1) * p.ph * p.pw * 64 * sizeof(bf16));
  size_t splitk = 0;
  int blocks = 0;
  for (int s = 0; s < n.nsteps; ++s) {
    const LpStep& st = n.step[s];
    const size_t px = size_t(2) * p.h[s] * p.w[s];
    if (st.buf == s) {
      if (st.tap >= 0) p.f[s] = take(px * st.ldo * sizeof(float));
      if (st.bf16_out) p.act[s] = take(px * st.ldo * sizeof(bf16));
    }
    if (st.op != LP_CONV) continue;
    const LpConv& c = n.conv[st.conv];
    int tw, th;
    conv_tile_shape(p.h[s], p.w[s], &tw, &th);
    const int m_tiles = 2 * ((p.w[s] + tw - 1) / tw) * ((p.h[s] + th - 1) / th);
    choose_tile(m_tiles, c.n, conv_taps(st.kind) * c.cin_pad / 64, EPI_RELU, true, &p.bn[s], &p.splits[s], &p.stages[s]);
    if (p.splits[s] > 1) splitk = std::max(splitk, size_t(p.splits[s]) * px * c.n * sizeof(float));
    if (st.tap >= 0 && st.buf == s) {
      const int l = st.tap;
      p.tap_step[l] = s;
      p.head.npix[l] = p.h[s] * p.w[s];
      p.head.C[l] = n.C[l];
      p.head.lin_off[l] = l == 0 ? 0 : p.head.lin_off[l - 1] + n.C[l - 1];
      p.head.block0[l] = blocks;
      blocks += (p.head.npix[l] + kHeadPix - 1) / kHeadPix;
    }
  }
  p.head.L = n.L;
  for (int l = n.L; l <= kLpMaxLayers; ++l) p.head.block0[l] = blocks;
  p.splitk = take(splitk);
  p.part = take(size_t(blocks) * sizeof(double));
  p.flags = take(kFlags * sizeof(unsigned));
  p.out = take(8 * sizeof(double));
  p.total = o;
  return p;
}

size_t lpips_ws_bytes(const LpNet& n, int H, int W) {
  return H >= n.min_size && W >= n.min_size ? lpips_plan(n, H, W).total : 0;
}
const void* lpips_out(const LpNet& n, const void* ws, int H, int W) {
  return static_cast<const char*>(ws) + lpips_plan(n, H, W).out;
}
const float* lpips_features(const LpNet& n, const void* ws, int H, int W, int l, int dims[3]) {
  const LpipsPlan p = lpips_plan(n, H, W);
  const int s = p.tap_step[l];
  dims[0] = p.h[s]; dims[1] = p.w[s]; dims[2] = n.C[l];
  return reinterpret_cast<const float*>(static_cast<const char*>(ws) + p.f[s]);
}
const bf16* lpips_step_output(const LpNet& n, const void* ws, int H, int W, int s, int dims[3]) {
  const LpipsPlan p = lpips_plan(n, H, W);
  const char* w = static_cast<const char*>(ws);
  if (s < 0) {
    dims[0] = p.ph; dims[1] = p.pw; dims[2] = 64;
    return reinterpret_cast<const bf16*>(w + p.pre);
  }
  const int b = n.step[s].buf;
  dims[0] = p.h[b]; dims[1] = p.w[b]; dims[2] = n.step[b].ldo;
  return n.step[b].bf16_out ? reinterpret_cast<const bf16*>(w + p.act[b]) : nullptr;
}

int launch_lpips(const LpNet& n, const float* pred, const float* gt, const uint8_t* mask, int H, int W, int transform,
                 const float* sk, const LpipsWeights& wts, void* ws, cudaStream_t stream) {
  if (H < n.min_size || W < n.min_size) {
    set_error("LPIPS (%s) needs H, W >= %d, got %d x %d", n.name, n.min_size, H, W);
    return MGB_ERR_INVALID;
  }
  LpipsPlan p = lpips_plan(n, H, W);
  char* w = static_cast<char*>(ws);
  auto at = [&](size_t off) { return w + off; };
  unsigned* flags = reinterpret_cast<unsigned*>(at(p.flags));
  CUDA_TRY(cudaMemsetAsync(flags, 0, kFlags * sizeof(unsigned), stream));
  bf16* pre = reinterpret_cast<bf16*>(at(p.pre));
  if (n.prep == LP_PREP_S2D4) {
    TRY(launch_plain("lpips_prep", lpips_prep_kernel, grid_for(size_t(4) * p.ph * p.pw, kPrepThreads), kPrepThreads, 0,
                     stream, pred, gt, mask, H, W, transform, sk, p.ph, p.pw, pre, flags));
  } else {
    const int parity = n.prep == LP_PREP_PARITY;
    TRY(launch_plain("lpips_prep64", lpips_prep64_kernel, grid_for(size_t(parity ? 4 : 1) * p.ph * p.pw, kPrepThreads),
                     kPrepThreads, 0, stream, pred, gt, mask, H, W, transform, sk, parity, p.ph, p.pw, pre, flags));
  }
  auto act = [&](int s) { return s < 0 ? pre : reinterpret_cast<bf16*>(at(p.act[s])); };
  for (int s = 0; s < n.nsteps; ++s) {
    const LpStep& st = n.step[s];
    const bf16* x = act(st.in);
    if (st.op != LP_CONV) {
      const int hi = p.h[st.in], wi = p.w[st.in];
      const dim3 grid = grid_for(size_t(2) * p.h[s] * p.w[s] * st.ldo / 8, kPoolThreads);
      if (st.op == LP_POOL2)
        TRY(launch_plain("lpips_pool2", lpips_pool_kernel<2>, grid, kPoolThreads, 0, stream, x, act(s), hi, wi, st.ldo,
                         p.h[s], p.w[s]));
      else
        TRY(launch_plain("lpips_pool", lpips_pool_kernel<3>, grid, kPoolThreads, 0, stream, x, act(s), hi, wi, st.ldo,
                         p.h[s], p.w[s]));
      continue;
    }
    const LpConv& c = n.conv[st.conv];
    // the source extent of the first conv: the blocks (kind 4) or one parity plane (kind 3)
    const bool first = st.in < 0 && n.prep != LP_PREP_PLAIN;
    GemmParams g;
    TRY(fill_conv_params(&g, x, wts.w[st.conv], 2, p.h[s], p.w[s], c.cin_pad, c.n, st.kind, p.bn[s], p.splits[s],
                         p.stages[s], first ? p.ph : 0, first ? p.pw : 0));
    memset(&g.epi, 0, sizeof(g.epi));
    g.epi.bias = wts.b[st.conv];
    g.epi.out_f32 = st.tap >= 0 ? reinterpret_cast<float*>(at(p.f[st.buf])) + st.col : nullptr;
    g.epi.out_bf16 = st.bf16_out ? act(st.buf) + st.col : nullptr;
    g.epi.ldo = st.ldo;
    g.epi.flags = EPI_RELU;
    g.epi.hw = p.h[s] * p.w[s];
    TRY(run_gemm(g, p.bn[s], reinterpret_cast<float*>(at(p.splitk)), stream));
  }
  LpipsHead head = p.head;
  for (int l = 0; l < n.L; ++l) head.f[l] = reinterpret_cast<const float*>(at(p.f[p.tap_step[l]]));
  head.lin = wts.lin;
  double* part = reinterpret_cast<double*>(at(p.part));
  TRY(launch_plain("lpips_head", lpips_head_kernel, head.block0[n.L], kHeadThreads, 0, stream, head, part));
  return launch_plain("lpips_final", lpips_final_kernel, 1, 32, 0, stream, part, head, flags,
                      reinterpret_cast<double*>(at(p.out)));
}

}  // namespace mgb
