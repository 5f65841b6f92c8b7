// Streaming (HBM-bound) helpers around the tensor-core kernels: layout changes that feed TMA
// (space-to-depth parity planes for stride-2 convs, nearest x2 upsampling, latent
// packing), the ABI's NCHW<->NHWC conversions, the tiny dense layers (time MLP, text K/V) and a row softmax. All use 128-bit accesses where the layout allows.
#include "common.cuh"
#include "kernels.h"
#include "launch.h"

namespace mgb {

// x fp32 [NB, H, W, C] -> y bf16 [NB, 4, ceil(H/2), ceil(W/2), C], plane = (h & 1) * 2 + (w & 1); plane elements whose
// source pixel lies outside the image (odd H or W) are zero = the convolution's zero padding there.
__global__ void s2d_kernel(const float4* __restrict__ x, uint2* __restrict__ y, int NB, int H, int W, int Q) {
  pdl_launch_dependents();
  pdl_wait();
  const int H2 = (H + 1) / 2, W2 = (W + 1) / 2;
  const size_t total = (size_t)NB * 4 * H2 * W2 * Q;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = int(i % Q);
    size_t r = i / Q;
    const int w2 = int(r % W2); r /= W2;
    const int h2 = int(r % H2); r /= H2;
    const int plane = int(r & 3);
    const int n = int(r >> 2);
    const int h = 2 * h2 + (plane >> 1), w = 2 * w2 + (plane & 1);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (h < H && w < W) v = __ldg(x + (((size_t)n * H + h) * W + w) * Q + q);
    y[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
}
int launch_space_to_depth(const float* x, bf16* y, int NB, int H, int W, int C, cudaStream_t stream) {
  if (C % 4 || H < 1 || W < 1) { set_error("space_to_depth: C %% 4 == 0 required"); return MGB_ERR_INVALID; }
  const size_t n = (size_t)NB * 4 * ((H + 1) / 2) * ((W + 1) / 2) * (C / 4);
  return launch_pdl("space_to_depth", s2d_kernel, grid_for(n, 256), 256, 0, stream, reinterpret_cast<const float4*>(x),
                    reinterpret_cast<uint2*>(y), NB, H, W, C / 4);
}

// nearest upsampling to Ho x Wo with Ho in {2H - 1, 2H} (same for W): x fp32 [NB, H, W, C] -> y bf16 [NB, Ho, Wo, C].
// F.interpolate(scale_factor=2, mode="nearest"), or F.interpolate(size=(Ho, Wo), mode="nearest") as diffusers'
// Upsample2D does when the UNet forwards `upsample_size`: for Ho = 2H - 1 the source index floor(d * H / Ho) equals
// d >> 1 for every d < Ho (d = 2k + 1: k + (k + H) / (2H - 1) < k + 1 because k <= H - 2), i.e. x2 then crop.
__global__ void upsample2x_kernel(const float4* __restrict__ x, uint2* __restrict__ y, int NB, int H, int W, int Ho, int Wo,
                                  int Q) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t total = (size_t)NB * Ho * Wo * Q;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = int(i % Q);
    size_t r = i / Q;
    const int w = int(r % Wo); r /= Wo;
    const int h = int(r % Ho);
    const int n = int(r / Ho);
    const float4 v = __ldg(x + (((size_t)n * H + (h >> 1)) * W + (w >> 1)) * Q + q);
    y[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
}
int launch_upsample2x(const float* x, bf16* y, int NB, int H, int W, int C, int Ho, int Wo, cudaStream_t stream) {
  if (C % 4 || (Ho != 2 * H && Ho != 2 * H - 1) || (Wo != 2 * W && Wo != 2 * W - 1)) {
    set_error("upsample2x: C %% 4 != 0 or target %d x %d is not 2x / 2x - 1 of %d x %d", Ho, Wo, H, W);
    return MGB_ERR_INVALID;
  }
  const size_t n = (size_t)NB * Ho * Wo * (C / 4);
  return launch_pdl("upsample2x", upsample2x_kernel, grid_for(n, 256), 256, 0, stream, reinterpret_cast<const float4*>(x),
                    reinterpret_cast<uint2*>(y), NB, H, W, Ho, Wo, C / 4);
}

__global__ void cast_bf16_kernel(const float4* __restrict__ x, uint2* __restrict__ y, size_t n4) {
  pdl_launch_dependents();
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(x + i);
    y[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
}
int launch_cast_bf16(const float* x, bf16* y, size_t n, cudaStream_t stream) {
  if (n % 4) { set_error("cast_bf16: n = %zu is not a multiple of 4", n); return MGB_ERR_INVALID; }
  return launch_pdl("cast bf16", cast_bf16_kernel, grid_for(n / 4, 256), 256, 0, stream,
                    reinterpret_cast<const float4*>(x), reinterpret_cast<uint2*>(y), n / 4);
}

// One thread per output 16-byte group (8 channels): rows [r0, r1) of the 2x image, each a copy of its source group.
__global__ void upsample2x_rows_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int W, int Q, int r0,
                                       size_t total) {
  pdl_launch_dependents();
  pdl_wait();
  const int Wo = 2 * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = int(i % Q);
    const size_t r = i / Q;
    const int w = int(r % Wo);
    const int h = r0 + int(r / Wo);
    y[i] = __ldg(x + ((size_t)(h >> 1) * W + (w >> 1)) * Q + q);
  }
}
int launch_upsample2x_rows(const bf16* x, bf16* y, int H, int W, int C, int r0, int r1, cudaStream_t stream) {
  if (C % 8 || r0 < 0 || r1 <= r0 || r1 > 2 * H) {
    set_error("upsample2x rows: C = %d (a multiple of 8), rows [%d, %d) of %d", C, r0, r1, 2 * H);
    return MGB_ERR_INVALID;
  }
  const size_t n = size_t(r1 - r0) * 2 * W * (C / 8);
  return launch_pdl("upsample2x rows", upsample2x_rows_kernel, grid_for(n, 256), 256, 0, stream,
                    reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), W, C / 8, r0, n);
}

__global__ void copy_rows_kernel(const float4* __restrict__ x, float4* __restrict__ y, size_t n4) {
  pdl_launch_dependents();
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
    y[i] = __ldg(x + i);
}
int launch_copy_rows(const float* x, float* y, long long M, int C, cudaStream_t stream) {
  if (C & 3) { set_error("copy_rows: C = %d is not a multiple of 4", C); return MGB_ERR_INVALID; }
  const size_t n4 = size_t(M) * (C / 4);
  return launch_pdl("copy rows", copy_rows_kernel, grid_for(n4, 256), 256, 0, stream, reinterpret_cast<const float4*>(x),
                    reinterpret_cast<float4*>(y), n4);
}

// UNet conv_in operand (reference marigold_depth_pipeline.py:456-458, marigold_iid_pipeline.py:538-540: rgb latent FIRST):
// out bf16 [M, 64] = [rgb(4) | target(Ct) | zeros], Ct = 4 (depth / normals) or 4 n (IID with n targets), 4 + Ct <= 64
__global__ void pack_latents_kernel(const float4* __restrict__ rgb, const float4* __restrict__ tgt,
                                    uint2* __restrict__ out, int M, int Qt) {
  pdl_launch_dependents();
  pdl_wait();
  const int total = M * 16;  // 16 x 8 B (4 bf16) per 64-channel row
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int m = i >> 4, part = i & 15;
    uint2 o = make_uint2(0, 0);
    if (part == 0) {
      const float4 a = __ldg(rgb + m);
      o = make_uint2(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w));
    } else if (part <= Qt) {
      const float4 b = __ldg(tgt + (size_t)m * Qt + (part - 1));
      o = make_uint2(pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
    }
    out[i] = o;
  }
}
int launch_pack_latents(const float* rgb, const float* tgt, bf16* out, int M, int Ct, cudaStream_t stream) {
  if (Ct < 4 || (Ct & 3) || 4 + Ct > 64) { set_error("pack_latents: target channels %d", Ct); return MGB_ERR_INVALID; }
  return launch_pdl("pack_latents", pack_latents_kernel, grid_for(size_t(M) * 16, 256), 256, 0, stream,
                    reinterpret_cast<const float4*>(rgb), reinterpret_cast<const float4*>(tgt),
                    reinterpret_cast<uint2*>(out), M, Ct / 4);
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int NB, int C, int HW,
                                    float scale) {
  const size_t total = (size_t)NB * C * HW;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = int(i % C);
    const size_t r = i / C;
    const size_t p = r % HW, n = r / HW;
    y[i] = __ldg(x + (n * C + c) * HW + p) * scale;
  }
}
int launch_nchw_to_nhwc(const float* x, float* y, int NB, int C, int HW, float scale, cudaStream_t stream) {
  return launch_plain("nchw_to_nhwc", nchw_to_nhwc_kernel, grid_for((size_t)NB * C * HW, 256), 256, 0, stream, x, y, NB,
                      C, HW, scale);
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int NB, int C, int HW,
                                    float scale) {
  const size_t total = (size_t)NB * C * HW;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t p = i % HW;
    const size_t r = i / HW;
    const int c = int(r % C);
    const size_t n = r / C;
    y[i] = __ldg(x + (n * HW + p) * C + c) * scale;
  }
}
int launch_nhwc_to_nchw(const float* x, float* y, int NB, int C, int HW, float scale, cudaStream_t stream) {
  return launch_plain("nhwc_to_nchw", nhwc_to_nchw_kernel, grid_for((size_t)NB * C * HW, 256), 256, 0, stream, x, y, NB,
                      C, HW, scale);
}

// rgb fp32 NCHW [NB, 3, HW] -> bf16 NHWC-64 (3 real channels + zeros): the VAE encoder conv_in operand
__global__ void pack_rgb_kernel(const float* __restrict__ rgb, uint4* __restrict__ out, int NB, size_t HW) {
  const size_t total = (size_t)NB * HW * 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t m = i >> 3;
    const int part = int(i & 7);
    uint4 o = make_uint4(0, 0, 0, 0);
    if (part == 0) {
      const size_t n = m / HW, p = m % HW;
      const float r = __ldg(rgb + (n * 3 + 0) * HW + p), g = __ldg(rgb + (n * 3 + 1) * HW + p),
                  b = __ldg(rgb + (n * 3 + 2) * HW + p);
      o.x = pack_bf16x2(r, g);
      o.y = pack_bf16x2(b, 0.f);
    }
    out[i] = o;
  }
}
int launch_pack_rgb(const float* rgb_nchw, bf16* out, int NB, int HW, cudaStream_t stream) {
  return launch_plain("pack_rgb", pack_rgb_kernel, grid_for((size_t)NB * HW * 8, 256), 256, 0, stream, rgb_nchw,
                      reinterpret_cast<uint4*>(out), NB, size_t(HW));
}

// One-time weight folding: P[M, N] = A[M, K] B[K, N] in fp32 (32 x 32 tiles through shared memory), written as bf16 into
// a wider row-major matrix: out[m * ldo + col0 + n]. Used at finalize_weights for W_proj_out . W_ff2 (see net.cu).
__global__ void __launch_bounds__(1024) fold_matmul_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                            bf16* __restrict__ out, int M, int N, int K, int ldo, int col0) {
  __shared__ float sa[32][33], sb[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int m = blockIdx.y * 32 + ty, n = blockIdx.x * 32 + tx;
  float acc = 0.f;
  for (int k0 = 0; k0 < K; k0 += 32) {
    sa[ty][tx] = (m < M && k0 + tx < K) ? A[(size_t)m * K + k0 + tx] : 0.f;
    sb[ty][tx] = (k0 + ty < K && n < N) ? B[(size_t)(k0 + ty) * N + n] : 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 32; ++k) acc = fmaf(sa[ty][k], sb[k][tx], acc);
    __syncthreads();
  }
  if (m < M && n < N) out[(size_t)m * ldo + col0 + n] = __float2bfloat16(acc);
}
int launch_fold_matmul(const float* A, const float* B, bf16* out, int M, int N, int K, int ldo, int col0, cudaStream_t stream) {
  dim3 grid((N + 31) / 32, (M + 31) / 32);
  return launch_plain("fold_matmul", fold_matmul_kernel, grid, 1024, 0, stream, A, B, out, M, N, K, ldo, col0);
}

// y[M, N] = act_out(act_in(x)[M, K] W[N, K]^T + b); fp32 everywhere; one warp per output element.
__global__ void __launch_bounds__(256) linear_small_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                           const float* __restrict__ b, float* __restrict__ y, int M,
                                                           int N, int K, int silu_in, int silu_out) {
  const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (long long)M * N) return;
  const int m = int(gw / N), n = int(gw - (long long)m * N);
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) {
    float xv = __ldg(x + (size_t)m * K + k);
    if (silu_in) xv = xv / (1.0f + expf(-xv));
    acc += xv * __ldg(w + (size_t)n * K + k);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    acc += b ? __ldg(b + n) : 0.f;
    if (silu_out) acc = acc / (1.0f + expf(-acc));
    y[(size_t)m * N + n] = acc;
  }
}
int launch_linear_small(const float* x, const float* w, const float* b, float* y, int M, int N, int K, int silu_in,
                        int silu_out, cudaStream_t stream) {
  const long long warps = (long long)M * N;
  return launch_plain("linear_small", linear_small_kernel, int((warps + 7) / 8), 256, 0, stream, x, w, b, y, M, N, K,
                      silu_in, silu_out);
}

// diffusers get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0): emb = [cos(t f) | sin(t f)],
// f_i = exp(-ln(10000) * i / half)   (SURVEY.md App. A.1 step 1)
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ emb, int M, int dim) {
  const int half = dim / 2;
  const int total = M * half;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int m = i / half, j = i - m * half;
    const float f = expf(-logf(10000.0f) * float(j) / float(half));
    const float a = t[m] * f;
    emb[(size_t)m * dim + j] = cosf(a);
    emb[(size_t)m * dim + half + j] = sinf(a);
  }
}
int launch_timestep_embedding(const float* t, float* emb, int M, int dim, cudaStream_t stream) {
  return launch_plain("timestep_embedding", timestep_embedding_kernel, grid_for(size_t(M) * dim / 2, 128), 128, 0, stream,
                      t, emb, M, dim);
}

// Row softmax of fp32 scores s[M, ld] (first n columns valid) -> bf16 probabilities p[M, ld], columns [n, ld) zeroed
// (ld is the K extent of the P V GEMM that follows: a multiple of 64). One CTA per row; the row is read three times
// from L2 (max, sum, write), all math fp32 on unrounded logits.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, bf16* __restrict__ p, int n, int ld) {
  __shared__ float red[32];
  const float* row = s + (size_t)blockIdx.x * ld;
  bf16* out = p + (size_t)blockIdx.x * ld;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, row[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < int(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) sum += __expf(row[i] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < int(blockDim.x >> 5); ++i) sum += red[i];
  const float inv = 1.f / sum;
  for (int i = threadIdx.x; i < ld; i += blockDim.x)
    out[i] = i < n ? __float2bfloat16(__expf(row[i] - mx) * inv) : __float2bfloat16(0.f);
}
int launch_softmax_rows(const float* s, bf16* p, int M, int n, int ld, cudaStream_t stream) {
  return launch_plain("softmax_rows", softmax_rows_kernel, M, 256, 0, stream, s, p, n, ld);
}

// x bf16 [M, N] -> y bf16 [N, ld] (ld >= M; columns [M, ld) zeroed) through a padded smem tile
__global__ void transpose_bf16_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int M, int N, int ld) {
  __shared__ bf16 tile[32][33];
  const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int m = m0 + r, n = n0 + threadIdx.x;
    tile[r][threadIdx.x] = (m < M && n < N) ? x[(size_t)m * N + n] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int n = n0 + r, m = m0 + threadIdx.x;
    if (m < ld && n < N) y[(size_t)n * ld + m] = tile[threadIdx.x][r];
  }
}
int launch_transpose_bf16(const bf16* x, bf16* y, int M, int N, int ld, cudaStream_t stream) {
  dim3 grid((N + 31) / 32, (ld + 31) / 32), block(32, 8);
  return launch_plain("transpose_bf16", transpose_bf16_kernel, grid, block, 0, stream, x, y, M, N, ld);
}

// Decoder input: z = post_quant_conv(latent / scale) (1x1, 4 -> 4, fp32) packed as bf16 NHWC-64.
// reference marigold_depth_pipeline.py:510-512. latent fp32 NCHW [NB, 4, HW].
__global__ void pack_decoder_latent_kernel(const float* __restrict__ lat, const float* __restrict__ w,
                                           const float* __restrict__ b, float inv_scale, uint4* __restrict__ out,
                                           int NB, size_t HW) {
  const size_t total = (size_t)NB * HW * 8;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t m = i >> 3;
    const int part = int(i & 7);
    uint4 o = make_uint4(0, 0, 0, 0);
    if (part == 0) {
      const size_t n = m / HW, p = m % HW;
      float x[4], z[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) x[c] = __ldg(lat + (n * 4 + c) * HW + p) * inv_scale;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float a = __ldg(b + c);
#pragma unroll
        for (int j = 0; j < 4; ++j) a += __ldg(w + c * 4 + j) * x[j];
        z[c] = a;
      }
      o.x = pack_bf16x2(z[0], z[1]);
      o.y = pack_bf16x2(z[2], z[3]);
    }
    out[i] = o;
  }
}
int launch_pack_decoder_latent(const float* latent_nchw, const float* w, const float* b, float inv_scale, bf16* out,
                               int NB, int HW, cudaStream_t stream) {
  return launch_plain("pack_decoder_latent", pack_decoder_latent_kernel, grid_for((size_t)NB * HW * 8, 256), 256, 0,
                      stream, latent_nchw, w, b, inv_scale, reinterpret_cast<uint4*>(out), NB, size_t(HW));
}

__global__ void select_step_kernel(const float* __restrict__ table, int total, const float* __restrict__ sched_k,
                                   float* __restrict__ cur_bias, float* __restrict__ cur_k,
                                   const int* __restrict__ counter, int step) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = step >= 0 ? step : *counter;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < total; j += gridDim.x * blockDim.x)
    cur_bias[j] = table[(size_t)i * total + j];
  if (blockIdx.x == 0 && threadIdx.x < 3) cur_k[threadIdx.x] = sched_k[(size_t)i * 3 + threadIdx.x];
}
int launch_select_step(const float* bias_table, int bias_total, const float* sched_k, float* cur_bias, float* cur_k,
                       const int* counter, int step, cudaStream_t stream) {
  return launch_pdl("select_step", select_step_kernel, grid_for(size_t(bias_total), 256), 256, 0, stream, bias_table,
                    bias_total, sched_k, cur_bias, cur_k, counter, step);
}
__global__ void advance_counter_kernel(int* counter) {
  pdl_launch_dependents();
  pdl_wait();
  *counter += 1;
}
int launch_advance_counter(int* counter, cudaStream_t stream) {
  return launch_pdl("advance_counter", advance_counter_kernel, 1, 1, 0, stream, counter);
}

}  // namespace mgb
