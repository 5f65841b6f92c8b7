// GroupNorm (+SiLU) and LayerNorm over NHWC / token-major fp32 activations -> bf16 GEMM operands.
//
// GroupNorm is ONE launch with a grid-wide barrier in the middle (all CTAs of the grid are co-resident by
// construction: the host caps the grid at the occupancy the kernel is compiled for):
//   phase 1  every CTA reduces its pixel chunk to per-group (sum, sum of squares) in a FIXED order (per-thread
//            fp32 sums -> per-channel slots in shared memory -> 8 lanes per group -> shuffle tree) and stores
//            the 2 G floats to its own slot of a partial buffer: no atomics on data;
//   barrier  one arrival counter per image (RED + acquire spin by one thread per CTA);
//   phase 2  every CTA sums the partials of its image in CTA order (double), which makes the statistics — and
//            with them the whole denoising path — bit-reproducible from run to run (the first version accumulated
//            with fp32 atomics: ~1e-2 run-to-run differences at the worst pixel after bf16 rounding), then
//            normalises + affine (+SiLU) + casts its chunk, whose first round of pixels is still in registers.
// The concat [a | b] of diffusers' up-block resnets is consumed directly (torch.cat is never materialised), and
// the raw bf16 copy for a ResnetBlock's 1x1 shortcut conv is emitted in the same pass.
// Semantics: torch.nn.GroupNorm (biased variance) as used by diffusers ResnetBlock2D / Transformer2DModel / VAE
// blocks; SURVEY.md App. A.1-A.2. Reached from reference marigold_depth_pipeline.py:461-463,491-492,512-513.
#include <algorithm>
#include "common.cuh"
#include "kernels.h"
#include "launch.h"
#include "norm_geom.h"

namespace mgb {

constexpr int kGnPartLoads = 12;  // partial-sum loads in flight per lane in phase 2
constexpr int kGnCtasPerSm = 2;   // __launch_bounds__ below guarantees this residency (<= 128 registers, <= 40 KB smem)

static __device__ __noinline__ void gn_barrier_timeout(unsigned seen, unsigned want) {
  printf("mgb: groupnorm grid barrier timeout block=(%d,%d) arrived=%u of %u\n", blockIdx.x, blockIdx.y, seen, want);
  __trap();
}

template <int KQ>
__global__ void __launch_bounds__(kGnThreads, kGnCtasPerSm)
    gn_fused_kernel(const float* __restrict__ xa, int Ca, const float* __restrict__ xb, int Cb, bf16* __restrict__ y,
                    bf16* __restrict__ raw, const float* __restrict__ gamma, const float* __restrict__ beta, int HW, int G,
                    float eps, int silu, GnGeom g, float2* __restrict__ part /* [NB][chunks][G] */,
                    unsigned* __restrict__ counter /* [NB], zero on entry */) {
  constexpr int R = kGnLoads / KQ;
  extern __shared__ float2 s_ch[];   // phase 1: [Tp][C] per-channel (sum, sumsq); phase 2: mean[G] | rstd[G] as floats
  const int img = blockIdx.y, chunk = blockIdx.x, chunks = gridDim.x;
  const int C = Ca + Cb, cpg = C / G;
  const int tq = threadIdx.x % g.Tq, tp = threadIdx.x / g.Tq;
  const bool active = tp < g.Tp;
  const int p0 = chunk * g.P, p1 = min(HW, p0 + g.P);
  const int Qa = Ca / 4, Qb = Cb / 4;
  const float4* xai = reinterpret_cast<const float4*>(xa + (size_t)img * HW * Ca);
  const float4* xbi = xb ? reinterpret_cast<const float4*>(xb + (size_t)img * HW * Cb) : nullptr;
  pdl_wait();

  // ---- phase 1: first round of pixels (kept in registers for phase 2), further rounds streamed ----
  // quad qd of the concatenated channel space lives in source a (qd < Qa) or b
  auto px = [&](int k, int p) -> const float4* {
    const int qd = tq + k * g.Tq;
    return qd < Qa ? xai + (size_t)p * Qa + qd : xbi + (size_t)p * Qb + (qd - Qa);
  };
  float4 v[KQ][R];
  float sum[KQ][4], sq[KQ][4];
#pragma unroll
  for (int k = 0; k < KQ; ++k) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int p = p0 + tp + r * g.Tp;
      v[k][r] = (active && p < p1) ? __ldg(px(k, p)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { sum[k][j] = 0.f; sq[k][j] = 0.f; }
  }
#pragma unroll
  for (int k = 0; k < KQ; ++k)
#pragma unroll
    for (int r = 0; r < R; ++r) {
      sum[k][0] += v[k][r].x; sq[k][0] = fmaf(v[k][r].x, v[k][r].x, sq[k][0]);
      sum[k][1] += v[k][r].y; sq[k][1] = fmaf(v[k][r].y, v[k][r].y, sq[k][1]);
      sum[k][2] += v[k][r].z; sq[k][2] = fmaf(v[k][r].z, v[k][r].z, sq[k][2]);
      sum[k][3] += v[k][r].w; sq[k][3] = fmaf(v[k][r].w, v[k][r].w, sq[k][3]);
    }
  if (active) {
    for (int pb = p0 + tp + g.Tp * R; pb < p1; pb += g.Tp * R) {   // tensors too large for one round per CTA (VAE)
      float4 w[KQ][R];
#pragma unroll
      for (int k = 0; k < KQ; ++k)
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int p = pb + r * g.Tp;
          w[k][r] = p < p1 ? __ldg(px(k, p)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
      for (int k = 0; k < KQ; ++k)
#pragma unroll
        for (int r = 0; r < R; ++r) {
          sum[k][0] += w[k][r].x; sq[k][0] = fmaf(w[k][r].x, w[k][r].x, sq[k][0]);
          sum[k][1] += w[k][r].y; sq[k][1] = fmaf(w[k][r].y, w[k][r].y, sq[k][1]);
          sum[k][2] += w[k][r].z; sq[k][2] = fmaf(w[k][r].z, w[k][r].z, sq[k][2]);
          sum[k][3] += w[k][r].w; sq[k][3] = fmaf(w[k][r].w, w[k][r].w, sq[k][3]);
        }
    }
#pragma unroll
    for (int k = 0; k < KQ; ++k) {
      float2* dst = s_ch + (size_t)tp * C + 4 * (tq + k * g.Tq);
#pragma unroll
      for (int j = 0; j < 4; ++j) dst[j] = make_float2(sum[k][j], sq[k][j]);
    }
  }
  __syncthreads();
  const int gi = threadIdx.x >> 3, lane8 = threadIdx.x & 7;
  {
    // group partial of this CTA: 8 lanes per group, channels j = lane8, lane8 + 8, ... and pixel lanes in order
    float s = 0.f, q = 0.f;
    if (gi < G) {
      for (int j = lane8; j < cpg; j += 8)
        for (int t = 0; t < g.Tp; ++t) {
          const float2 e = s_ch[(size_t)t * C + gi * cpg + j];
          s += e.x; q += e.y;
        }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (gi < G && lane8 == 0) part[((size_t)img * chunks + chunk) * G + gi] = make_float2(s, q);
  }
  // ---- grid barrier over the CTAs of this image ----
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter + img, 1u);
    unsigned seen;
    const long long t0 = clock64();
    for (;;) {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter + img) : "memory");
      if (seen >= unsigned(chunks)) break;
      if (clock64() - t0 > (1ll << 31)) gn_barrier_timeout(seen, unsigned(chunks));
    }
  }
  __syncthreads();
  // only now may the next kernel's CTAs take SM resources: every CTA of this grid is resident
  pdl_launch_dependents();
  // affine parameters: in flight while the statistics are reduced
  float4 ga4[KQ], be4[KQ];
#pragma unroll
  for (int k = 0; k < KQ; ++k) {
    const int qd = tq + k * g.Tq;
    ga4[k] = gamma ? __ldg(reinterpret_cast<const float4*>(gamma) + qd) : make_float4(1.f, 1.f, 1.f, 1.f);
    be4[k] = beta ? __ldg(reinterpret_cast<const float4*>(beta) + qd) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float* s_stat = reinterpret_cast<float*>(s_ch);
  {
    // every CTA of the image sums the same partials in the same (CTA index) order: identical statistics everywhere,
    // independent of scheduling. Loads bypass L1 (written by other SMs) and are issued kGnPartLoads at a time (this phase
    // is a chain of L2 round trips right behind the barrier: 192 chunks / 8 lanes = 24 entries per lane).
    double s = 0.0, q = 0.0;
    if (gi < G) {
      const float2* pp = part + (size_t)img * chunks * G + gi;
      for (int c0 = lane8; c0 < chunks; c0 += 8 * kGnPartLoads) {
        float2 t[kGnPartLoads];
#pragma unroll
        for (int u = 0; u < kGnPartLoads; ++u) {
          const int c = c0 + 8 * u;
          t[u] = c < chunks ? __ldcg(pp + (size_t)c * G) : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < kGnPartLoads; ++u) { s += double(t[u].x); q += double(t[u].y); }
      }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    __syncthreads();   // s_ch (phase 1) is dead: reuse as s_stat
    if (gi < G && lane8 == 0) {
      const double n = double(HW) * cpg;
      const double mean = s / n;
      double var = q / n - mean * mean;
      if (var < 0.0) var = 0.0;
      s_stat[gi] = float(mean);
      s_stat[G + gi] = rsqrtf(float(var) + eps);
    }
  }
  __syncthreads();
  if (!active) return;
  // ---- phase 2: normalise + affine (+SiLU) + cast ----
  float sc[KQ][4], sh[KQ][4];
#pragma unroll
  for (int k = 0; k < KQ; ++k) {
    const int qd = tq + k * g.Tq;
    const float gav[4] = {ga4[k].x, ga4[k].y, ga4[k].z, ga4[k].w}, bev[4] = {be4[k].x, be4[k].y, be4[k].z, be4[k].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gj = (4 * qd + j) / cpg;
      const float rstd = s_stat[G + gj];
      sc[k][j] = rstd * gav[j];
      sh[k][j] = bev[j] - s_stat[gj] * rstd * gav[j];
    }
  }
  uint2* yo = reinterpret_cast<uint2*>(y + (size_t)img * HW * C);
  uint2* ro = raw ? reinterpret_cast<uint2*>(raw + (size_t)img * HW * C) : nullptr;
  for (int pb = p0 + tp;;) {
#pragma unroll
    for (int k = 0; k < KQ; ++k)
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int p = pb + r * g.Tp;
        if (p < p1) {
          const size_t idx = (size_t)p * g.Q + tq + k * g.Tq;
          const float4 t = v[k][r];
          float o0 = fmaf(t.x, sc[k][0], sh[k][0]), o1 = fmaf(t.y, sc[k][1], sh[k][1]),
                o2 = fmaf(t.z, sc[k][2], sh[k][2]), o3 = fmaf(t.w, sc[k][3], sh[k][3]);
          if (silu) { o0 = silu_f(o0); o1 = silu_f(o1); o2 = silu_f(o2); o3 = silu_f(o3); }
          yo[idx] = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
          if (ro) ro[idx] = make_uint2(pack_bf16x2(t.x, t.y), pack_bf16x2(t.z, t.w));
        }
      }
    pb += g.Tp * R;
    if (pb >= p1) break;
#pragma unroll
    for (int k = 0; k < KQ; ++k)
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int p = pb + r * g.Tp;
        v[k][r] = p < p1 ? __ldg(px(k, p)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
  }
}

// CTAs that are guaranteed co-resident (the grid barrier needs all of them on the device at once)
static int gn_max_ctas() {
  static int v = -1;
  if (v < 0) {
    int dev = 0, sms = 0, occ = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int worst = kGnCtasPerSm;
    const size_t smem = 40 * 1024;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fused_kernel<1>, kGnThreads, smem) == cudaSuccess) worst = std::min(worst, occ);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fused_kernel<2>, kGnThreads, smem) == cudaSuccess) worst = std::min(worst, occ);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gn_fused_kernel<4>, kGnThreads, smem) == cudaSuccess) worst = std::min(worst, occ);
    v = std::max(1, worst) * std::max(1, sms);
  }
  return v;
}

static bool gn_plan(int NB, int HW, int C, int G, GnGeom* g) {
  if (C % G != 0 || G * 8 > kGnThreads || NB < 1) return false;
  const int per_img = std::max(1, std::min(kGnMaxChunks, gn_max_ctas() / NB));
  if (gn_max_ctas() < NB) return false;
  return gn_geometry(HW, C, g, per_img);
}

// scratch of one GroupNorm call: [NB][chunks][G] float2 partials
size_t groupnorm_part_bytes(int NB, int HW, int C, int G) {
  GnGeom g;
  if (!gn_plan(NB, HW, C, G, &g)) return 0;
  return size_t(NB) * g.chunks * G * sizeof(float2);
}
// stand-alone workspace: partials + NB barrier counters
size_t groupnorm_ws_bytes(int NB, int HW, int C, int G) {
  return ((groupnorm_part_bytes(NB, HW, C, G) + 255) & ~size_t(255)) + size_t(NB) * sizeof(unsigned);
}

// GroupNorm(+SiLU) over the channel concat [a | b] (b optional). part: groupnorm_part_bytes() of scratch; counters: NB
// unsigned, ZERO on entry (the network zeroes all counters of a forward with one memset).
int launch_gn_fused(const float* xa, int Ca, const float* xb, int Cb, bf16* y, bf16* raw_copy, const float* gamma,
                    const float* beta, int NB, int HW, int G, float eps, int silu, void* part, unsigned* counters,
                    cudaStream_t stream) {
  GnGeom g;
  const int C = Ca + Cb;
  if ((Ca & 3) || (Cb & 3) || !gn_plan(NB, HW, C, G, &g)) {
    set_error("groupnorm: unsupported NB=%d C=%d+%d G=%d", NB, Ca, Cb, G);
    return MGB_ERR_INVALID;
  }
  dim3 grid(g.chunks, NB);
  const size_t smem = std::max(size_t(g.Tp) * C * sizeof(float2), size_t(2) * G * sizeof(float));
  if (smem > 40 * 1024) { set_error("groupnorm: C=%d needs %zu B of shared memory", C, smem); return MGB_ERR_INVALID; }
  float2* pp = static_cast<float2*>(part);
  auto kern = g.Kq == 1 ? gn_fused_kernel<1> : g.Kq == 2 ? gn_fused_kernel<2> : gn_fused_kernel<4>;
  return launch_pdl("groupnorm", kern, grid, kGnThreads, smem, stream, xa, Ca, xb, Cb, y, raw_copy, gamma, beta, HW, G, eps,
                    silu, g, pp, counters);
}

// Stand-alone GroupNorm (operator-level ABI): ws = groupnorm_ws_bytes() of scratch (counters zeroed here).
int launch_groupnorm(const float* x, bf16* y, bf16* raw_copy, const float* gamma, const float* beta, float* ws,
                     int NB, int HW, int C, int G, float eps, int silu, cudaStream_t stream) {
  const size_t pb = (groupnorm_part_bytes(NB, HW, C, G) + 255) & ~size_t(255);
  unsigned* counters = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(ws) + pb);
  cudaError_t e = cudaMemsetAsync(counters, 0, size_t(NB) * sizeof(unsigned), stream);
  if (e != cudaSuccess) { set_error("groupnorm memset: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  return launch_gn_fused(x, C, nullptr, 0, y, raw_copy, gamma, beta, NB, HW, G, eps, silu, ws, counters, stream);
}

// -------------------------------------------------------------------------------------------------
// LayerNorm: one warp per token, values held in registers (C <= 1280 -> <= 10 float4 per lane).
// Two-pass (mean, then centred variance) like torch.nn.LayerNorm.
// -------------------------------------------------------------------------------------------------
constexpr int kLnMaxQ = 10;
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, bf16* __restrict__ y,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, int M, int C, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= M) return;
  const int Q = C / 4;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)warp * C);
  float4 v[kLnMaxQ];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kLnMaxQ; ++k) {
    const int q = lane + 32 * k;
    if (q < Q) {
      v[k] = __ldg(xr + q);
      s += v[k].x + v[k].y + v[k].z + v[k].w;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < kLnMaxQ; ++k) {
    const int q = lane + 32 * k;
    if (q < Q) {
      const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
      ss += a * a + b * b + c * c + d * d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rstd = rsqrtf(ss / C + eps);
  uint2* yr = reinterpret_cast<uint2*>(y + (size_t)warp * C);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int k = 0; k < kLnMaxQ; ++k) {
    const int q = lane + 32 * k;
    if (q < Q) {
      const float4 ga = __ldg(g4 + q), be = __ldg(b4 + q);
      const float o0 = (v[k].x - mean) * rstd * ga.x + be.x, o1 = (v[k].y - mean) * rstd * ga.y + be.y;
      const float o2 = (v[k].z - mean) * rstd * ga.z + be.z, o3 = (v[k].w - mean) * rstd * ga.w + be.w;
      yr[q] = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
    }
  }
}

// -------------------------------------------------------------------------------------------------
// Cross attention against the FIXED two-token empty-prompt context, collapsed algebraically, fused with the LayerNorm
// before it (norm2) and the one after it (norm3) — one launch instead of LayerNorm + to_q GEMM + attention + to_out GEMM
// + LayerNorm (reference: attn2 of diffusers' BasicTransformerBlock, reached from marigold_depth_pipeline.py:461-463; the
// context is always CLIP(""), :381-394,438-442).
//   softmax over 2 keys: w0 = sigmoid((q . (k0 - k1)) / sqrt(64)) per head, w1 = 1 - w0, and with q = Wq z:
//       q_h . dk_h = z . G_h,            G_h = Wq[h-block, :]^T dk_h                    (G: [H, C])
//   attention output per head = v1_h + w0_h (v0_h - v1_h), and through to_out:
//       Wo a + bo = c1 + sum_h w0_h U_h, c1 = Wo v1 + bo,  U_h = Wo[:, h-block] (v0 - v1)_h   (U: [H, C])
//   so the block is   y = x + c1 + sum_h sigmoid(scale * LN2(x) . G_h) U_h   — exact, C (2 H) MACs per token instead of
//   2 C^2, all in fp32 (the two GEMMs it replaces rounded z, q, a to bf16).
// x fp32 [M, C] -> y bf16 [M, C] (the trunk after attn2: first K-operand of the folded ff.net.2 + proj_out GEMM) and
// a_out bf16 [M, C] = LN3(y) (operand of the feed-forward GEMM).
// -------------------------------------------------------------------------------------------------
// Persistent blocks with the folded tables in shared memory (G, U as bf16 [H][C]; c1 and the two LayerNorm affines fp32):
// re-reading G and U from L1 / L2 for every token would move 13-205 KB per token against 1-5 KB of activations; from
// shared memory the tables cost one conflict-free LDS.64 per quad and head.
// One warp per token, tokens strided over the grid.
__device__ __forceinline__ float4 bf16x4_to_f4(uint2 v) {
  const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(&v.x), b = *reinterpret_cast<const __nv_bfloat162*>(&v.y);
  return make_float4(__bfloat162float(a.x), __bfloat162float(a.y), __bfloat162float(b.x), __bfloat162float(b.y));
}

// QL: quads per lane (ceil(C / 128)): 3 / 5 / 10 for C = 320 / 640 / 1280 — sized exactly so that the small-C levels run at
// 4 blocks per SM (the generic 10-slot version needed 128 registers: 16 warps per SM for a latency-bound kernel)
template <int QL>
__global__ void __launch_bounds__(256, QL <= 3 ? 4 : QL <= 5 ? 3 : 1)
    xattn2_fused_kernel(const float* __restrict__ x, bf16* __restrict__ y, bf16* __restrict__ a_out,
                        const float* __restrict__ g2, const float* __restrict__ b2, const float* __restrict__ g3,
                        const float* __restrict__ b3, const bf16* __restrict__ GU /* [2][H][C] */,
                        const float* __restrict__ c1, int M, int C, int H, float scale, float eps) {
  extern __shared__ __align__(16) uint8_t xs_raw[];
  pdl_launch_dependents();
  const int Q = C / 4;
  uint2* sG = reinterpret_cast<uint2*>(xs_raw);                       // [H][Q] bf16x4
  uint2* sU = sG + (size_t)H * Q;
  float4* sP = reinterpret_cast<float4*>(sU + (size_t)H * Q);         // [5][Q]: c1, g2, b2, g3, b3
  {
    // static weights (may be read before the predecessor kernel has finished): six 1-D bulk copies (TMA) issued by one
    // thread, completion counted on an mbarrier. (A per-thread copy loop would serialise ~50 L2 round trips.)
    __shared__ __align__(8) uint64_t bar;
    if (threadIdx.x == 0) {
      mbar_init(&bar, 1);
      fence_mbar_init();
      const uint32_t gu_bytes = uint32_t(2) * H * C * 2, p_bytes = uint32_t(C) * 4;
      mbar_arrive_expect_tx(&bar, gu_bytes + 5 * p_bytes);
      bulk_copy_g2s(sG, GU, gu_bytes, &bar);
      const float* ps[5] = {c1, g2, b2, g3, b3};
      for (int k = 0; k < 5; ++k) bulk_copy_g2s(sP + (size_t)k * Q, ps[k], p_bytes, &bar);
    }
    __syncthreads();
    mbar_wait(&bar, 0);
  }
  __syncthreads();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int tok = blockIdx.x * wpb + (threadIdx.x >> 5); tok < M; tok += gridDim.x * wpb) {
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)tok * C);
    float4 z[QL], acc[QL];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < QL; ++k) {
      const int q = lane + 32 * k;
      if (q < Q) { acc[k] = __ldg(xr + q); s += acc[k].x + acc[k].y + acc[k].z + acc[k].w; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    float mean = s / C, ss = 0.f;
#pragma unroll
    for (int k = 0; k < QL; ++k) {
      const int q = lane + 32 * k;
      if (q < Q) {
        const float a = acc[k].x - mean, b = acc[k].y - mean, c = acc[k].z - mean, d = acc[k].w - mean;
        ss += a * a + b * b + c * c + d * d;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    float rstd = rsqrtf(ss / C + eps);
    // z = LN2(x); acc becomes x + c1
#pragma unroll
    for (int k = 0; k < QL; ++k) {
      const int q = lane + 32 * k;
      if (q < Q) {
        const float4 cc = sP[q], ga = sP[Q + q], be = sP[2 * Q + q];
        z[k] = make_float4((acc[k].x - mean) * rstd * ga.x + be.x, (acc[k].y - mean) * rstd * ga.y + be.y,
                           (acc[k].z - mean) * rstd * ga.z + be.z, (acc[k].w - mean) * rstd * ga.w + be.w);
        acc[k] = make_float4(acc[k].x + cc.x, acc[k].y + cc.y, acc[k].z + cc.z, acc[k].w + cc.w);
      }
    }
    for (int h0 = 0; h0 < H; h0 += 4) {
      float d[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        d[j] = 0.f;
        if (h0 + j < H) {
          const uint2* Gh = sG + (size_t)(h0 + j) * Q;
#pragma unroll
          for (int k = 0; k < QL; ++k) {
            const int q = lane + 32 * k;
            if (q < Q) {
              const float4 g = bf16x4_to_f4(Gh[q]);
              d[j] += z[k].x * g.x + z[k].y * g.y + z[k].z * g.z + z[k].w * g.w;
            }
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int j = 0; j < 4; ++j) d[j] += __shfl_xor_sync(0xffffffffu, d[j], o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (h0 + j < H) {
          const float w0 = 1.0f / (1.0f + __expf(-d[j] * scale));
          const uint2* Uh = sU + (size_t)(h0 + j) * Q;
#pragma unroll
          for (int k = 0; k < QL; ++k) {
            const int q = lane + 32 * k;
            if (q < Q) {
              const float4 u = bf16x4_to_f4(Uh[q]);
              acc[k].x = fmaf(w0, u.x, acc[k].x); acc[k].y = fmaf(w0, u.y, acc[k].y);
              acc[k].z = fmaf(w0, u.z, acc[k].z); acc[k].w = fmaf(w0, u.w, acc[k].w);
            }
          }
        }
      }
    }
    // store the trunk, then LN3 of the same row
    uint2* yr = reinterpret_cast<uint2*>(y + (size_t)tok * C);
    s = 0.f;
#pragma unroll
    for (int k = 0; k < QL; ++k) {
      const int q = lane + 32 * k;
      if (q < Q) {
        yr[q] = make_uint2(pack_bf16x2(acc[k].x, acc[k].y), pack_bf16x2(acc[k].z, acc[k].w));
        s += acc[k].x + acc[k].y + acc[k].z + acc[k].w;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    mean = s / C; ss = 0.f;
#pragma unroll
    for (int k = 0; k < QL; ++k) {
      const int q = lane + 32 * k;
      if (q < Q) {
        const float a = acc[k].x - mean, b = acc[k].y - mean, c = acc[k].z - mean, d2 = acc[k].w - mean;
        ss += a * a + b * b + c * c + d2 * d2;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    rstd = rsqrtf(ss / C + eps);
    uint2* ar = reinterpret_cast<uint2*>(a_out + (size_t)tok * C);
#pragma unroll
    for (int k = 0; k < QL; ++k) {
      const int q = lane + 32 * k;
      if (q < Q) {
        const float4 ga = sP[3 * Q + q], be = sP[4 * Q + q];
        const float o0 = (acc[k].x - mean) * rstd * ga.x + be.x, o1 = (acc[k].y - mean) * rstd * ga.y + be.y;
        const float o2 = (acc[k].z - mean) * rstd * ga.z + be.z, o3 = (acc[k].w - mean) * rstd * ga.w + be.w;
        ar[q] = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
      }
    }
  }
}

// Wide rows (C = 1280, few tokens): FOUR warps per token, each owning a contiguous quarter of the channels; LayerNorm
// sums and the per-head partial dot products meet in shared memory behind a 128-thread named barrier per token group.
// (One warp per token leaves 576 tokens x a 20-head serial chain on few warps per SM.)
constexpr int kXwMaxH = 32;
// Token count up to which the wide kernel is used. Four warps per token pay while the launch is latency-bound (few
// tokens: one member's 24^2 / 12^2 levels); with many tokens (batched members) one warp per token has the higher
// throughput.
constexpr int kXwMaxTokens = 1024;
__device__ __forceinline__ void xw_barrier(int g) {
  if (g == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}
__device__ __forceinline__ float xw_allsum(float v, float* red /* [4] of this group */, int w, int lane, int g) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  xw_barrier(g);                 // previous readers of red[] are done
  if (lane == 0) red[w] = v;
  xw_barrier(g);
  return (red[0] + red[1]) + (red[2] + red[3]);     // same order in all four warps
}

__global__ void __launch_bounds__(256, 1)
    xattn2_wide_kernel(const float* __restrict__ x, bf16* __restrict__ y, bf16* __restrict__ a_out,
                       const float* __restrict__ g2, const float* __restrict__ b2, const float* __restrict__ g3,
                       const float* __restrict__ b3, const bf16* __restrict__ GU, const float* __restrict__ c1, int M,
                       int C, int H, float scale, float eps) {
  constexpr int QW = 3;                          // quads per lane within a warp's channel quarter (C / 16 <= 96 quads)
  extern __shared__ __align__(16) uint8_t xs_raw[];
  pdl_launch_dependents();
  const int Q = C / 4, Qq = Q / 4;               // quads per row, per warp quarter
  uint2* sG = reinterpret_cast<uint2*>(xs_raw);
  uint2* sU = sG + (size_t)H * Q;
  float4* sP = reinterpret_cast<float4*>(sU + (size_t)H * Q);
  __shared__ __align__(8) uint64_t bar;
  __shared__ float s_red[2][4];
  __shared__ float s_dot[2][4][kXwMaxH];
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
    const uint32_t gu_bytes = uint32_t(2) * H * C * 2, p_bytes = uint32_t(C) * 4;
    mbar_arrive_expect_tx(&bar, gu_bytes + 5 * p_bytes);
    bulk_copy_g2s(sG, GU, gu_bytes, &bar);
    const float* ps[5] = {c1, g2, b2, g3, b3};
    for (int k = 0; k < 5; ++k) bulk_copy_g2s(sP + (size_t)k * Q, ps[k], p_bytes, &bar);
  }
  __syncthreads();
  mbar_wait(&bar, 0);
  pdl_wait();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = warp >> 2, w = warp & 3;         // token group of this block (0 / 1), channel quarter
  const int q0 = w * Qq;
  float* red = s_red[g];
  const int iters = (M + 2 * gridDim.x - 1) / (2 * gridDim.x);
  for (int it = 0; it < iters; ++it) {
    const int tok = (it * gridDim.x + blockIdx.x) * 2 + g;
    const bool live = tok < M;                   // dead groups still take part in their own barriers
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)(live ? tok : 0) * C) + q0;
    float4 z[QW], acc[QW];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < QW; ++k) {
      const int q = lane + 32 * k;
      acc[k] = (live && q < Qq) ? __ldg(xr + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      s += acc[k].x + acc[k].y + acc[k].z + acc[k].w;
    }
    float mean = xw_allsum(s, red, w, lane, g) / C, ss = 0.f;
#pragma unroll
    for (int k = 0; k < QW; ++k) {
      if (lane + 32 * k < Qq) {
        const float a = acc[k].x - mean, b = acc[k].y - mean, c = acc[k].z - mean, d = acc[k].w - mean;
        ss += a * a + b * b + c * c + d * d;
      }
    }
    float rstd = rsqrtf(xw_allsum(ss, red, w, lane, g) / C + eps);
#pragma unroll
    for (int k = 0; k < QW; ++k) {
      const int q = lane + 32 * k;
      if (q < Qq) {
        const float4 cc = sP[q0 + q], ga = sP[Q + q0 + q], be = sP[2 * Q + q0 + q];
        z[k] = make_float4((acc[k].x - mean) * rstd * ga.x + be.x, (acc[k].y - mean) * rstd * ga.y + be.y,
                           (acc[k].z - mean) * rstd * ga.z + be.z, (acc[k].w - mean) * rstd * ga.w + be.w);
        acc[k] = make_float4(acc[k].x + cc.x, acc[k].y + cc.y, acc[k].z + cc.z, acc[k].w + cc.w);
      } else {
        z[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    // partial logits of every head over this warp's channel quarter
    for (int h0 = 0; h0 < H; h0 += 4) {
      float d[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        d[j] = 0.f;
        if (h0 + j < H) {
          const uint2* Gh = sG + (size_t)(h0 + j) * Q + q0;
#pragma unroll
          for (int k = 0; k < QW; ++k) {
            const int q = lane + 32 * k;
            if (q < Qq) {
              const float4 gg = bf16x4_to_f4(Gh[q]);
              d[j] += z[k].x * gg.x + z[k].y * gg.y + z[k].z * gg.z + z[k].w * gg.w;
            }
          }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int j = 0; j < 4; ++j) d[j] += __shfl_xor_sync(0xffffffffu, d[j], o);
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) if (h0 + j < H) s_dot[g][w][h0 + j] = d[j];
      }
    }
    xw_barrier(g);
    for (int h = 0; h < H; ++h) {
      const float dsum = (s_dot[g][0][h] + s_dot[g][1][h]) + (s_dot[g][2][h] + s_dot[g][3][h]);
      const float w0 = 1.0f / (1.0f + __expf(-dsum * scale));
      const uint2* Uh = sU + (size_t)h * Q + q0;
#pragma unroll
      for (int k = 0; k < QW; ++k) {
        const int q = lane + 32 * k;
        if (q < Qq) {
          const float4 u = bf16x4_to_f4(Uh[q]);
          acc[k].x = fmaf(w0, u.x, acc[k].x); acc[k].y = fmaf(w0, u.y, acc[k].y);
          acc[k].z = fmaf(w0, u.z, acc[k].z); acc[k].w = fmaf(w0, u.w, acc[k].w);
        }
      }
    }
    // trunk (bf16) and LN3
    uint2* yr = reinterpret_cast<uint2*>(y + (size_t)(live ? tok : 0) * C) + q0;
    s = 0.f;
#pragma unroll
    for (int k = 0; k < QW; ++k) {
      const int q = lane + 32 * k;
      if (q < Qq) {
        if (live) yr[q] = make_uint2(pack_bf16x2(acc[k].x, acc[k].y), pack_bf16x2(acc[k].z, acc[k].w));
        s += acc[k].x + acc[k].y + acc[k].z + acc[k].w;
      }
    }
    mean = xw_allsum(s, red, w, lane, g) / C; ss = 0.f;
#pragma unroll
    for (int k = 0; k < QW; ++k) {
      if (lane + 32 * k < Qq) {
        const float a = acc[k].x - mean, b = acc[k].y - mean, c = acc[k].z - mean, d2 = acc[k].w - mean;
        ss += a * a + b * b + c * c + d2 * d2;
      }
    }
    rstd = rsqrtf(xw_allsum(ss, red, w, lane, g) / C + eps);
    uint2* ar = reinterpret_cast<uint2*>(a_out + (size_t)(live ? tok : 0) * C) + q0;
#pragma unroll
    for (int k = 0; k < QW; ++k) {
      const int q = lane + 32 * k;
      if (live && q < Qq) {
        const float4 ga = sP[3 * Q + q0 + q], be = sP[4 * Q + q0 + q];
        const float o0 = (acc[k].x - mean) * rstd * ga.x + be.x, o1 = (acc[k].y - mean) * rstd * ga.y + be.y;
        const float o2 = (acc[k].z - mean) * rstd * ga.z + be.z, o3 = (acc[k].w - mean) * rstd * ga.w + be.w;
        ar[q] = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
      }
    }
    xw_barrier(g);               // s_dot is rewritten by the next token
  }
}

int launch_xattn2_fused(const float* x, bf16* y, bf16* a_out, const float* g2, const float* b2, const float* g3,
                        const float* b3, const bf16* GU, const float* c1, int M, int C, int H, float scale, float eps,
                        cudaStream_t stream) {
  if (C % 4 != 0 || C / 4 > 32 * kLnMaxQ || H < 1) { set_error("xattn2: unsupported C=%d H=%d", C, H); return MGB_ERR_INVALID; }
  const size_t smem = size_t(2) * H * C * 2 + size_t(5) * C * 4;
  if (smem > 200 * 1024) { set_error("xattn2: C=%d H=%d needs %zu B of shared memory", C, H, smem); return MGB_ERR_INVALID; }
  if (C % 16 == 0 && C / 16 > 40 && C / 16 <= 96 && H <= kXwMaxH && M <= kXwMaxTokens) {
    // wide rows: four warps per token (C = 1280: 80 quads per warp quarter)
    TRY(raise_smem_limit_once<xattn2_wide_kernel>("xattn2", 200 * 1024));
    const int blocks = std::max(1, std::min((M + 1) / 2, kNumSMs));
    return launch_pdl("xattn2", xattn2_wide_kernel, blocks, 256, smem, stream, x, y, a_out, g2, b2, g3, b3, GU, c1, M, C, H,
                      scale, eps);
  }
  const int ql = (C / 4 + 31) / 32;
  auto kern = ql <= 3 ? xattn2_fused_kernel<3> : ql <= 5 ? xattn2_fused_kernel<5> : xattn2_fused_kernel<10>;
  TRY(ql <= 3   ? raise_smem_limit_once<xattn2_fused_kernel<3>>("xattn2", 200 * 1024)
      : ql <= 5 ? raise_smem_limit_once<xattn2_fused_kernel<5>>("xattn2", 200 * 1024)
                : raise_smem_limit_once<xattn2_fused_kernel<10>>("xattn2", 200 * 1024));
  const int warps_per_block = 8;
  // one wave of resident blocks, each loading the tables once
  const int by_regs = ql <= 3 ? 4 : ql <= 5 ? 3 : 1;
  const int per_sm = std::max(1, std::min<int>(by_regs, int((220 * 1024) / (smem + 1024))));
  const int blocks = std::max(1, std::min((M + warps_per_block - 1) / warps_per_block, kNumSMs * per_sm));
  return launch_pdl("xattn2", kern, blocks, 256, smem, stream, x, y, a_out, g2, b2, g3, b3, GU, c1, M, C, H, scale, eps);
}

// One-time folding of the empty-prompt context into the bf16 tables GU = [G | U] ([2][H][C]) and c1 [C] (see above). wq, wo fp32 [C, C] in the
// PyTorch [out, in] layout; kv fp32 [2 (k | v), 2 tokens, C]; bo fp32 [C].
__global__ void xattn2_fold_kernel(const float* __restrict__ wq, const float* __restrict__ wo, const float* __restrict__ bo,
                                   const float* __restrict__ kv, bf16* __restrict__ GU /* [2][H][C] */,
                                   float* __restrict__ c1, int C, int H) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * (H + 1)) return;
  const int c = i % C, h = i / C;
  const float* k0 = kv; const float* k1 = kv + C; const float* v0 = kv + 2 * C; const float* v1 = kv + 3 * C;
  if (h < H) {
    float g = 0.f, u = 0.f;
    for (int d = 0; d < 64; ++d) {
      const int j = h * 64 + d;
      g = fmaf(wq[(size_t)j * C + c], k0[j] - k1[j], g);
      u = fmaf(wo[(size_t)c * C + j], v0[j] - v1[j], u);
    }
    GU[(size_t)h * C + c] = __float2bfloat16(g);
    GU[((size_t)H + h) * C + c] = __float2bfloat16(u);
  } else {
    float a = bo ? bo[c] : 0.f;
    for (int j = 0; j < C; ++j) a = fmaf(wo[(size_t)c * C + j], v1[j], a);
    c1[c] = a;
  }
}
int launch_xattn2_fold(const float* wq, const float* wo, const float* bo, const float* kv, bf16* GU, float* c1, int C,
                       cudaStream_t stream) {
  const int H = C / 64, n = C * (H + 1);
  return launch_plain("xattn2 fold", xattn2_fold_kernel, (n + 255) / 256, 256, 0, stream, wq, wo, bo, kv, GU, c1, C, H);
}

int launch_layernorm(const float* x, bf16* y, const float* gamma, const float* beta, int M, int C, float eps,
                     cudaStream_t stream) {
  if (C % 4 != 0 || C / 4 > 32 * kLnMaxQ) {
    set_error("layernorm: unsupported C=%d", C);
    return MGB_ERR_INVALID;
  }
  const int warps_per_block = 8;
  const int blocks = (M + warps_per_block - 1) / warps_per_block;
  return launch_pdl("layernorm", layernorm_kernel, blocks, 256, 0, stream, x, y, gamma, beta, M, C, eps);
}

}  // namespace mgb
