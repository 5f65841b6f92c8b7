// Flash self-attention for head_dim 64 on sm_90a (wgmma + TMA).
//
// Replaces F.scaled_dot_product_attention under diffusers' Attention (attn1 of every
// BasicTransformerBlock) reached from reference marigold/marigold_depth_pipeline.py:461-463.
//
//   qkv : bf16 [NB * T, 3C]   (Q | K | V column blocks; head h owns columns h*64 .. h*64+63)
//   out : bf16 [NB * T, C]
//
// One CTA = 128 queries of one (image, head), KV processed in blocks of 64 tokens; 288 threads:
//   warps 0-7  two consumer warpgroups, 64 query rows each:
//                S  = Q K_j^T    wgmma m64n64k16 x 4, both operands K-major in shared memory, S in registers
//                softmax         online, in registers: a row lives in the four lanes of a quad (two shuffles per
//                                max / sum), O and l rescaled when the row max grows
//                O += P V_j      wgmma m64n64k16 x 4, A = P (bf16) straight from the S registers (the accumulator
//                                fragment of 16 columns is the A fragment of one k16 step), B = V in its natural
//                                [token, d] layout as an MN-major (transposed) operand: no transpose pass
//   warp 8     TMA producer: Q tile (128 x 64) once, K / V tiles (64 x 64) through 3-stage rings
// Two CTAs per SM (~66 KB of shared memory and <= 113 registers per thread each): the softmax of one warpgroup
// overlaps the MMAs of the others.
#include <cstdlib>
#include "common.cuh"
#include "kernels.h"
#include "launch.h"

namespace mgb {

constexpr int kAttnConsumers = 256;
constexpr int kAttnThreads = kAttnConsumers + 32;
constexpr int kQBytes = 128 * 128;       // 128 rows x 64 bf16
constexpr int kKvBytes = 64 * 128;       // 64 rows x 64 bf16
constexpr int kKvStages = 3;
struct AttnParams {
  CUtensorMap tmap_q;   // 3D {3C, T, NB}, box {64, 128, 1}
  CUtensorMap tmap_kv;  // 3D {3C, T, NB}, box {64, 64, 1}
  bf16* out;
  int T, C;
  float scale_log2;
  // split-KV (balances the last wave of CTAs): blockIdx.z = img * splits + split; split s covers KV blocks
  // [s * nkv / splits, (s+1) * ...). With splits > 1 the CTA writes un-normalised fp32 O plus (m, l) per row;
  // attn_combine_kernel merges them.
  int splits;
  float* part_o;    // [splits][NB][C/64][T][64]
  float* part_ml;   // [splits][NB][C/64][T][2]   (m in log2 units incl. the softmax scale, l)
};

__global__ void __launch_bounds__(kAttnThreads, 2) flash_attn64_kernel(const __grid_constant__ AttnParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kQBytes;
  uint8_t* sV = sK + kKvStages * kKvBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kKvStages * kKvBytes);
  uint64_t* q_full = bars;                   // 1
  uint64_t* k_full = bars + 1;               // [3]
  uint64_t* k_empty = bars + 4;              // [3]  one arrival per consumer warpgroup
  uint64_t* v_full = bars + 7;               // [3]
  uint64_t* v_empty = bars + 10;             // [3]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 128, head = blockIdx.y, img = blockIdx.z / p.splits, split = blockIdx.z % p.splits;
  const int nkv_all = (p.T + 63) / 64;
  const int jb0 = split * nkv_all / p.splits;                 // first KV block of this CTA
  const int nkv = (split + 1) * nkv_all / p.splits - jb0;     // its number of KV blocks (>= 1: host keeps splits <= nkv_all)

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&p.tmap_q);
    tma_prefetch_desc(&p.tmap_kv);
    mbar_init(q_full, 1);
    for (int s = 0; s < kKvStages; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], 2);
      mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    // ===================== TMA producer =====================
    // One thread running a latency chain: whole loop inside one elected thread, shared-window addresses
    // precomputed, counters instead of % and /.
    if (elect_one()) {
      const uint32_t kfull = smem_u32(k_full), kempty = smem_u32(k_empty), vfull = smem_u32(v_full),
                     vempty = smem_u32(v_empty);
      const uint32_t sK_a = smem_u32(sK), sV_a = smem_u32(sV);
      mbar_arrive_expect_tx(q_full, kQBytes);
      tma_load_3d(sQ, &p.tmap_q, q_full, head * 64, q0, img);
      const int ck = p.C + head * 64, cv = 2 * p.C + head * 64;
      uint32_t s = 0, ph = 0;
      for (int j = 0; j < nkv; ++j) {
        mbar_wait_wg(kempty + s * 8, ph ^ 1);
        mbar_expect_tx_a(kfull + s * 8, kKvBytes);
        tma_load_3d_a(sK_a + s * kKvBytes, &p.tmap_kv, kfull + s * 8, ck, (jb0 + j) * 64, img);
        mbar_wait_wg(vempty + s * 8, ph ^ 1);
        mbar_expect_tx_a(vfull + s * 8, kKvBytes);
        tma_load_3d_a(sV_a + s * kKvBytes, &p.tmap_kv, vfull + s * 8, cv, (jb0 + j) * 64, img);
        if (++s == kKvStages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers =====================
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  // this thread's two query rows (accumulator fragment rows l/4 and l/4 + 8 of its warp's 16) and column pairs
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cpair = (lane & 3) * 2;
  constexpr uint32_t kHi = uint32_t(kDescSw128Hi >> 32), kLbo = 1u << 16;
  const uint32_t dq_lo = ((smem_u32(sQ) + uint32_t(wg) * 64u * 128u) >> 4) | kLbo;
  const uint32_t dk_lo0 = (smem_u32(sK) >> 4) | kLbo, dv_lo0 = (smem_u32(sV) >> 4) | kLbo;
  const uint32_t kfull = smem_u32(k_full), vfull = smem_u32(v_full);

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running max (log2 units) and partial sums, rows lo / hi
  mbar_wait_wg(smem_u32(q_full), 0);
  uint32_t s = 0, ph = 0;
  for (int j = 0; j < nkv; ++j) {
    // ---- S = Q K^T
    float sc[32];
    mbar_wait_wg(kfull + s * 8, ph);
    const uint32_t dk_lo = dk_lo0 + s * uint32_t(kKvBytes >> 4);
    wgmma_fence();
    Wgmma<64>::ss(sc, make_u64(dq_lo, kHi), make_u64(dk_lo, kHi), 0u);
    Wgmma<64>::ss(sc, make_u64(dq_lo + 2, kHi), make_u64(dk_lo + 2, kHi), 1u);
    Wgmma<64>::ss(sc, make_u64(dq_lo + 4, kHi), make_u64(dk_lo + 4, kHi), 1u);
    Wgmma<64>::ss(sc, make_u64(dq_lo + 6, kHi), make_u64(dk_lo + 6, kHi), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    if (wg_leader) mbar_arrive(&k_empty[s]);

    // ---- online softmax (exp2 domain: the softmax scale folded into scale_log2)
    const int kv_valid = p.T - (jb0 + j) * 64;     // >= 64 except possibly in the last block
    if (kv_valid < 64) {                           // ragged tail (T % 64 != 0)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int c = 8 * jj + cpair;
        if (c >= kv_valid) { sc[4 * jj] = -INFINITY; sc[4 * jj + 2] = -INFINITY; }
        if (c + 1 >= kv_valid) { sc[4 * jj + 1] = -INFINITY; sc[4 * jj + 3] = -INFINITY; }
      }
    }
    float mx0 = sc[0], mx1 = sc[2];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      mx0 = fmaxf(mx0, fmaxf(sc[4 * jj], sc[4 * jj + 1]));
      mx1 = fmaxf(mx1, fmaxf(sc[4 * jj + 2], sc[4 * jj + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0 * p.scale_log2), mn1 = fmaxf(m1, mx1 * p.scale_log2);
    const float a0 = ex2_approx(m0 - mn0), a1 = ex2_approx(m1 - mn1);   // 0 on the first block (m = -inf)
    m0 = mn0; m1 = mn1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      o[4 * jj] *= a0; o[4 * jj + 1] *= a0;
      o[4 * jj + 2] *= a1; o[4 * jj + 3] *= a1;
    }
    // P = exp2(S * c - m) (exp2(-inf) = 0 masks the tail), packed to bf16 pairs in the wgmma A-fragment order:
    // k16 step kk takes accumulator column groups 2 kk and 2 kk + 1
    uint32_t pa[4][4];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float e0 = ex2_approx(fmaf(sc[4 * jj], p.scale_log2, -m0));
      const float e1 = ex2_approx(fmaf(sc[4 * jj + 1], p.scale_log2, -m0));
      const float e2 = ex2_approx(fmaf(sc[4 * jj + 2], p.scale_log2, -m1));
      const float e3 = ex2_approx(fmaf(sc[4 * jj + 3], p.scale_log2, -m1));
      l0 += e0 + e1;
      l1 += e2 + e3;
      pa[jj >> 1][(jj & 1) * 2] = pack_bf16x2(e0, e1);
      pa[jj >> 1][(jj & 1) * 2 + 1] = pack_bf16x2(e2, e3);
    }

    // ---- O += P V: V [kv, d] d-contiguous (MN-major B): 16 kv rows = 2048 B per k16 step
    mbar_wait_wg(vfull + s * 8, ph);
    const uint32_t dv_lo = dv_lo0 + s * uint32_t(kKvBytes >> 4);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) Wgmma<64>::rs_tb(o, pa[kk], make_u64(dv_lo + 128 * kk, kHi), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (wg_leader) mbar_arrive(&v_empty[s]);
    if (++s == kKvStages) { s = 0; ph ^= 1; }
  }

  // ---- epilogue: the quad's partial sums give the row sums; O / l
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qrow = q0 + r_lo + 8 * h;
    if (qrow >= p.T) continue;
    const float m = h ? m1 : m0, l = h ? l1 : l0;
    if (p.splits == 1) {
      const float inv = 1.f / l;
      bf16* dst = p.out + ((size_t)img * p.T + qrow) * p.C + head * 64 + cpair;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    } else {
      const size_t prow = ((size_t(split) * gridDim.z / p.splits + img) * gridDim.y + head) * p.T + qrow;
      float* dst = p.part_o + prow * 64 + cpair;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<float2*>(dst + 8 * jj) = make_float2(o[4 * jj + 2 * h], o[4 * jj + 2 * h + 1]);
      if ((lane & 3) == 0) *reinterpret_cast<float2*>(p.part_ml + prow * 2) = make_float2(m, l);
    }
  }
}

// Merge the split-KV partials: out[row, :] = sum_s w_s O_s / sum_s w_s l_s, w_s = 2^(m_s - max m). One thread per
// (row, 8 columns).
__global__ void __launch_bounds__(256) attn_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                                                           bf16* __restrict__ out, int splits, int NB, int heads, int T, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t rows = size_t(NB) * heads * T;
  const size_t gid = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t r = gid >> 3;
  const int c8 = int(gid & 7) * 8;
  if (r >= rows) return;
  float m = -INFINITY;
  for (int s = 0; s < splits; ++s) m = fmaxf(m, __ldg(part_ml + (size_t(s) * rows + r) * 2));
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, l = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float2 ml = __ldg(reinterpret_cast<const float2*>(part_ml + (size_t(s) * rows + r) * 2));
    const float w = ex2_approx(ml.x - m);
    l = fmaf(ml.y, w, l);
    const float4* po = reinterpret_cast<const float4*>(part_o + (size_t(s) * rows + r) * 64 + c8);
    const float4 a = __ldg(po), b = __ldg(po + 1);
    acc[0] = fmaf(a.x, w, acc[0]); acc[1] = fmaf(a.y, w, acc[1]); acc[2] = fmaf(a.z, w, acc[2]); acc[3] = fmaf(a.w, w, acc[3]);
    acc[4] = fmaf(b.x, w, acc[4]); acc[5] = fmaf(b.y, w, acc[5]); acc[6] = fmaf(b.z, w, acc[6]); acc[7] = fmaf(b.w, w, acc[7]);
  }
  const float inv = 1.f / l;
  const size_t t = r % T, ih = r / T;
  const size_t img = ih / heads, head = ih % heads;
  uint4* dst = reinterpret_cast<uint4*>(out + (img * T + t) * C + head * 64 + c8);
  *dst = make_uint4(pack_bf16x2(acc[0] * inv, acc[1] * inv), pack_bf16x2(acc[2] * inv, acc[3] * inv),
                    pack_bf16x2(acc[4] * inv, acc[5] * inv), pack_bf16x2(acc[6] * inv, acc[7] * inv));
}

// KV splits that minimise the number of CTA rounds (2 CTAs per SM) weighted by the split's length
int flash_attn64_splits(int NB, int T, int C) {
  const int units = ((T + 127) / 128) * (C / 64) * NB, nkv = (T + 63) / 64, slots = kNumSMs * 2;
  int best = 1;
  double best_t = 1e30;
  for (int s = 1; s <= 8; ++s) {
    if (s > 1 && nkv / s < 6) break;
    const double rounds = double((units * s + slots - 1) / slots);
    // cost model: a CTA's fixed cost (prologue, Q load, first S, epilogue) is worth ~15 KV blocks, the combine
    // pass ~8 (estimates, not measured on the H100)
    const double t = rounds * (double(nkv) / s + 15.0) + (s > 1 ? 8.0 : 0.0);
    if (t < best_t - 1e-9) { best_t = t; best = s; }
  }
  return best;
}
size_t flash_attn64_ws_bytes(int NB, int T, int C) {
  const int s = flash_attn64_splits(NB, T, C);
  if (s == 1) return 0;
  return size_t(s) * NB * (C / 64) * T * (64 + 2) * sizeof(float);
}

int launch_flash_attn64(const bf16* qkv, bf16* out, int NB, int T, int C, float scale, float* ws, size_t ws_bytes,
                        cudaStream_t stream) {
  if (C % 64 != 0 || T <= 0) {
    set_error("flash_attn64: C %% 64 != 0 or bad T");
    return MGB_ERR_INVALID;
  }
  AttnParams p;
  const uint64_t dims[3] = {uint64_t(3 * C), uint64_t(T), uint64_t(NB)};
  const uint64_t strides[2] = {uint64_t(3 * C) * 2, uint64_t(T) * 3 * C * 2};
  const uint32_t box_q[3] = {64, 128, 1}, box_kv[3] = {64, 64, 1};
  int rc = make_tmap_3d(&p.tmap_q, qkv, dims, strides, box_q);
  if (rc) return rc;
  rc = make_tmap_3d(&p.tmap_kv, qkv, dims, strides, box_kv);
  if (rc) return rc;
  p.out = out; p.T = T; p.C = C;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.splits = 1; p.part_o = nullptr; p.part_ml = nullptr;
  {
    const int sp = flash_attn64_splits(NB, T, C);
    if (sp > 1 && ws != nullptr && ws_bytes >= flash_attn64_ws_bytes(NB, T, C)) {
      p.splits = sp;
      p.part_o = ws;
      p.part_ml = ws + size_t(sp) * NB * (C / 64) * T * 64;
    }
  }
  const size_t smem = 1024 + kQBytes + 2 * kKvStages * kKvBytes + 256;
  TRY(raise_smem_limit_once<flash_attn64_kernel>("flash_attn64", int(smem)));
  dim3 grid((T + 127) / 128, C / 64, NB * p.splits);
  TRY(launch_pdl("flash_attn64", flash_attn64_kernel, grid, kAttnThreads, smem, stream, p));
  if (p.splits == 1) return MGB_OK;
  const size_t threads = size_t(NB) * (C / 64) * T * 8;
  return launch_pdl("attn_combine", attn_combine_kernel, dim3(unsigned((threads + 255) / 256)), 256, 0, stream,
                    (const float*)p.part_o, (const float*)p.part_ml, out, p.splits, NB, C / 64, T, C);
}

}  // namespace mgb
