// Warpgroup-MMA (wgmma) GEMM / implicit-GEMM convolution for sm_90a.
//
//   D[M, N] = A[M, K] * B[N, K]^T,  bf16 operands, fp32 accumulation in registers.
//
// One 128 x BLOCK_N output tile per CTA. Warp roles (288 threads):
//   warps 0..7  two consumer warpgroups. Warpgroup g issues 4 x wgmma m64 n BLOCK_N k16 per pipeline stage on rows
//               [64 g, 64 g + 64) of the A tile and the whole B tile, keeps one stage of MMAs in flight
//               (wgmma.wait_group 1) and releases a stage once its MMAs have completed. Then the fused epilogue
//               (bias / activation / GEGLU / residual / scheduler step / output cast) from its accumulator registers.
//   warp 8      TMA producer: A tile (128 rows x 64 K, SWIZZLE_128B) + B tile (BLOCK_N x 64 K)
//               per pipeline stage, completion signalled on an mbarrier (complete_tx).
//
// A operand addressing:
//   mode 0  rows: 2D tensor map {K, M}; tile m covers rows [128 m, 128 m + 128).
//   mode 1  conv: 5D tensor map {C, W, H, P, NB} over an NHWC image (P parity planes; P = 1 for
//           stride-1). A CTA's 128 rows are a tile_h x tile_w pixel rectangle; K block kb maps to
//           (tap, channel block); the tap shifts the box by (dy, dx) and TMA zero-fills the halo, so
//           padding costs nothing and no im2col buffer exists.
// Replaces (behaviourally) the cuDNN/cuBLAS calls under torch.nn.Conv2d / Linear reached from
// reference marigold/marigold_depth_pipeline.py:461-463,491-492,512-513.
#include <algorithm>
#include "common.cuh"
#include "kernels.h"
#include "launch.h"

namespace mgb {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int kConsumerThreads = 256;                 // two warpgroups of 64 tile rows each
constexpr int kProducerWarp = kConsumerThreads / 32;
constexpr int kGemmThreads = kConsumerThreads + 32;

__host__ __device__ constexpr int a_stage_bytes() { return BLOCK_M * BLOCK_K * 2; }
__host__ __device__ constexpr int b_stage_bytes(int block_n) { return block_n * BLOCK_K * 2; }
// Epilogue scratch: every consumer warp stages its 16 accumulator rows in fp32 at this pitch (floats). The 8-float pad
// makes the fragment's 64-bit stores and the row-contiguous 128-bit reloads bank-conflict free.
__host__ __device__ constexpr int epi_pitch(int block_n) { return block_n + 8; }
size_t gemm_epi_scratch_bytes(int block_n) { return size_t(kConsumerThreads / 32) * 16 * epi_pitch(block_n) * sizeof(float); }

size_t gemm_smem_bytes(int block_n, int stages) {
  // 1024 B alignment slack + A ring + B ring + barriers
  return 1024 + size_t(stages) * (a_stage_bytes() + b_stage_bytes(block_n)) + 256;
}

// -------------------------------------------------------------------------------------------------
// Fused epilogue for one row and one chunk of CH accumulator columns.
// -------------------------------------------------------------------------------------------------
struct RowCtx {
  bool valid;    // row inside the problem
  long long m;   // output row index (token / pixel)
};

template <int CH>
__device__ __forceinline__ void epilogue_chunk(const GemmEpilogue& e, const RowCtx& rc, float (&v)[CH], int col0,
                                               int n_valid /* valid output columns from col0 */) {
  // v[] already holds activation-applied values for output columns col0 .. col0 + CH
  if (!rc.valid || n_valid <= 0) return;
  const long long base = rc.m * (long long)e.ldo + col0;
  const bool full = (n_valid >= CH) && ((e.ldo & 3) == 0) && ((col0 & 3) == 0);
  if (e.residual) {
    if (full) {
      const float4* r4 = reinterpret_cast<const float4*>(e.residual + base);
#pragma unroll
      for (int i = 0; i < CH / 4; ++i) {
        float4 r = __ldg(r4 + i);
        v[4 * i + 0] += r.x; v[4 * i + 1] += r.y; v[4 * i + 2] += r.z; v[4 * i + 3] += r.w;
      }
    } else {
#pragma unroll
      for (int i = 0; i < CH; ++i)
        if (i < n_valid) v[i] += __ldg(e.residual + base + i);
    }
  }
  if (e.out_f32) {
    if (full) {
      float4* o4 = reinterpret_cast<float4*>(e.out_f32 + base);
#pragma unroll
      for (int i = 0; i < CH / 4; ++i) o4[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < CH; ++i)
        if (i < n_valid) e.out_f32[base + i] = v[i];
    }
  }
  if (e.out_bf16) {
    if (full && ((e.ldo & 7) == 0) && ((col0 & 7) == 0)) {
      uint4* o4 = reinterpret_cast<uint4*>(e.out_bf16 + base);
#pragma unroll
      for (int i = 0; i < CH / 8; ++i)
        o4[i] = make_uint4(pack_bf16x2(v[8 * i], v[8 * i + 1]), pack_bf16x2(v[8 * i + 2], v[8 * i + 3]),
                           pack_bf16x2(v[8 * i + 4], v[8 * i + 5]), pack_bf16x2(v[8 * i + 6], v[8 * i + 7]));
    } else {
#pragma unroll
      for (int i = 0; i < CH; ++i)
        if (i < n_valid) e.out_bf16[base + i] = __float2bfloat16(v[i]);
    }
  }
}

// Special small-N epilogues (N <= 16 accumulator columns, whole row in one chunk).
__device__ __forceinline__ void epilogue_special(const GemmEpilogue& e, const RowCtx& rc, float (&v)[16], int N) {
  if (!rc.valid) return;
  if (e.flags & EPI_SCHED) {
    const float kx = __ldg(e.sched_k + 0), kv = __ldg(e.sched_k + 1), kz = __ldg(e.sched_k + 2);
    const long long base = rc.m * (long long)e.ldo;
    for (int c = 0; c < N; ++c) {
      float x = __ldg(e.sched_x + base + c);
      float z = e.sched_z ? __ldg(e.sched_z + base + c) : 0.0f;
      if (e.aux_out) e.aux_out[base + c] = v[c];
      // written so that kz == 0 with z == 0 is exact
      e.out_f32[base + c] = kx * x + kv * v[c] + kz * z;
    }
    return;
  }
  const long long img = rc.m / e.hw, pix = rc.m % e.hw;
  if (e.flags & EPI_DEPTH) {
    // reference marigold_depth_pipeline.py:515 (channel mean), :473 (clip), :475 (shift to [0,1])
    float d = (v[0] + v[1] + v[2]) / 3.0f;
    d = fminf(fmaxf(d, -1.0f), 1.0f);
    e.out_f32[img * e.hw + pix] = (d + 1.0f) / 2.0f;
    return;
  }
  if (e.flags & EPI_NORMALS) {
    // reference marigold_normals_pipeline.py:438-440
    float a = fminf(fmaxf(v[0], -1.0f), 1.0f), b = fminf(fmaxf(v[1], -1.0f), 1.0f),
          c = fminf(fmaxf(v[2], -1.0f), 1.0f);
    float nrm = fmaxf(sqrtf(a * a + b * b + c * c), 1e-6f);
    float* o = e.out_f32 + img * 3 * e.hw + pix;
    o[0] = a / nrm; o[e.hw] = b / nrm; o[2 * (long long)e.hw] = c / nrm;
    return;
  }
  if (e.flags & EPI_NCHW) {
    // EPI_UNIT: reference marigold_iid_pipeline.py:562-565 (clip to [-1, 1], shift to [0, 1])
    const bool unit = (e.flags & EPI_UNIT) != 0;
    for (int c = 0; c < N; ++c)
      e.out_f32[(img * N + c) * e.hw + pix] = unit ? (fminf(fmaxf(v[c], -1.0f), 1.0f) + 1.0f) / 2.0f : v[c];
    return;
  }
}

// -------------------------------------------------------------------------------------------------
// Coalesced epilogue. A warp's accumulator fragment (16 rows; a lane holds pairs of columns of two rows) is staged
// through shared memory so that 8 lanes cover one row's 128 contiguous bytes and a warp instruction moves four full
// lines; bias, activation, residual and the casts are applied after the reload, where a lane owns 4 fixed columns.
// The store loop is deliberately rolled and small: it runs once per CTA, i.e. from a cold instruction cache.
// -------------------------------------------------------------------------------------------------
struct TileGeom {
  int mode;
  long long m_base;
  int M;
  int img, ty, tx, H, W, tile_w_shift, tile_w_mask, tile_h, out_y0;   // ty: the image's tile row
};

__device__ __forceinline__ bool tile_row_index(const TileGeom& g, int row, long long* m) {
  if (g.mode == 0) {
    *m = g.m_base + row;
    return *m < g.M;
  }
  const int hh = row >> g.tile_w_shift, ww = row & g.tile_w_mask;
  const int h = g.ty * g.tile_h + hh, w = (g.tx << g.tile_w_shift) + ww;
  *m = ((long long)g.img * g.H + h - g.out_y0) * g.W + w;
  return (h < g.H) && (w < g.W);
}

// Unaligned / ragged tail: rare, kept out of line.
static __device__ __noinline__ void store_tail(float4 x, int nv, const float* residual, float* out_f32, bf16* out_bf16,
                                        long long o, long long o32) {
  const float xs[4] = {x.x, x.y, x.z, x.w};
  for (int k = 0; k < 4 && k < nv; ++k) {
    float a = xs[k];
    if (residual) a += __ldg(residual + o + k);
    if (out_f32) out_f32[o32 + k] = a;
    if (out_bf16) out_bf16[o + k] = __float2bfloat16(a);
  }
}

// -------------------------------------------------------------------------------------------------
// The kernel
// -------------------------------------------------------------------------------------------------
// kBand: the instantiation that reads GemmParams' row-band fields (ty0, src_y0, out_y0) and the split output
// (GemmEpilogue::out_f32_hi); the others take them as absent, so that the network's other GEMMs pay nothing for them.
// MINB = CTAs per SM the kernel is compiled for. 1: the register file of an SM for one CTA (accumulators of up to
// 128 x 256), deep operand ring, one output tile per SM at a time. 2: <= 113 registers per thread and <= 113 KB of
// shared memory, so TWO CTAs share an SM and the epilogue of one tile runs under the K loop of the other. Used for
// multi-wave grids with block_n <= 128 (GEGLU feed-forward, QKV, VAE convs).
template <int BLOCK_N, int MINB, bool kBand>
__global__ void __launch_bounds__(kGemmThreads, MINB) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  pdl_launch_dependents();
  const long long t_entry = clock64();
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024 B alignment
  // pointer + integer keeps the shared address space (a uintptr_t round trip decays to generic ld/st)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int stages = p.stages;
  constexpr int kABytes = a_stage_bytes();
  constexpr int kBBytes = b_stage_bytes(BLOCK_N);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + size_t(stages) * kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_b + size_t(stages) * kBBytes);
  uint64_t* empty_bar = full_bar + stages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, n_tile = blockIdx.y, split = blockIdx.z;
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);

  // conv tile decomposition
  int img = 0, ty = 0, tx = 0;
  if (p.mode != 0) {
    const int per_img = p.tiles_x * p.tiles_y;
    img = m_tile / per_img;
    const int r = m_tile - img * per_img;
    ty = r / p.tiles_x;
    tx = r - ty * p.tiles_x;
  }

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&p.tmap_a);
    tma_prefetch_desc(&p.tmap_b);
    if (p.num_kb1 < p.num_kb) tma_prefetch_desc(&p.tmap_a2);
#pragma unroll 1
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);          // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Weights never depend on a predecessor kernel: start streaming the first B tiles of the pipeline
  // before waiting on it (the A operand and residuals are read only after pdl_wait()).
  const int n_pre = min(stages, kb1 - kb0);
  if (warp == kProducerWarp && elect_one()) {
    for (int i = 0; i < n_pre; ++i) {
      mbar_arrive_expect_tx(&full_bar[i], kABytes + kBBytes);
      tma_load_2d(smem_b + size_t(i) * kBBytes, &p.tmap_b, &full_bar[i], (kb0 + i) * BLOCK_K, n_tile * BLOCK_N);
    }
  }
  // everything above overlapped the previous kernel's tail; operands / residuals are read below
  pdl_wait();
  long long* dbg = p.dbg ? p.dbg + ((size_t(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * 8 : nullptr;
  if (dbg && threadIdx.x == 0) { dbg[0] = t_entry; dbg[1] = clock64(); }

  // The producer is ONE thread running a latency chain per K block: whole loop inside one elected thread,
  // shared-window addresses precomputed, counters instead of divisions.
  const uint32_t full_a = smem_u32(full_bar), empty_a = smem_u32(empty_bar);
  if (warp == kProducerWarp) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      uint32_t stage = 0, phase = 0;
      const uint32_t sa0 = smem_u32(smem_a), sb0 = smem_u32(smem_b);
      const int ncol = n_tile * BLOCK_N;
      const uint32_t ustages = uint32_t(stages);
      if (p.mode == 0) {
        const int mrow = m_tile * BLOCK_M;
        int kc = kb0 * BLOCK_K;
        for (int kb = kb0; kb < kb1; ++kb, kc += BLOCK_K) {
          mbar_wait_wg(empty_a + stage * 8, phase ^ 1);
          const uint32_t fb = full_a + stage * 8;
          if (kb - kb0 >= n_pre) {        // (the first n_pre weight tiles were issued before pdl_wait)
            mbar_expect_tx_a(fb, kABytes + kBBytes);
            tma_load_2d_a(sb0 + stage * kBBytes, &p.tmap_b, fb, kc, ncol);
          }
          // K concatenation of two row-major operands (A = [A1 | A2]): blocks past num_kb1 come from the second map
          if (kb < p.num_kb1) tma_load_2d_a(sa0 + stage * kABytes, &p.tmap_a, fb, kc, mrow);
          else tma_load_2d_a(sa0 + stage * kABytes, &p.tmap_a2, fb, (kb - p.num_kb1) * BLOCK_K, mrow);
          if (++stage == ustages) { stage = 0; phase ^= 1; }
        }
      } else {
        const int cblocks = p.cblocks, x0 = tx * p.tile_w;
        const int y0 = ((kBand ? p.ty0 : 0) + ty) * p.tile_h, ya = y0 - (kBand ? p.src_y0 : 0);
        int tap = kb0 / cblocks, cb = kb0 - tap * cblocks;
        int kc = kb0 * BLOCK_K;
        for (int kb = kb0; kb < kb1; ++kb, kc += BLOCK_K) {
          mbar_wait_wg(empty_a + stage * 8, phase ^ 1);
          const uint32_t fb = full_a + stage * 8;
          if (kb - kb0 >= n_pre) {
            mbar_expect_tx_a(fb, kABytes + kBBytes);
            tma_load_2d_a(sb0 + stage * kBBytes, &p.tmap_b, fb, kc, ncol);
          }
          if (kb < p.num_kb1) {
            tma_load_5d_a(sa0 + stage * kABytes, &p.tmap_a, fb, cb * BLOCK_K, x0 + p.tap_dx[tap], ya + p.tap_dy[tap],
                          p.tap_p[tap], img);
            if (++cb == cblocks) { cb = 0; ++tap; }
          } else {
            // K blocks of the second operand (the 1x1 shortcut over the block input): same pixels, no tap shift
            tma_load_5d_a(sa0 + stage * kABytes, &p.tmap_a2, fb, (kb - p.num_kb1) * BLOCK_K, x0, y0, 0, img);
          }
          if (++stage == ustages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: MMA =====================
  const int wg = warp >> 2;                          // rows [64 wg, 64 wg + 64) of the tile
  const bool wg_leader = (threadIdx.x & 127) == 0;
  float acc[BLOCK_N / 2];
#pragma unroll
  for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
  {
    constexpr uint32_t kDescHi = uint32_t(kDescSw128Hi >> 32);       // SBO 1024, SWIZZLE_128B
    constexpr uint32_t kLbo = 1u << 16;
    const uint32_t ustages = uint32_t(stages);
    const uint32_t b_lo0 = (smem_u32(smem_b) >> 4) | kLbo;
    uint32_t stage = 0, phase = 0;
    int prev = -1;         // stage of the previous K block: released once wgmma.wait_group 1 shows its MMAs complete
    // the A tile's rows are 128 B apart (conv tiles: pixels in TMA box order), so rows 64.. start 8 KB in
    const uint32_t a_lo0 = ((smem_u32(smem_a) + uint32_t(wg) * 64u * 128u) >> 4) | kLbo;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait_wg(full_a + stage * 8, phase);
      if (dbg && kb == kb0 && threadIdx.x == 0) dbg[2] = clock64();
      const uint32_t al = a_lo0 + stage * uint32_t(kABytes >> 4), bl = b_lo0 + stage * uint32_t(kBBytes >> 4);
      wgmma_fence();
      // K advance: +32 B (2 descriptor units) inside the 128 B swizzle atom
      Wgmma<BLOCK_N>::ss(acc, make_u64(al, kDescHi), make_u64(bl, kDescHi), 1u);
      Wgmma<BLOCK_N>::ss(acc, make_u64(al + 2, kDescHi), make_u64(bl + 2, kDescHi), 1u);
      Wgmma<BLOCK_N>::ss(acc, make_u64(al + 4, kDescHi), make_u64(bl + 4, kDescHi), 1u);
      Wgmma<BLOCK_N>::ss(acc, make_u64(al + 6, kDescHi), make_u64(bl + 6, kDescHi), 1u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
      prev = int(stage);
      if (++stage == ustages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }

  // ===================== consumers: epilogue =====================
  // Every MMA of both warpgroups has completed and every issued stage was consumed: the operand ring is free and
  // becomes the staging scratch, 16 rows x epi_pitch floats per warp (the host sizes the ring to hold it).
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
  if (dbg && threadIdx.x == 0) dbg[3] = clock64();
  constexpr int kPitch = epi_pitch(BLOCK_N);
  const int row0 = wg * 64 + (warp & 3) * 16;       // first tile row of this warp
  float* s_base = reinterpret_cast<float*>(smem_a) + warp * 16 * kPitch;
  {
    const int r = lane >> 2, c2 = (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      *reinterpret_cast<float2*>(s_base + r * kPitch + 8 * j + c2) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(s_base + (r + 8) * kPitch + 8 * j + c2) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  __syncwarp();
  TileGeom tg;
  tg.mode = p.mode; tg.m_base = (long long)m_tile * BLOCK_M; tg.M = p.M;
  tg.img = img; tg.ty = (kBand ? p.ty0 : 0) + ty; tg.tx = tx; tg.H = p.H; tg.W = p.W;
  tg.tile_w_shift = p.tile_w_shift; tg.tile_w_mask = p.tile_w - 1; tg.tile_h = p.tile_h;
  tg.out_y0 = kBand ? p.out_y0 : 0;
  const GemmEpilogue& e = p.epi;
  const int n0 = n_tile * BLOCK_N;

  if constexpr (BLOCK_N == 16) {
    // one lane per row: the whole row (<= 16 accumulator columns) in registers
    if (lane < 16) {
      RowCtx rc;
      rc.valid = tile_row_index(tg, row0 + lane, &rc.m);
      const float* src = s_base + lane * kPitch;
      if (p.partial != nullptr) {
        float* dst = p.partial + ((long long)split * p.M + rc.m) * p.N + n0;
        if (rc.valid) {
#pragma unroll
          for (int i = 0; i < 16; ++i)
            if (n0 + i < p.N) dst[i] = src[i];
        }
      } else {
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          v[i] = src[i];
          if (e.flags & EPI_SCALE) v[i] *= e.scale;
          if (e.bias && (n0 + i) < p.N) v[i] += __ldg(e.bias + n0 + i);
          if (e.flags & EPI_SILU) v[i] = silu_f(v[i]);
          if (e.flags & EPI_RELU) v[i] = fmaxf(v[i], 0.f);
        }
        if (e.flags & (EPI_SCHED | EPI_DEPTH | EPI_NORMALS | EPI_NCHW)) {
          epilogue_special(e, rc, v, p.N);
        } else {
          epilogue_chunk<16>(e, rc, v, n0, p.N - n0);
        }
      }
    }
  } else {
    // after the reload this lane owns columns c4 .. c4 + 3 of a 32-column chunk in rows it * 4 + (lane >> 3), it = 0..3
    const int sub = lane >> 3, c4 = (lane & 7) * 4;
    const float* s_rd = s_base + sub * kPitch + c4;
    const bool raw = p.partial != nullptr;                 // split-K: raw accumulators, epilogue deferred
    const bool geglu = !raw && (e.flags & EPI_GEGLU);
    float* out_f32 = raw ? p.partial + (long long)split * p.M * p.N : e.out_f32;
    bf16* out_bf16 = raw ? nullptr : e.out_bf16;
    const float* residual = raw ? nullptr : e.residual;
    const float* bias = raw ? nullptr : e.bias;
    const int ldo = raw ? p.N : e.ldo;
    const int n_out = geglu ? p.N / 2 : p.N;               // output columns
    const int half = BLOCK_N / 2;
    const int chunks = geglu ? half / 32 : BLOCK_N / 32;
    const float scale = (!raw && (e.flags & EPI_SCALE)) ? e.scale : 1.0f;
    const bool silu = !raw && (e.flags & EPI_SILU);
    const bool relu = !raw && (e.flags & EPI_RELU);
    const bool ld_vec = (ldo & 3) == 0;
    long long off[4];
    uint32_t vmask = 0;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      long long m;
      const bool ok = tile_row_index(tg, row0 + it * 4 + sub, &m);
      off[it] = m * (long long)ldo;
      vmask |= uint32_t(ok) << it;
    }
#pragma unroll 1
    for (int j = 0; j < chunks; ++j) {
      const int acc_col = n0 + j * 32 + c4;                                   // accumulator column (bias index)
      const int col = geglu ? n_tile * half + j * 32 + c4 : acc_col;          // output column
      const int nv = n_out - col;
      float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f), g4 = b4;
      if (bias && nv >= 4) {
        b4 = __ldg(reinterpret_cast<const float4*>(bias + acc_col));
        if (geglu) g4 = __ldg(reinterpret_cast<const float4*>(bias + acc_col + half));
      } else if (bias && nv > 0) {
        b4.x = __ldg(bias + acc_col);
        if (nv > 1) b4.y = __ldg(bias + acc_col + 1);
        if (nv > 2) b4.z = __ldg(bias + acc_col + 2);
      }
      // warp-uniform: the whole 32-column chunk is inside the matrix
      const int chunk_nv = n_out - (col - c4);
      if (chunk_nv <= 0) break;
      // split output: the whole chunk lies on one side of split_col (both multiples of 32)
      const bool hi = kBand && !raw && e.out_f32_hi != nullptr && col - c4 >= e.split_col;
      float* const o32 = hi ? e.out_f32_hi : out_f32;
      const int ocol = hi ? col - e.split_col : col;
      const float* s_chunk = s_rd + j * 32;
      const bool vec = ld_vec && nv >= 4;
      if (!geglu && !silu && !relu && ld_vec && chunk_nv >= 32) {
        // fast path: all scratch and residual loads of the lane's 4 rows are issued before anything is consumed
        float4 x[4], rr[4];
#pragma unroll
        for (int it = 0; it < 4; ++it) x[it] = *reinterpret_cast<const float4*>(s_chunk + it * (4 * kPitch));
        if (residual) {
#pragma unroll
          for (int it = 0; it < 4; ++it)
            rr[it] = ((vmask >> it) & 1u) ? __ldg(reinterpret_cast<const float4*>(residual + off[it] + col))
                                          : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          float4 v = make_float4(__fmaf_rn(x[it].x, scale, b4.x), __fmaf_rn(x[it].y, scale, b4.y),
                                 __fmaf_rn(x[it].z, scale, b4.z), __fmaf_rn(x[it].w, scale, b4.w));
          if (residual) {
            v.x = __fadd_rn(v.x, rr[it].x); v.y = __fadd_rn(v.y, rr[it].y);
            v.z = __fadd_rn(v.z, rr[it].z); v.w = __fadd_rn(v.w, rr[it].w);
          }
          if ((vmask >> it) & 1u) {
            const long long o = off[it] + col;
            if (o32) *reinterpret_cast<float4*>(o32 + off[it] + ocol) = v;
            if (out_bf16)
              *reinterpret_cast<uint2*>(out_bf16 + o) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
          }
        }
      } else {
        // general path (GEGLU's erf polynomial, SiLU, ragged / unaligned tails): rolled to stay small
#pragma unroll 1
        for (int it = 0; it < 4; ++it) {
          float4 x = *reinterpret_cast<const float4*>(s_chunk + it * (4 * kPitch));
          if (geglu) {
            const float4 g = *reinterpret_cast<const float4*>(s_chunk + half + it * (4 * kPitch));
            // (value + bias) * gelu(gate + bias)
            x.x = __fmul_rn(__fadd_rn(x.x, b4.x), gelu_erf(__fadd_rn(g.x, g4.x)));
            x.y = __fmul_rn(__fadd_rn(x.y, b4.y), gelu_erf(__fadd_rn(g.y, g4.y)));
            x.z = __fmul_rn(__fadd_rn(x.z, b4.z), gelu_erf(__fadd_rn(g.z, g4.z)));
            x.w = __fmul_rn(__fadd_rn(x.w, b4.w), gelu_erf(__fadd_rn(g.w, g4.w)));
          } else {
            x.x = fmaf(x.x, scale, b4.x); x.y = fmaf(x.y, scale, b4.y);
            x.z = fmaf(x.z, scale, b4.z); x.w = fmaf(x.w, scale, b4.w);
            if (silu) { x.x = silu_f(x.x); x.y = silu_f(x.y); x.z = silu_f(x.z); x.w = silu_f(x.w); }
            if (relu) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
          }
          if (!((vmask >> it) & 1u) || nv <= 0) continue;
          const long long o = off[it] + col;
          if (vec) {
            if (residual) {
              const float4 rr = __ldg(reinterpret_cast<const float4*>(residual + o));
              x.x += rr.x; x.y += rr.y; x.z += rr.z; x.w += rr.w;
            }
            if (o32) *reinterpret_cast<float4*>(o32 + off[it] + ocol) = x;
            if (out_bf16)
              *reinterpret_cast<uint2*>(out_bf16 + o) = make_uint2(pack_bf16x2(x.x, x.y), pack_bf16x2(x.z, x.w));
          } else {
            store_tail(x, nv, residual, o32, out_bf16, o, off[it] + ocol);
          }
        }
      }
    }
  }
  if (dbg && threadIdx.x == 0) { dbg[4] = clock64(); dbg[5] = clock64(); }
}

// -------------------------------------------------------------------------------------------------
// Split-K deferred epilogue: sum the partials, then the same fused epilogue on CUDA cores.
// Column-owner mapping: a thread owns up to kSkQuads column quads and walks a block of rows (fixed summation order
// over the splits: deterministic).
// -------------------------------------------------------------------------------------------------
constexpr int kSkThreads = 256;
constexpr int kSkQuads = 3;      // N <= 3072

__global__ void __launch_bounds__(kSkThreads) splitk_epilogue_kernel(const GemmParams p, int splits, int rows_per_block,
                                                                     int blocks_per_img, int rows_per_img) {
  pdl_launch_dependents();
  pdl_wait();
  const GemmEpilogue& e = p.epi;
  const int nq = p.N / 4;
  const int img = blockIdx.x / blocks_per_img;
  const int r0 = img * rows_per_img + (blockIdx.x % blocks_per_img) * rows_per_block;
  const int r1 = min(r0 + rows_per_block, (img + 1) * rows_per_img);
  const size_t slab = (size_t)p.M * p.N;
#pragma unroll
  for (int k = 0; k < kSkQuads; ++k) {
    const int q = threadIdx.x + k * kSkThreads;
    if (q >= nq) break;
    const int c = q * 4;
    float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (e.bias) b4 = __ldg(reinterpret_cast<const float4*>(e.bias + c));
    for (int m = r0; m < r1; ++m) {
      const float* src = p.partial + (size_t)m * p.N + c;
      float4 a = __ldg(reinterpret_cast<const float4*>(src));
      for (int s = 1; s < splits; ++s) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(src + (size_t)s * slab));
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      }
      float v[4] = {a.x, a.y, a.z, a.w};
      if (e.flags & EPI_SCALE) { v[0] *= e.scale; v[1] *= e.scale; v[2] *= e.scale; v[3] *= e.scale; }
      v[0] += b4.x; v[1] += b4.y; v[2] += b4.z; v[3] += b4.w;
      if (e.flags & EPI_SILU) { v[0] = silu_f(v[0]); v[1] = silu_f(v[1]); v[2] = silu_f(v[2]); v[3] = silu_f(v[3]); }
      if (e.flags & EPI_RELU) { v[0] = fmaxf(v[0], 0.f); v[1] = fmaxf(v[1], 0.f); v[2] = fmaxf(v[2], 0.f); v[3] = fmaxf(v[3], 0.f); }
      const long long o = (long long)m * e.ldo + c;
      if (e.residual) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(e.residual + o));
        v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
      }
      if (e.out_f32) *reinterpret_cast<float4*>(e.out_f32 + o) = make_float4(v[0], v[1], v[2], v[3]);
      if (e.out_bf16) *reinterpret_cast<uint2*>(e.out_bf16 + o) = make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]));
    }
  }
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------
static long long* g_gemm_dbg = nullptr;
void set_gemm_debug_buffer(long long* dev_ptr) { g_gemm_dbg = dev_ptr; }

template <int BN, int MINB, bool kBand = false>
static int launch_one(const GemmParams& p_in, int splits, cudaStream_t stream) {
  GemmParams p = p_in;
  p.dbg = g_gemm_dbg;
  const size_t smem = gemm_smem_bytes(BN, p.stages);
  constexpr auto kernel = gemm_tc_kernel<BN, MINB, kBand>;
  TRY(raise_smem_limit_once<kernel>("gemm_tc", 227 * 1024));
  int m_tiles;
  if (p.mode == 0) {
    m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  } else {
    m_tiles = (p.M / (p.H * p.W)) * p.tiles_x * p.tiles_y;
  }
  dim3 grid(m_tiles, (p.N + BN - 1) / BN, splits);
  return launch_pdl("gemm_tc", kernel, grid, kGemmThreads, smem, stream, p);
}

int launch_gemm_tc(const GemmParams& p, int block_n, int splits, int ctas_per_sm, cudaStream_t stream) {
  if (p.epi.out_f32_hi || p.ty0 || p.src_y0 || p.out_y0) {
    switch (block_n * 4 + ctas_per_sm) {
      case 64 * 4 + 2: return launch_one<64, 2, true>(p, splits, stream);
      case 128 * 4 + 2: return launch_one<128, 2, true>(p, splits, stream);
      case 64 * 4 + 1: return launch_one<64, 1, true>(p, splits, stream);
      case 128 * 4 + 1: return launch_one<128, 1, true>(p, splits, stream);
      case 160 * 4 + 1: return launch_one<160, 1, true>(p, splits, stream);
      case 256 * 4 + 1: return launch_one<256, 1, true>(p, splits, stream);
      default: set_error("gemm_tc: no row-band kernel for block_n %d", block_n); return MGB_ERR_INVALID;
    }
  }
  if (ctas_per_sm == 2) {
    switch (block_n) {
      case 64: return launch_one<64, 2>(p, splits, stream);
      case 128: return launch_one<128, 2>(p, splits, stream);
      default: break;
    }
  }
  switch (block_n) {
    case 16: return launch_one<16, 1>(p, splits, stream);
    case 32: return launch_one<32, 1>(p, splits, stream);
    case 64: return launch_one<64, 1>(p, splits, stream);
    case 128: return launch_one<128, 1>(p, splits, stream);
    case 160: return launch_one<160, 1>(p, splits, stream);
    case 256: return launch_one<256, 1>(p, splits, stream);
    default: set_error("gemm_tc: no kernel for block_n %d", block_n); return MGB_ERR_CUDA;
  }
}

int launch_splitk_epilogue(const GemmParams& p_in, int block_n, int splits, cudaStream_t stream) {
  (void)block_n;
  GemmParams p = p_in;
  if ((p.epi.flags & EPI_GEGLU) || (p.N & 3) || (p.epi.ldo & 3) || p.N / 4 > kSkThreads * kSkQuads) {
    set_error("split-K epilogue: unsupported shape/flags (N=%d ldo=%d flags=%d)", p.N, p.epi.ldo, p.epi.flags);
    return MGB_ERR_CUDA;
  }
  // blocks never straddle images (rows_per_img = hw when known, else the whole M)
  const int rows_per_img = (p.epi.hw > 0 && p.M % p.epi.hw == 0) ? p.epi.hw : p.M;
  const int imgs = p.M / rows_per_img;
  int blocks_per_img = std::max(1, std::min(rows_per_img, (kNumSMs * 2) / imgs));
  const int rows_per_block = (rows_per_img + blocks_per_img - 1) / blocks_per_img;
  blocks_per_img = (rows_per_img + rows_per_block - 1) / rows_per_block;
  return launch_pdl("splitk epilogue", splitk_epilogue_kernel, imgs * blocks_per_img, kSkThreads, 0, stream, p, splits,
                    rows_per_block, blocks_per_img, rows_per_img);
}

// ---- tensor maps ----
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

static int make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                     const uint32_t* box) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point unavailable");
    return MGB_ERR_CUDA;
  }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1; }
  for (int i = 0; i < rank - 1; ++i) gstr[i] = strides[i];
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,..] box=[%u,%u,..] base=%p", int(r), rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1], base);
    return MGB_ERR_CUDA;
  }
  return MGB_OK;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                 uint32_t box_inner, uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {row_stride_bytes};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap(out, base, 2, dims, strides, box);
}
int make_tmap_3d(CUtensorMap* out, const void* base, const uint64_t dims[3], const uint64_t strides_bytes[2],
                 const uint32_t box[3]) {
  return make_tmap(out, base, 3, dims, strides_bytes, box);
}
int make_tmap_5d(CUtensorMap* out, const void* base, const uint64_t dims[5], const uint64_t strides_bytes[4],
                 const uint32_t box[5]) {
  return make_tmap(out, base, 5, dims, strides_bytes, box);
}

}  // namespace mgb
