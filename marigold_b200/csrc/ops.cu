// Host-side operator builders: turn "linear" / "conv2d" requests into GemmParams (tensor maps, tile
// geometry, tap tables) and pick tile shapes. Used by the network composition (net.cu) and by the
// operator-level C ABI (api.cu).
#include <algorithm>
#include <cstring>

#include "device.h"
#include "kernels.h"
#include "ops.h"

namespace mgb {

void conv_tile_shape(int Hout, int Wout, int* tile_w, int* tile_h) {
  int best_w = 16, best_tiles = 1 << 30;
  const int cands[5] = {128, 64, 32, 16, 8};
  for (int tw : cands) {
    const int th = 128 / tw;
    const int tiles = ((Wout + tw - 1) / tw) * ((Hout + th - 1) / th);
    if (tiles < best_tiles) { best_tiles = tiles; best_w = tw; }
  }
  *tile_w = best_w;
  *tile_h = 128 / best_w;
}

int fill_linear_params(GemmParams* p, const bf16* a, const bf16* w, int M, int N, int K, int block_n, int splits,
                       int stages, const bf16* a2, int K2) {
  // a2 (optional): second row-major operand [M, K2]; the weight is [N, K + K2] (K concatenation)
  memset(p, 0, sizeof(*p));
  if (K % 64 != 0 || M <= 0 || N <= 0 || (a2 && (K2 % 64 != 0 || K2 <= 0))) {
    set_error("linear: need K %% 64 == 0 (got M=%d N=%d K=%d K2=%d)", M, N, K, K2);
    return MGB_ERR_INVALID;
  }
  if (!a2) K2 = 0;
  p->mode = 0;
  p->M = M; p->N = N;
  p->num_kb1 = K / 64;
  p->num_kb = (K + K2) / 64;
  if (splits < 1) splits = 1;
  splits = std::min(splits, p->num_kb);
  p->kb_per_split = (p->num_kb + splits - 1) / splits;
  p->stages = stages;
  int rc = make_tmap_2d(&p->tmap_a, a, uint64_t(K), uint64_t(M), uint64_t(K) * 2, 64, 128);
  if (rc) return rc;
  if (a2) {
    rc = make_tmap_2d(&p->tmap_a2, a2, uint64_t(K2), uint64_t(M), uint64_t(K2) * 2, 64, 128);
    if (rc) return rc;
  }
  rc = make_tmap_2d(&p->tmap_b, w, uint64_t(K + K2), uint64_t(N), uint64_t(K + K2) * 2, 64, uint32_t(block_n));
  return rc;
}

int fill_conv_params(GemmParams* p, const bf16* x, const bf16* w, int NB, int Hout, int Wout, int Cin, int Cout,
                     int kind, int block_n, int splits, int stages, int Hsrc, int Wsrc, const bf16* x2, int Cin2) {
  // x2 (optional): bf16 NHWC [NB, Hout, Wout, Cin2], the operand of a 1x1 convolution over the same output pixels whose
  // weight columns follow the taps in w ([Cout, ntaps * Cin + Cin2]): K concatenation (stride-1 kinds only)
  // Hsrc x Wsrc: spatial extent of the tensor the taps address (the image for stride 1; one parity plane for
  // stride 2, i.e. ceil(Hin / 2) x ceil(Win / 2), which exceeds the output by one for the VAE's pad-(0,1,0,1) conv
  // on an odd input). <= 0: same as the output.
  if (Hsrc <= 0) Hsrc = Hout;
  if (Wsrc <= 0) Wsrc = Wout;
  memset(p, 0, sizeof(*p));
  if (Cin % 64 != 0 || NB <= 0 || Hout <= 0 || Wout <= 0) {
    set_error("conv2d: need Cin %% 64 == 0 (got NB=%d H=%d W=%d Cin=%d)", NB, Hout, Wout, Cin);
    return MGB_ERR_INVALID;
  }
  p->mode = 1;
  p->M = NB * Hout * Wout;
  p->N = Cout;
  p->H = Hout; p->W = Wout;
  conv_tile_shape(Hout, Wout, &p->tile_w, &p->tile_h);
  p->tile_w_shift = 0;
  while ((1 << p->tile_w_shift) < p->tile_w) ++p->tile_w_shift;
  p->tiles_x = (Wout + p->tile_w - 1) / p->tile_w;
  p->tiles_y = (Hout + p->tile_h - 1) / p->tile_h;
  p->cblocks = Cin / 64;
  int planes = 1;
  if (kind == 0) {
    p->ntaps = 9;
    for (int kh = 0; kh < 3; ++kh)
      for (int kw = 0; kw < 3; ++kw) {
        const int t = kh * 3 + kw;
        p->tap_p[t] = 0; p->tap_dy[t] = int8_t(kh - 1); p->tap_dx[t] = int8_t(kw - 1);
      }
  } else if (kind == 1) {
    p->ntaps = 1;
  } else if (kind == 2 || kind == 3) {
    // stride-2 over the 4 parity planes p = (h & 1) * 2 + (w & 1) of the input
    //   kind 2 (pad 1):          input row 2*oh + kh - 1 -> kh=0: (odd, -1)  kh=1: (even, 0)  kh=2: (odd, 0)
    //   kind 3 (pad (0,1,0,1)):  input row 2*oh + kh     -> kh=0: (even, 0)  kh=1: (odd, 0)   kh=2: (even, +1)
    planes = 4;
    p->ntaps = 9;
    const int par2[3] = {1, 0, 1}, off2[3] = {-1, 0, 0};
    const int par3[3] = {0, 1, 0}, off3[3] = {0, 0, 1};
    for (int kh = 0; kh < 3; ++kh)
      for (int kw = 0; kw < 3; ++kw) {
        const int t = kh * 3 + kw;
        const int ph = kind == 2 ? par2[kh] : par3[kh], pw = kind == 2 ? par2[kw] : par3[kw];
        p->tap_p[t] = int8_t(ph * 2 + pw);
        p->tap_dy[t] = int8_t(kind == 2 ? off2[kh] : off3[kh]);
        p->tap_dx[t] = int8_t(kind == 2 ? off2[kw] : off3[kw]);
      }
  } else {
    set_error("conv2d: unknown kind %d", kind);
    return MGB_ERR_INVALID;
  }
  p->num_kb1 = p->ntaps * p->cblocks;
  if (x2 != nullptr && (Cin2 % 64 != 0 || Cin2 <= 0 || (kind != 0 && kind != 1))) {
    set_error("conv2d: second operand needs Cin2 %% 64 == 0 and a stride-1 kind (got %d, kind %d)", Cin2, kind);
    return MGB_ERR_INVALID;
  }
  p->num_kb = p->num_kb1 + (x2 ? Cin2 / 64 : 0);
  if (splits < 1) splits = 1;
  splits = std::min(splits, p->num_kb);
  p->kb_per_split = (p->num_kb + splits - 1) / splits;
  p->stages = stages;

  const uint64_t C2 = uint64_t(Cin) * 2;
  const uint64_t dims[5] = {uint64_t(Cin), uint64_t(Wsrc), uint64_t(Hsrc), uint64_t(planes), uint64_t(NB)};
  const uint64_t strides[4] = {C2, C2 * Wsrc, C2 * Wsrc * Hsrc, C2 * Wsrc * Hsrc * planes};
  const uint32_t box[5] = {64, uint32_t(p->tile_w), uint32_t(p->tile_h), 1, 1};
  int rc = make_tmap_5d(&p->tmap_a, x, dims, strides, box);
  if (rc) return rc;
  if (x2) {
    const uint64_t C22 = uint64_t(Cin2) * 2;
    const uint64_t dims2[5] = {uint64_t(Cin2), uint64_t(Wout), uint64_t(Hout), 1, uint64_t(NB)};
    const uint64_t strides2[4] = {C22, C22 * Wout, C22 * Wout * Hout, C22 * Wout * Hout};
    const uint32_t box2[5] = {64, uint32_t(p->tile_w), uint32_t(p->tile_h), 1, 1};
    rc = make_tmap_5d(&p->tmap_a2, x2, dims2, strides2, box2);
    if (rc) return rc;
  }
  const uint64_t Ktot = uint64_t(p->ntaps) * Cin + (x2 ? uint64_t(Cin2) : 0);
  rc = make_tmap_2d(&p->tmap_b, w, Ktot, uint64_t(Cout), Ktot * 2, 64, uint32_t(block_n));
  return rc;
}

int effective_splits(const GemmParams& p) { return (p.num_kb + p.kb_per_split - 1) / p.kb_per_split; }

int run_gemm(GemmParams& p, int block_n, float* splitk_ws, cudaStream_t stream) {
  const int splits = effective_splits(p);
  // The special epilogues exist only in the 16-wide instantiation, where one lane holds a whole output row: any other
  // width would silently take the plain NHWC epilogue, and N > 16 would index past that row.
  const int special = p.epi.flags & kSpecialEpilogues;
  if (special) {
    const bool three = (special & (EPI_DEPTH | EPI_NORMALS)) != 0;
    if (block_n != 16 || p.N > 16 || (three && p.N != 3) || !p.epi.out_f32 ||
        ((special & EPI_SCHED) ? (!p.epi.sched_x || !p.epi.sched_k) : p.epi.hw <= 0)) {
      set_error("special epilogue (flags %d) needs block_n 16 (got %d), N <= 16 (N == 3 for depth / normals; got %d), "
                "out_f32, and sched_x + sched_k or hw", p.epi.flags, block_n, p.N);
      return MGB_ERR_INVALID;
    }
  }
  if ((p.epi.flags & EPI_GEGLU) && (block_n % 64 != 0)) {
    set_error("GEGLU epilogue needs block_n %% 64 == 0 (got %d)", block_n);
    return MGB_ERR_INVALID;
  }
  // Multi-wave grids run two CTAs per SM (gemm_tc.cu, MINB = 2): shallow operand rings of <= 113 KB, the epilogue of
  // one tile under the K loop of its neighbour. Single-wave grids, and tiles whose accumulators do not fit half the
  // register file (block_n > 128), keep one CTA per SM with a deep ring.
  // the drained operand ring doubles as the epilogue's staging scratch: it must hold gemm_epi_scratch_bytes()
  const int need = block_n > 16 ? int(gemm_epi_scratch_bytes(block_n)) : 0;
  int ctas_per_sm = 1;
  {
    const long long m_tiles = p.mode == 0 ? (p.M + 127) / 128 : (long long)(p.M / (p.H * p.W)) * p.tiles_x * p.tiles_y;
    const long long ctas = m_tiles * ((p.N + block_n - 1) / block_n) * splits;
    if (block_n >= 64 && block_n <= 128 && ctas > kNumSMs) {
      const int stage_bytes = 16384 + block_n * 128;
      const int max_st = (113 * 1024 - 1280) / stage_bytes;
      const int st = std::min(max_st, std::max(p.stages, (need + stage_bytes - 1) / stage_bytes));
      if (st >= 2 && st * stage_bytes >= need) { p.stages = st; ctas_per_sm = 2; }
    }
  }
  const int kernel_minb = ctas_per_sm == 1 ? 1 : 2;
  if (block_n > 16 && ctas_per_sm == 1) {
    // deepen the pipeline until the ring holds the epilogue scratch
    for (;;) {
      const int ring = p.stages * (16384 + block_n * 128);
      if (ring >= need || p.stages >= 16) break;
      ++p.stages;
    }
  }
  if (p.stages < 2 || p.stages > 8 || gemm_smem_bytes(block_n, p.stages) > 227 * 1024) {
    set_error("gemm: stages=%d does not fit shared memory for block_n=%d", p.stages, block_n);
    return MGB_ERR_INVALID;
  }
  if (splits > 1) {
    if (!splitk_ws) {
      set_error("split-K requested without a workspace");
      return MGB_ERR_INVALID;
    }
    if (p.epi.flags & (EPI_SCHED | EPI_DEPTH | EPI_NORMALS | EPI_NCHW | EPI_GEGLU)) {
      set_error("split-K is not supported with GEGLU or the small-N special epilogues");
      return MGB_ERR_INVALID;
    }
    p.partial = splitk_ws;
  } else {
    p.partial = nullptr;
  }
  TRY(launch_gemm_tc(p, block_n, splits, kernel_minb, stream));
  return splits > 1 ? launch_splitk_epilogue(p, block_n, splits, stream) : MGB_OK;
}

// Tile-shape heuristic. Cost model (SM cycles): per CTA  num_kb * K-block time + epilogue + prologue; CTAs run in waves
// of kNumSMs (1 CTA/SM). The H100's dense bf16 rate is 2048 MAC per cycle and SM, so a 128 x BN x 64 K block cannot take
// less than 4*BN cycles (the tensor-core floor).
// Measured on an H100 SXM (400 W) with the clock stamps of tools/gemm_phases.py, K = 2880, one CTA per SM:
// K block 1030 cycles at BN = 256 (floor 1024), 814 at BN = 160 (floor 640), i.e. max(4*BN + 40, ~800);
// epilogue 6.1 k cycles at BN = 128 / 160 and 9.8 k at BN = 256, ~2.5 k per 64 columns; prologue + first
// operand ~3.6 k. The split-K reduce launch (~9000 cycles + its traffic) is an estimate, not measured.
void choose_tile(int m_tiles, int N, int num_kb, int flags, bool allow_split, int* block_n, int* splits,
                 int* stages) {
  const int cands[6] = {256, 160, 128, 64, 32, 16};
  const bool geglu = (flags & EPI_GEGLU) != 0;
  // the special epilogues run only in the 16-wide instantiation and never under split-K (run_gemm enforces both)
  const bool special = (flags & kSpecialEpilogues) != 0;
  double best = 1e30;
  int bbn = special ? 16 : 128, bsp = 1;
  for (int bn : cands) {
    if (special) break;
    if (geglu && (bn % 64 != 0)) continue;
    if (bn > 64 && N < bn / 2 + 1) continue;  // mostly padding
    if (bn < 64 && N >= 64) continue;         // 16 / 32 wide tiles are for the tiny heads only (N <= 32)
    const int n_tiles = (N + bn - 1) / bn;
    for (int sp = 1; sp <= (allow_split ? 16 : 1); ++sp) {
      if (sp > 1 && num_kb / sp < 4) break;
      const long long ctas = (long long)m_tiles * n_tiles * sp;
      const long long waves = (ctas + kNumSMs - 1) / kNumSMs;
      const int kb = (num_kb + sp - 1) / sp;
      const double per_kb = std::max(4.0 * bn + 40.0, 800.0);
      const double cta_cycles = double(kb) * per_kb + double((bn + 63) / 64) * 2500.0 + 3600.0;
      double t = waves * cta_cycles;
      if (sp > 1) t += 9000.0 + double(m_tiles) * 128.0 * N * sp * 4.0 / (double(kNumSMs) * 64.0);
      if (t < best) { best = t; bbn = bn; bsp = sp; }
    }
  }
  *block_n = bbn;
  *splits = bsp;
  const int stage_bytes = 16384 + bbn * 128;
  const int kb = (num_kb + bsp - 1) / bsp;
  // Deep pipelines (the whole 200 KB) only pay off for long K loops. Short-K GEMMs are dominated by
  // prologue / first-load / epilogue latency: cap them near 110 KB so that the NEXT kernel's CTA (launched
  // early through PDL) can become resident on the same SM and overlap its prologue and first operand loads
  // with this kernel's epilogue.
  const int budget = kb <= 12 ? 110 * 1024 : 200 * 1024;
  int st = int((budget - 2048) / stage_bytes);
  st = std::max(2, std::min(st, 8));
  st = std::min(st, std::max(2, kb));
  *stages = st;
}

}  // namespace mgb
