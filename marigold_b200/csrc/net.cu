// Forward graphs of the Marigold hot path, as sequences of kernels.h launches on one stream:
//   UNet step   (diffusers UNet2DConditionModel, SD-2 config)   reference call: marigold_depth_pipeline.py:461-463
//   VAE encode  (AutoencoderKL.encoder + quant_conv)            reference call: marigold_depth_pipeline.py:491-495
//   VAE decode  (post_quant_conv + AutoencoderKL.decoder)       reference call: marigold_depth_pipeline.py:510-515
// Architecture per SURVEY.md App. A (restated; diffusers itself is not available offline).
//
// Numerics: bf16 tensor-core operands, fp32 accumulation, fp32 residual trunk and latent state;
// GroupNorm/LayerNorm/softmax statistics in fp32.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "launch.h"
#include "net.h"

namespace mgb {

// ---------------------------------------------------------------------------------------------
// arena
// ---------------------------------------------------------------------------------------------
static size_t align1k(size_t x) { return (x + 1023) & ~size_t(1023); }
static constexpr uintptr_t kDryBase = 0x100000;   // a dry run's addresses: kDryBase + bump offset, never dereferenced

void Arena::start() {
  off = 0; n = 0; events = 0;
  rec.clear(); live.clear();
}

void* Arena::alloc(size_t bytes) {
  const size_t a = align1k(off);
  off = a + bytes;
  if (off > peak) peak = off;
  const size_t i = n++;
  if (dry) {
    rec.push_back({bytes, a, events++, 0});
    live.push_back(i);
    return reinterpret_cast<void*>(kDryBase + a);
  }
  if (status != MGB_OK) return nullptr;
  if (plan) {
    if (i >= plan->size() || (*plan)[i].bytes != bytes) {
      set_error("arena: allocation %zu of %zu bytes is not the plan's (%zu buffers)", i, bytes, plan->size());
      status = MGB_ERR_STATE;
      return nullptr;
    }
    const ArenaBuf& b = (*plan)[i];
    if (b.off + b.bytes > cap) { set_error("arena overflow"); status = MGB_ERR_NOMEM; return nullptr; }
    return base + b.off;
  }
  if (off > cap) { set_error("arena overflow"); status = MGB_ERR_NOMEM; return nullptr; }
  return base + a;
}

void Arena::free(const void* p) {
  if (!dry || !p) return;
  const size_t a = size_t(reinterpret_cast<uintptr_t>(p) - kDryBase);
  for (size_t k = live.size(); k-- > 0;) {
    if (rec[live[k]].off == a) {
      rec[live[k]].t_free = events++;
      live.erase(live.begin() + k);
      return;
    }
  }
}

void Arena::release(size_t m) {
  off = m;
  if (!dry) return;
  // everything allocated since the mark: the live buffers at bump offsets >= m, newest first
  for (size_t k = live.size(); k-- > 0;) {
    if (rec[live[k]].off < m) continue;
    rec[live[k]].t_free = events++;
    live.erase(live.begin() + k);
  }
}

void Arena::finish() {
  for (size_t i : live) rec[i].t_free = events;
  live.clear();
  ++events;
}

// First fit in the given order: each buffer at the lowest aligned offset clear of every buffer already placed whose
// lifetime overlaps its own.
static size_t place_in_order(std::vector<ArenaBuf>& b, const std::vector<size_t>& order) {
  std::vector<size_t> placed;
  std::vector<std::pair<size_t, size_t>> busy;
  placed.reserve(b.size());
  size_t peak = 0;
  for (size_t i : order) {
    busy.clear();
    for (size_t j : placed)
      if (b[j].bytes && b[j].t_alloc < b[i].t_free && b[i].t_alloc < b[j].t_free)
        busy.push_back({b[j].off, b[j].off + b[j].bytes});
    std::sort(busy.begin(), busy.end());
    size_t o = 0;
    for (const auto& r : busy) {
      if (o + b[i].bytes <= r.first) break;
      o = std::max(o, align1k(r.second));
    }
    b[i].off = o;
    placed.push_back(i);
    peak = std::max(peak, o + b[i].bytes);
  }
  return peak;
}

size_t arena_place(std::vector<ArenaBuf>& bufs, int placement) {
  std::vector<size_t> order(bufs.size());
  for (size_t i = 0; i < order.size(); ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(),
                   [&](size_t x, size_t y) { return bufs[x].t_alloc < bufs[y].t_alloc; });
  if (placement == 1) {
    std::reverse(order.begin(), order.end());
    return place_in_order(bufs, order);
  }
  // In allocation order, every aligned offset below the top of a stack is taken, so a stack-shaped sequence lands
  // where the bump allocator puts it, whose aligned peak no placement beats. Largest first replaces it only where it
  // needs strictly less memory (rounded to the alignment).
  std::vector<ArenaBuf> by_size = bufs;
  const size_t peak = place_in_order(bufs, order);
  std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return bufs[x].bytes > bufs[y].bytes; });
  const size_t peak2 = place_in_order(by_size, order);
  if (align1k(peak2) >= align1k(peak)) return peak;
  bufs.swap(by_size);
  return peak2;
}

// Arena memory for n T's. A failed allocation turns the rest of the forward into a dry run: nothing more is launched,
// and the caller reports the arena's status.
template <typename T>
static T* aalloc(Ctx& c, size_t n) {
  void* p = c.arena->alloc(n * sizeof(T));
  if (c.dry) return reinterpret_cast<T*>(p);
  if (!p) {
    c.dry = true;
  } else if (c.opt.poison && cudaMemsetAsync(p, 0xFF, n * sizeof(T), c.stream) != cudaSuccess) {
    set_error("arena poison memset failed");
    c.arena->status = MGB_ERR_CUDA;
    c.dry = true;
  }
  return reinterpret_cast<T*>(p);
}

// ---------------------------------------------------------------------------------------------
// launch wrappers (skipped in dry-run mode, which only measures arena / split-K needs)
// ---------------------------------------------------------------------------------------------
struct Epi {
  const float* bias = nullptr;
  const float* residual = nullptr;
  float* out_f32 = nullptr;
  bf16* out_bf16 = nullptr;
  int flags = 0;
  float scale = 1.f;
  int hw = 0;
  const float* sched_x = nullptr;
  const float* sched_z = nullptr;
  const float* sched_k = nullptr;
  float* aux_out = nullptr;
  float* out_f32_hi = nullptr;   // columns [split_col, N) of an fp32 output (GemmEpilogue::out_f32_hi)
  int split_col = 0;
};

// Debug only (tools/marginal_cost.py): MGB_SKIP=gn,ln,attn,xattn,gemm drops a kernel family from the graph so
// that its marginal in-graph cost can be read from the step time. Results are garbage when set.
static bool skip_family(const char* name) {
  static const char* env = getenv("MGB_SKIP");
  return env && strstr(env, name) != nullptr;
}

static void set_epi(GemmParams& p, const Epi& e, int ldo) {
  p.epi.bias = e.bias; p.epi.residual = e.residual; p.epi.out_f32 = e.out_f32; p.epi.out_bf16 = e.out_bf16;
  p.epi.ldo = ldo; p.epi.flags = e.flags; p.epi.hw = e.hw; p.epi.scale = e.scale;
  p.epi.sched_x = e.sched_x; p.epi.sched_z = e.sched_z; p.epi.sched_k = e.sched_k; p.epi.aux_out = e.aux_out;
  p.epi.out_f32_hi = e.out_f32_hi; p.epi.split_col = e.split_col;
}

static int gemm_common(Ctx& c, GemmParams& p, int bn, int splits, const Epi& e, int ldo) {
  if (skip_family("gemm")) return MGB_OK;
  set_epi(p, e, ldo);
  if (splits > 1) {
    const size_t need = size_t(splits) * p.M * p.N * sizeof(float);
    if (need > c.splitk_cap) {
      set_error("split-K workspace too small (%zu > %zu)", need, c.splitk_cap);
      return MGB_ERR_STATE;
    }
  }
  return run_gemm(p, bn, c.splitk_ws, c.stream);
}

struct Tile { int bn, sp, st; };

// the tile of an M-row linear over W: choose_tile's, or GEGLU's fixed one
static Tile linear_tile(int M, const LinW& W, int flags) {
  Tile t;
  choose_tile((M + 127) / 128, W.n, W.k / 64, flags, true, &t.bn, &t.sp, &t.st);
  if (flags & EPI_GEGLU) t = {256, 1, (W.k / 64 <= 12) ? 2 : 4};
  return t;
}

// y = a[M,K] W^T (+ epilogue); ldo = row stride of the outputs (0: W.n, or W.n / 2 for GEGLU)
// tile (or null: linear_tile's): a block of rows of a larger problem passes that problem's tile, so that its rows come
// out bit for bit as they do in the whole (the K split and the epilogue path depend on the tile, never on the row)
static int linear(Ctx& c, const bf16* a, int M, const LinW& W, const Epi& e, int ldo = 0, const bf16* a2 = nullptr,
                  int K1 = 0, const Tile* tile = nullptr) {
  // a2 != nullptr: K concatenation, A = [a (K1 columns) | a2 (W.k - K1 columns)]
  const bool geglu = (e.flags & EPI_GEGLU) != 0;
  const Tile t = tile ? *tile : linear_tile(M, W, e.flags);
  const int bn = t.bn, sp = t.sp, st = t.st;
  if (sp > 1) c.splitk_need = std::max(c.splitk_need, size_t(sp) * M * W.n * sizeof(float));
  if (c.dry) return MGB_OK;
  GemmParams p;
  if (a2) TRY(fill_linear_params(&p, a, W.w, M, W.n, K1, bn, sp, st, a2, W.k - K1));
  else TRY(fill_linear_params(&p, a, W.w, M, W.n, W.k, bn, sp, st));
  return gemm_common(c, p, bn, effective_splits(p), e, ldo > 0 ? ldo : (geglu ? W.n / 2 : W.n));
}

// generic A[M,K] x B[N,K]^T with raw pointers (attention score / PV GEMMs in the VAE)
static int matmul_nt(Ctx& c, const bf16* a, const bf16* b, int M, int N, int K, const Epi& e, int ldo,
                     const Tile& tile) {
  LinW W; W.w = const_cast<bf16*>(b); W.n = N; W.k = K;
  // B is an activation written by an earlier kernel of this stream (K, or V^T straight out of the transpose): the
  // GEMM's pre-wait B prefetch must not run ahead of its producer, so no programmatic early launch here.
  PlainLaunchScope no_early_launch;
  return linear(c, a, M, W, e, ldo, nullptr, 0, &tile);
}
static Tile matmul_tile(int M, int N, int K, int flags) {
  LinW W; W.n = N; W.k = K;
  return linear_tile(M, W, flags);
}

// the tile of a conv3x3 over NB images of Hout x Wout (choose_tile's), and the image's tile rows
static Tile conv_tile(int NB, int Hout, int Wout, const ConvW& W, int flags, int* tile_h = nullptr,
                      int* tiles_y = nullptr) {
  int tw, th;
  conv_tile_shape(Hout, Wout, &tw, &th);
  const int m_tiles = NB * ((Wout + tw - 1) / tw) * ((Hout + th - 1) / th);
  Tile t;
  choose_tile(m_tiles, W.cout, (9 * W.cin_pad + W.k_extra) / 64, flags, true, &t.bn, &t.sp, &t.st);
  if (tile_h) *tile_h = th;
  if (tiles_y) *tiles_y = (Hout + th - 1) / th;
  return t;
}

// 3x3 conv on NHWC bf16; Hout x Wout output; kind per ops.cu
static int conv3x3(Ctx& c, const bf16* x, int NB, int Hout, int Wout, const ConvW& W, int kind, const Epi& e,
                   int Hsrc = 0, int Wsrc = 0, const bf16* x2 = nullptr) {
  if ((x2 != nullptr) != (W.k_extra > 0)) { set_error("conv3x3: second operand / weight layout mismatch"); return MGB_ERR_STATE; }
  const Tile t = conv_tile(NB, Hout, Wout, W, e.flags);
  const int bn = t.bn, sp = t.sp, st = t.st;
  const size_t M = size_t(NB) * Hout * Wout;
  if (sp > 1) c.splitk_need = std::max(c.splitk_need, size_t(sp) * M * W.cout * sizeof(float));
  if (c.dry) return MGB_OK;
  GemmParams p;
  TRY(fill_conv_params(&p, x, W.w, NB, Hout, Wout, W.cin_pad, W.cout, kind, bn, sp, st, Hsrc, Wsrc, x2, W.k_extra));
  Epi e2 = e;
  e2.hw = Hout * Wout;
  return gemm_common(c, p, bn, effective_splits(p), e2, W.cout);
}

// Tile rows [ty0, ty0 + tiles) of one H x W image of a pad-1 3x3 conv run with tile t, the tile of the whole conv
// (conv_tile over all its images): every output pixel comes out bit for bit as the whole conv computes it, since a
// tile's arithmetic depends on the tile and never on where the tile is. x holds the operand's image rows
// [src_y0, src_y0 + src_rows), which must include every row of the band and its one-row halo that lies in the image;
// the output's row 0 is image row out_y0.
static int conv3x3_band(Ctx& c, const bf16* x, int src_y0, int src_rows, int H, int W, const ConvW& Wt, const Tile& t,
                        const Epi& e, int ldo, int ty0, int tiles, int out_y0) {
  if (t.sp != 1 || Wt.k_extra) { set_error("conv band: the conv splits K or has a second operand"); return MGB_ERR_STATE; }
  if (c.dry) return MGB_OK;
  GemmParams p;
  TRY(fill_conv_params(&p, x, Wt.w, 1, H, W, Wt.cin_pad, Wt.cout, 0, t.bn, 1, t.st, src_rows, W));
  TRY(set_conv_band(&p, ty0, tiles, src_y0, out_y0));
  Epi e2 = e;
  e2.hw = H * W;
  return gemm_common(c, p, t.bn, 1, e2, ldo);
}

#define LAUNCH(call)               \
  do {                             \
    if (!c.dry) TRY(call);         \
  } while (0)

// fp32 trunk tensor [M, C]
static Act act_alloc(Ctx& c, size_t M, int C) {
  Act a;
  a.p = aalloc<float>(c, M * C);
  a.C = C;
  return a;
}

// GroupNorm (+SiLU) over [a | b] (b == nullptr: single source) -> bf16 operand; one deterministic launch (norm.cu).
// Scratch: partials from the arena (freed on return in a planned forward, else released by the caller's mark), one
// barrier counter per image from the per-forward
// counter slab (zeroed once per forward by zero_counters()).
static int groupnorm(Ctx& c, const Act& a, const Act* b, bf16* y, bf16* raw, const NormW& n, int NB, int HW, float eps,
                     int silu) {
  if (skip_family("gn")) return MGB_OK;
  const int Cb = (b && b->p) ? b->C : 0;
  void* part = aalloc<char>(c, groupnorm_part_bytes(NB, HW, a.C + Cb, c.groups));
  const size_t coff = c.sync_off;
  c.sync_off += size_t(NB);
  if (c.sync_off > c.sync_need) c.sync_need = c.sync_off;
  int rc = MGB_OK;
  if (!c.dry) {
    if (c.sync_off > c.sync_cap) { set_error("groupnorm: barrier counter slab exhausted"); return MGB_ERR_STATE; }
    rc = launch_gn_fused(a.p, a.C, Cb ? b->p : nullptr, Cb, y, raw, n.g, n.b, NB, HW, c.groups, eps, silu, part,
                         c.sync_base + coff, c.stream);
  }
  if (c.planned) c.arena->free(part);   // read by this launch alone
  return rc;
}

// ---------------------------------------------------------------------------------------------
// ResnetBlock2D: GN -> SiLU -> conv3x3 (+temb) -> GN -> SiLU -> conv3x3 ; + (1x1 shortcut | x)
//   x fp32 [M, cin] -> y fp32 [M, cout] (y preallocated by the caller, or in a planned forward allocated here if y.p
//   is null)
// In a planned forward (c.planned) each buffer is allocated where it is first written and freed after its last read,
// and with consume_x so is x: after the first GroupNorm where the shortcut reads GroupNorm's raw copy instead, else
// after conv2. Otherwise (the UNet step) the scratch is allocated at entry, the stack layout its captured graph holds.
// ---------------------------------------------------------------------------------------------
static int resnet_forward(Ctx& c, const ResnetW& R, Act& x, Act* skip, Act& y, int NB, int H, int W,
                          bool consume_x = false) {
  const bool planned = c.planned;
  // input = x, or the channel concat [x | skip] of an up block (never materialised in fp32: GroupNorm reads both
  // sources, and the 1x1 shortcut reads the bf16 copy GroupNorm emits)
  const size_t M = size_t(NB) * H * W;
  const size_t mk = c.arena->mark();
  bf16* t1 = aalloc<bf16>(c, M * R.cin);
  bf16* raw = R.has_sc ? aalloc<bf16>(c, M * R.cin) : nullptr;
  Act h;
  bf16* t2 = nullptr;
  if (!planned) {
    h = act_alloc(c, M, R.cout);
    t2 = aalloc<bf16>(c, M * R.cout);
  }
  TRY(groupnorm(c, x, skip, t1, raw, R.n1, NB, H * W, R.eps, 1));
  if (consume_x && R.has_sc) c.arena->free(x.p);
  if (planned) h = act_alloc(c, M, R.cout);
  Epi e1;
  e1.bias = (R.bias_off >= 0 && c.cur_bias) ? c.cur_bias + R.bias_off : R.c1.b;
  e1.out_f32 = h.p;
  TRY(conv3x3(c, t1, NB, H, W, R.c1, 0, e1));
  if (planned) {
    c.arena->free(t1);
    t2 = aalloc<bf16>(c, M * R.cout);
  }
  TRY(groupnorm(c, h, nullptr, t2, nullptr, R.n2, NB, H * W, R.eps, 1));
  if (planned) c.arena->free(h.p);
  if (!y.p) y = act_alloc(c, M, R.cout);
  // conv2 (+ residual). Where the block changes the channel count, diffusers adds conv_shortcut(x), a 1x1 convolution:
  // its K blocks are appended to conv2's implicit GEMM (weights [W2 | Wsc], bias b2 + bsc, second A operand = the raw
  // bf16 copy of the block input), which removes a GEMM launch (plus a split-K reduce on the small levels) and the
  // fp32 round trip of its output
  Epi e2; e2.bias = R.c2.b; e2.out_f32 = y.p;
  if (!R.has_sc) e2.residual = x.p;
  TRY(conv3x3(c, t2, NB, H, W, R.c2, 0, e2, 0, 0, R.has_sc ? raw : nullptr));
  if (planned) {
    c.arena->free(t2);
    c.arena->free(raw);
    if (consume_x && !R.has_sc) c.arena->free(x.p);
  } else {
    c.arena->release(mk);
  }
  return MGB_OK;
}

// GroupNorm statistics of [x | xb] (launch_gn_stats; or x alone) into stats, with groupnorm()'s scratch and barrier
// counter
static int groupnorm_stats(Ctx& c, const float* x, int Ca, const float* xb, int Cb, float2* stats,
                           const NormW& n, int NB, int HW, float eps) {
  void* part = aalloc<char>(c, groupnorm_part_bytes(NB, HW, Ca + Cb, c.groups));
  const size_t coff = c.sync_off;
  c.sync_off += size_t(NB);
  if (c.sync_off > c.sync_need) c.sync_need = c.sync_off;
  int rc = MGB_OK;
  if (!c.dry) {
    if (c.sync_off > c.sync_cap) { set_error("groupnorm: barrier counter slab exhausted"); return MGB_ERR_STATE; }
    rc = launch_gn_stats(x, Ca, xb, Cb, stats, n.g, n.b, NB, HW, c.groups, eps, part, c.sync_base + coff, c.stream);
  }
  c.arena->free(part);
  return rc;
}

// Tile rows per band of the decoder's banded full-resolution convs: about an eighth of the image, or as a test forces.
static int band_tiles(int tiles_y, int force) {
  return force > 0 ? std::min(force, tiles_y) : std::max(1, (tiles_y + 7) / 8);
}

// ---------------------------------------------------------------------------------------------
// The decoder's last up-conv (Upsample2D: nearest 2x, then a 3x3 conv, cin = cout = 2 * 128) in low memory. h, the
// half-resolution fp32 input, is rounded to bf16 once (a quarter of U; the same bits as upsample2x, a copy plus one
// rounding) and freed with its ping-pong partner. The 2x operand then exists one band of tile rows (plus its halo rows)
// at a time, and the conv runs that band's tiles through a map that starts at the band's first halo row. The epilogue
// splits the output: channels [0, 128) to a, [128, 256) to b, each a packed fp32 128-channel map of its own.
// Peak: a + b + the bf16 input + one band, 2.25 U plus a band. Same tile, split and K order as the whole conv.
// ---------------------------------------------------------------------------------------------
static int up_conv_low_memory(Ctx& c, const ConvW& Wt, Act& h, Act& partner, Act& a, Act& b, int NB, int H, int W) {
  const int cin = Wt.cin_pad, half = Wt.cout / 2;
  if (cin != Wt.cout || half % 32 || !c.planned) {
    set_error("up-conv in low memory: needs a planned arena and cin = cout, a multiple of 64 (got %d -> %d)", cin, Wt.cout);
    return MGB_ERR_STATE;
  }
  const int Hh = H / 2, Wh = W / 2, HW = H * W;
  bf16* xh = aalloc<bf16>(c, size_t(NB) * Hh * Wh * cin);
  LAUNCH(launch_cast_bf16(h.p, xh, size_t(NB) * Hh * Wh * cin, c.stream));
  c.arena->free(h.p);
  c.arena->free(partner.p);
  h = partner = Act();
  a = act_alloc(c, size_t(NB) * HW, half);
  b = act_alloc(c, size_t(NB) * HW, half);
  int th, tiles_y;
  const Tile t = conv_tile(NB, H, W, Wt, 0, &th, &tiles_y);
  const int bt = band_tiles(tiles_y, c.opt.band_up_tiles);
  bf16* band = aalloc<bf16>(c, size_t(std::min(H, bt * th + 2)) * W * cin);
  Epi e; e.bias = Wt.b; e.split_col = half;
  for (int n = 0; n < NB; ++n) {
    e.out_f32 = a.p + size_t(n) * HW * half;
    e.out_f32_hi = b.p + size_t(n) * HW * half;
    for (int ty0 = 0; ty0 < tiles_y; ty0 += bt) {
      const int tiles = std::min(bt, tiles_y - ty0);
      const int lo = std::max(0, ty0 * th - 1), hi = std::min(H, (ty0 + tiles) * th + 1);
      LAUNCH(launch_upsample2x_rows(xh + size_t(n) * Hh * Wh * cin, band, Hh, Wh, cin, lo, hi, c.stream));
      TRY(conv3x3_band(c, band, lo, hi - lo, H, W, Wt, t, e, half, ty0, tiles, 0));
    }
  }
  c.arena->free(band);
  c.arena->free(xh);
  return MGB_OK;
}

// ---------------------------------------------------------------------------------------------
// The ResnetBlock2D with a 1x1 shortcut over cin = 2 cout channels after up_conv_low_memory, on its input as the two
// packed fp32 halves a = channels [0, cout) and b = [cout, cin), in 2.5 U. Same operands, tiles, splits and K order as
// resnet_forward, hence the same bits. Planned arena only; consumes a, and y is b.
//   GroupNorm 1  statistics over [a | b], then the row apply: each warp reads both halves of its row, then writes the
//                shortcut's operand raw = bf16([a | b]) (2 cin bytes) over a's row and conv1's operand t1 over b's.
//   conv1        in bands of tile rows, each into one of two staging bands; band k's output is copied over b's rows
//                of band k only after band k + 1's conv is enqueued, the last conv that reads t1 rows of band k.
//   GroupNorm 2  over h (b) into t2; conv2 reads t2 and raw (a) and writes y over b.
// Peak: a + b + t2.
// ---------------------------------------------------------------------------------------------
static int resnet_shortcut_halves(Ctx& c, const ResnetW& R, Act& a, Act& b, Act& y, int NB, int H, int W) {
  if (R.cin != 2 * R.cout || !R.has_sc || !c.planned || a.C != R.cout || b.C != R.cout) {
    set_error("resnet on halves: needs a planned arena and a 1x1 shortcut over cin = 2 cout (got %d -> %d)", R.cin, R.cout);
    return MGB_ERR_STATE;
  }
  const int HW = H * W, cin = R.cin, cout = R.cout;
  const size_t M = size_t(NB) * HW;
  float2* st = aalloc<float2>(c, size_t(NB) * cin);
  TRY(groupnorm_stats(c, a.p, cout, b.p, cout, st, R.n1, NB, HW, R.eps));
  bf16* raw = reinterpret_cast<bf16*>(a.p);
  bf16* t1 = reinterpret_cast<bf16*>(b.p);
  LAUNCH(launch_gn_apply_rows(a.p, b.p, cout, st, t1, raw, NB, HW, cin, 1, c.stream));
  c.arena->free(st);
  int th, tiles_y;
  const Tile t = conv_tile(NB, H, W, R.c1, 0, &th, &tiles_y);
  const int bt = band_tiles(tiles_y, c.opt.band_conv1_tiles);
  const size_t band_px = size_t(std::min(H, bt * th)) * W;
  float* stage[2] = {aalloc<float>(c, band_px * cout), aalloc<float>(c, band_px * cout)};
  Epi e1;
  e1.bias = (R.bias_off >= 0 && c.cur_bias) ? c.cur_bias + R.bias_off : R.c1.b;
  for (int n = 0; n < NB; ++n) {
    const bf16* x = t1 + size_t(n) * HW * cin;
    float* hn = b.p + size_t(n) * HW * cout;
    int prev = -1;   // first tile row of the band whose output waits in its staging band
    for (int ty0 = 0;; ty0 += bt) {
      if (ty0 < tiles_y) {
        e1.out_f32 = stage[(ty0 / bt) & 1];
        TRY(conv3x3_band(c, x, 0, H, H, W, R.c1, t, e1, cout, ty0, std::min(bt, tiles_y - ty0), ty0 * th));
      }
      if (prev >= 0) {
        const int r0 = prev * th, r1 = std::min(H, (prev + bt) * th);
        LAUNCH(launch_copy_rows(stage[(prev / bt) & 1], hn + size_t(r0) * W * cout, (long long)(r1 - r0) * W, cout,
                                c.stream));
      }
      if (ty0 >= tiles_y) break;
      prev = ty0;
    }
  }
  c.arena->free(stage[1]);
  c.arena->free(stage[0]);
  st = aalloc<float2>(c, size_t(NB) * cout);
  TRY(groupnorm_stats(c, b.p, cout, nullptr, 0, st, R.n2, NB, HW, R.eps));
  bf16* t2 = aalloc<bf16>(c, M * cout);
  LAUNCH(launch_gn_apply_rows(b.p, nullptr, 0, st, t2, nullptr, NB, HW, cout, 1, c.stream));
  c.arena->free(st);
  Epi e2; e2.bias = R.c2.b; e2.out_f32 = b.p;
  TRY(conv3x3(c, t2, NB, H, W, R.c2, 0, e2, 0, 0, raw));
  c.arena->free(t2);
  c.arena->free(a.p);
  y = b;
  a = b = Act();
  return MGB_OK;
}

// ---------------------------------------------------------------------------------------------
// Row split (Ctx::split_world > 0, one image): an attention's output o holds world chunks of row_split_chunk(T) rows;
// this rank computes the rows of its chunk, and the exchange function fills the others in place (an all-gather).
// ---------------------------------------------------------------------------------------------
static size_t attn_out_rows(const Ctx& c, size_t M, int T) {
  return c.split_world > 0 ? std::max(M, size_t(c.split_world) * row_split_chunk(T, c.split_world)) : M;
}
static void split_rows(const Ctx& c, int T, int* begin, int* end) {
  if (c.split_world <= 0) { *begin = 0; *end = T; return; }
  const int chunk = row_split_chunk(T, c.split_world);
  *begin = std::min(T, c.split_rank * chunk);
  *end = std::min(T, *begin + chunk);
}
static int exchange_rows(Ctx& c, bf16* o, int T, int C) {
  if (c.split_world <= 0 || c.dry) return MGB_OK;
  const size_t chunk_bytes = size_t(row_split_chunk(T, c.split_world)) * C * sizeof(bf16);
  const int st = c.exchange_fn(c.exchange_ctx, o, chunk_bytes, c.split_rank, c.split_world, c.stream);
  if (st != 0) {
    set_error("row split: the exchange function returned %d (rank %d of %d, %zu bytes per rank)", st, c.split_rank,
              c.split_world, chunk_bytes);
    return MGB_ERR_STATE;
  }
  return MGB_OK;
}

// ---------------------------------------------------------------------------------------------
// Transformer2DModel (1 BasicTransformerBlock, linear projections). x fp32 [M, C] -> y fp32 [M, C]
// ---------------------------------------------------------------------------------------------
static int xfmr_forward(Ctx& c, const XfmrW& X, Act& x, Act& y, int NB, int T) {
  const int C = X.C;
  const size_t M = size_t(NB) * T;
  const size_t mk = c.arena->mark();
  bf16* a = aalloc<bf16>(c, M * C);          // normalised operand (reused)
  float* hs0 = aalloc<float>(c, M * C);
  float* hs1 = aalloc<float>(c, M * C);
  bf16* qkv = aalloc<bf16>(c, M * 3 * C);
  bf16* o = aalloc<bf16>(c, attn_out_rows(c, M, T) * C);
  bf16* ffm = aalloc<bf16>(c, M * 4 * C);
  bf16* hsb = aalloc<bf16>(c, M * C);
  const size_t attn_ws_bytes = flash_attn64_ws_bytes(NB, T, C);
  float* attn_ws = attn_ws_bytes ? aalloc<float>(c, attn_ws_bytes / sizeof(float)) : nullptr;

  TRY(groupnorm(c, x, nullptr, a, nullptr, X.gn, NB, T, 1e-6f, 0));
  { Epi e; e.bias = X.proj_in.b; e.out_f32 = hs0; TRY(linear(c, a, int(M), X.proj_in, e)); }
  // self attention
  const bool no_ln = skip_family("ln"), no_attn = skip_family("attn"), no_x = skip_family("xattn");
  if (!no_ln) LAUNCH(launch_layernorm(hs0, a, X.ln1.g, X.ln1.b, int(M), C, 1e-5f, c.stream));
  { Epi e; e.out_bf16 = qkv; TRY(linear(c, a, int(M), X.qkv, e)); }
  {
    int r0, r1;
    split_rows(c, T, &r0, &r1);
    // a rank without rows (r0 = r1 = T) launches an empty range, not the partial last block another rank owns
    const int qb0 = r0 / 128, qb1 = r1 > r0 ? (r1 + 127) / 128 : qb0;
    if (!no_attn) LAUNCH(launch_flash_attn64(qkv, o, NB, T, C, 0.125f, attn_ws, attn_ws_bytes, c.stream, qb0, qb1));
    TRY(exchange_rows(c, o, T, C));
  }
  { Epi e; e.bias = X.o1.b; e.residual = hs0; e.out_f32 = hs1; TRY(linear(c, o, int(M), X.o1, e)); }
  // cross attention against the empty-prompt context, collapsed (norm.cu: xattn2_fused_kernel): LN2, to_q, the 2-key
  // softmax, to_out + residual and LN3 are one launch; hsb = bf16 trunk after attn2, a = LN3 of it for the feed-forward
  if (!no_x) {
    LAUNCH(launch_xattn2_fused(hs1, hsb, a, X.ln2.g, X.ln2.b, X.ln3.g, X.ln3.b, X.xGU, X.xc1, int(M), C, C / 64, 0.125f,
                               1e-5f, c.stream));
  }
  // GEGLU feed-forward
  { Epi e; e.bias = X.ff1.b; e.out_bf16 = ffm; e.flags = EPI_GEGLU; TRY(linear(c, a, int(M), X.ff1, e)); }
  // ff.net.2 + proj_out + the block residual: ONE GEMM over [hs0 | ffm] with the folded weight (api_net.cu)
  {
    Epi e; e.bias = X.ffpo.b; e.residual = x.p; e.out_f32 = y.p;
    TRY(linear(c, hsb, int(M), X.ffpo, e, 0, ffm, C));
  }
  c.arena->release(mk);
  return MGB_OK;
}

// ---------------------------------------------------------------------------------------------
// VAE mid-block attention: single head, dim C (512), over T = h*w tokens. x, y fp32 [NB*T, C].
// Per image: fp32 scores S = Q K^T / sqrt(C) (T x Tp, Tp = T rounded up to 64), fp32 row softmax -> bf16 P with the
// pad columns zeroed, O = P V through V^T [C, Tp] (pad zeroed): any T works, and the logits are never rounded to bf16.
// The queries of an image are taken in blocks of R rows (vae_attn_rows), so S and P take R x Tp, not T x Tp. Both GEMMs
// run every block with the tile of the whole T-row problem: each row is the same kernel's same arithmetic whatever R
// is, and the softmax is row-local, so the output is bit-identical to one block. R = T is exactly the unblocked launch
// sequence.
// ---------------------------------------------------------------------------------------------
int vae_attn_rows(int T, int C, size_t budget, int force_rows) {
  if (force_rows > 0) return std::min(force_rows, T);
  const int Tp = (T + 63) / 64 * 64;
  const size_t row_bytes = size_t(Tp) * (sizeof(float) + sizeof(bf16));
  if (size_t(T) * row_bytes <= budget) return T;
  const Tile pv = matmul_tile(T, C, Tp, 0);
  const int ctas_per_128_rows = (C + pv.bn - 1) / pv.bn * pv.sp;
  const int wave_rows = (kNumSMs + ctas_per_128_rows - 1) / ctas_per_128_rows * 128;
  const int budget_rows = int(std::min(budget / row_bytes, size_t(T))) / 128 * 128;
  return std::min(T, std::max(budget_rows, wave_rows));
}

int vae_attn_core(Ctx& c, const bf16* q, const bf16* k, const bf16* v, bf16* o, int NB, int T, int C, int row_begin,
                  int row_end) {
  if (row_end < 0) row_end = T;
  const int Tp = (T + 63) / 64 * 64;
  const int R = vae_attn_rows(T, C, c.opt.attn_budget, c.opt.attn_rows);
  const Tile tile_s = matmul_tile(T, T, C, EPI_SCALE), tile_pv = matmul_tile(T, C, Tp, 0);
  const size_t mk = c.arena->mark();
  bf16* vt = aalloc<bf16>(c, size_t(C) * Tp);
  float* s = aalloc<float>(c, size_t(R) * Tp);
  bf16* pr = aalloc<bf16>(c, size_t(R) * Tp);
  const float scale = 1.0f / sqrtf(float(C));
  for (int n = 0; n < NB; ++n) {
    const size_t off = size_t(n) * T * C;
    for (int r0 = row_begin; r0 < row_end; r0 += R) {
      const int rows = std::min(R, row_end - r0);
      const size_t qo = off + size_t(r0) * C;
      { Epi e; e.out_f32 = s; e.flags = EPI_SCALE; e.scale = scale; TRY(matmul_nt(c, q + qo, k + off, rows, T, C, e, Tp, tile_s)); }
      LAUNCH(launch_softmax_rows(s, pr, rows, T, Tp, c.stream));
      if (r0 == row_begin) LAUNCH(launch_transpose_bf16(v + off, vt, T, C, Tp, c.stream));
      { Epi e; e.out_bf16 = o + qo; TRY(matmul_nt(c, pr, vt, rows, C, Tp, e, 0, tile_pv)); }
    }
  }
  c.arena->release(mk);
  return MGB_OK;
}

static int vae_attn_forward(Ctx& c, const VaeAttnW& A, Act& x, Act& y, int NB, int T) {
  const int C = A.C;
  const size_t M = size_t(NB) * T;
  const size_t mk = c.arena->mark();
  bf16* a = aalloc<bf16>(c, M * C);
  bf16* q = aalloc<bf16>(c, M * C);
  bf16* k = aalloc<bf16>(c, M * C);
  bf16* v = aalloc<bf16>(c, M * C);
  bf16* o = aalloc<bf16>(c, attn_out_rows(c, M, T) * C);
  TRY(groupnorm(c, x, nullptr, a, nullptr, A.gn, NB, T, 1e-6f, 0));
  { Epi e; e.bias = A.q.b; e.out_bf16 = q; TRY(linear(c, a, int(M), A.q, e)); }
  { Epi e; e.bias = A.k.b; e.out_bf16 = k; TRY(linear(c, a, int(M), A.k, e)); }
  { Epi e; e.bias = A.v.b; e.out_bf16 = v; TRY(linear(c, a, int(M), A.v, e)); }
  int r0, r1;
  split_rows(c, T, &r0, &r1);
  TRY(vae_attn_core(c, q, k, v, o, NB, T, C, r0, r1));
  TRY(exchange_rows(c, o, T, C));
  { Epi e; e.bias = A.o.b; e.residual = x.p; e.out_f32 = y.p; TRY(linear(c, o, int(M), A.o, e)); }
  c.arena->release(mk);
  return MGB_OK;
}

// ---------------------------------------------------------------------------------------------
// UNet step. rgb: fp32 NHWC [NB, lh, lw, 4]; tgt: fp32 NHWC [NB, lh, lw, Ct] (Ct = unet_out_channels: 4, or 4 n for the
// n-target IID models), updated in place by the fused conv_out + scheduler epilogue. raw_out (or null): fp32 NHWC
// [NB, lh, lw, Ct] model output.
// ---------------------------------------------------------------------------------------------
static int zero_counters(Ctx& c) {
  // one memset (a memset node under capture) for the grid-barrier counters of every GroupNorm of this forward
  c.sync_off = 0;
  if (c.dry || !c.sync_base || c.sync_cap == 0) return MGB_OK;
  if (cudaMemsetAsync(c.sync_base, 0, c.sync_cap * sizeof(unsigned), c.stream) != cudaSuccess) {
    set_error("barrier counter memset failed");
    return MGB_ERR_CUDA;
  }
  return MGB_OK;
}

int unet_forward(mgb_handle* hd, Ctx& c, const float* rgb, float* tgt, const float* noise, float* raw_out, int step,
                 int NB, int lh, int lw) {
  const UNetW& U = hd->unet;
  const mgb_config& cfg = hd->cfg;
  const int L = cfg.unet_layers_per_block;
  const int* ch = cfg.unet_block_channels;
  int H = lh, W = lw;
  size_t M = size_t(NB) * H * W;
  TRY(zero_counters(c));
  // level sizes: a stride-2 pad-1 conv gives ceil(s / 2); coming back up the target is the skip connection's size
  // (diffusers forwards `upsample_size` when a latent dim is not a multiple of 8), i.e. 2s or 2s - 1
  int lvH[4] = {lh, 0, 0, 0}, lvW[4] = {lw, 0, 0, 0};
  for (int i = 1; i < 4; ++i) { lvH[i] = (lvH[i - 1] + 1) / 2; lvW[i] = (lvW[i - 1] + 1) / 2; }

  std::vector<Act> skips;
  size_t ri = 0, xi = 0;

  // step < 0: the step index is read from the device counter (CUDA-graph replay)
  LAUNCH(launch_select_step(hd->bias_table, hd->bias_total, hd->sched_k, hd->cur_bias, hd->cur_sched_k,
                            hd->step_counter, step, c.stream));
  c.cur_bias = hd->cur_bias;
  bf16* x0 = aalloc<bf16>(c, M * 64);
  LAUNCH(launch_pack_latents(rgb, tgt, x0, int(M), cfg.unet_out_channels, c.stream));
  Act h = act_alloc(c, M, ch[0]);
  {
    Epi e; e.bias = U.conv_in.b; e.out_f32 = h.p;
    TRY(conv3x3(c, x0, NB, H, W, U.conv_in, 0, e));
  }
  skips.push_back(h);
  int cur = ch[0];
  // down path
  for (int i = 0; i < 4; ++i) {
    const bool last = i == 3;
    for (int j = 0; j < L; ++j) {
      Act y = act_alloc(c, M, ch[i]);
      TRY(resnet_forward(c, U.resnets[ri++], h, nullptr, y, NB, H, W));
      h = y; cur = ch[i];
      if (!last) {
        Act y2 = act_alloc(c, M, cur);
        TRY(xfmr_forward(c, U.xfmrs[xi++], h, y2, NB, H * W));
        h = y2;
      }
      skips.push_back(h);
    }
    if (!last) {
      const int Hn = lvH[i + 1], Wn = lvW[i + 1];
      bf16* planes = aalloc<bf16>(c, size_t(NB) * 4 * Hn * Wn * cur);
      LAUNCH(launch_space_to_depth(h.p, planes, NB, H, W, cur, c.stream));
      H = Hn; W = Wn; M = size_t(NB) * H * W;
      Act y = act_alloc(c, M, cur);
      {
        Epi e; e.bias = U.downs[i].b; e.out_f32 = y.p;
        TRY(conv3x3(c, planes, NB, H, W, U.downs[i], 2, e));
      }
      h = y;
      skips.push_back(h);
    }
  }
  // mid
  {
    Act y = act_alloc(c, M, cur);
    TRY(resnet_forward(c, U.resnets[ri++], h, nullptr, y, NB, H, W));
    Act y2 = act_alloc(c, M, cur);
    TRY(xfmr_forward(c, U.xfmrs[xi++], y, y2, NB, H * W));
    Act y3 = act_alloc(c, M, cur);
    TRY(resnet_forward(c, U.resnets[ri++], y2, nullptr, y3, NB, H, W));
    h = y3;
  }
  // up path: the concat [h | skip] is consumed directly by the resnet's GroupNorm
  for (int i = 0; i < 4; ++i) {
    const int cout = ch[3 - i];
    for (int j = 0; j < L + 1; ++j) {
      Act sk = skips.back();
      skips.pop_back();
      Act y = act_alloc(c, M, cout);
      TRY(resnet_forward(c, U.resnets[ri++], h, &sk, y, NB, H, W));
      h = y; cur = cout;
      if (i > 0) {
        Act y2 = act_alloc(c, M, cur);
        TRY(xfmr_forward(c, U.xfmrs[xi++], h, y2, NB, H * W));
        h = y2;
      }
    }
    if (i < 3) {
      const int Hn = lvH[2 - i], Wn = lvW[2 - i];
      bf16* up = aalloc<bf16>(c, size_t(NB) * Hn * Wn * cur);
      LAUNCH(launch_upsample2x(h.p, up, NB, H, W, cur, Hn, Wn, c.stream));
      H = Hn; W = Wn; M = size_t(NB) * H * W;
      Act y = act_alloc(c, M, cur);
      {
        Epi e; e.bias = U.ups[i].b; e.out_f32 = y.p;
        TRY(conv3x3(c, up, NB, H, W, U.ups[i], 0, e));
      }
      h = y;
    }
  }
  // out: GN -> SiLU -> conv_out fused with the scheduler step
  bf16* t = aalloc<bf16>(c, M * cur);
  TRY(groupnorm(c, h, nullptr, t, nullptr, U.norm_out, NB, H * W, 1e-5f, 1));
  {
    Epi e;
    e.bias = U.conv_out.b;
    e.flags = EPI_SCHED;
    e.out_f32 = tgt; e.sched_x = tgt; e.sched_z = noise; e.aux_out = raw_out;
    e.sched_k = hd->cur_sched_k;
    TRY(conv3x3(c, t, NB, H, W, U.conv_out, 0, e));
  }
  if (step < 0) LAUNCH(launch_advance_counter(hd->step_counter, c.stream));
  return MGB_OK;
}

// ---------------------------------------------------------------------------------------------
// VAE forwards. Their arena is lifetime-planned (api_net.cu): every buffer is allocated where it is first written and
// freed after its last read, so the memory live at once stays near the largest working set of one step. At full
// resolution that is the decoder's first up-level resnet's GroupNorm: its 256-channel fp32 input and the two bf16
// copies it writes, 4 U (U = one fp32 128-channel map). With c.dec_low_memory the last up-conv runs in bands into two
// 128-channel halves (up_conv_low_memory), that resnet runs on the halves in their own memory
// (resnet_shortcut_halves), the two after it free their input and allocate their output as late as they can, and the
// decoder's peak is 2.5 U (plus GroupNorm scratch): that resnet's second GroupNorm and conv2 (both halves and t2), and
// each 128-channel resnet (input, output and one operand). The encoder's peak is 2.5 U too.
// ---------------------------------------------------------------------------------------------
// mid block: resnet, attention, resnet; consumes h and leaves the result in it
static int vae_mid_forward(Ctx& c, const ResnetW& r0, const VaeAttnW& A, const ResnetW& r1, Act& h, int NB, int H,
                           int W) {
  Act y1, y3;
  TRY(resnet_forward(c, r0, h, nullptr, y1, NB, H, W, true));
  Act y2 = act_alloc(c, size_t(NB) * H * W, y1.C);
  TRY(vae_attn_forward(c, A, y1, y2, NB, H * W));
  c.arena->free(y1.p);
  TRY(resnet_forward(c, r1, y2, nullptr, y3, NB, H, W, true));
  h = y3;
  return MGB_OK;
}

// VAE encoder: rgb fp32 NCHW [NB,3,H,W] -> latent fp32 NCHW [NB,4,H/8,W/8] (mean * latent_scale)
int vae_encode_forward(mgb_handle* hd, Ctx& c, const float* rgb, float* latent_out, int NB, int H, int W) {
  const VaeW& V = hd->vae;
  const mgb_config& cfg = hd->cfg;
  const int* ch = cfg.vae_block_channels;
  const int L = cfg.vae_layers_per_block;
  size_t M = size_t(NB) * H * W;
  size_t ri = 0;
  TRY(zero_counters(c));
  const size_t mk0 = c.arena->mark();
  bf16* x0 = aalloc<bf16>(c, M * 64);
  LAUNCH(launch_pack_rgb(rgb, x0, NB, H * W, c.stream));
  Act h = act_alloc(c, M, ch[0]);
  { Epi e; e.bias = V.enc_in.b; e.out_f32 = h.p; TRY(conv3x3(c, x0, NB, H, W, V.enc_in, 0, e)); }
  c.arena->free(x0);
  int cur = ch[0];
  for (int i = 0; i < 4; ++i) {
    // ping-pong trunk buffers for this resolution, each allocated by the resnet that first writes it
    Act buf[2];
    for (int j = 0; j < L; ++j) {
      TRY(resnet_forward(c, V.enc_res[ri++], h, nullptr, buf[j & 1], NB, H, W, j == 0));
      h = buf[j & 1]; cur = ch[i];
    }
    if (i < 3) {
      // F.pad(x, (0,1,0,1)) + 3x3 stride 2 pad 0: floor(s / 2) outputs; the parity planes hold ceil(s / 2) entries
      const int Hp = (H + 1) / 2, Wp = (W + 1) / 2;
      bf16* planes = aalloc<bf16>(c, size_t(NB) * 4 * Hp * Wp * cur);
      LAUNCH(launch_space_to_depth(h.p, planes, NB, H, W, cur, c.stream));
      c.arena->free(buf[0].p);
      c.arena->free(buf[1].p);
      H /= 2; W /= 2; M = size_t(NB) * H * W;
      Act y = act_alloc(c, M, cur);
      { Epi e; e.bias = V.enc_down[i].b; e.out_f32 = y.p; TRY(conv3x3(c, planes, NB, H, W, V.enc_down[i], 3, e, Hp, Wp)); }
      c.arena->free(planes);
      h = y;
    } else {
      c.arena->free(buf[L & 1].p);   // h's partner; h goes on into the mid block
    }
  }
  TRY(vae_mid_forward(c, V.enc_res[ri], V.enc_attn, V.enc_res[ri + 1], h, NB, H, W));
  bf16* t = aalloc<bf16>(c, M * cur);
  TRY(groupnorm(c, h, nullptr, t, nullptr, V.enc_norm_out, NB, H * W, 1e-6f, 1));
  c.arena->free(h.p);
  {
    // conv_out with quant_conv folded in; mean half only; * latent_scale; NCHW output
    Epi e; e.bias = V.enc_out.b; e.out_f32 = latent_out; e.flags = EPI_NCHW | EPI_SCALE; e.scale = cfg.latent_scale;
    TRY(conv3x3(c, t, NB, H, W, V.enc_out, 0, e));
  }
  c.arena->release(mk0);
  return MGB_OK;
}

// VAE decoder: latent fp32 NCHW [NB,4,lh,lw] -> out fp32 NCHW (depth: 1 plane, normals/raw: 3 planes)
int vae_decode_forward(mgb_handle* hd, Ctx& c, const float* latent, float* out, int NB, int lh, int lw, int mode) {
  const VaeW& V = hd->vae;
  const mgb_config& cfg = hd->cfg;
  const int* ch = cfg.vae_block_channels;
  const int L = cfg.vae_layers_per_block;
  int H = lh, W = lw;
  size_t M = size_t(NB) * H * W;
  TRY(zero_counters(c));
  const size_t mk0 = c.arena->mark();
  bf16* z = aalloc<bf16>(c, M * 64);
  LAUNCH(launch_pack_decoder_latent(latent, V.pq_w, V.pq_b, 1.0f / cfg.latent_scale, z, NB, H * W, c.stream));
  int cur = ch[3];
  Act h = act_alloc(c, M, cur);
  { Epi e; e.bias = V.dec_in.b; e.out_f32 = h.p; TRY(conv3x3(c, z, NB, H, W, V.dec_in, 0, e)); }
  c.arena->free(z);
  TRY(vae_mid_forward(c, V.dec_res[0], V.dec_attn, V.dec_res[1], h, NB, H, W));
  size_t ri = 2;
  Act buf[2], half_a, half_b;   // half_a, half_b: the last up-conv's output in low memory (up_conv_low_memory)
  for (int i = 0; i < 4; ++i) {
    const int cout = ch[3 - i];
    buf[0] = buf[1] = Act();   // ping-pong trunk buffers, each allocated by the resnet that first writes it
    if (c.dec_low_memory && i == 3) {
      // Full resolution in 2.5 U: the first resnet on the up-conv's two halves, and every block's output a buffer of
      // its own, allocated after the block's conv1 output is freed, with the block's input freed after its last read.
      // (The ping-pong pair below holds both 128-channel trunk maps through every block: 3.5 U in the next two.)
      for (int j = 0; j < L + 1; ++j) {
        Act y;
        if (j == 0) TRY(resnet_shortcut_halves(c, V.dec_res[ri++], half_a, half_b, y, NB, H, W));
        else TRY(resnet_forward(c, V.dec_res[ri++], h, nullptr, y, NB, H, W, true));
        h = y; cur = cout;
      }
      buf[0] = h;     // freed after dec_norm_out below
      continue;
    }
    for (int j = 0; j < L + 1; ++j) {
      TRY(resnet_forward(c, V.dec_res[ri++], h, nullptr, buf[j & 1], NB, H, W, j == 0));
      h = buf[j & 1]; cur = cout;
    }
    if (c.dec_low_memory && i == 2) {
      Act& partner = buf[0].p == h.p ? buf[1] : buf[0];
      H *= 2; W *= 2; M = size_t(NB) * H * W;
      TRY(up_conv_low_memory(c, V.dec_up[i], h, partner, half_a, half_b, NB, H, W));
      buf[0] = buf[1] = Act();
      continue;
    }
    if (i < 3) {
      bf16* up = aalloc<bf16>(c, M * 4 * cur);
      LAUNCH(launch_upsample2x(h.p, up, NB, H, W, cur, 2 * H, 2 * W, c.stream));
      c.arena->free(buf[0].p);
      c.arena->free(buf[1].p);
      H *= 2; W *= 2; M = size_t(NB) * H * W;
      Act next = act_alloc(c, M, cur);
      { Epi e; e.bias = V.dec_up[i].b; e.out_f32 = next.p; TRY(conv3x3(c, up, NB, H, W, V.dec_up[i], 0, e)); }
      c.arena->free(up);
      h = next;
    }
  }
  bf16* t = aalloc<bf16>(c, M * cur);
  TRY(groupnorm(c, h, nullptr, t, nullptr, V.dec_norm_out, NB, H * W, 1e-6f, 1));
  c.arena->free(buf[0].p);
  c.arena->free(buf[1].p);
  {
    Epi e; e.bias = V.dec_out.b; e.out_f32 = out;
    e.flags = mode == MGB_DECODE_DEPTH ? EPI_DEPTH : mode == MGB_DECODE_NORMALS ? EPI_NORMALS
              : mode == MGB_DECODE_UNIT3 ? (EPI_NCHW | EPI_UNIT) : EPI_NCHW;
    TRY(conv3x3(c, t, NB, H, W, V.dec_out, 0, e));
  }
  c.arena->release(mk0);
  return MGB_OK;
}

}  // namespace mgb
