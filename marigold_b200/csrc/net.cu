// Forward graphs of the Marigold hot path, as sequences of kernels.h launches on one stream:
//   UNet step   (diffusers UNet2DConditionModel, SD-2 config)   reference call: marigold_depth_pipeline.py:461-463
//   VAE encode  (AutoencoderKL.encoder + quant_conv)            reference call: marigold_depth_pipeline.py:491-495
//   VAE decode  (post_quant_conv + AutoencoderKL.decoder)       reference call: marigold_depth_pipeline.py:510-515
// Architecture per SURVEY.md App. A (restated; diffusers itself is not available offline).
//
// Numerics: bf16 tensor-core operands, fp32 accumulation, fp32 residual trunk and latent state;
// GroupNorm/LayerNorm/softmax statistics in fp32.
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "launch.h"
#include "net.h"

namespace mgb {

// ---------------------------------------------------------------------------------------------
// arena
// ---------------------------------------------------------------------------------------------
void* Arena::alloc(size_t bytes) {
  const size_t a = (off + 1023) & ~size_t(1023);
  off = a + bytes;
  if (off > peak) peak = off;
  if (dry) return reinterpret_cast<void*>(uintptr_t(0x100000) + a);
  if (off > cap) { overflow = true; return nullptr; }
  return base + a;
}
template <typename T>
static T* aalloc(Ctx& c, size_t n) { return reinterpret_cast<T*>(c.arena->alloc(n * sizeof(T))); }

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

// y = a[M,K] W^T (+ epilogue); ldo = row stride of the outputs (0: W.n, or W.n / 2 for GEGLU)
static int linear(Ctx& c, const bf16* a, int M, const LinW& W, const Epi& e, int ldo = 0, const bf16* a2 = nullptr,
                  int K1 = 0) {
  // a2 != nullptr: K concatenation, A = [a (K1 columns) | a2 (W.k - K1 columns)]
  int bn, sp, st;
  const bool geglu = (e.flags & EPI_GEGLU) != 0;
  choose_tile((M + 127) / 128, W.n, W.k / 64, e.flags, true, &bn, &sp, &st);
  if (geglu) { bn = 256; sp = 1; st = (W.k / 64 <= 12) ? 2 : 4; }
  if (sp > 1) c.splitk_need = std::max(c.splitk_need, size_t(sp) * M * W.n * sizeof(float));
  if (c.dry) return MGB_OK;
  GemmParams p;
  if (a2) TRY(fill_linear_params(&p, a, W.w, M, W.n, K1, bn, sp, st, a2, W.k - K1));
  else TRY(fill_linear_params(&p, a, W.w, M, W.n, W.k, bn, sp, st));
  return gemm_common(c, p, bn, effective_splits(p), e, ldo > 0 ? ldo : (geglu ? W.n / 2 : W.n));
}

// generic A[M,K] x B[N,K]^T with raw pointers (attention score / PV GEMMs in the VAE)
static int matmul_nt(Ctx& c, const bf16* a, const bf16* b, int M, int N, int K, const Epi& e, int ldo = 0) {
  LinW W; W.w = const_cast<bf16*>(b); W.n = N; W.k = K;
  // B is an activation written by an earlier kernel of this stream (K, or V^T straight out of the transpose): the
  // GEMM's pre-wait B prefetch must not run ahead of its producer, so no programmatic early launch here.
  PlainLaunchScope no_early_launch;
  return linear(c, a, M, W, e, ldo);
}

// 3x3 conv on NHWC bf16; Hout x Wout output; kind per ops.cu
static int conv3x3(Ctx& c, const bf16* x, int NB, int Hout, int Wout, const ConvW& W, int kind, const Epi& e,
                   int Hsrc = 0, int Wsrc = 0, const bf16* x2 = nullptr) {
  int tw, th;
  conv_tile_shape(Hout, Wout, &tw, &th);
  const int m_tiles = NB * ((Wout + tw - 1) / tw) * ((Hout + th - 1) / th);
  int bn, sp, st;
  if ((x2 != nullptr) != (W.k_extra > 0)) { set_error("conv3x3: second operand / weight layout mismatch"); return MGB_ERR_STATE; }
  choose_tile(m_tiles, W.cout, (9 * W.cin_pad + W.k_extra) / 64, e.flags, true, &bn, &sp, &st);
  const size_t M = size_t(NB) * Hout * Wout;
  if (sp > 1) c.splitk_need = std::max(c.splitk_need, size_t(sp) * M * W.cout * sizeof(float));
  if (c.dry) return MGB_OK;
  GemmParams p;
  TRY(fill_conv_params(&p, x, W.w, NB, Hout, Wout, W.cin_pad, W.cout, kind, bn, sp, st, Hsrc, Wsrc, x2, W.k_extra));
  Epi e2 = e;
  e2.hw = Hout * Wout;
  return gemm_common(c, p, bn, effective_splits(p), e2, W.cout);
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
// Scratch: partials from the arena (released by the caller's mark), one barrier counter per image from the per-forward
// counter slab (zeroed once per forward by zero_counters()).
static int groupnorm(Ctx& c, const Act& a, const Act* b, bf16* y, bf16* raw, const NormW& n, int NB, int HW, float eps,
                     int silu) {
  if (skip_family("gn")) return MGB_OK;
  const int Cb = (b && b->p) ? b->C : 0;
  void* part = c.arena->alloc(groupnorm_part_bytes(NB, HW, a.C + Cb, c.groups));
  const size_t coff = c.sync_off;
  c.sync_off += size_t(NB);
  if (c.sync_off > c.sync_need) c.sync_need = c.sync_off;
  if (c.dry) return MGB_OK;
  if (c.sync_off > c.sync_cap) { set_error("groupnorm: barrier counter slab exhausted"); return MGB_ERR_STATE; }
  return launch_gn_fused(a.p, a.C, Cb ? b->p : nullptr, Cb, y, raw, n.g, n.b, NB, HW, c.groups, eps, silu, part,
                         c.sync_base + coff, c.stream);
}

// ---------------------------------------------------------------------------------------------
// ResnetBlock2D: GN -> SiLU -> conv3x3 (+temb) -> GN -> SiLU -> conv3x3 ; + (1x1 shortcut | x)
//   x fp32 [M, cin] -> y fp32 [M, cout] (y preallocated by the caller)
// ---------------------------------------------------------------------------------------------
static int resnet_forward(Ctx& c, const ResnetW& R, Act& x, Act* skip, Act& y, int NB, int H, int W) {
  // input = x, or the channel concat [x | skip] of an up block (never materialised in fp32: GroupNorm reads both
  // sources, and the 1x1 shortcut reads the bf16 copy GroupNorm emits)
  const size_t M = size_t(NB) * H * W;
  const size_t mk = c.arena->mark();
  bf16* t1 = aalloc<bf16>(c, M * R.cin);
  bf16* raw = R.has_sc ? aalloc<bf16>(c, M * R.cin) : nullptr;
  Act h = act_alloc(c, M, R.cout);
  bf16* t2 = aalloc<bf16>(c, M * R.cout);
  TRY(groupnorm(c, x, skip, t1, raw, R.n1, NB, H * W, R.eps, 1));
  Epi e1;
  e1.bias = (R.bias_off >= 0 && c.cur_bias) ? c.cur_bias + R.bias_off : R.c1.b;
  e1.out_f32 = h.p;
  TRY(conv3x3(c, t1, NB, H, W, R.c1, 0, e1));
  TRY(groupnorm(c, h, nullptr, t2, nullptr, R.n2, NB, H * W, R.eps, 1));
  // conv2 (+ residual). Where the block changes the channel count, diffusers adds conv_shortcut(x), a 1x1 convolution:
  // its K blocks are appended to conv2's implicit GEMM (weights [W2 | Wsc], bias b2 + bsc, second A operand = the raw
  // bf16 copy of the block input), which removes a GEMM launch (plus a split-K reduce on the small levels) and the
  // fp32 round trip of its output
  Epi e2; e2.bias = R.c2.b; e2.out_f32 = y.p;
  if (!R.has_sc) e2.residual = x.p;
  TRY(conv3x3(c, t2, NB, H, W, R.c2, 0, e2, 0, 0, R.has_sc ? raw : nullptr));
  c.arena->release(mk);
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
  bf16* o = aalloc<bf16>(c, M * C);
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
  if (!no_attn) LAUNCH(launch_flash_attn64(qkv, o, NB, T, C, 0.125f, attn_ws, attn_ws_bytes, c.stream));
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
// ---------------------------------------------------------------------------------------------
static int vae_attn_forward(Ctx& c, const VaeAttnW& A, Act& x, Act& y, int NB, int T) {
  const int C = A.C;
  const size_t M = size_t(NB) * T;
  const int Tp = (T + 63) / 64 * 64;
  const size_t mk = c.arena->mark();
  bf16* a = aalloc<bf16>(c, M * C);
  bf16* q = aalloc<bf16>(c, M * C);
  bf16* k = aalloc<bf16>(c, M * C);
  bf16* v = aalloc<bf16>(c, M * C);
  bf16* vt = aalloc<bf16>(c, size_t(C) * Tp);
  float* s = aalloc<float>(c, size_t(T) * Tp);
  bf16* pr = aalloc<bf16>(c, size_t(T) * Tp);
  bf16* o = aalloc<bf16>(c, M * C);
  TRY(groupnorm(c, x, nullptr, a, nullptr, A.gn, NB, T, 1e-6f, 0));
  { Epi e; e.bias = A.q.b; e.out_bf16 = q; TRY(linear(c, a, int(M), A.q, e)); }
  { Epi e; e.bias = A.k.b; e.out_bf16 = k; TRY(linear(c, a, int(M), A.k, e)); }
  { Epi e; e.bias = A.v.b; e.out_bf16 = v; TRY(linear(c, a, int(M), A.v, e)); }
  const float scale = 1.0f / sqrtf(float(C));
  for (int n = 0; n < NB; ++n) {
    const size_t off = size_t(n) * T * C;
    { Epi e; e.out_f32 = s; e.flags = EPI_SCALE; e.scale = scale; TRY(matmul_nt(c, q + off, k + off, T, T, C, e, Tp)); }
    LAUNCH(launch_softmax_rows(s, pr, T, T, Tp, c.stream));
    LAUNCH(launch_transpose_bf16(v + off, vt, T, C, Tp, c.stream));
    { Epi e; e.out_bf16 = o + off; TRY(matmul_nt(c, pr, vt, T, C, Tp, e)); }
  }
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
// VAE encoder: rgb fp32 NCHW [NB,3,H,W] -> latent fp32 NCHW [NB,4,H/8,W/8] (mean * latent_scale)
// ---------------------------------------------------------------------------------------------
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
  int cur = ch[0];
  for (int i = 0; i < 4; ++i) {
    // ping-pong trunk buffers for this resolution
    Act buf[2] = {act_alloc(c, M, ch[i]), act_alloc(c, M, ch[i])};
    for (int j = 0; j < L; ++j) {
      Act y = buf[j & 1];
      TRY(resnet_forward(c, V.enc_res[ri++], h, nullptr, y, NB, H, W));
      h = y; cur = ch[i];
    }
    if (i < 3) {
      // F.pad(x, (0,1,0,1)) + 3x3 stride 2 pad 0: floor(s / 2) outputs; the parity planes hold ceil(s / 2) entries
      const int Hp = (H + 1) / 2, Wp = (W + 1) / 2;
      bf16* planes = aalloc<bf16>(c, size_t(NB) * 4 * Hp * Wp * cur);
      LAUNCH(launch_space_to_depth(h.p, planes, NB, H, W, cur, c.stream));
      H /= 2; W /= 2; M = size_t(NB) * H * W;
      Act y = act_alloc(c, M, cur);
      { Epi e; e.bias = V.enc_down[i].b; e.out_f32 = y.p; TRY(conv3x3(c, planes, NB, H, W, V.enc_down[i], 3, e, Hp, Wp)); }
      h = y;
    }
  }
  {
    Act y1 = act_alloc(c, M, cur);
    TRY(resnet_forward(c, V.enc_res[ri++], h, nullptr, y1, NB, H, W));
    Act y2 = act_alloc(c, M, cur);
    TRY(vae_attn_forward(c, V.enc_attn, y1, y2, NB, H * W));
    Act y3 = act_alloc(c, M, cur);
    TRY(resnet_forward(c, V.enc_res[ri++], y2, nullptr, y3, NB, H, W));
    h = y3;
  }
  bf16* t = aalloc<bf16>(c, M * cur);
  TRY(groupnorm(c, h, nullptr, t, nullptr, V.enc_norm_out, NB, H * W, 1e-6f, 1));
  {
    // conv_out with quant_conv folded in; mean half only; * latent_scale; NCHW output
    Epi e; e.bias = V.enc_out.b; e.out_f32 = latent_out; e.flags = EPI_NCHW | EPI_SCALE; e.scale = cfg.latent_scale;
    TRY(conv3x3(c, t, NB, H, W, V.enc_out, 0, e));
  }
  c.arena->release(mk0);
  return MGB_OK;
}

// ---------------------------------------------------------------------------------------------
// VAE decoder: latent fp32 NCHW [NB,4,lh,lw] -> out fp32 NCHW (depth: 1 plane, normals/raw: 3 planes)
// ---------------------------------------------------------------------------------------------
int vae_decode_forward(mgb_handle* hd, Ctx& c, const float* latent, float* out, int NB, int lh, int lw, int mode) {
  const VaeW& V = hd->vae;
  const mgb_config& cfg = hd->cfg;
  const int* ch = cfg.vae_block_channels;
  const int L = cfg.vae_layers_per_block;
  int H = lh, W = lw;
  size_t M = size_t(NB) * H * W;
  size_t ri = 0;
  TRY(zero_counters(c));
  const size_t mk0 = c.arena->mark();
  bf16* z = aalloc<bf16>(c, M * 64);
  LAUNCH(launch_pack_decoder_latent(latent, V.pq_w, V.pq_b, 1.0f / cfg.latent_scale, z, NB, H * W, c.stream));
  int cur = ch[3];
  Act h = act_alloc(c, M, cur);
  { Epi e; e.bias = V.dec_in.b; e.out_f32 = h.p; TRY(conv3x3(c, z, NB, H, W, V.dec_in, 0, e)); }
  {
    Act y1 = act_alloc(c, M, cur);
    TRY(resnet_forward(c, V.dec_res[ri++], h, nullptr, y1, NB, H, W));
    Act y2 = act_alloc(c, M, cur);
    TRY(vae_attn_forward(c, V.dec_attn, y1, y2, NB, H * W));
    Act y3 = act_alloc(c, M, cur);
    TRY(resnet_forward(c, V.dec_res[ri++], y2, nullptr, y3, NB, H, W));
    h = y3;
  }
  for (int i = 0; i < 4; ++i) {
    const int cout = ch[3 - i];
    Act buf[2] = {act_alloc(c, M, cout), act_alloc(c, M, cout)};
    for (int j = 0; j < L + 1; ++j) {
      Act y = buf[j & 1];
      TRY(resnet_forward(c, V.dec_res[ri++], h, nullptr, y, NB, H, W));
      h = y; cur = cout;
    }
    if (i < 3) {
      bf16* up = aalloc<bf16>(c, M * 4 * cur);
      LAUNCH(launch_upsample2x(h.p, up, NB, H, W, cur, 2 * H, 2 * W, c.stream));
      H *= 2; W *= 2; M = size_t(NB) * H * W;
      Act y = act_alloc(c, M, cur);
      { Epi e; e.bias = V.dec_up[i].b; e.out_f32 = y.p; TRY(conv3x3(c, up, NB, H, W, V.dec_up[i], 0, e)); }
      h = y;
    }
  }
  bf16* t = aalloc<bf16>(c, M * cur);
  TRY(groupnorm(c, h, nullptr, t, nullptr, V.dec_norm_out, NB, H * W, 1e-6f, 1));
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
