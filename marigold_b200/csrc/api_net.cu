// C ABI, handle part: weights (load / repack), conditioning, schedule, encode / denoise / decode.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "debug.h"
#include "launch.h"
#include "net.h"

namespace mgb {
int unet_forward(mgb_handle* hd, Ctx& c, const float* rgb, float* tgt, const float* noise, float* raw_out, int step,
                 int NB, int lh, int lw);
int vae_encode_forward(mgb_handle* hd, Ctx& c, const float* rgb, float* latent_out, int NB, int H, int W);
int vae_decode_forward(mgb_handle* hd, Ctx& c, const float* latent, float* out, int NB, int lh, int lw, int mode);
}  // namespace mgb

using namespace mgb;

// -------------------------------------------------------------------------------------------------
// host helpers
// -------------------------------------------------------------------------------------------------
static void invalidate_step_graph(mgb_handle* h) { h->step_graph.exec.reset(); }

// Grows a buffer the step graph may have captured: waits for the device and drops the graph before freeing it.
template <class T>
static int grow_captured(mgb_handle* h, DevBuf<T>& buf, size_t need) {
  if (need <= buf.bytes()) return MGB_OK;
  CUDA_TRY(cudaDeviceSynchronize());
  invalidate_step_graph(h);
  return buf.grow(need);
}

static inline uint16_t f2bf(float f) {  // round-to-nearest-even, NaN preserved
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return uint16_t((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return uint16_t(u >> 16);
}
static inline float half2f(uint16_t h) {
  const uint32_t s = (h >> 15) & 1, e = (h >> 10) & 0x1f, m = h & 0x3ff;
  uint32_t u;
  if (e == 0) {
    if (m == 0) u = s << 31;
    else {
      int ee = -1; uint32_t mm = m;
      do { mm <<= 1; ++ee; } while (!(mm & 0x400));
      u = (s << 31) | ((127 - 15 - ee) << 23) | ((mm & 0x3ff) << 13);
    }
  } else if (e == 31) u = (s << 31) | 0x7f800000u | (m << 13);
  else u = (s << 31) | ((e - 15 + 127) << 23) | (m << 13);
  float f; memcpy(&f, &u, 4); return f;
}

struct Loader {
  const std::map<std::string, HostTensor>& host;
  std::vector<DevBuf<void>> weights;   // handed to the handle only if every upload succeeds
  int rc = MGB_OK;
  const HostTensor* get(const std::string& key) {
    auto it = host.find(key);
    if (it == host.end()) {
      if (rc == MGB_OK) { set_error("finalize_weights: tensor '%s' was not loaded", key.c_str()); rc = MGB_ERR_STATE; }
      return nullptr;
    }
    return &it->second;
  }
  // A new device array, filled from src unless null. Nothing more is allocated after a failure: it keeps its text.
  void* upload(const void* src, size_t bytes) {
    DevBuf<void> b;
    if (rc != MGB_OK || (rc = b.grow(bytes)) != MGB_OK) return nullptr;
    if (src && cudaMemcpy(b, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("cudaMemcpy H2D failed"); rc = MGB_ERR_CUDA;
      return nullptr;
    }
    weights.push_back(std::move(b));
    return weights.back();
  }
  float* up_f32(const std::vector<float>& v) { return static_cast<float*>(upload(v.data(), v.size() * 4)); }
  bf16* up_bf16(const std::vector<float>& v) {
    std::vector<uint16_t> b(v.size());
    for (size_t i = 0; i < v.size(); ++i) b[i] = f2bf(v[i]);
    return static_cast<bf16*>(upload(b.data(), b.size() * 2));
  }
  bool shape_is(const HostTensor* t, std::initializer_list<int64_t> s, const std::string& key) {
    if (!t) return false;
    if (t->shape.size() != s.size() || !std::equal(s.begin(), s.end(), t->shape.begin())) {
      if (rc == MGB_OK) {
        std::string got, want;
        for (auto d : t->shape) got += std::to_string(d) + ",";
        for (auto d : s) want += std::to_string(d) + ",";
        set_error("tensor '%s' has shape [%s], expected [%s]", key.c_str(), got.c_str(), want.c_str());
        rc = MGB_ERR_INVALID;
      }
      return false;
    }
    return true;
  }
  // [cout, cin, 3, 3] -> tap-major [cout, 9 * cin_pad]
  static std::vector<float> pack_conv(const std::vector<float>& w, int cout, int cin, int cin_pad) {
    std::vector<float> o(size_t(cout) * 9 * cin_pad, 0.f);
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < cin; ++ci)
        for (int t = 0; t < 9; ++t)
          o[(size_t(co) * 9 + t) * cin_pad + ci] = w[(size_t(co) * cin + ci) * 9 + t];
    return o;
  }
  ConvW conv(const std::string& p, int cin, int cout) {
    ConvW c; c.cin = cin; c.cout = cout; c.cin_pad = (cin + 63) / 64 * 64;
    const HostTensor* w = get(p + ".weight");
    const HostTensor* b = get(p + ".bias");
    if (!shape_is(w, {cout, cin, 3, 3}, p + ".weight") || !shape_is(b, {cout}, p + ".bias")) return c;
    c.w = up_bf16(pack_conv(w->data, cout, cin, c.cin_pad));
    c.b = up_f32(b->data);
    return c;
  }
  LinW lin(const std::string& p, int n, int k, bool bias, bool conv1x1 = false) {
    LinW l; l.n = n; l.k = k;
    const HostTensor* w = get(p + ".weight");
    if (conv1x1) { if (!shape_is(w, {n, k, 1, 1}, p + ".weight")) return l; }
    else if (!shape_is(w, {n, k}, p + ".weight")) return l;
    l.w = up_bf16(w->data);
    if (bias) {
      const HostTensor* b = get(p + ".bias");
      if (!shape_is(b, {n}, p + ".bias")) return l;
      l.b = up_f32(b->data);
    }
    return l;
  }
  NormW norm(const std::string& p, int c) {
    NormW n; n.c = c;
    const HostTensor* w = get(p + ".weight");
    const HostTensor* b = get(p + ".bias");
    if (!shape_is(w, {c}, p + ".weight") || !shape_is(b, {c}, p + ".bias")) return n;
    n.g = up_f32(w->data); n.b = up_f32(b->data);
    return n;
  }
  ResnetW resnet(const std::string& p, int cin, int cout, int temb_dim, float eps) {
    ResnetW r; r.cin = cin; r.cout = cout; r.eps = eps;
    r.n1 = norm(p + ".norm1", cin);
    r.c1 = conv(p + ".conv1", cin, cout);
    r.n2 = norm(p + ".norm2", cout);
    if (cin == cout) {
      r.c2 = conv(p + ".conv2", cout, cout);
    } else {
      // conv2 and the 1x1 conv_shortcut as one K-concatenated weight [cout, 9 * cout + cin], bias b2 + bsc
      r.has_sc = true;
      r.c2.cin = cout; r.c2.cin_pad = cout; r.c2.cout = cout; r.c2.k_extra = cin;
      const HostTensor *w2 = get(p + ".conv2.weight"), *b2 = get(p + ".conv2.bias"),
                       *ws = get(p + ".conv_shortcut.weight"), *bs = get(p + ".conv_shortcut.bias");
      if (cin % 64 != 0) { if (rc == MGB_OK) { set_error("resnet %s: shortcut input channels %d not a multiple of 64", p.c_str(), cin); rc = MGB_ERR_UNSUPPORTED; } }
      else if (shape_is(w2, {cout, cout, 3, 3}, p + ".conv2.weight") && shape_is(b2, {cout}, p + ".conv2.bias") &&
               shape_is(ws, {cout, cin, 1, 1}, p + ".conv_shortcut.weight") && shape_is(bs, {cout}, p + ".conv_shortcut.bias")) {
        const std::vector<float> taps = pack_conv(w2->data, cout, cout, cout);
        const size_t k1 = size_t(9) * cout, kt = k1 + cin;
        std::vector<float> w(size_t(cout) * kt), b(cout);
        for (int co = 0; co < cout; ++co) {
          memcpy(&w[co * kt], &taps[co * k1], k1 * 4);
          memcpy(&w[co * kt + k1], &ws->data[size_t(co) * cin], size_t(cin) * 4);
          b[co] = b2->data[co] + bs->data[co];
        }
        r.c2.w = up_bf16(w);
        r.c2.b = up_f32(b);
      }
    }
    if (temb_dim > 0) {
      const HostTensor* w = get(p + ".time_emb_proj.weight");
      const HostTensor* b = get(p + ".time_emb_proj.bias");
      const HostTensor* cb = get(p + ".conv1.bias");
      if (shape_is(w, {cout, temb_dim}, p + ".time_emb_proj.weight") && shape_is(b, {cout}, p + ".time_emb_proj.bias") &&
          cb) {
        r.temb_w = up_f32(w->data);
        std::vector<float> bb(cout);
        for (int i = 0; i < cout; ++i) bb[i] = b->data[i] + cb->data[i];  // fold conv1.bias
        r.temb_b = up_f32(bb);
      }
    }
    return r;
  }
  XfmrW xfmr(const std::string& p, int C, int ctx) {
    XfmrW x; x.C = C;
    x.gn = norm(p + ".norm", C);
    x.proj_in = lin(p + ".proj_in", C, C, true);

    const std::string t = p + ".transformer_blocks.0";
    x.ln1 = norm(t + ".norm1", C); x.ln2 = norm(t + ".norm2", C); x.ln3 = norm(t + ".norm3", C);
    // fused QKV [3C, C]
    const HostTensor *q = get(t + ".attn1.to_q.weight"), *k = get(t + ".attn1.to_k.weight"),
                     *v = get(t + ".attn1.to_v.weight");
    if (shape_is(q, {C, C}, t + ".attn1.to_q.weight") && shape_is(k, {C, C}, t + ".attn1.to_k.weight") &&
        shape_is(v, {C, C}, t + ".attn1.to_v.weight")) {
      std::vector<float> w;
      w.reserve(size_t(3) * C * C);
      w.insert(w.end(), q->data.begin(), q->data.end());
      w.insert(w.end(), k->data.begin(), k->data.end());
      w.insert(w.end(), v->data.begin(), v->data.end());
      x.qkv.n = 3 * C; x.qkv.k = C; x.qkv.w = up_bf16(w);
    }
    x.o1 = lin(t + ".attn1.to_out.0", C, C, true);
    {
      const HostTensor *q2 = get(t + ".attn2.to_q.weight"), *o2 = get(t + ".attn2.to_out.0.weight"),
                       *ob = get(t + ".attn2.to_out.0.bias");
      if (shape_is(q2, {C, C}, t + ".attn2.to_q.weight") && shape_is(o2, {C, C}, t + ".attn2.to_out.0.weight") &&
          shape_is(ob, {C}, t + ".attn2.to_out.0.bias")) {
        x.q2w = up_f32(q2->data); x.o2w = up_f32(o2->data); x.o2b = up_f32(ob->data);
      }
    }
    const HostTensor *k2 = get(t + ".attn2.to_k.weight"), *v2 = get(t + ".attn2.to_v.weight");
    if (shape_is(k2, {C, ctx}, t + ".attn2.to_k.weight") && shape_is(v2, {C, ctx}, t + ".attn2.to_v.weight")) {
      x.k2w = up_f32(k2->data); x.v2w = up_f32(v2->data);
    }
    // folded against the empty prompt's two tokens by set_text_embedding, in place
    x.kv = static_cast<float*>(upload(nullptr, size_t(2) * 2 * C * 4));
    x.xGU = static_cast<bf16*>(upload(nullptr, size_t(2) * (C / 64) * C * 2));
    x.xc1 = static_cast<float*>(upload(nullptr, size_t(C) * 4));
    // GEGLU: interleave [value | gate] per 256-column accumulator tile
    const HostTensor *fw = get(t + ".ff.net.0.proj.weight"), *fb = get(t + ".ff.net.0.proj.bias");
    if (shape_is(fw, {8 * C, C}, t + ".ff.net.0.proj.weight") && shape_is(fb, {8 * C}, t + ".ff.net.0.proj.bias")) {
      const int N = 8 * C, half = 128, tiles = N / 256;
      std::vector<float> w(size_t(N) * C), b(N);
      for (int nt = 0; nt < tiles; ++nt)
        for (int r = 0; r < 256; ++r) {
          const int src = r < half ? nt * half + r : 4 * C + nt * half + (r - half);
          memcpy(&w[(size_t(nt) * 256 + r) * C], &fw->data[size_t(src) * C], size_t(C) * 4);
          b[nt * 256 + r] = fb->data[src];
        }
      x.ff1.n = N; x.ff1.k = C; x.ff1.geglu = true;
      x.ff1.w = up_bf16(w); x.ff1.b = up_f32(b);
    }
    {
      // y = x + proj_out(hs0 + ff.net.2(m)) = x + hs0 W_po^T + m (W_po W_ff2)^T + (b_po + W_po b_ff2): one GEMM over the
      // K-concatenated operand [hs0 | m] with the folded weight (product in fp32 on the device, then bf16)
      const HostTensor *wpo = get(p + ".proj_out.weight"), *bpo = get(p + ".proj_out.bias"),
                       *w2 = get(t + ".ff.net.2.weight"), *b2 = get(t + ".ff.net.2.bias");
      if (shape_is(wpo, {C, C}, p + ".proj_out.weight") && shape_is(bpo, {C}, p + ".proj_out.bias") &&
          shape_is(w2, {C, 4 * C}, t + ".ff.net.2.weight") && shape_is(b2, {C}, t + ".ff.net.2.bias")) {
        const int K = 5 * C;
        std::vector<float> wl(size_t(C) * K, 0.f), b(C);
        for (int n = 0; n < C; ++n) {
          memcpy(&wl[size_t(n) * K], &wpo->data[size_t(n) * C], size_t(C) * 4);
          double acc = bpo->data[n];
          for (int j = 0; j < C; ++j) acc += double(wpo->data[size_t(n) * C + j]) * b2->data[j];
          b[n] = float(acc);
        }
        x.ffpo.n = C; x.ffpo.k = K;
        x.ffpo.w = up_bf16(wl);
        x.ffpo.b = up_f32(b);
        DevBuf<float> dA, dB;
        if (x.ffpo.w && dA.grow(size_t(C) * C * 4) == MGB_OK && dB.grow(size_t(C) * 4 * C * 4) == MGB_OK &&
            cudaMemcpy(dA, wpo->data.data(), size_t(C) * C * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
            cudaMemcpy(dB, w2->data.data(), size_t(C) * 4 * C * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
            launch_fold_matmul(dA, dB, x.ffpo.w, C, 4 * C, C, K, C, nullptr) == MGB_OK &&
            cudaDeviceSynchronize() == cudaSuccess) {
        } else if (rc == MGB_OK) { set_error("folding proj_out . ff.net.2 failed for %s", p.c_str()); rc = MGB_ERR_CUDA; }
      }
    }
    return x;
  }
  VaeAttnW vae_attn(const std::string& p, int C) {
    VaeAttnW a; a.C = C;
    a.gn = norm(p + ".group_norm", C);
    a.q = lin(p + ".to_q", C, C, true);
    a.k = lin(p + ".to_k", C, C, true);
    a.v = lin(p + ".to_v", C, C, true);
    a.o = lin(p + ".to_out.0", C, C, true);
    return a;
  }
};

extern "C" {

int mgb_create(const mgb_config* cfg, mgb_handle** out) {
  if (!cfg || !out) { set_error("mgb_create: null argument"); return MGB_ERR_INVALID; }
  for (int i = 0; i < 4; ++i) {
    if (cfg->unet_block_channels[i] <= 0 || cfg->unet_block_channels[i] % 64 || cfg->vae_block_channels[i] <= 0 ||
        cfg->vae_block_channels[i] % 64) {
      set_error("mgb_create: block channels must be positive multiples of 64");
      return MGB_ERR_INVALID;
    }
  }
  // depth / normals: in 8 = rgb(4) | target(4), out 4. IID with n targets (marigold_iid_pipeline.py:467-585,
  // src/trainer/marigold_iid_trainer.py:203-246): in 4 (n + 1), out 4 n; the scheduler epilogue handles <= 16 columns
  if (cfg->vae_latent_channels != 4 || cfg->unet_out_channels < 4 || cfg->unet_out_channels % 4 || cfg->unet_out_channels > 16 ||
      cfg->unet_in_channels != 4 + cfg->unet_out_channels) {
    set_error("mgb_create: need latent=4, out=4n (n <= 4), in=4+out (got in=%d out=%d latent=%d)", cfg->unet_in_channels,
              cfg->unet_out_channels, cfg->vae_latent_channels);
    return MGB_ERR_UNSUPPORTED;
  }
  if (cfg->norm_groups <= 0 || cfg->unet_cross_dim <= 0 || cfg->unet_layers_per_block <= 0 ||
      cfg->vae_layers_per_block <= 0) {
    set_error("mgb_create: bad config");
    return MGB_ERR_INVALID;
  }
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) {
    set_error("mgb_create: no CUDA device (this library has no CPU fallback)");
    return MGB_ERR_CUDA;
  }
  mgb_handle* h = new mgb_handle();
  h->cfg = *cfg;
  *out = h;
  return MGB_OK;
}

void mgb_destroy(mgb_handle* h) { delete h; }

int mgb_load_tensor(mgb_handle* h, const char* key, const void* data, const int64_t* shape, int32_t ndim,
                    int32_t dtype) {
  if (!h || !key || !data || !shape || ndim < 0 || ndim > 8) { set_error("load_tensor: bad argument"); return MGB_ERR_INVALID; }
  if (h->finalized) { set_error("load_tensor after finalize_weights"); return MGB_ERR_STATE; }
  HostTensor t;
  size_t n = 1;
  for (int i = 0; i < ndim; ++i) { t.shape.push_back(shape[i]); n *= size_t(shape[i]); }
  t.data.resize(n);
  if (dtype == MGB_F32) memcpy(t.data.data(), data, n * 4);
  else if (dtype == MGB_BF16) {
    const uint16_t* s = static_cast<const uint16_t*>(data);
    for (size_t i = 0; i < n; ++i) { uint32_t u = uint32_t(s[i]) << 16; memcpy(&t.data[i], &u, 4); }
  } else if (dtype == MGB_F16) {
    const uint16_t* s = static_cast<const uint16_t*>(data);
    for (size_t i = 0; i < n; ++i) t.data[i] = half2f(s[i]);
  } else { set_error("load_tensor: unknown dtype %d", dtype); return MGB_ERR_INVALID; }
  h->host[key] = std::move(t);
  return MGB_OK;
}

// All or nothing: a failed call leaves the handle unfinalized and holding none of its uploads, so it can be retried.
int mgb_finalize_weights(mgb_handle* h) {
  if (!h) { set_error("null handle"); return MGB_ERR_INVALID; }
  if (h->finalized) { set_error("finalize_weights called twice"); return MGB_ERR_STATE; }
  Loader L{h->host, {}};
  const mgb_config& cfg = h->cfg;
  const int* ch = cfg.unet_block_channels;
  const int nl = cfg.unet_layers_per_block;
  const int temb = ch[0] * 4, ctx = cfg.unet_cross_dim;
  UNetW U;
  U.temb_dim = temb;
  U.conv_in = L.conv("unet.conv_in", cfg.unet_in_channels, ch[0]);
  {
    const HostTensor *w1 = L.get("unet.time_embedding.linear_1.weight"), *b1 = L.get("unet.time_embedding.linear_1.bias"),
                     *w2 = L.get("unet.time_embedding.linear_2.weight"), *b2 = L.get("unet.time_embedding.linear_2.bias");
    if (L.shape_is(w1, {temb, ch[0]}, "unet.time_embedding.linear_1.weight") && L.shape_is(b1, {temb}, "…linear_1.bias") &&
        L.shape_is(w2, {temb, temb}, "unet.time_embedding.linear_2.weight") && L.shape_is(b2, {temb}, "…linear_2.bias")) {
      U.te_w1 = L.up_f32(w1->data); U.te_b1 = L.up_f32(b1->data);
      U.te_w2 = L.up_f32(w2->data); U.te_b2 = L.up_f32(b2->data);
    }
  }
  // down blocks (execution order)
  std::vector<int> skip_ch = {ch[0]};
  int prev = ch[0];
  for (int i = 0; i < 4; ++i) {
    const std::string b = "unet.down_blocks." + std::to_string(i);
    for (int j = 0; j < nl; ++j) {
      U.resnets.push_back(L.resnet(b + ".resnets." + std::to_string(j), j == 0 ? prev : ch[i], ch[i], temb, 1e-5f));
      if (i < 3) U.xfmrs.push_back(L.xfmr(b + ".attentions." + std::to_string(j), ch[i], ctx));
      skip_ch.push_back(ch[i]);
    }
    if (i < 3) { U.downs.push_back(L.conv(b + ".downsamplers.0.conv", ch[i], ch[i])); skip_ch.push_back(ch[i]); }
    prev = ch[i];
  }
  U.resnets.push_back(L.resnet("unet.mid_block.resnets.0", ch[3], ch[3], temb, 1e-5f));
  U.xfmrs.push_back(L.xfmr("unet.mid_block.attentions.0", ch[3], ctx));
  U.resnets.push_back(L.resnet("unet.mid_block.resnets.1", ch[3], ch[3], temb, 1e-5f));
  prev = ch[3];
  for (int i = 0; i < 4; ++i) {
    const int cout = ch[3 - i];
    const std::string b = "unet.up_blocks." + std::to_string(i);
    for (int j = 0; j < nl + 1; ++j) {
      const int sc = skip_ch.back(); skip_ch.pop_back();
      U.resnets.push_back(L.resnet(b + ".resnets." + std::to_string(j), (j == 0 ? prev : cout) + sc, cout, temb, 1e-5f));
      if (i > 0) U.xfmrs.push_back(L.xfmr(b + ".attentions." + std::to_string(j), cout, ctx));
    }
    if (i < 3) U.ups.push_back(L.conv(b + ".upsamplers.0.conv", cout, cout));
    prev = cout;
  }
  U.norm_out = L.norm("unet.conv_norm_out", ch[0]);
  U.conv_out = L.conv("unet.conv_out", ch[0], cfg.unet_out_channels);

  // ---- VAE ----
  VaeW V;
  const int* vc = cfg.vae_block_channels;
  const int vl = cfg.vae_layers_per_block;
  V.enc_in = L.conv("vae.encoder.conv_in", 3, vc[0]);
  prev = vc[0];
  for (int i = 0; i < 4; ++i) {
    const std::string b = "vae.encoder.down_blocks." + std::to_string(i);
    for (int j = 0; j < vl; ++j)
      V.enc_res.push_back(L.resnet(b + ".resnets." + std::to_string(j), j == 0 ? prev : vc[i], vc[i], 0, 1e-6f));
    if (i < 3) V.enc_down.push_back(L.conv(b + ".downsamplers.0.conv", vc[i], vc[i]));
    prev = vc[i];
  }
  V.enc_res.push_back(L.resnet("vae.encoder.mid_block.resnets.0", vc[3], vc[3], 0, 1e-6f));
  V.enc_attn = L.vae_attn("vae.encoder.mid_block.attentions.0", vc[3]);
  V.enc_res.push_back(L.resnet("vae.encoder.mid_block.resnets.1", vc[3], vc[3], 0, 1e-6f));
  V.enc_norm_out = L.norm("vae.encoder.conv_norm_out", vc[3]);
  {
    // conv_out (C -> 8) followed by quant_conv (1x1, 8 -> 8): fold, keep the 4 mean channels
    // (reference marigold_depth_pipeline.py:491-495); the bias is pre-multiplied by latent_scale
    // because the epilogue computes acc * scale + bias.
    const int C = vc[3];
    const HostTensor *cw = L.get("vae.encoder.conv_out.weight"), *cb = L.get("vae.encoder.conv_out.bias"),
                     *qw = L.get("vae.quant_conv.weight"), *qb = L.get("vae.quant_conv.bias");
    if (L.shape_is(cw, {8, C, 3, 3}, "vae.encoder.conv_out.weight") && L.shape_is(cb, {8}, "vae.encoder.conv_out.bias") &&
        L.shape_is(qw, {8, 8, 1, 1}, "vae.quant_conv.weight") && L.shape_is(qb, {8}, "vae.quant_conv.bias")) {
      std::vector<float> w(size_t(4) * C * 9, 0.f), b(4, 0.f);
      for (int o = 0; o < 4; ++o) {
        double bb = qb->data[o];
        for (int j = 0; j < 8; ++j) {
          const float q = qw->data[o * 8 + j];
          bb += double(q) * cb->data[j];
          for (size_t e = 0; e < size_t(C) * 9; ++e) w[size_t(o) * C * 9 + e] += q * cw->data[size_t(j) * C * 9 + e];
        }
        b[o] = float(bb * cfg.latent_scale);
      }
      V.enc_out.cin = C; V.enc_out.cin_pad = C; V.enc_out.cout = 4;
      V.enc_out.w = L.up_bf16(Loader::pack_conv(w, 4, C, C));
      V.enc_out.b = L.up_f32(b);
    }
  }
  {
    const HostTensor *pw = L.get("vae.post_quant_conv.weight"), *pb = L.get("vae.post_quant_conv.bias");
    if (L.shape_is(pw, {4, 4, 1, 1}, "vae.post_quant_conv.weight") && L.shape_is(pb, {4}, "vae.post_quant_conv.bias")) {
      V.pq_w = L.up_f32(pw->data); V.pq_b = L.up_f32(pb->data);
    }
  }
  V.dec_in = L.conv("vae.decoder.conv_in", 4, vc[3]);
  V.dec_res.push_back(L.resnet("vae.decoder.mid_block.resnets.0", vc[3], vc[3], 0, 1e-6f));
  V.dec_attn = L.vae_attn("vae.decoder.mid_block.attentions.0", vc[3]);
  V.dec_res.push_back(L.resnet("vae.decoder.mid_block.resnets.1", vc[3], vc[3], 0, 1e-6f));
  prev = vc[3];
  for (int i = 0; i < 4; ++i) {
    const int cout = vc[3 - i];
    const std::string b = "vae.decoder.up_blocks." + std::to_string(i);
    for (int j = 0; j < vl + 1; ++j)
      V.dec_res.push_back(L.resnet(b + ".resnets." + std::to_string(j), j == 0 ? prev : cout, cout, 0, 1e-6f));
    if (i < 3) V.dec_up.push_back(L.conv(b + ".upsamplers.0.conv", cout, cout));
    prev = cout;
  }
  V.dec_norm_out = L.norm("vae.decoder.conv_norm_out", vc[0]);
  V.dec_out = L.conv("vae.decoder.conv_out", vc[0], 3);

  if (L.rc != MGB_OK) return L.rc;
  // what the step graph selects each step into: a row of every resnet's (conv1.bias + time_emb_proj(silu(temb))),
  // {kx, kv, kz}, and the step counter. Their sizes are fixed by the network, so a retried call reuses them.
  int total = 0;
  for (ResnetW& r : U.resnets) { r.bias_off = total; total += r.cout; }
  TRY(h->cur_bias.grow(size_t(total) * 4));
  TRY(h->cur_sched_k.grow(3 * 4));
  TRY(h->step_counter.grow(4));
  CUDA_TRY(cudaMemset(h->step_counter, 0, 4));
  CUDA_TRY(cudaDeviceSynchronize());
  h->weights = std::move(L.weights);
  h->unet = std::move(U);
  h->vae = std::move(V);
  h->bias_total = total;
  h->host.clear();
  h->finalized = true;
  return MGB_OK;
}

// The folded kv / xGU / xc1 are rewritten in place: a captured step graph reads them.
int mgb_set_text_embedding(mgb_handle* h, const float* embed_host, int32_t n_tokens) {
  if (!h || !embed_host) { set_error("set_text_embedding: null argument"); return MGB_ERR_INVALID; }
  if (!h->finalized) { set_error("set_text_embedding before finalize_weights"); return MGB_ERR_STATE; }
  if (n_tokens != 2) {
    set_error("set_text_embedding: the cross-attention kernel is specialised to the empty prompt's 2 tokens (got %d)",
              n_tokens);
    return MGB_ERR_UNSUPPORTED;
  }
  h->text_set = false;
  const int ctx = h->cfg.unet_cross_dim;
  DevBuf<float> d_ctx;
  TRY(d_ctx.grow(size_t(n_tokens) * ctx * 4));
  CUDA_TRY(cudaMemcpy(d_ctx, embed_host, size_t(n_tokens) * ctx * 4, cudaMemcpyHostToDevice));
  for (XfmrW& x : h->unet.xfmrs) {
    TRY(launch_linear_small(d_ctx, x.k2w, nullptr, x.kv, n_tokens, x.C, ctx, 0, 0, nullptr));
    TRY(launch_linear_small(d_ctx, x.v2w, nullptr, x.kv + size_t(n_tokens) * x.C, n_tokens, x.C, ctx, 0, 0, nullptr));
    TRY(launch_xattn2_fold(x.q2w, x.o2w, x.o2b, x.kv, x.xGU, x.xc1, x.C, nullptr));
  }
  CUDA_TRY(cudaDeviceSynchronize());
  h->text_set = true;
  return MGB_OK;
}

int mgb_set_schedule(mgb_handle* h, int32_t n, const int32_t* timesteps, const float* kx, const float* kv,
                     const float* kz) {
  if (!h || n <= 0 || !timesteps || !kx || !kv || !kz) { set_error("set_schedule: bad argument"); return MGB_ERR_INVALID; }
  if (!h->finalized) { set_error("set_schedule before finalize_weights"); return MGB_ERR_STATE; }
  const UNetW& U = h->unet;
  const int c0 = h->cfg.unet_block_channels[0], temb = U.temb_dim, total = h->bias_total;
  std::vector<float> t(n), k(size_t(n) * 3);
  for (int i = 0; i < n; ++i) { t[i] = float(timesteps[i]); k[3 * i] = kx[i]; k[3 * i + 1] = kv[i]; k[3 * i + 2] = kz[i]; }
  int max_c = 0;
  for (const ResnetW& r : U.resnets) max_c = std::max(max_c, r.cout);
  DevBuf<float> sched_k, d_t, d_emb, d_h1, d_temb, bias_table, tmp;
  TRY(sched_k.grow(k.size() * 4));
  CUDA_TRY(cudaMemcpy(sched_k, k.data(), k.size() * 4, cudaMemcpyHostToDevice));
  TRY(d_t.grow(size_t(n) * 4));
  TRY(d_emb.grow(size_t(n) * c0 * 4));
  TRY(d_h1.grow(size_t(n) * temb * 4));
  TRY(d_temb.grow(size_t(n) * temb * 4));
  CUDA_TRY(cudaMemcpy(d_t, t.data(), n * 4, cudaMemcpyHostToDevice));
  TRY(launch_timestep_embedding(d_t, d_emb, n, c0, nullptr));
  TRY(launch_linear_small(d_emb, U.te_w1, U.te_b1, d_h1, n, temb, c0, 0, 1, nullptr));
  TRY(launch_linear_small(d_h1, U.te_w2, U.te_b2, d_temb, n, temb, temb, 0, 0, nullptr));
  // one contiguous table [n, bias_total]: row i = every resnet's (conv1.bias + time_emb_proj(silu(temb_i)))
  TRY(bias_table.grow(size_t(n) * total * 4));
  TRY(tmp.grow(size_t(n) * max_c * 4));
  for (const ResnetW& r : U.resnets) {
    TRY(launch_linear_small(d_temb, r.temb_w, r.temb_b, tmp, n, r.cout, temb, 1, 0, nullptr));
    CUDA_TRY(cudaMemcpy2DAsync(bias_table.get() + r.bias_off, size_t(total) * 4, tmp, size_t(r.cout) * 4,
                               size_t(r.cout) * 4, n, cudaMemcpyDeviceToDevice, nullptr));
  }
  CUDA_TRY(cudaDeviceSynchronize());
  invalidate_step_graph(h);
  h->sched_k = std::move(sched_k);
  h->bias_table = std::move(bias_table);
  h->kz_host.assign(kz, kz + n);
  h->n_steps = n;
  return MGB_OK;
}

// -------------------------------------------------------------------------------------------------
// workspace management: dry-run the requested graph to size the arena and split-K workspace
// -------------------------------------------------------------------------------------------------
enum { OP_UNET = 0, OP_ENCODE = 1, OP_DECODE = 2 };

// The UNet step's NHWC staging buffers, carved from the start of the arena in this order (a braced list is evaluated
// left to right). The captured step graph bakes in their addresses, so the single step and the denoising loop must
// lay them out identically.
struct UNetStaging { float *rgb, *tgt, *nz, *raw; };
static UNetStaging stage_unet(mgb_handle* h, Arena& a, int NB, int HW) {
  const size_t n = size_t(NB) * HW * h->cfg.unet_out_channels * 4;
  auto f32 = [&a](size_t bytes) { return reinterpret_cast<float*>(a.alloc(bytes)); };
  a.off = 0;
  return {f32(size_t(NB) * HW * 4 * 4), f32(n), f32(n), f32(n)};
}

static size_t weight_bytes(const mgb_handle* h) {
  size_t n = 0;
  for (const auto& w : h->weights) n += w.bytes();
  return n;
}

// What any call that decodes needs beside the workspace and the weights, at least: the CUDA context of a process that has
// loaded torch and this library (measured 0.90 GB on an H100 80GB HBM3), and per output pixel the smallest reserve a
// pipeline call holds, one depth member's (pipeline.call_reserve_bytes(h, w, 1, 1): 4 (1 * 4 + 3) bytes).
constexpr size_t kDecodeContextBytes = size_t(768) << 20;
constexpr size_t kDecodeReservePerPixel = 28;

// The handle's row split (mgb_set_row_split) into a forward's context, or none
static void set_split(const mgb_handle* h, Ctx& c) {
  const mgb_handle::RowSplit& r = h->row_split;
  c.split_world = r.fn ? r.world : 0;
  c.split_rank = r.rank;
  c.exchange_fn = r.fn;
  c.exchange_ctx = r.ctx;
}

// The context of a real run on `stream`, in the handle's arena and workspaces
static Ctx make_ctx(mgb_handle* h, void* stream) {
  Ctx c;
  c.stream = reinterpret_cast<cudaStream_t>(stream);
  c.arena = &h->arena;
  c.arena->base = h->arena_buf; c.arena->cap = h->arena_buf.bytes();
  c.arena->dry = false; c.arena->status = MGB_OK; c.arena->plan = nullptr;
  c.dry = false;
  c.opt = h->opt;
  c.splitk_ws = h->splitk_ws; c.splitk_cap = h->splitk_ws.bytes();
  c.groups = h->cfg.norm_groups;
  c.sync_base = h->sync_slab;
  c.sync_cap = h->sync_slab.bytes() / sizeof(unsigned);
  set_split(h, c);
  return c;
}

// The context of a dry run: it launches nothing, records its allocations in *dry and sums its workspace needs
static Ctx dry_ctx(const mgb_handle* h, Arena* dry) {
  dry->dry = true;
  Ctx c;
  c.arena = dry;
  c.dry = true;
  c.opt = h->opt;
  c.splitk_cap = ~size_t(0);
  c.groups = h->cfg.norm_groups;
  set_split(h, c);
  return c;
}

// Whether a decode of lh x lw latents runs its full-resolution 256-channel stage in low memory (Ctx::dec_low_memory):
// where one member's decode on the default path cannot be admitted on this device, i.e. needs more than its memory
// less the weights, kDecodeContextBytes and kDecodeReservePerPixel per pixel. No decode that the default path could
// run is moved, since each needs at least that much beside its workspace; or as mgb_debug_vae_low_memory sets it. The
// decision depends on the shape and the VAE attention's row blocking alone, and is kept for the last shape asked.
static int decode_low_memory(mgb_handle* h, int lh, int lw, bool* on) {
  if (h->opt.low_memory != 0) { *on = h->opt.low_memory > 0; return MGB_OK; }
  mgb_handle::DecodeRule& k = h->decode_rule;
  if (k.valid && k.lh == lh && k.lw == lw && k.attn_budget == h->opt.attn_budget && k.attn_rows == h->opt.attn_rows) {
    *on = k.low_memory;
    return MGB_OK;
  }
  if (h->device_bytes == 0) {
    size_t free_b = 0, total = 0;
    CUDA_TRY(cudaMemGetInfo(&free_b, &total));
    h->device_bytes = total;
  }
  Arena dry;
  Ctx c = dry_ctx(h, &dry);
  // the rule prices one member's whole decode on the default path: no rank's share of the rows, and no bands
  c.split_world = 0;
  c.opt.band_up_tiles = c.opt.band_conv1_tiles = 0;
  c.arena->start();
  c.planned = true;
  TRY(vae_decode_forward(h, c, nullptr, nullptr, 1, lh, lw, 0));
  dry.finish();
  const size_t need = arena_place(dry.rec, 0) + c.splitk_need;
  const size_t pixels = size_t(64) * lh * lw;
  *on = need + weight_bytes(h) + kDecodeContextBytes + kDecodeReservePerPixel * pixels > h->device_bytes;
  k = {true, lh, lw, h->opt.attn_budget, h->opt.attn_rows, *on};
  return MGB_OK;
}

// a0..a3 meaning per op:
//   UNET:   a0 = rgb latent NCHW, a1 = target NCHW (in/out), a2 = noise NCHW or null, a3 = model_out NCHW or null
//   ENCODE: a0 = rgb NCHW, a1 = latent out NCHW
//   DECODE: a0 = latent NCHW, a1 = out NCHW
static int run_graph(mgb_handle* h, Ctx& c, int op, const float* a0, float* a1, const float* a2, float* a3, int step,
                     int NB, int d0, int d1, int mode) {
  c.arena->start();
  c.planned = op != OP_UNET;
  if (op == OP_ENCODE) return vae_encode_forward(h, c, a0, a1, NB, d0, d1);
  if (op == OP_DECODE) {
    TRY(decode_low_memory(h, d0, d1, &c.dec_low_memory));
    return vae_decode_forward(h, c, a0, a1, NB, d0, d1, mode);
  }
  // UNET single step through NCHW <-> NHWC conversions
  const int HW = d0 * d1, Ct = h->cfg.unet_out_channels;
  const UNetStaging s = stage_unet(h, *c.arena, NB, HW);
  if (!c.dry) {
    TRY(launch_nchw_to_nhwc(a0, s.rgb, NB, 4, HW, 1.f, c.stream));
    TRY(launch_nchw_to_nhwc(a1, s.tgt, NB, Ct, HW, 1.f, c.stream));
    if (a2) TRY(launch_nchw_to_nhwc(a2, s.nz, NB, Ct, HW, 1.f, c.stream));
  }
  TRY(unet_forward(h, c, s.rgb, s.tgt, a2 ? s.nz : nullptr, a3 ? s.raw : nullptr, step, NB, d0, d1));
  if (!c.dry) {
    TRY(launch_nhwc_to_nchw(s.tgt, a1, NB, Ct, HW, 1.f, c.stream));
    if (a3) TRY(launch_nhwc_to_nchw(s.raw, a3, NB, Ct, HW, 1.f, c.stream));
  }
  return MGB_OK;
}

struct WorkspaceNeed { size_t arena = 0, splitk = 0, sync = 0; };   // bytes

// Dry-runs one graph: its arena peak, split-K workspace and GroupNorm barrier counters. The VAE forwards' arena is
// planned: their buffers, placed by lifetime (arena_place with the handle's placement), go to *bufs and the arena
// peak is the plan's. The UNet step keeps the bump allocator's stack layout, which its captured graph holds; *bufs
// then receives the buffers at their bump offsets.
static int workspace_need(mgb_handle* h, int op, int NB, int d0, int d1, WorkspaceNeed* need,
                          std::vector<ArenaBuf>* bufs = nullptr) {
  Arena dry;
  Ctx c = dry_ctx(h, &dry);
  TRY(run_graph(h, c, op, nullptr, nullptr, nullptr, nullptr, 0, NB, d0, d1, 0));
  dry.finish();
  const size_t arena = op == OP_UNET ? dry.peak : arena_place(dry.rec, h->opt.placement);
  *need = {arena, c.splitk_need, c.sync_need * sizeof(unsigned)};
  if (bufs) bufs->swap(dry.rec);
  return MGB_OK;
}

static int ensure_workspace(mgb_handle* h, int op, int NB, int d0, int d1) {
  WorkspaceNeed need;
  TRY(workspace_need(h, op, NB, d0, d1, &need, op == OP_UNET ? nullptr : &h->arena_plan));
  TRY(grow_captured(h, h->arena_buf, need.arena + (1 << 20)));
  TRY(grow_captured(h, h->splitk_ws, need.splitk));
  return grow_captured(h, h->sync_slab, need.sync);
}

static int check_ready(mgb_handle* h, bool need_sched) {
  if (!h) { set_error("null handle"); return MGB_ERR_INVALID; }
  if (!h->finalized) { set_error("weights not finalized"); return MGB_ERR_STATE; }
  if (need_sched && (!h->text_set || h->n_steps == 0)) {
    set_error("set_text_embedding and set_schedule must be called before denoising");
    return MGB_ERR_STATE;
  }
  return MGB_OK;
}

// B images of H x W pixels (a decode's output size) within kMaxPixels, checked before anything is sized or launched
static int check_pixels(const char* what, int B, int H, int W) {
  if (size_t(B) * size_t(H) * size_t(W) > kMaxPixels) {
    set_error("%s: %d x %d x %d pixels exceed the supported maximum of %zu per call", what, B, H, W, kMaxPixels);
    return MGB_ERR_UNSUPPORTED;
  }
  return MGB_OK;
}

// A row-split handle runs one image per call
static int check_split_batch(const mgb_handle* h, const char* what, int B) {
  if (h->row_split.fn && B != 1) {
    set_error("%s: the handle splits attention rows over %d ranks, which takes one image per call (got %d)", what,
              h->row_split.world, B);
    return MGB_ERR_INVALID;
  }
  return MGB_OK;
}

// Sizes the workspace for one graph, then runs it once on `stream` (run_graph's arguments).
static int run_once(mgb_handle* h, void* stream, int op, const float* a0, float* a1, const float* a2, float* a3,
                    int step, int NB, int d0, int d1, int mode) {
  TRY(ensure_workspace(h, op, NB, d0, d1));
  Ctx c = make_ctx(h, stream);
  if (op != OP_UNET) c.arena->plan = &h->arena_plan;
  TRY(run_graph(h, c, op, a0, a1, a2, a3, step, NB, d0, d1, mode));
  TRY(h->arena.status);
  if (c.arena->plan && c.arena->n != h->arena_plan.size()) {
    set_error("arena: the forward made %zu allocations, its plan %zu", c.arena->n, h->arena_plan.size());
    return MGB_ERR_STATE;
  }
  return MGB_OK;
}

int mgb_encode(mgb_handle* h, const float* rgb, int32_t B, int32_t H, int32_t W, float* latent, void* stream) {
  TRY(check_ready(h, false));
  if (!rgb || !latent || B <= 0 || H < 8 || W < 8) {
    set_error("mgb_encode: need B > 0 and H, W >= 8 (got %d x %d)", H, W);
    return MGB_ERR_INVALID;
  }
  TRY(check_pixels("mgb_encode", B, H, W));
  TRY(check_split_batch(h, "mgb_encode", B));
  return run_once(h, stream, OP_ENCODE, rgb, latent, nullptr, nullptr, 0, B, H, W, 0);
}

int mgb_unet_step(mgb_handle* h, const float* rgb_latent, float* target, const float* noise, float* model_out,
                  int32_t step_index, int32_t B, int32_t lh, int32_t lw, void* stream) {
  TRY(check_ready(h, true));
  if (!rgb_latent || !target || B <= 0 || lh <= 0 || lw <= 0) {
    set_error("mgb_unet_step: bad argument (latent %d x %d)", lh, lw);
    return MGB_ERR_INVALID;
  }
  if (step_index < 0 || step_index >= h->n_steps) { set_error("step_index %d outside schedule of %d", step_index, h->n_steps); return MGB_ERR_INVALID; }
  if (h->kz_host[step_index] != 0.f && !noise) { set_error("step %d needs noise (kz != 0)", step_index); return MGB_ERR_INVALID; }
  TRY(check_split_batch(h, "mgb_unet_step", B));
  return run_once(h, stream, OP_UNET, rgb_latent, target, noise, model_out, step_index, B, lh, lw, 0);
}

int mgb_denoise_range(mgb_handle* h, const float* rgb_latent, float* target, const float* step_noise,
                      int32_t first_step, int32_t num_steps, int32_t B, int32_t lh, int32_t lw, void* stream) {
  TRY(check_ready(h, true));
  if (!rgb_latent || !target || B <= 0 || lh <= 0 || lw <= 0) {
    set_error("mgb_denoise: bad argument (latent %d x %d)", lh, lw);
    return MGB_ERR_INVALID;
  }
  if (first_step < 0 || num_steps < 0 || first_step + num_steps > h->n_steps) {
    set_error("mgb_denoise_range: steps [%d, %d) outside schedule of %d", first_step, first_step + num_steps, h->n_steps);
    return MGB_ERR_INVALID;
  }
  for (int i = first_step; i < first_step + num_steps; ++i)
    if (h->kz_host[i] != 0.f && !step_noise) { set_error("schedule step %d injects noise but step_noise is NULL", i); return MGB_ERR_INVALID; }
  TRY(check_split_batch(h, "mgb_denoise", B));
  TRY(ensure_workspace(h, OP_UNET, B, lh, lw));
  Ctx c = make_ctx(h, stream);
  const int HW = lh * lw, Ct = h->cfg.unet_out_channels;
  const size_t n = size_t(B) * HW * Ct;
  const UNetStaging s = stage_unet(h, *c.arena, B, HW);
  const size_t base = c.arena->mark();
  TRY(launch_nchw_to_nhwc(rgb_latent, s.rgb, B, 4, HW, 1.f, c.stream));
  TRY(launch_nchw_to_nhwc(target, s.tgt, B, Ct, HW, 1.f, c.stream));
  const bool any_noise = step_noise != nullptr;
  if (!any_noise) CUDA_TRY(cudaMemsetAsync(s.nz, 0, n * 4, c.stream));   // kz * 0 must stay finite
  static const bool graphs_env = getenv("MGB_NO_GRAPH") == nullptr;
  // a row-split step calls the exchange function from the host between kernels: it runs eagerly, and leaves the
  // graph of the unsplit shape as it is (unless ensure_workspace grew a buffer the graph holds, which drops it)
  const bool graphs = graphs_env && !h->row_split.fn;
  mgb_handle::StepGraph& G = h->step_graph;
  for (int i = first_step; i < first_step + num_steps; ++i) {
    if (h->kz_host[i] != 0.f) TRY(launch_nchw_to_nhwc(step_noise + size_t(i) * n, s.nz, B, Ct, HW, 1.f, c.stream));
    if (graphs && G.exec && G.NB == B && G.lh == lh && G.lw == lw) {
      // arm the device step counter for this replay (pageable 4-byte H2D: staged by the driver, so the
      // source may be reused immediately)
      CUDA_TRY(cudaMemcpyAsync(h->step_counter, &i, 4, cudaMemcpyHostToDevice, c.stream));
      CUDA_TRY(cudaGraphLaunch(G.exec.get(), c.stream));
      count_launch(G.launches);
      continue;
    }
    c.arena->release(base);
    TRY(unet_forward(h, c, s.rgb, s.tgt, s.nz, nullptr, i, B, lh, lw));  // eager (also warms one-time attributes)
    TRY(h->arena.status);   // a step the arena cut short launched only part of its kernels: never capture it
    if (graphs && !G.exec_failed) {
      // capture one step (reads the step index from the device counter) for all later steps of this shape
      invalidate_step_graph(h);
      Ctx cc = c;
      cc.stream = h->capture_stream.get();
      if (!cc.stream) {
        CUDA_TRY(cudaStreamCreateWithFlags(&cc.stream, cudaStreamNonBlocking));
        h->capture_stream.reset(cc.stream);
      }
      const long long l0 = launch_count();
      cudaGraph_t graph = nullptr;
      cudaError_t ce = cudaStreamBeginCapture(cc.stream, cudaStreamCaptureModeThreadLocal);
      int rc = MGB_OK;
      if (ce == cudaSuccess) {
        c.arena->release(base);
        rc = unet_forward(h, cc, s.rgb, s.tgt, s.nz, nullptr, -1, B, lh, lw);
        ce = cudaStreamEndCapture(cc.stream, &graph);
      }
      const long long nl = launch_count() - l0;
      count_launch(-nl);                                                 // capture launched nothing
      cudaGraphExec_t exec = nullptr;
      if (rc == MGB_OK && ce == cudaSuccess && graph) ce = cudaGraphInstantiate(&exec, graph, 0);
      if (graph) cudaGraphDestroy(graph);
      if (rc == MGB_OK && ce == cudaSuccess && exec && h->arena.status == MGB_OK) {
        G.exec.reset(exec); G.NB = B; G.lh = lh; G.lw = lw; G.launches = nl;
      } else {
        cudaGetLastError();
        G.exec_failed = true;                                            // stay on the eager path
      }
    }
  }
  TRY(launch_nhwc_to_nchw(s.tgt, target, B, Ct, HW, 1.f, c.stream));
  return h->arena.status;
}

int mgb_denoise(mgb_handle* h, const float* rgb_latent, float* target, const float* step_noise, int32_t B, int32_t lh,
                int32_t lw, void* stream) {
  if (!h) { set_error("null handle"); return MGB_ERR_INVALID; }
  return mgb_denoise_range(h, rgb_latent, target, step_noise, 0, h->n_steps, B, lh, lw, stream);
}

int mgb_decode(mgb_handle* h, const float* latent, int32_t B, int32_t lh, int32_t lw, int32_t mode, float* out,
               void* stream) {
  TRY(check_ready(h, false));
  if (!latent || !out || B <= 0 || lh <= 0 || lw <= 0 || mode < 0 || mode > 3) {
    set_error("mgb_decode: bad argument (latent %d x %d, mode %d)", lh, lw, mode);
    return MGB_ERR_INVALID;
  }
  TRY(check_pixels("mgb_decode", B, 8 * lh, 8 * lw));
  TRY(check_split_batch(h, "mgb_decode", B));
  return run_once(h, stream, OP_DECODE, latent, out, nullptr, nullptr, 0, B, lh, lw, mode);
}

}  // extern "C"

// -------------------------------------------------------------------------------------------------
// read-back of the handle's device tables (mgb_debug_read): field paths name the structs above in execution order
// -------------------------------------------------------------------------------------------------
namespace {
struct FieldRef {
  const void* p = nullptr;
  size_t bytes = 0;
  bool found = false;
};

// A dotted field path ("unet.resnets.3.c1.w"), matched one part at a time.
struct FieldPath {
  std::vector<std::string> parts;
  size_t pos = 0;
  explicit FieldPath(const std::string& s) {
    for (size_t a = 0;;) {
      const size_t b = s.find('.', a);
      parts.push_back(s.substr(a, b == std::string::npos ? std::string::npos : b - a));
      if (b == std::string::npos) break;
      a = b + 1;
    }
  }
  bool take(const char* name) {
    if (pos >= parts.size() || parts[pos] != name) return false;
    ++pos;
    return true;
  }
  // the next part as a decimal index below n
  bool index(size_t n, size_t* i) {
    if (pos >= parts.size()) return false;
    const std::string& s = parts[pos];
    if (s.empty() || s.size() > 9 || s.find_first_not_of("0123456789") != std::string::npos) return false;
    *i = std::stoul(s);
    if (*i >= n) return false;
    ++pos;
    return true;
  }
  // The last part is `name`. A weight whose pointer is null does not exist (a bias-free GEMM, a VAE resnet's time
  // projection); handle state always does, and is empty until it is first set.
  bool leaf(const char* name, const void* p, size_t bytes, FieldRef* r, bool state = false) {
    if (pos + 1 != parts.size() || parts[pos] != name) return false;
    if (p || state) *r = {p, p ? bytes : 0, true};
    return true;
  }
};

void read_norm(FieldPath& f, const NormW& n, FieldRef* r) {
  f.leaf("g", n.g, size_t(n.c) * 4, r) || f.leaf("b", n.b, size_t(n.c) * 4, r);
}
void read_conv(FieldPath& f, const ConvW& c, FieldRef* r) {
  f.leaf("w", c.w, size_t(c.cout) * (9 * c.cin_pad + c.k_extra) * 2, r) || f.leaf("b", c.b, size_t(c.cout) * 4, r);
}
void read_lin(FieldPath& f, const LinW& l, FieldRef* r) {
  f.leaf("w", l.w, size_t(l.n) * l.k * 2, r) || f.leaf("b", l.b, size_t(l.n) * 4, r);
}
void read_resnet(FieldPath& f, const ResnetW& x, int temb_dim, FieldRef* r) {
  if (f.take("n1")) read_norm(f, x.n1, r);
  else if (f.take("n2")) read_norm(f, x.n2, r);
  else if (f.take("c1")) read_conv(f, x.c1, r);
  else if (f.take("c2")) read_conv(f, x.c2, r);
  else f.leaf("temb_w", x.temb_w, size_t(x.cout) * temb_dim * 4, r) || f.leaf("temb_b", x.temb_b, size_t(x.cout) * 4, r);
}
void read_xfmr(FieldPath& f, const XfmrW& x, int ctx, FieldRef* r) {
  const size_t C = x.C;
  if (f.take("gn")) read_norm(f, x.gn, r);
  else if (f.take("ln1")) read_norm(f, x.ln1, r);
  else if (f.take("ln2")) read_norm(f, x.ln2, r);
  else if (f.take("ln3")) read_norm(f, x.ln3, r);
  else if (f.take("proj_in")) read_lin(f, x.proj_in, r);
  else if (f.take("qkv")) read_lin(f, x.qkv, r);
  else if (f.take("o1")) read_lin(f, x.o1, r);
  else if (f.take("ff1")) read_lin(f, x.ff1, r);
  else if (f.take("ffpo")) read_lin(f, x.ffpo, r);
  else f.leaf("q2w", x.q2w, C * C * 4, r) || f.leaf("o2w", x.o2w, C * C * 4, r) || f.leaf("o2b", x.o2b, C * 4, r) ||
       f.leaf("k2w", x.k2w, C * ctx * 4, r) || f.leaf("v2w", x.v2w, C * ctx * 4, r) ||
       f.leaf("kv", x.kv, 4 * C * 4, r) || f.leaf("xGU", x.xGU, 2 * (C / 64) * C * 2, r) || f.leaf("xc1", x.xc1, C * 4, r);
}
void read_vae_attn(FieldPath& f, const VaeAttnW& a, FieldRef* r) {
  if (f.take("gn")) read_norm(f, a.gn, r);
  else if (f.take("q")) read_lin(f, a.q, r);
  else if (f.take("k")) read_lin(f, a.k, r);
  else if (f.take("v")) read_lin(f, a.v, r);
  else if (f.take("o")) read_lin(f, a.o, r);
}
template <class T, class Read>
void read_list(FieldPath& f, const std::vector<T>& v, Read read) {
  size_t i;
  if (f.index(v.size(), &i)) read(v[i]);
}

FieldRef find_field(const mgb_handle* h, const std::string& name) {
  FieldPath f(name);
  FieldRef r;
  auto conv = [&](const ConvW& c) { read_conv(f, c, &r); };
  auto resnet = [&](const ResnetW& x) { read_resnet(f, x, 0, &r); };
  if (f.take("unet")) {
    const UNetW& U = h->unet;
    const size_t T = U.temb_dim, c0 = h->cfg.unet_block_channels[0];
    if (f.take("conv_in")) conv(U.conv_in);
    else if (f.take("conv_out")) conv(U.conv_out);
    else if (f.take("norm_out")) read_norm(f, U.norm_out, &r);
    else if (f.take("resnets")) read_list(f, U.resnets, [&](const ResnetW& x) { read_resnet(f, x, U.temb_dim, &r); });
    else if (f.take("xfmrs")) read_list(f, U.xfmrs, [&](const XfmrW& x) { read_xfmr(f, x, h->cfg.unet_cross_dim, &r); });
    else if (f.take("downs")) read_list(f, U.downs, conv);
    else if (f.take("ups")) read_list(f, U.ups, conv);
    else f.leaf("te_w1", U.te_w1, T * c0 * 4, &r) || f.leaf("te_b1", U.te_b1, T * 4, &r) ||
         f.leaf("te_w2", U.te_w2, T * T * 4, &r) || f.leaf("te_b2", U.te_b2, T * 4, &r);
  } else if (f.take("vae")) {
    const VaeW& V = h->vae;
    if (f.take("enc_in")) conv(V.enc_in);
    else if (f.take("enc_out")) conv(V.enc_out);
    else if (f.take("enc_norm_out")) read_norm(f, V.enc_norm_out, &r);
    else if (f.take("enc_res")) read_list(f, V.enc_res, resnet);
    else if (f.take("enc_down")) read_list(f, V.enc_down, conv);
    else if (f.take("enc_attn")) read_vae_attn(f, V.enc_attn, &r);
    else if (f.take("dec_in")) conv(V.dec_in);
    else if (f.take("dec_out")) conv(V.dec_out);
    else if (f.take("dec_norm_out")) read_norm(f, V.dec_norm_out, &r);
    else if (f.take("dec_res")) read_list(f, V.dec_res, resnet);
    else if (f.take("dec_up")) read_list(f, V.dec_up, conv);
    else if (f.take("dec_attn")) read_vae_attn(f, V.dec_attn, &r);
    else f.leaf("pq_w", V.pq_w, 16 * 4, &r) || f.leaf("pq_b", V.pq_b, 4 * 4, &r);
  } else {
    const size_t n = h->n_steps, total = h->bias_total;
    f.leaf("bias_table", h->bias_table, n * total * 4, &r, true) || f.leaf("sched_k", h->sched_k, n * 3 * 4, &r, true) ||
        f.leaf("cur_bias", h->cur_bias, total * 4, &r, true) || f.leaf("cur_sched_k", h->cur_sched_k, 3 * 4, &r, true) ||
        f.leaf("step_counter", h->step_counter, 4, &r, true);
  }
  return r;
}
}  // namespace

extern "C" {

int mgb_set_row_split(mgb_handle* h, int32_t rank, int32_t world, mgb_exchange_fn fn, void* ctx) {
  if (!h) { set_error("set_row_split: null handle"); return MGB_ERR_INVALID; }
  if (!fn) { h->row_split = mgb_handle::RowSplit(); return MGB_OK; }
  if (world < 1 || rank < 0 || rank >= world) {
    set_error("set_row_split: rank %d of world %d", rank, world);
    return MGB_ERR_INVALID;
  }
  h->row_split = {rank, world, fn, ctx};
  return MGB_OK;
}

/* debug hooks (declared in debug.h) */

int64_t mgb_debug_read(mgb_handle* h, const char* field, void* dst, int64_t cap_bytes, uint64_t* dev_addr) {
  if (!h || !field) { set_error("debug_read: null argument"); return MGB_ERR_INVALID; }
  if (!h->finalized) { set_error("debug_read('%s') before finalize_weights", field); return MGB_ERR_STATE; }
  const FieldRef r = find_field(h, field);
  if (!r.found) { set_error("debug_read: unknown field '%s'", field); return MGB_ERR_INVALID; }
  if (dev_addr) *dev_addr = uint64_t(reinterpret_cast<uintptr_t>(r.p));
  if (dst && r.bytes) {
    if (cap_bytes < int64_t(r.bytes)) {
      set_error("debug_read: field '%s' has %zu bytes, the destination %lld", field, r.bytes, (long long)cap_bytes);
      return MGB_ERR_INVALID;
    }
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(dst, r.p, r.bytes, cudaMemcpyDeviceToHost));
  }
  return int64_t(r.bytes);
}

int32_t mgb_debug_weight_buffers(mgb_handle* h, uint64_t* addr, int64_t* bytes, int32_t cap) {
  if (!h) { set_error("debug_weight_buffers: null handle"); return MGB_ERR_INVALID; }
  if (!h->finalized) { set_error("debug_weight_buffers before finalize_weights"); return MGB_ERR_STATE; }
  const int32_t n = int32_t(h->weights.size());
  for (int32_t i = 0; i < n && i < cap; ++i) {
    if (addr) addr[i] = uint64_t(reinterpret_cast<uintptr_t>(h->weights[i].get()));
    if (bytes) bytes[i] = int64_t(h->weights[i].bytes());
  }
  return n;
}

int mgb_debug_vae_attn_blocks(mgb_handle* h, int64_t budget_bytes, int32_t force_rows, int32_t NB, int32_t T,
                              int32_t* rows, int32_t* blocks) {
  if (!h || NB <= 0 || T <= 0) { set_error("debug_vae_attn_blocks: bad argument"); return MGB_ERR_INVALID; }
  h->opt.attn_budget = budget_bytes > 0 ? size_t(budget_bytes) : kVaeAttnBudget;
  h->opt.attn_rows = force_rows > 0 ? force_rows : 0;
  const int R = vae_attn_rows(T, h->cfg.vae_block_channels[3], h->opt.attn_budget, h->opt.attn_rows);
  if (rows) *rows = R;
  if (blocks) *blocks = NB * ((T + R - 1) / R);
  return MGB_OK;
}

int mgb_debug_vae_attn_core(mgb_handle* h, const void* q, const void* k, const void* v, void* o, int32_t NB,
                            int32_t T) {
  TRY(check_ready(h, false));
  if (!q || !k || !v || !o || NB <= 0 || T <= 0) { set_error("debug_vae_attn_core: bad argument"); return MGB_ERR_INVALID; }
  const int C = h->cfg.vae_block_channels[3];
  auto in = [](const void* p) { return reinterpret_cast<const bf16*>(p); };
  Arena dry;
  Ctx d = dry_ctx(h, &dry);
  TRY(vae_attn_core(d, in(q), in(k), in(v), reinterpret_cast<bf16*>(o), NB, T, C));
  TRY(grow_captured(h, h->arena_buf, dry.peak + (1 << 20)));
  TRY(grow_captured(h, h->splitk_ws, d.splitk_need));
  Ctx c = make_ctx(h, nullptr);
  c.arena->start();
  TRY(vae_attn_core(c, in(q), in(k), in(v), reinterpret_cast<bf16*>(o), NB, T, C));
  return h->arena.status;
}

int mgb_debug_arena(mgb_handle* h, int32_t poison, int32_t placement) {
  if (!h || placement < 0 || placement > 1) { set_error("debug_arena: bad argument"); return MGB_ERR_INVALID; }
  h->opt.poison = poison != 0;
  h->opt.placement = placement;
  return MGB_OK;
}

int mgb_debug_vae_low_memory(mgb_handle* h, int32_t mode) {
  if (!h || mode < -1 || mode > 1) { set_error("debug_vae_low_memory: bad argument"); return MGB_ERR_INVALID; }
  h->opt.low_memory = mode;
  return MGB_OK;
}

int mgb_debug_vae_bands(mgb_handle* h, int32_t up_tiles, int32_t conv1_tiles) {
  if (!h) { set_error("debug_vae_bands: bad argument"); return MGB_ERR_INVALID; }
  h->opt.band_up_tiles = std::max(0, int(up_tiles));
  h->opt.band_conv1_tiles = std::max(0, int(conv1_tiles));
  return MGB_OK;
}

int64_t mgb_debug_arena_place(int64_t n, const int64_t* bytes, const int64_t* t_alloc, const int64_t* t_free,
                              int32_t placement, int64_t* off) {
  if (n < 0 || (n > 0 && (!bytes || !t_alloc || !t_free || !off)) || placement < 0 || placement > 1) {
    set_error("debug_arena_place: bad argument");
    return MGB_ERR_INVALID;
  }
  std::vector<ArenaBuf> b(static_cast<size_t>(n));
  for (int64_t i = 0; i < n; ++i) {
    if (bytes[i] < 0 || t_free[i] <= t_alloc[i]) {
      set_error("debug_arena_place: buffer %lld has bytes %lld, lifetime [%lld, %lld)", (long long)i,
                (long long)bytes[i], (long long)t_alloc[i], (long long)t_free[i]);
      return MGB_ERR_INVALID;
    }
    b[i].bytes = size_t(bytes[i]); b[i].t_alloc = t_alloc[i]; b[i].t_free = t_free[i];
  }
  const size_t peak = arena_place(b, placement);
  for (int64_t i = 0; i < n; ++i) off[i] = int64_t(b[i].off);
  return int64_t(peak);
}

int64_t mgb_debug_arena_plan(mgb_handle* h, int32_t op, int32_t B, int32_t d0, int32_t d1, int64_t* bytes,
                             int64_t* t_alloc, int64_t* t_free, int64_t* off, int64_t cap) {
  if (!h || op < OP_UNET || op > OP_DECODE || B <= 0 || d0 <= 0 || d1 <= 0) {
    set_error("debug_arena_plan: bad argument");
    return MGB_ERR_INVALID;
  }
  TRY(check_ready(h, false));
  TRY(check_pixels("debug_arena_plan", B, op == OP_ENCODE ? d0 : 8 * d0, op == OP_ENCODE ? d1 : 8 * d1));
  WorkspaceNeed need;
  std::vector<ArenaBuf> bufs;
  TRY(workspace_need(h, op, B, d0, d1, &need, &bufs));
  for (size_t i = 0; i < bufs.size() && int64_t(i) < cap; ++i) {
    if (bytes) bytes[i] = int64_t(bufs[i].bytes);
    if (t_alloc) t_alloc[i] = bufs[i].t_alloc;
    if (t_free) t_free[i] = bufs[i].t_free;
    if (off) off[i] = int64_t(bufs[i].off);
  }
  return int64_t(bufs.size());
}

size_t mgb_workspace_bytes(mgb_handle* h, int32_t B, int32_t H, int32_t W) {
  if (!h || !h->finalized || B <= 0 || H < 8 || W < 8 || size_t(B) * size_t(H) * size_t(W) > kMaxPixels) return 0;
  size_t peak = 0;
  for (int op = 0; op < 3; ++op) {
    const int d0 = op == OP_ENCODE ? H : H / 8, d1 = op == OP_ENCODE ? W : W / 8;
    WorkspaceNeed need;
    if (workspace_need(h, op, B, d0, d1, &need) != MGB_OK) return 0;
    peak = std::max(peak, need.arena + need.splitk);
  }
  return peak;
}

size_t mgb_workspace_held_bytes(mgb_handle* h) {
  if (!h) return 0;
  return h->arena_buf.bytes() + h->splitk_ws.bytes() + h->sync_slab.bytes();
}

}  // extern "C"
