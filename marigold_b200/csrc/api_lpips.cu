// C ABI of the LPIPS evaluation: the weight handle (the AlexNet, VGG16 or SqueezeNet 1.1 features + the lin heads) and the
// IID evaluation with LPIPS (lpips.cu after eval.cu's IID passes, one synchronisation).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "debug.h"
#include "device.h"
#include "kernels.h"

using namespace mgb;

struct mgb_lpips {
  const LpNet* net;
  DevBuf<bf16> w[kLpMaxConvs];
  DevBuf<float> b[kLpMaxConvs];
  DevBuf<float> lin;
};

namespace {

int upload(DevBuf<bf16>& dst, const std::vector<bf16>& src) {
  TRY(dst.grow(src.size() * sizeof(bf16)));
  CUDA_TRY(cudaMemcpy(dst.get(), src.data(), src.size() * sizeof(bf16), cudaMemcpyHostToDevice));
  return MGB_OK;
}
int upload(DevBuf<float>& dst, const std::vector<float>& src) {
  TRY(dst.grow(src.size() * sizeof(float)));
  CUDA_TRY(cudaMemcpy(dst.get(), src.data(), src.size() * sizeof(float), cudaMemcpyHostToDevice));
  return MGB_OK;
}

// Conv weight [cout, cin, k, k] as the bf16 implicit-GEMM operand [n, taps * cin_pad], tap-major, zero in the padded
// rows (a Fire squeeze's n = 64 > cout) and channels (cin < cin_pad). AlexNet's conv1: the 3 x 3 block taps (kb_h, kb_w)
// over 64 block channels, w[o, c, 4 kb_h + rh, 4 kb_w + rw] at s2d_channel(rh, rw, c), zero where the 12 x 12 block
// window overhangs the 11 x 11 kernel and in channels 48..63.
std::vector<bf16> repack(const LpNet& net, int ci_index, const float* w) {
  const LpConv& c = net.conv[ci_index];
  const int co = c.cout, ci = c.cin, k = c.k;
  if (net.prep == LP_PREP_S2D4 && ci_index == 0) {
    std::vector<bf16> out(size_t(co) * 9 * kLpipsS2dC, __float2bfloat16(0.f));
    for (int o = 0; o < co; ++o)
      for (int t = 0; t < 9; ++t)
        for (int rh = 0; rh < 4; ++rh)
          for (int rw = 0; rw < 4; ++rw) {
            const int kh = 4 * (t / 3) + rh, kw = 4 * (t % 3) + rw;
            if (kh >= k || kw >= k) continue;
            for (int ch = 0; ch < ci; ++ch)
              out[(size_t(o) * 9 + t) * kLpipsS2dC + s2d_channel(rh, rw, ch)] =
                  __float2bfloat16(w[((size_t(o) * ci + ch) * k + kh) * k + kw]);
          }
    return out;
  }
  const int taps = k * k;
  std::vector<bf16> out(size_t(c.n) * taps * c.cin_pad, __float2bfloat16(0.f));
  for (int o = 0; o < co; ++o)
    for (int t = 0; t < taps; ++t)
      for (int ch = 0; ch < ci; ++ch)
        out[(size_t(o) * taps + t) * c.cin_pad + ch] = __float2bfloat16(w[(size_t(o) * ci + ch) * taps + t]);
  return out;
}

size_t iid_part(int H, int W) { return (eval_iid_ws_bytes(H, W) + 255) & ~size_t(255); }

}  // namespace

extern "C" {

int mgb_lpips_create_net(int32_t net_type, int32_t n_conv, const float* const* conv_w, const int32_t* conv_w_shape,
                         const float* const* conv_b, int32_t n_lin, const float* const* lin_w, const int32_t* lin_channels,
                         mgb_lpips** out) {
  if (!conv_w || !conv_w_shape || !conv_b || !lin_w || !lin_channels || !out) {
    set_error("mgb_lpips_create_net: null argument");
    return MGB_ERR_INVALID;
  }
  *out = nullptr;
  const LpNet* net = lpips_net(net_type);
  if (!net) {
    set_error("mgb_lpips_create_net: unknown net type %d", net_type);
    return MGB_ERR_INVALID;
  }
  if (n_conv != net->nconv || n_lin != net->L) {
    set_error("mgb_lpips_create_net: %s has %d convolutions and %d lin layers, got %d and %d", net->name, net->nconv,
              net->L, n_conv, n_lin);
    return MGB_ERR_INVALID;
  }
  for (int i = 0; i < n_conv; ++i) {
    const int32_t* s = conv_w_shape + 4 * i;
    const LpConv& c = net->conv[i];
    if (s[0] != c.cout || s[1] != c.cin || s[2] != c.k || s[3] != c.k) {
      set_error("mgb_lpips_create_net: conv %d: weight [%d, %d, %d, %d], expected [%d, %d, %d, %d] (torchvision %s)", i,
                s[0], s[1], s[2], s[3], c.cout, c.cin, c.k, c.k, net->name);
      return MGB_ERR_INVALID;
    }
    if (!conv_w[i] || !conv_b[i]) {
      set_error("mgb_lpips_create_net: conv %d: null weight", i);
      return MGB_ERR_INVALID;
    }
  }
  for (int l = 0; l < n_lin; ++l) {
    if (lin_channels[l] != net->C[l] || !lin_w[l]) {
      set_error("mgb_lpips_create_net: lin %d: %d channels, expected %d (%s)", l, lin_channels[l], net->C[l], net->name);
      return MGB_ERR_INVALID;
    }
  }
  mgb_lpips* h = new mgb_lpips();
  h->net = net;
  std::vector<float> lin;
  int rc = MGB_OK;
  for (int i = 0; i < n_conv && rc == MGB_OK; ++i) {
    const LpConv& c = net->conv[i];
    rc = upload(h->w[i], repack(*net, i, conv_w[i]));
    std::vector<float> bias(conv_b[i], conv_b[i] + c.cout);
    bias.resize(c.n, 0.f);                        // a Fire squeeze's padded columns: ReLU(0 + 0) = 0
    if (rc == MGB_OK) rc = upload(h->b[i], bias);
  }
  for (int l = 0; l < n_lin; ++l) lin.insert(lin.end(), lin_w[l], lin_w[l] + net->C[l]);
  if (rc == MGB_OK) rc = upload(h->lin, lin);
  if (rc != MGB_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return MGB_OK;
}

int mgb_lpips_create(const float* const conv_w[5], const int32_t conv_w_shape[5][4], const float* const conv_b[5],
                     const float* const lin_w[5], const int32_t lin_channels[5], mgb_lpips** out) {
  if (!conv_w_shape) {
    set_error("mgb_lpips_create: null argument");
    return MGB_ERR_INVALID;
  }
  return mgb_lpips_create_net(MGB_LPIPS_ALEX, kLpipsLayers, conv_w, &conv_w_shape[0][0], conv_b, kLpipsLayers, lin_w,
                              lin_channels, out);
}

void mgb_lpips_destroy(mgb_lpips* h) { delete h; }

int32_t mgb_lpips_min_size(int32_t net_type) {
  const LpNet* net = lpips_net(net_type);
  return net ? net->min_size : 0;
}

size_t mgb_lpips_ws_bytes_h(const mgb_lpips* h, int32_t H, int32_t W) {
  if (!h || H < h->net->min_size || W < h->net->min_size) return 0;
  return iid_part(H, W) + lpips_ws_bytes(*h->net, H, W);
}

size_t mgb_lpips_ws_bytes(int32_t H, int32_t W) {
  const LpNet& alex = *lpips_net(MGB_LPIPS_ALEX);
  return H >= alex.min_size && W >= alex.min_size ? iid_part(H, W) + lpips_ws_bytes(alex, H, W) : 0;
}

int mgb_eval_iid_lpips(const float* pred, const float* gt, const uint8_t* mask, int32_t H, int32_t W, int32_t up_to_scale,
                       int32_t transform, const mgb_lpips* lp, void* ws, double* out_host, void* stream) {
  const int min_size = lp ? lp->net->min_size : kLpipsMinSize;
  if (!pred || !gt || !ws || !out_host || !lp || H < min_size || W < min_size || transform < 0 || transform > 2) {
    set_error("mgb_eval_iid_lpips: bad argument (H=%d W=%d transform=%d; H and W must be >= %d)", H, W, transform,
              min_size);
    return MGB_ERR_INVALID;
  }
  const LpNet& net = *lp->net;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  char* lws = static_cast<char*>(ws) + iid_part(H, W);
  TRY(launch_eval_iid(pred, gt, mask, H, W, up_to_scale != 0, transform, ws, s));
  LpipsWeights wts;
  for (int i = 0; i < net.nconv; ++i) { wts.w[i] = lp->w[i]; wts.b[i] = lp->b[i]; }
  wts.lin = lp->lin;
  TRY(launch_lpips(net, pred, gt, mask, H, W, transform, up_to_scale ? eval_iid_sk(ws, H, W) : nullptr, wts, lws, s));
  double res[7], lres[6];
  cudaError_t e = cudaMemcpyAsync(res, eval_iid_out(ws, H, W), sizeof(res), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(lres, lpips_out(net, lws, H, W), sizeof(lres), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) { set_error("mgb_eval_iid_lpips: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  if (up_to_scale && res[6] == 0.0) {
    set_error("mgb_eval_iid_lpips: no pixel is valid in channel 0 of the mask, so the brightness quantile is undefined");
    return MGB_ERR_INVALID;
  }
  if (lres[1] != 0.0) {      // torchmetrics' _lpips_update with normalize=True
    set_error("Expected both input arguments to be normalized tensors with shape [N, 3, H, W]. Got input with shape "
              "torch.Size([1, 3, %d, %d]) and torch.Size([1, 3, %d, %d]) and values in range [%.4f, %.4f] and "
              "[%.4f, %.4f] when all values are expected to be in the [0, 1] range.",
              H, W, H, W, lres[2], lres[3], lres[4], lres[5]);
    return MGB_ERR_INVALID;
  }
  for (int i = 0; i < 6; ++i) out_host[i] = res[i];
  out_host[6] = lres[0];
  return MGB_OK;
}

/* debug hooks (declared in debug.h) */
int mgb_debug_lpips_features(const void* ws, int32_t H, int32_t W, int32_t layer, float* dst_dev, int32_t dims_out[3]) {
  if (!ws || !dims_out || layer < 0 || layer >= kLpipsLayers || H < kLpipsMinSize || W < kLpipsMinSize) {
    set_error("mgb_debug_lpips_features: bad argument");
    return MGB_ERR_INVALID;
  }
  int d[3];
  const float* f = lpips_features(*lpips_net(MGB_LPIPS_ALEX), static_cast<const char*>(ws) + iid_part(H, W), H, W, layer, d);
  for (int i = 0; i < 3; ++i) dims_out[i] = d[i];
  if (dst_dev) CUDA_TRY(cudaMemcpy(dst_dev, f, size_t(2) * d[0] * d[1] * d[2] * sizeof(float), cudaMemcpyDeviceToDevice));
  return MGB_OK;
}

int mgb_debug_lpips_net_features(const mgb_lpips* h, const void* ws, int32_t H, int32_t W, int32_t layer, float* dst_dev,
                                 int32_t dims_out[3]) {
  if (!h || !ws || !dims_out || layer < 0 || layer >= h->net->L || H < h->net->min_size || W < h->net->min_size) {
    set_error("mgb_debug_lpips_net_features: bad argument");
    return MGB_ERR_INVALID;
  }
  int d[3];
  const float* f = lpips_features(*h->net, static_cast<const char*>(ws) + iid_part(H, W), H, W, layer, d);
  for (int i = 0; i < 3; ++i) dims_out[i] = d[i];
  if (dst_dev) CUDA_TRY(cudaMemcpy(dst_dev, f, size_t(2) * d[0] * d[1] * d[2] * sizeof(float), cudaMemcpyDeviceToDevice));
  return MGB_OK;
}

int mgb_debug_lpips_step(const mgb_lpips* h, const void* ws, int32_t H, int32_t W, int32_t step, void* dst_dev,
                         int32_t info_out[11]) {
  if (!h || !ws || !info_out || step < -1 || step >= h->net->nsteps || H < h->net->min_size || W < h->net->min_size) {
    set_error("mgb_debug_lpips_step: bad argument");
    return MGB_ERR_INVALID;
  }
  const LpNet& n = *h->net;
  int d[3];
  const bf16* x = lpips_step_output(n, static_cast<const char*>(ws) + iid_part(H, W), H, W, step, d);
  const LpStep st = step < 0 ? LpStep{-1, -1, -1, 0, 64, -1, -1, -1, true} : n.step[step];
  const int32_t info[11] = {st.op, st.in, st.buf, st.col, st.conv, st.kind, st.tap, d[0], d[1], d[2], n.nsteps};
  for (int i = 0; i < 11; ++i) info_out[i] = info[i];
  if (!dst_dev) return MGB_OK;
  if (!x) {
    set_error("mgb_debug_lpips_step: step %d writes no bf16 output", step);
    return MGB_ERR_INVALID;
  }
  const size_t planes = step < 0 && n.prep == LP_PREP_PARITY ? 4 : 1;
  CUDA_TRY(cudaMemcpy(dst_dev, x, size_t(2) * planes * d[0] * d[1] * d[2] * sizeof(bf16), cudaMemcpyDeviceToDevice));
  return MGB_OK;
}

}  // extern "C"
