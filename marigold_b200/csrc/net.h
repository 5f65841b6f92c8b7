// Network composition for the Marigold hot path: weights, activation arena, and the forward graphs of
// the SD-2 UNet step and the SD VAE encoder / decoder, expressed as sequences of the kernels in
// kernels.h. Host-side C++ only; no torch.
#pragma once
#include <map>
#include <string>
#include <unordered_set>
#include <vector>

#include "device.h"
#include "kernels.h"
#include "ops.h"

namespace mgb {

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> shape;
  size_t numel() const { return data.size(); }
};

// ---- device-side weights ------------------------------------------------------------------------
struct ConvW {   // 3x3 conv, tap-major bf16 [cout, 9 * cin_pad (+ k_extra)]
  bf16* w = nullptr;
  float* b = nullptr;
  int cin = 0, cin_pad = 0, cout = 0;
  int k_extra = 0;   // columns of a 1x1 convolution over a second operand appended after the taps (conv2 + conv_shortcut)
};
struct LinW {    // bf16 [n, k]
  bf16* w = nullptr;
  float* b = nullptr;
  int n = 0, k = 0;
  bool geglu = false;
};
struct NormW {
  float* g = nullptr;
  float* b = nullptr;
  int c = 0;
};
struct ResnetW {
  NormW n1, n2;
  ConvW c1, c2;
  bool has_sc = false;
  int cin = 0, cout = 0;
  // time embedding projection (UNet only): fp32 [cout, temb_dim]; bias already includes conv1.bias
  float* temb_w = nullptr;
  float* temb_b = nullptr;
  int bias_off = -1;           // offset of this resnet's row in the per-step bias table (UNet only)
  float eps = 1e-5f;
};
struct XfmrW {
  int C = 0;
  NormW gn, ln1, ln2, ln3;
  LinW proj_in, qkv, o1, ff1;
  LinW ffpo;             // ff.net.2 folded with proj_out: bf16 [C, C + 4C] = [W_po | W_po W_ff2], bias b_po + W_po b_ff2
  // cross attention (attn2): fp32 masters, folded against the empty-prompt context at set_text_embedding
  float* q2w = nullptr;  // to_q   fp32 [C, C]
  float* o2w = nullptr;  // to_out fp32 [C, C]
  float* o2b = nullptr;  // to_out bias [C]
  float* k2w = nullptr;  // to_k   fp32 [C, ctx]
  float* v2w = nullptr;  // to_v
  float* kv = nullptr;   // fp32 [2 (k|v), n_ctx, C]
  bf16* xGU = nullptr;   // [2][H, C]  G_h = Wq[h-block]^T (k0 - k1)_h ; U_h = Wo[:, h-block] (v0 - v1)_h
  float* xc1 = nullptr;  // [C]        Wo v1 + bo
};
struct VaeAttnW {
  int C = 0;
  NormW gn;
  LinW q, k, v, o;
};

struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0, peak = 0;
  bool dry = false;
  bool overflow = false;
  void* alloc(size_t bytes);
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
};

// A trunk activation: fp32 [M, C]
struct Act {
  float* p = nullptr;
  int C = 0;
};

struct Ctx {
  cudaStream_t stream = nullptr;
  Arena* arena = nullptr;
  bool dry = false;
  float* splitk_ws = nullptr;
  size_t splitk_cap = 0;   // bytes available
  size_t splitk_need = 0;  // bytes needed (dry run)
  int groups = 32;
  const float* cur_bias = nullptr;  // current step's concatenated resnet conv1 biases (device)
  // grid-barrier counters of the GroupNorm launches of one forward (one per image and launch; zeroed once per forward)
  unsigned* sync_base = nullptr;
  size_t sync_off = 0, sync_cap = 0, sync_need = 0;
};

struct UNetW {
  ConvW conv_in, conv_out;
  NormW norm_out;
  float *te_w1 = nullptr, *te_b1 = nullptr, *te_w2 = nullptr, *te_b2 = nullptr;
  int temb_dim = 0;
  std::vector<ResnetW> resnets;   // execution order
  std::vector<XfmrW> xfmrs;       // execution order
  std::vector<ConvW> downs, ups;
};
struct VaeW {
  // encoder
  ConvW enc_in, enc_out;          // enc_out has quant_conv folded in, mean half only
  NormW enc_norm_out;
  std::vector<ResnetW> enc_res;   // execution order (down blocks then mid 0, mid 1)
  std::vector<ConvW> enc_down;
  VaeAttnW enc_attn;
  // decoder
  float* pq_w = nullptr;          // post_quant_conv fp32 [4,4]
  float* pq_b = nullptr;
  ConvW dec_in, dec_out;
  NormW dec_norm_out;
  std::vector<ResnetW> dec_res;   // mid 0, mid 1, then up blocks
  std::vector<ConvW> dec_up;
  VaeAttnW dec_attn;
};

}  // namespace mgb

struct mgb_handle {
  mgb_config cfg;
  std::map<std::string, mgb::HostTensor> host;  // until finalize
  bool finalized = false;
  std::vector<mgb::DevBuf<void>> weights;  // every device array the UNetW / VaeW raw pointers point into
  mgb::UNetW unet;
  mgb::VaeW vae;
  mgb::DevBuf<char> arena_buf;
  mgb::Arena arena;                 // view of arena_buf, refreshed by each call that runs a graph
  mgb::DevBuf<float> splitk_ws;
  mgb::DevBuf<unsigned> sync_slab;  // GroupNorm grid-barrier counters of one forward
  // conditioning / schedule
  bool text_set = false;
  int n_steps = 0;
  mgb::DevBuf<float> sched_k;       // device [n_steps, 3]
  std::vector<float> kz_host;
  // per-step tables selected on the device (so one CUDA graph serves every step)
  mgb::DevBuf<float> bias_table;    // device [n_steps, bias_total]
  int bias_total = 0;
  mgb::DevBuf<float> cur_bias;      // device [bias_total]
  mgb::DevBuf<float> cur_sched_k;   // device [3]
  mgb::DevBuf<int> step_counter;    // device
  // ensemble scratch
  mgb::DevBuf<float> ens_ws;
  mgb::PinnedBuf<double> ens_pinned;  // pinned host staging (api_ens.cu)
  mgb::DevBuf<float> ens_v3;          // per-pixel order statistics for the forward-difference objective
  // Cached CUDA graph of one UNet step. It is keyed by (NB, lh, lw) alone: whatever replaces a buffer whose address
  // the graph captured (arena, split-K workspace, sync slab, sched_k, bias_table) calls invalidate_step_graph first.
  // Declared after the buffers so that it is destroyed before them.
  struct StepGraph {
    mgb::GraphExec exec;
    int NB = 0, lh = 0, lw = 0;
    long long launches = 0;
    bool exec_failed = false;
  } step_graph;
  mgb::Stream capture_stream;
};
