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

// One activation buffer of a forward: its size, its lifetime [t_alloc, t_free) in events (allocations and frees,
// counted from the forward's start) and its offset in the arena: the bump offset while a dry run records it, the
// planned one once arena_place has placed it.
struct ArenaBuf {
  size_t bytes = 0, off = 0;
  int64_t t_alloc = 0, t_free = 0;
};

// Gives each buffer a 1024-aligned offset such that no two buffers whose lifetimes overlap share a byte; returns the
// peak (the largest off + bytes). Placement 0 places first fit in allocation order, which puts a stack-shaped sequence
// exactly where the bump allocator does, or first fit largest first where that needs less memory. Placement 1 places
// first fit in reverse allocation order (tests: results must not depend on where buffers are).
size_t arena_place(std::vector<ArenaBuf>& bufs, int placement);

// Activation memory of one forward. Without a plan it is a bump allocator: mark / release give back everything
// allocated since the mark, and free() gives back nothing. A dry run records every allocation's size and lifetime
// (release() and free() end lifetimes); a real run given that dry run's placed records (`plan`) hands out the planned
// offsets, so a buffer holds its bytes only from its allocation to its free.
struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0, peak = 0;
  bool dry = false;
  int status = MGB_OK;   // MGB_ERR_NOMEM past cap, MGB_ERR_STATE when a real run leaves its plan
  std::vector<ArenaBuf> rec;                  // dry run: every allocation so far
  std::vector<size_t> live;                   // dry run: indices into rec not yet freed
  int64_t events = 0;
  const std::vector<ArenaBuf>* plan = nullptr;
  size_t n = 0;                               // allocations so far
  void start();                               // begins one forward
  void* alloc(size_t bytes);
  void free(const void* p);
  void finish();                              // dry run: ends the lifetimes still open
  size_t mark() const { return off; }
  void release(size_t m);
};

// A trunk activation: fp32 [M, C]
struct Act {
  float* p = nullptr;
  int C = 0;
};

// Largest image batch one encode / decode call accepts: NB * H * W output pixels (e.g. one 8192 x 8192 image, or
// one 12 MP photo and four more). Below it every 32-bit count of the VAE graph (pixels, GEMM rows, per-row sizes,
// grid dimensions) stays in range; element counts and offsets are 64-bit.
constexpr size_t kMaxPixels = size_t(1) << 26;

// Workspace target of the VAE mid-block attention's score rows: fp32 S + bf16 P, 6 bytes per logit. An image whose
// whole T x Tp score matrix fits runs as one block (every size up to 1024 x 1024 does); above it the query rows are
// processed in blocks (vae_attn_rows).
constexpr size_t kVaeAttnBudget = size_t(2) << 30;

// Query rows per block of the VAE mid-block attention over T tokens of width C: T when T * Tp * 6 bytes fit `budget`;
// else the largest multiple of 128 that fits, raised where needed so that each block's P V GEMM still fills one wave
// of the SMs. force_rows > 0 overrides the choice (tests).
int vae_attn_rows(int T, int C, size_t budget, int force_rows);

// A handle's settings of its forwards: the library's defaults unless a debug hook (debug.h) sets them. Each forward's
// Ctx holds a copy.
struct ForwardOptions {
  // VAE mid-block attention row blocking: vae_attn_rows' budget and forced rows (mgb_debug_vae_attn_blocks)
  size_t attn_budget = kVaeAttnBudget;
  int attn_rows = 0;
  // fill every buffer the arena hands out with 0xFF bytes (NaN in fp32 and bf16) first; arena_place's placement of the
  // VAE forwards' plans (mgb_debug_arena)
  bool poison = false;
  int placement = 0;
  // The decoder's full-resolution stage in low memory (Ctx::dec_low_memory): 0 where one member's default decode does
  // not fit the device beside the weights (decode_low_memory, api_net.cu), 1 always, -1 never (mgb_debug_vae_low_memory)
  int low_memory = 0;
  // Tile rows per band of the low-memory decoder's banded up-conv and conv1: 0 the library's choice, else forced
  // (mgb_debug_vae_bands)
  int band_up_tiles = 0, band_conv1_tiles = 0;
};

struct Ctx {
  cudaStream_t stream = nullptr;
  Arena* arena = nullptr;
  bool dry = false;
  ForwardOptions opt;      // the handle's
  bool planned = false;    // the arena is lifetime-planned (the VAE forwards): buffers are freed after their last read
  bool dec_low_memory = false;   // the decoder's full-resolution 256-channel stage runs in 2.5 U (net.cu)
  float* splitk_ws = nullptr;
  size_t splitk_cap = 0;   // bytes available
  size_t splitk_need = 0;  // bytes needed (dry run)
  int groups = 32;
  const float* cur_bias = nullptr;  // current step's concatenated resnet conv1 biases (device)
  // grid-barrier counters of the GroupNorm launches of one forward (one per image and launch; zeroed once per forward)
  unsigned* sync_base = nullptr;
  size_t sync_off = 0, sync_cap = 0, sync_need = 0;
  // row split (mgb_set_row_split): split_world > 0 runs this rank's share of every attention's query rows, then
  // exchange(); 0 runs them whole
  int split_rank = 0, split_world = 0;
  mgb_exchange_fn exchange_fn = nullptr;
  void* exchange_ctx = nullptr;
};

// Query rows per rank of a T-row attention split over `world` ranks: whole 128-row blocks, ceil(ceil(T / 128) / world)
// of them. Rank r owns rows [r chunk, (r + 1) chunk) within [0, T).
inline int row_split_chunk(int T, int world) { return ((T + 127) / 128 + world - 1) / world * 128; }

// The VAE mid-block attention between its projections: o = softmax(q k^T / sqrt(C)) v per image, on bf16 q, k, v, o
// [NB * T, C], in blocks of vae_attn_rows(T, C, c.opt.attn_budget, c.opt.attn_rows) query rows. Its scratch (V^T, one block's
// fp32 scores and bf16 probabilities) comes from the arena and is released on return.
// Query rows [row_begin, row_end) only (row_end < 0: through T), in the blocks and tiles of the whole T-row problem,
// so each row is bit-identical to the whole call's; row_begin a multiple of 128 (or of the block rows).
int vae_attn_core(Ctx& c, const bf16* q, const bf16* k, const bf16* v, bf16* o, int NB, int T, int C,
                  int row_begin = 0, int row_end = -1);

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
  mgb::ForwardOptions opt;
  // The VAE forwards' arena plan: placed by the dry run that sizes each call's workspace, replayed by its real run.
  std::vector<mgb::ArenaBuf> arena_plan;
  size_t device_bytes = 0;          // the device's memory, read once
  struct DecodeRule {                // the rule's last decision (decode_low_memory)
    bool valid = false;
    int lh = 0, lw = 0;
    size_t attn_budget = 0;
    int attn_rows = 0;
    bool low_memory = false;
  } decode_rule;
  // row split (mgb_set_row_split): installed while fn != null
  struct RowSplit {
    int rank = 0, world = 0;
    mgb_exchange_fn fn = nullptr;
    void* ctx = nullptr;
  } row_split;
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
