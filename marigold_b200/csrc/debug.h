// Debug entry points of libmarigold_b200.so: exported, but not part of the public header (include/marigold_b200.h).
// Tests and tools reach them through marigold_b200._lib.DEBUG_SIGNATURES, which restates this file for ctypes. The
// files that define them include it, so a definition that drifts from its declaration does not compile.
#pragma once
#include "../../include/marigold_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- api_ops.cu ---- */

/* per-CTA clock64 phase stamps of subsequent GEMM launches */
void mgb_debug_gemm_timing(void* dev_buffer);
/* bytes of device and pinned host memory the library's buffers hold now */
int64_t mgb_debug_live_device_bytes(void);

// GroupNorm in two launches over the concat [a | b] of two packed fp32 maps of Ch channels each, in their own memory as
// the decoder's low-memory resnet runs it: raw = bf16([a | b]) [NB * HW, 2 Ch] over a, y [NB * HW, 2 Ch] over b.
// ws: mgb_op_groupnorm_ws_bytes(NB, HW, 2 Ch, G); stats: NB * 2 Ch float2.
int mgb_debug_groupnorm_halves(float* a, float* b, int32_t Ch, const float* gamma, const float* beta, float* ws,
                               void* stats, int32_t NB, int32_t HW, int32_t G, float eps, int32_t silu, void* stream);

// One band of the decoder's banded 3x3 pad-1 convs (net.cu, conv3x3_band): tile rows [ty0, ty0 + tiles) of one
// H x W image, with the tile the network gives the whole conv over NB_tile such images. x: bf16 [src_rows, W, Cin],
// image rows [src_y0, src_y0 + src_rows); output pixel (y, x) to fp32 row (y - out_y0) W + x at a row stride of ldo,
// columns >= split_col to out_hi (or null: all to out). geom (or null) receives {tile_h, tiles_y}; x == null only
// fills it.
int mgb_debug_conv2d_band(const void* x, int32_t src_y0, int32_t src_rows, const void* w, const float* bias, float* out,
                          float* out_hi, int32_t split_col, int32_t ldo, int32_t out_y0, int32_t NB_tile, int32_t H,
                          int32_t W, int32_t Cin, int32_t Cout, int32_t ty0, int32_t tiles, int32_t* geom, void* stream);

/* ---- api_lpips.cu ---- */

/* copies the fp32 post-ReLU features of AlexNet layer `layer` (0..4) that the last mgb_eval_iid_lpips call on ws left
 * there, [2, h, w, C] (pred, then gt), to dst_dev; dims_out = {h, w, C}. dst_dev NULL: only the dims. A
 * device-to-device copy; nothing is launched. */
int mgb_debug_lpips_features(const void* ws, int32_t H, int32_t W, int32_t layer, float* dst_dev, int32_t dims_out[3]);

/* the same for the tapped layer `layer` (0 .. L - 1) of the handle's net. */
int mgb_debug_lpips_net_features(const mgb_lpips* h, const void* ws, int32_t H, int32_t W, int32_t layer, float* dst_dev,
                                 int32_t dims_out[3]);

/* step `step` of the handle's net (-1: the prep operand). info_out = {op, input step, output buffer's step, column,
 * conv index (-1 for a pool), conv kind, tap (-1: none), h, w, ldo, nsteps}; with dst_dev, copies the bf16 output
 * buffer the step writes into, [2, h, w, ldo] (the prep operand of SqueezeNet: [2, 4, h, w, 64]); MGB_ERR_INVALID when
 * the step writes no bf16 output. */
int mgb_debug_lpips_step(const mgb_lpips* h, const void* ws, int32_t H, int32_t W, int32_t step, void* dst_dev,
                         int32_t info_out[11]);

/* ---- api_net.cu ---- */

// Copies the device array behind one field (find_field's paths) into dst, when dst is not null, and returns its size in
// bytes; *dev_addr receives its device address. It copies memory only: no kernel runs and no handle state changes.
int64_t mgb_debug_read(mgb_handle* h, const char* field, void* dst, int64_t cap_bytes, uint64_t* dev_addr);

// Every device array the weights own (h->weights): addresses and sizes of the first `cap`; returns how many there are.
int32_t mgb_debug_weight_buffers(mgb_handle* h, uint64_t* addr, int64_t* bytes, int32_t cap);

// VAE mid-block attention row blocking of this handle: sets its workspace budget (budget_bytes <= 0: the library's,
// kVaeAttnBudget) and forced rows per block (force_rows <= 0: none), then reports the rows per block (*rows) and the
// blocks over all NB images (*blocks) that an (NB, T)-token attention of the VAE's width runs with.
int mgb_debug_vae_attn_blocks(mgb_handle* h, int64_t budget_bytes, int32_t force_rows, int32_t NB, int32_t T,
                              int32_t* rows, int32_t* blocks);

// The VAE mid-block attention's core (vae_attn_core) alone, as vae_attn_forward runs it: bf16 q, k, v [NB * T, C] ->
// bf16 o, C = the VAE's mid-block width, in this handle's arena and split-K workspace (grown to a dry pass's need) with
// the row blocking mgb_debug_vae_attn_blocks set, on the default stream.
int mgb_debug_vae_attn_core(mgb_handle* h, const void* q, const void* k, const void* v, void* o, int32_t NB, int32_t T);

// Debug switches of this handle's arena: poison != 0 fills every buffer a forward's arena hands out with 0xFF bytes
// (NaN in fp32 and bf16) before the forward uses it; placement is arena_place's placement of the VAE forwards' plans
// (0: the library's, 1: first fit in reverse allocation order). No result may depend on either.
int mgb_debug_arena(mgb_handle* h, int32_t poison, int32_t placement);

// The decoder's full-resolution stage of this handle: mode 1 runs it in low memory (the banded up-conv into two halves
// and the first resnet on them) at every size, -1 never, 0 where the library's rule (decode_low_memory) asks for it.
// Outputs are the same bits either way.
int mgb_debug_vae_low_memory(mgb_handle* h, int32_t mode);

// Tile rows per band of the low-memory decoder's banded up-conv and conv1 on this handle (<= 0: the library's choice,
// about an eighth of the image). Outputs are the same bits at every band height.
int mgb_debug_vae_bands(mgb_handle* h, int32_t up_tiles, int32_t conv1_tiles);

// arena_place on n buffers, a pure host function: sizes and lifetimes [t_alloc, t_free) in, offsets out. Returns the
// peak, or a negative status.
int64_t mgb_debug_arena_place(int64_t n, const int64_t* bytes, const int64_t* t_alloc, const int64_t* t_free,
                              int32_t placement, int64_t* off);

// The arena of one forward at this shape (op 0: UNet step on a d0 x d1 latent, 1: encode of d0 x d1 pixels, 2: decode
// of a d0 x d1 latent), as workspace_need lays it out: per buffer in allocation order its size, lifetime and offset,
// for the first `cap` buffers. Returns the buffer count, or a negative status.
int64_t mgb_debug_arena_plan(mgb_handle* h, int32_t op, int32_t B, int32_t d0, int32_t d1, int64_t* bytes,
                             int64_t* t_alloc, int64_t* t_free, int64_t* off, int64_t cap);

#ifdef __cplusplus
}
#endif
