// C ABI: error plumbing + operator-level entry points (layer parity tests call these).
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "debug.h"
#include "device.h"
#include "kernels.h"
#include "launch.h"
#include "ops.h"

namespace mgb {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }
}  // namespace mgb

using namespace mgb;

extern "C" {

const char* mgb_last_error(void) { return get_error(); }
const char* mgb_build_info(void) {
  return "libmarigold_b200 sm_90a: wgmma.mma_async bf16 (fp32 register accumulators), cp.async.bulk.tensor (TMA) "
         "SWIZZLE_128B, mbarrier pipelines; no CPU fallback";
}
int64_t mgb_launch_count(void) { return launch_count(); }
/* debug hooks (declared in debug.h) */
void mgb_debug_gemm_timing(void* dev_buffer) { set_gemm_debug_buffer(reinterpret_cast<long long*>(dev_buffer)); }
int64_t mgb_debug_live_device_bytes(void) { return g_live_bytes.load(); }

static void fill_epi(GemmEpilogue* e, const float* bias, const float* residual, float* out_f32, void* out_bf16,
                     int ldo, int flags, float scale, const float* sched_x, const float* sched_z, const float* sched_k,
                     float* aux_out) {
  memset(e, 0, sizeof(*e));
  e->bias = bias; e->residual = residual; e->out_f32 = out_f32;
  e->out_bf16 = reinterpret_cast<bf16*>(out_bf16);
  e->ldo = ldo; e->flags = flags; e->scale = scale;
  e->sched_x = sched_x; e->sched_z = sched_z; e->sched_k = sched_k; e->aux_out = aux_out;
}

int mgb_op_linear_ex(const void* a, const void* a2, const void* w, const float* bias, const float* residual,
                     float* out_f32, void* out_bf16, int32_t M, int32_t N, int32_t K, int32_t K2, int32_t ldo,
                     int32_t flags, float scale, const float* sched_x, const float* sched_z, const float* sched_k,
                     float* aux_out, int32_t block_n, int32_t splits, int32_t stages, float* splitk_ws, void* stream) {
  if (!a || !w || (!out_f32 && !out_bf16) || (a2 && K2 <= 0)) { set_error("op_linear: null pointer or K2"); return MGB_ERR_INVALID; }
  if (!a2) K2 = 0;
  const int n_out = (flags & EPI_GEGLU) ? N / 2 : N;
  if (ldo <= 0) ldo = n_out;
  if (ldo < n_out) { set_error("op_linear: ldo %d < %d output columns", ldo, n_out); return MGB_ERR_INVALID; }
  if (block_n <= 0) {
    int bn, sp, st;
    choose_tile((M + 127) / 128, N, (K + K2) / 64, flags, splitk_ws != nullptr && !(flags & EPI_GEGLU), &bn, &sp, &st);
    block_n = bn; if (splits <= 0) splits = sp; if (stages <= 0) stages = st;
  }
  if (splits <= 0) splits = 1;
  if (stages <= 0) stages = 4;
  GemmParams p;
  int rc = fill_linear_params(&p, reinterpret_cast<const bf16*>(a), reinterpret_cast<const bf16*>(w), M, N, K, block_n,
                              splits, stages, reinterpret_cast<const bf16*>(a2), K2);
  if (rc) return rc;
  fill_epi(&p.epi, bias, residual, out_f32, out_bf16, ldo, flags, scale, sched_x, sched_z, sched_k, aux_out);
  return run_gemm(p, block_n, splitk_ws, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_linear(const void* a, const void* w, const float* bias, const float* residual, float* out_f32,
                  void* out_bf16, int32_t M, int32_t N, int32_t K, int32_t flags, int32_t block_n, int32_t splits,
                  int32_t stages, float* splitk_ws, void* stream) {
  return mgb_op_linear_ex(a, nullptr, w, bias, residual, out_f32, out_bf16, M, N, K, 0, 0, flags, 1.0f, nullptr, nullptr,
                          nullptr, nullptr, block_n, splits, stages, splitk_ws, stream);
}

int mgb_op_conv2d_ex(const void* x, const void* x2, const void* w, const float* bias, const float* residual,
                     float* out_f32, void* out_bf16, int32_t NB, int32_t Hout, int32_t Wout, int32_t Cin, int32_t Cin2,
                     int32_t Cout, int32_t kind, int32_t Hsrc, int32_t Wsrc, int32_t flags, float scale,
                     const float* sched_x, const float* sched_z, const float* sched_k, float* aux_out, int32_t block_n,
                     int32_t splits, int32_t stages, float* splitk_ws, void* stream) {
  if (!x || !w || (!out_f32 && !out_bf16) || (x2 && Cin2 <= 0)) { set_error("op_conv2d: null pointer or Cin2"); return MGB_ERR_INVALID; }
  if (!x2) Cin2 = 0;
  const int taps = kind == 1 ? 1 : kind == 5 ? 25 : 9;
  if (block_n <= 0) {
    int tw, th;
    conv_tile_shape(Hout, Wout, &tw, &th);
    const int m_tiles = NB * ((Wout + tw - 1) / tw) * ((Hout + th - 1) / th);
    int bn, sp, st;
    choose_tile(m_tiles, Cout, (taps * Cin + Cin2) / 64, flags, splitk_ws != nullptr, &bn, &sp, &st);
    block_n = bn; if (splits <= 0) splits = sp; if (stages <= 0) stages = st;
  }
  if (splits <= 0) splits = 1;
  if (stages <= 0) stages = 4;
  GemmParams p;
  int rc = fill_conv_params(&p, reinterpret_cast<const bf16*>(x), reinterpret_cast<const bf16*>(w), NB, Hout, Wout,
                            Cin, Cout, kind, block_n, splits, stages, Hsrc, Wsrc, reinterpret_cast<const bf16*>(x2), Cin2);
  if (rc) return rc;
  fill_epi(&p.epi, bias, residual, out_f32, out_bf16, Cout, flags, scale, sched_x, sched_z, sched_k, aux_out);
  p.epi.hw = Hout * Wout;
  return run_gemm(p, block_n, splitk_ws, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_conv2d(const void* x, const void* w, const float* bias, const float* residual, float* out_f32,
                  void* out_bf16, int32_t NB, int32_t Hout, int32_t Wout, int32_t Cin, int32_t Cout, int32_t kind,
                  int32_t flags, int32_t block_n, int32_t splits, int32_t stages, float* splitk_ws, void* stream) {
  return mgb_op_conv2d_ex(x, nullptr, w, bias, residual, out_f32, out_bf16, NB, Hout, Wout, Cin, 0, Cout, kind, 0, 0, flags,
                          1.0f, nullptr, nullptr, nullptr, nullptr, block_n, splits, stages, splitk_ws, stream);
}

int mgb_op_flash_attn64_ex(const void* qkv, void* out, int32_t NB, int32_t T, int32_t C, float scale,
                           int32_t q_block_begin, int32_t q_block_end, void* stream) {
  if (q_block_end < 0) { set_error("op_flash_attn64_ex: q_block_end %d < 0", q_block_end); return MGB_ERR_INVALID; }
  // split-KV workspace of the operator-level entry point: a process-wide buffer grown on demand (the network
  // path carves it out of its arena instead). Never destroyed, so it is not freed during static destruction,
  // after the CUDA runtime may have unloaded.
  static DevBuf<float>& ws = *new DevBuf<float>();
  const size_t need = flash_attn64_ws_bytes(NB, T, C);
  if (need > ws.bytes()) {
    cudaDeviceSynchronize();
    if (int rc = ws.grow(need)) return rc;
  }
  return launch_flash_attn64(reinterpret_cast<const bf16*>(qkv), reinterpret_cast<bf16*>(out), NB, T, C, scale,
                             need ? ws.get() : nullptr, need ? ws.bytes() : 0, reinterpret_cast<cudaStream_t>(stream),
                             q_block_begin, q_block_end);
}

int mgb_op_flash_attn64(const void* qkv, void* out, int32_t NB, int32_t T, int32_t C, float scale, void* stream) {
  return mgb_op_flash_attn64_ex(qkv, out, NB, T, C, scale, 0, T > 0 ? (T + 127) / 128 : 0, stream);
}

size_t mgb_op_groupnorm_ws_bytes(int32_t NB, int32_t HW, int32_t C, int32_t G) { return groupnorm_ws_bytes(NB, HW, C, G); }

int mgb_op_groupnorm(const float* x, void* y, const float* gamma, const float* beta, float* ws, int32_t NB, int32_t HW,
                     int32_t C, int32_t G, float eps, int32_t silu, void* stream) {
  return launch_groupnorm(x, reinterpret_cast<bf16*>(y), nullptr, gamma, beta, ws, NB, HW, C, G, eps, silu,
                          reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_groupnorm_ex(const float* xa, int32_t Ca, const float* xb, int32_t Cb, void* y, void* raw_copy,
                        const float* gamma, const float* beta, float* ws, int32_t NB, int32_t HW, int32_t G, float eps,
                        int32_t silu, void* stream) {
  if (!xa || !y || !ws || (xb == nullptr) != (Cb == 0)) { set_error("op_groupnorm_ex: null pointer or Cb"); return MGB_ERR_INVALID; }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const size_t pb = (groupnorm_part_bytes(NB, HW, Ca + Cb, G) + 255) & ~size_t(255);
  unsigned* counters = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(ws) + pb);
  if (cudaMemsetAsync(counters, 0, size_t(NB) * sizeof(unsigned), s) != cudaSuccess) {
    set_error("op_groupnorm_ex: counter memset failed");
    return MGB_ERR_CUDA;
  }
  return launch_gn_fused(xa, Ca, xb, Cb, reinterpret_cast<bf16*>(y), reinterpret_cast<bf16*>(raw_copy), gamma, beta, NB, HW,
                         G, eps, silu, ws, counters, s);
}

// debug hook (debug.h)
int mgb_debug_groupnorm_halves(float* a, float* b, int32_t Ch, const float* gamma, const float* beta, float* ws,
                               void* stats, int32_t NB, int32_t HW, int32_t G, float eps, int32_t silu, void* stream) {
  if (!a || !b || !ws || !stats || Ch <= 0) { set_error("debug_groupnorm_halves: bad argument"); return MGB_ERR_INVALID; }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const size_t pb = (groupnorm_part_bytes(NB, HW, 2 * Ch, G) + 255) & ~size_t(255);
  unsigned* counters = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(ws) + pb);
  if (cudaMemsetAsync(counters, 0, size_t(NB) * sizeof(unsigned), s) != cudaSuccess) {
    set_error("debug_groupnorm_halves: counter memset failed");
    return MGB_ERR_CUDA;
  }
  float2* st = reinterpret_cast<float2*>(stats);
  TRY(launch_gn_stats(a, Ch, b, Ch, st, gamma, beta, NB, HW, G, eps, ws, counters, s));
  return launch_gn_apply_rows(a, b, Ch, st, reinterpret_cast<bf16*>(b), reinterpret_cast<bf16*>(a), NB, HW, 2 * Ch, silu,
                              s);
}

// debug hook (debug.h)
int mgb_debug_conv2d_band(const void* x, int32_t src_y0, int32_t src_rows, const void* w, const float* bias, float* out,
                          float* out_hi, int32_t split_col, int32_t ldo, int32_t out_y0, int32_t NB_tile, int32_t H,
                          int32_t W, int32_t Cin, int32_t Cout, int32_t ty0, int32_t tiles, int32_t* geom, void* stream) {
  if (NB_tile <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) { set_error("debug_conv2d_band: bad argument"); return MGB_ERR_INVALID; }
  int tw, th, bn, sp, st;
  conv_tile_shape(H, W, &tw, &th);
  const int tiles_y = (H + th - 1) / th;
  choose_tile(NB_tile * ((W + tw - 1) / tw) * tiles_y, Cout, 9 * Cin / 64, 0, true, &bn, &sp, &st);
  if (geom) { geom[0] = th; geom[1] = tiles_y; }
  if (!x) return MGB_OK;
  if (!w || !out || ldo <= 0 || sp != 1) { set_error("debug_conv2d_band: bad argument or a split-K tile"); return MGB_ERR_INVALID; }
  GemmParams p;
  TRY(fill_conv_params(&p, reinterpret_cast<const bf16*>(x), reinterpret_cast<const bf16*>(w), 1, H, W, Cin, Cout, 0, bn,
                       1, st, src_rows, W));
  TRY(set_conv_band(&p, ty0, tiles, src_y0, out_y0));
  fill_epi(&p.epi, bias, nullptr, out, nullptr, ldo, 0, 1.0f, nullptr, nullptr, nullptr, nullptr);
  p.epi.out_f32_hi = out_hi;
  p.epi.split_col = out_hi ? split_col : 0;
  p.epi.hw = H * W;
  return run_gemm(p, bn, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_layernorm(const float* x, void* y, const float* gamma, const float* beta, int32_t M, int32_t C, float eps,
                     void* stream) {
  return launch_layernorm(x, reinterpret_cast<bf16*>(y), gamma, beta, M, C, eps, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_xattn2(const float* x, void* y, void* a_out, const float* ln2_g, const float* ln2_b, const float* ln3_g,
                  const float* ln3_b, const void* GU, const float* c1, int32_t M, int32_t C, int32_t H, float scale, float eps,
                  void* stream) {
  if (!x || !y || !a_out || !GU || !c1) { set_error("op_xattn2: null pointer"); return MGB_ERR_INVALID; }
  return launch_xattn2_fused(x, reinterpret_cast<bf16*>(y), reinterpret_cast<bf16*>(a_out), ln2_g, ln2_b, ln3_g, ln3_b,
                             reinterpret_cast<const bf16*>(GU), c1, M, C, H, scale, eps,
                             reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_pack_decoder_latent(const float* latent_dev, const float* w_dev, const float* b_dev, float inv_scale,
                               void* out_bf16_dev, int32_t NB, int32_t HW, void* stream) {
  if (!latent_dev || !w_dev || !b_dev || !out_bf16_dev || NB <= 0 || HW <= 0) {
    set_error("op_pack_decoder_latent: bad argument (NB=%d HW=%d)", NB, HW);
    return MGB_ERR_INVALID;
  }
  return launch_pack_decoder_latent(latent_dev, w_dev, b_dev, inv_scale, reinterpret_cast<bf16*>(out_bf16_dev), NB, HW,
                                    reinterpret_cast<cudaStream_t>(stream));
}

/* ---- pre / post-processing and evaluation (image.cu, eval.cu) ---- */
int mgb_resize_ex(const void* src, int32_t src_is_u8, int32_t NC, int32_t H, int32_t W, float* dst, int32_t h, int32_t w,
                  int32_t mode, int32_t arith, int32_t post, float* tmp, void* stream) {
  if (!src || !dst || !tmp) { set_error("mgb_resize_ex: null pointer"); return MGB_ERR_INVALID; }
  return launch_resize(src, src_is_u8, NC, H, W, dst, h, w, mode, arith, post, tmp, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_colorize(const float* depth, int64_t HW, float dmin, float dmax, const uint8_t* lut, uint8_t* out_hwc, void* stream) {
  return launch_colorize(depth, HW, dmin, dmax, lut, out_hwc, reinterpret_cast<cudaStream_t>(stream));
}

size_t mgb_eval_ws_bytes(void) { return eval_ws_bytes() + 16 * sizeof(double); }

static int eval_depth_run(const char* what, const float* pred, const float* gt, const uint8_t* mask, int64_t H, int64_t W,
                          int32_t alignment, const int32_t* rows, const int32_t* cols, int32_t fit_h, int32_t fit_w, float dmin,
                          float dmax, float* aligned_out, void* ws, double* out_host, void* stream) {
  double* out_dev = reinterpret_cast<double*>(static_cast<char*>(ws) + eval_ws_bytes());
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  TRY(launch_eval_depth(pred, gt, mask, H, W, alignment, rows, cols, fit_h, fit_w, dmin, dmax, aligned_out, ws, out_dev, s));
  cudaError_t e = cudaMemcpyAsync(out_host, out_dev, 13 * sizeof(double), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) { set_error("%s: %s", what, cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  return MGB_OK;
}

int mgb_eval_depth(const float* pred, const float* gt, const uint8_t* mask, int64_t HW, int32_t least_squares, float dmin,
                   float dmax, float* aligned_out, void* ws, double* out_host, void* stream) {
  if (!pred || !gt || !ws || !out_host || HW <= 0) { set_error("mgb_eval_depth: bad argument"); return MGB_ERR_INVALID; }
  return eval_depth_run("mgb_eval_depth", pred, gt, mask, 1, HW, least_squares ? 1 : 0, nullptr, nullptr, 0, 0, dmin, dmax,
                        aligned_out, ws, out_host, stream);
}

int mgb_eval_depth_ex(const float* pred, const float* gt, const uint8_t* mask, int32_t H, int32_t W, int32_t alignment,
                      const int32_t* fit_rows, const int32_t* fit_cols, int32_t fit_h, int32_t fit_w, float dmin, float dmax,
                      float* aligned_out, void* ws, double* out_host, void* stream) {
  const bool tables = fit_rows || fit_cols;
  if (!pred || !gt || !ws || !out_host || H <= 0 || W <= 0 || alignment < 0 || alignment > 2 ||
      (tables && (!fit_rows || !fit_cols || fit_h <= 0 || fit_w <= 0))) {
    set_error("mgb_eval_depth_ex: bad argument");
    return MGB_ERR_INVALID;
  }
  return eval_depth_run("mgb_eval_depth_ex", pred, gt, mask, H, W, alignment, fit_rows, fit_cols, fit_h, fit_w, dmin, dmax,
                        aligned_out, ws, out_host, stream);
}

size_t mgb_eval_normals_ws_bytes(int64_t HW) { return eval_normals_ws_bytes(HW); }

int mgb_eval_normals(const float* pred, const float* gt, const uint8_t* mask, int32_t H, int32_t W, float* error_out, void* ws,
                     double* out_host, void* stream) {
  if (!pred || !gt || !ws || !out_host || H <= 0 || W <= 0) { set_error("mgb_eval_normals: bad argument"); return MGB_ERR_INVALID; }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  TRY(launch_eval_normals(pred, gt, mask, int64_t(H) * W, error_out, ws, s));
  cudaError_t e = cudaMemcpyAsync(out_host, eval_normals_out(ws), 9 * sizeof(double), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) { set_error("mgb_eval_normals: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  return MGB_OK;
}

size_t mgb_eval_iid_ws_bytes(int32_t H, int32_t W) { return H > 0 && W > 0 ? eval_iid_ws_bytes(H, W) : 0; }

int mgb_eval_iid(const float* pred, const float* gt, const uint8_t* mask, int32_t H, int32_t W, int32_t up_to_scale,
                 int32_t transform, void* ws, double* out_host, void* stream) {
  if (!pred || !gt || !ws || !out_host || H < 11 || W < 11 || transform < 0 || transform > 2) {
    set_error("mgb_eval_iid: bad argument (H=%d W=%d transform=%d; H and W must be >= 11)", H, W, transform);
    return MGB_ERR_INVALID;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  TRY(launch_eval_iid(pred, gt, mask, H, W, up_to_scale != 0, transform, ws, s));
  double res[7];
  cudaError_t e = cudaMemcpyAsync(res, eval_iid_out(ws, H, W), sizeof(res), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) { set_error("mgb_eval_iid: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  if (up_to_scale && res[6] == 0.0) {
    set_error("mgb_eval_iid: no pixel is valid in channel 0 of the mask, so the brightness quantile is undefined");
    return MGB_ERR_INVALID;
  }
  for (int i = 0; i < 6; ++i) out_host[i] = res[i];
  return MGB_OK;
}

int mgb_op_space_to_depth(const float* x, void* y, int32_t NB, int32_t H, int32_t W, int32_t C, void* stream) {
  return launch_space_to_depth(x, reinterpret_cast<bf16*>(y), NB, H, W, C, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_upsample2x_ex(const float* x, void* y, int32_t NB, int32_t H, int32_t W, int32_t C, int32_t Ho, int32_t Wo,
                         void* stream) {
  return launch_upsample2x(x, reinterpret_cast<bf16*>(y), NB, H, W, C, Ho, Wo, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_upsample2x(const float* x, void* y, int32_t NB, int32_t H, int32_t W, int32_t C, void* stream) {
  return mgb_op_upsample2x_ex(x, y, NB, H, W, C, 2 * H, 2 * W, stream);
}

int mgb_op_softmax_rows(const float* s, void* p, int32_t M, int32_t n, int32_t ld, void* stream) {
  if (!s || !p || M <= 0 || n <= 0 || ld < n) { set_error("op_softmax_rows: bad argument (M=%d n=%d ld=%d)", M, n, ld); return MGB_ERR_INVALID; }
  return launch_softmax_rows(s, reinterpret_cast<bf16*>(p), M, n, ld, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_op_transpose_bf16(const void* x, void* y, int32_t M, int32_t N, int32_t ld, void* stream) {
  if (!x || !y || M <= 0 || N <= 0 || ld < M) { set_error("op_transpose_bf16: bad argument (M=%d N=%d ld=%d)", M, N, ld); return MGB_ERR_INVALID; }
  return launch_transpose_bf16(reinterpret_cast<const bf16*>(x), reinterpret_cast<bf16*>(y), M, N, ld,
                               reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
