// Device-side evaluation step that follows the hot path in dataset evaluation (SURVEY.md 8f-4): least-squares
// scale / shift alignment of a prediction to the ground truth over the valid pixels (reference
// src/util/alignment.py:35-82) and the masked depth metrics (src/util/metric.py:64-191) in two streaming passes and ONE
// host synchronisation per sample (the reference does a numpy lstsq on the host and one `.item()` per metric).
//   pass 1  sums n, sum p, sum p^2, sum g, sum p g over the fit's pixels (double) -> scale, shift from the 2 x 2 normal
//           equations. The fit is against gt, or against 1 / gt for least_square_disparity, over all pixels or over the
//           nearest-downsampled map of max_resolution (index tables)
//   pass 2  aligned = p * scale + shift; for disparity 1 / max(aligned, 1e-3); then clip(clip(., dmin, dmax), 1e-6)
//           (script/depth/eval.py:196-207) and the sums of every metric over the full-resolution mask; a last block turns
//           them into the metric values.
// HBM-bound: 9 bytes / pixel / pass (pred f32, gt f32, mask u8).
// The surface-normals evaluation (below) computes the angular error and the normals metrics with an exact median.
#include <cfloat>

#include "common.cuh"
#include "kernels.h"
#include "launch.h"

namespace mgb {

constexpr int kEvThreads = 256;
constexpr int kEvBlocks = kNumSMs * 2;
constexpr int kEvSums = 12;

__device__ __forceinline__ void block_reduce_store(double (&v)[kEvSums], int n, double* __restrict__ out) {
  __shared__ double sh[kEvThreads / 32][kEvSums];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = 0; k < n; ++k) {
    double d = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == 0) sh[warp][k] = d;
  }
  __syncthreads();
  if (threadIdx.x < n) {
    double t = 0.0;
    for (int w = 0; w < kEvThreads / 32; ++w) t += sh[w][threadIdx.x];
    out[(size_t)blockIdx.x * kEvSums + threadIdx.x] = t;
  }
}

// The fit's pixels: the full map (rows == nullptr), or the nearest-downsampled map of fit_h x fit_w pixels whose source row
// and column are rows[i], cols[j] (align_depth_least_square's max_resolution, alignment.py:48-59). disparity: fit against
// 1 / gt over valid & gt > 0 & pred > 0 (script/depth/eval.py:180-195; depth2disparity is fp32, alignment.py:85-94).
__global__ void __launch_bounds__(kEvThreads)
    eval_align_sums_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                           long long n_fit, long long W, const int* __restrict__ rows, const int* __restrict__ cols, int fit_w,
                           int disparity, double* __restrict__ part) {
  double v[kEvSums] = {0};
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n_fit; q += (long long)gridDim.x * blockDim.x) {
    const long long p = rows ? (long long)rows[q / fit_w] * W + cols[q % fit_w] : q;
    if (mask && !mask[p]) continue;
    const float pf = pred[p], gf = gt[p];
    if (disparity && !(gf > 0.f && pf > 0.f)) continue;
    const double a = pf, g = disparity ? __fdiv_rn(1.0f, gf) : gf;
    v[0] += 1.0; v[1] += a; v[2] += a * a; v[3] += g; v[4] += a * g;
  }
  block_reduce_store(v, 5, part);
}

// scale, shift of min || [p 1] [s t]^T - g ||^2 over the valid pixels (np.linalg.lstsq in alignment.py:66-69)
// Sum of quantity k over the blocks' partials by one warp: lane l takes blocks l, l + 32, ... (independent loads), xor tree.
// (A single thread would walk blocks x 12 dependent loads.)
__device__ __forceinline__ double warp_sum_partials(const double* __restrict__ part, int nblocks, int k) {
  double t = 0.0;
  for (int b = threadIdx.x & 31; b < nblocks; b += 32) t += part[(size_t)b * kEvSums + k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}

__global__ void eval_align_solve_kernel(const double* __restrict__ part, int nblocks, int do_align, double* __restrict__ st) {
  double s[5];
  for (int k = 0; k < 5; ++k) s[k] = warp_sum_partials(part, nblocks, k);
  if (threadIdx.x != 0) return;
  double scale = 1.0, shift = 0.0;
  if (do_align) {
    const double n = s[0], sp = s[1], spp = s[2], sg = s[3], spg = s[4];
    const double det = n * spp - sp * sp;
    if (n > 0 && fabs(det) > 1e-300) {
      scale = (n * spg - sp * sg) / det;
      shift = (spp * sg - sp * spg) / det;
    } else if (n > 0) {               // constant prediction: lstsq's minimum-norm solution of the rank-1 system
      const double m = sp / n, gm = sg / n;
      scale = gm * m / (m * m + 1.0);
      shift = gm / (m * m + 1.0);
    }
  }
  st[0] = scale; st[1] = shift; st[2] = s[0];
}

__global__ void __launch_bounds__(kEvThreads)
    eval_metric_sums_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                            long long HW, const double* __restrict__ st, int disparity, float dmin, float dmax,
                            float* __restrict__ aligned_out, double* __restrict__ part) {
  // numpy: float32 pred * float64 scale + float64 shift is float64, and torch promotes the float64 prediction against the
  // float32 ground truth (script/depth/eval.py:177-213), so the reference's metric arithmetic is double: so is this
  const double scale = st[0], shift = st[1];
  double v[kEvSums] = {0};
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    double a = double(pred[p]) * scale + shift;
    if (disparity) a = 1.0 / fmax(a, 1e-3);              // clip the disparity to >= 1e-3, back to depth (eval.py:196-200)
    a = fmin(fmax(a, double(dmin)), double(dmax));
    a = fmax(a, 1e-6);
    if (aligned_out) aligned_out[p] = float(a);
    if (mask && !mask[p]) continue;
    const double g = double(gt[p]);
    const double diff = a - g;
    const double dl = log(a) - log(g);
    const double r = fmax(a / g, g / a);
    const double di = 1.0 / a - 1.0 / g;
    v[0] += 1.0;
    v[1] += fabs(diff) / g;                               // abs_relative_difference
    v[2] += diff * diff / g;                              // squared_relative_difference
    v[3] += diff * diff;                                  // rmse_linear
    v[4] += dl * dl;                                      // rmse_log / silog first term
    v[5] += dl;                                           // silog second term
    v[6] += fabs(log10(a) - log10(g));                    // log10
    v[7] += r < 1.25 ? 1.0 : 0.0;                         // delta1
    v[8] += r < 1.25 * 1.25 ? 1.0 : 0.0;                  // delta2
    v[9] += r < 1.25 * 1.25 * 1.25 ? 1.0 : 0.0;           // delta3
    v[10] += di * di;                                     // i_rmse
  }
  block_reduce_store(v, 11, part);
}

__global__ void eval_metric_final_kernel(const double* __restrict__ part, int nblocks, const double* __restrict__ st,
                                         double* __restrict__ out) {
  double s[kEvSums] = {0};
  for (int k = 0; k < 11; ++k) s[k] = warp_sum_partials(part, nblocks, k);
  if (threadIdx.x != 0) return;
  const double n = s[0] > 0 ? s[0] : 1.0;
  out[0] = st[0]; out[1] = st[1]; out[2] = s[0];
  out[3] = s[1] / n;                                     // abs_relative_difference
  out[4] = s[2] / n;                                     // squared_relative_difference
  out[5] = sqrt(s[3] / n);                               // rmse_linear
  out[6] = sqrt(s[4] / n);                               // rmse_log
  out[7] = s[6] / n;                                     // log10
  out[8] = s[7] / n; out[9] = s[8] / n; out[10] = s[9] / n;   // delta1..3
  out[11] = sqrt(s[10] / n);                             // i_rmse
  const double t = s[4] / n - (s[5] * s[5]) / (n * n);
  out[12] = sqrt(t > 0 ? t : 0.0) * 100.0;               // silog_rmse
}

size_t eval_ws_bytes() { return size_t(kEvBlocks) * kEvSums * sizeof(double) + 16 * sizeof(double) + 64; }

// out_dev: 13 doubles {scale, shift, n_valid, abs_rel, sq_rel, rmse, rmse_log, log10, delta1, delta2, delta3, i_rmse, silog}
// align: 0 none, 1 least squares on depth, 2 least squares on disparity. rows / cols: the fit's index tables (fit_h x fit_w
// pixels) or nullptr for a fit over all H x W pixels.
int launch_eval_depth(const float* pred, const float* gt, const uint8_t* mask, long long H, long long W, int align,
                      const int* rows, const int* cols, int fit_h, int fit_w, float dmin, float dmax, float* aligned_out,
                      void* ws, double* out_dev, cudaStream_t stream) {
  double* part = static_cast<double*>(ws);
  double* st = part + size_t(kEvBlocks) * kEvSums;
  const long long HW = H * W, n_fit = rows ? (long long)fit_h * fit_w : HW;
  const int blocks = int(std::min<long long>((HW + kEvThreads - 1) / kEvThreads, kEvBlocks));
  const int fit_blocks = int(std::min<long long>((n_fit + kEvThreads - 1) / kEvThreads, kEvBlocks));
  TRY(launch_plain("eval_align_sums", eval_align_sums_kernel, fit_blocks, kEvThreads, 0, stream, pred, gt, mask, n_fit, W,
                   rows, cols, fit_w, align == 2, part));
  TRY(launch_plain("eval_align_solve", eval_align_solve_kernel, 1, 32, 0, stream, part, fit_blocks, align != 0, st));
  TRY(launch_plain("eval_metric_sums", eval_metric_sums_kernel, blocks, kEvThreads, 0, stream, pred, gt, mask, HW, st,
                   align == 2, dmin, dmax, aligned_out, part));
  return launch_plain("eval_metric_final", eval_metric_final_kernel, 1, 32, 0, stream, part, blocks, st, out_dev);
}

// ---------------------------------------------------------------------------------------------------------------------
// Surface-normals evaluation (script/normals/eval.py:145-157): compute_cosine_error(masked=True) (src/util/metric.py:
// 194-219) and the metrics of metric.py:222-257 in four launches and ONE synchronisation.
//   error    per-pixel angular error, written to the workspace (and error_out); fixed-order double sums of n, e, e^2 and
//            the five threshold counts; a histogram of the high 16 bits of the errors (shared memory, then global)
//   locate   one block: the high-16 bins holding the order statistics (n-1)/2 and n/2 and their ranks inside the bins
//   refine   histograms of the low 16 bits of the errors that fall in those two bins
//   final    one block: the two order statistics exactly, np.median's mean of them, the other metrics
// The errors are >= 0, so the unsigned order of their bit patterns is their numeric order, and integer counts do not
// depend on the order the atomics land in: the median is exact and every output is deterministic.
// locate / refine and the low-bin lookup of final (sel_*) serve any 32-bit keys whose unsigned order is the values'
// order: the intrinsic-image evaluation below selects its brightness quantile with them.
constexpr int kNrHiBins = 0x4335 + 1;       // high halves of [0, 180.00002]; the last bin takes anything above (NaN)
constexpr int kNrLoBins = 1 << 16;
constexpr int kNrSelThreads = 1024;
constexpr unsigned kNrInvalid = 0xFFFFFFFFu;  // workspace bits of a pixel that is not valid
constexpr float kInvPi = 1.0f / 3.14159265358979323846f;

struct NrSel {
  unsigned n;
  unsigned bin[2];    // high-16 bin of the two order statistics (kNrInvalid when n == 0)
  unsigned rank[2];   // rank inside that bin
  float frac;         // torch.quantile's interpolation weight between them (0 for the median)
};

// High-16 bin of a key; `top` takes every key above it.
__device__ __forceinline__ unsigned sel_bin(unsigned bits, unsigned top) { return min(bits >> 16, top); }
__device__ __forceinline__ unsigned nr_bin(unsigned bits) { return sel_bin(bits, unsigned(kNrHiBins - 1)); }

// torch.cosine_similarity(pred, gt, dim=0) (each vector over max(norm, 1e-8), then the products summed over the channels
// in order), clamp(-1, 1), acos, * 180.0, / pi. torch's CUDA division by a scalar multiplies by its fp32 reciprocal,
// which is what the reference's evaluation on the GPU computes. No contraction, in the reference's order.
__device__ __forceinline__ float angular_error(float x0, float x1, float x2, float y0, float y1, float y2, float ny) {
  const float nx = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x0, x0), __fmul_rn(x1, x1)), __fmul_rn(x2, x2)));
  const float dx = fmaxf(nx, 1e-8f), dy = fmaxf(ny, 1e-8f);
  float c = __fadd_rn(__fadd_rn(__fmul_rn(__fdiv_rn(x0, dx), __fdiv_rn(y0, dy)), __fmul_rn(__fdiv_rn(x1, dx), __fdiv_rn(y1, dy))),
                      __fmul_rn(__fdiv_rn(x2, dx), __fdiv_rn(y2, dy)));
  c = fminf(fmaxf(c, -1.0f), 1.0f);
  return __fmul_rn(__fmul_rn(acosf(c), 180.0f), kInvPi);
}

// The loops below step over whole warps (base is warp-uniform), so the warp-aggregated atomics can use the full mask:
// lanes with equal keys add once (heavy ties, e.g. pred == gt, would otherwise serialise on one counter).
__device__ __forceinline__ void warp_agg_add(unsigned* __restrict__ hist, unsigned key, bool take) {
  const unsigned k = take ? key : kNrInvalid;
  const unsigned peers = __match_any_sync(0xffffffffu, k);
  if (take && (threadIdx.x & 31) == unsigned(__ffs(peers) - 1)) atomicAdd(hist + key, unsigned(__popc(peers)));
}

__global__ void __launch_bounds__(kEvThreads)
    eval_normals_error_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                              long long HW, unsigned* __restrict__ err_bits, float* __restrict__ err_out,
                              unsigned* __restrict__ hist_hi, double* __restrict__ part) {
  extern __shared__ unsigned sh_hist[];
  for (int i = threadIdx.x; i < kNrHiBins; i += blockDim.x) sh_hist[i] = 0;
  __syncthreads();
  double v[kEvSums] = {0};
  for (long long base = (long long)blockIdx.x * blockDim.x; base < HW; base += (long long)gridDim.x * blockDim.x) {
    const long long p = base + threadIdx.x;
    bool valid = false;
    unsigned bits = kNrInvalid;
    if (p < HW) {
      const float y0 = gt[p], y1 = gt[p + HW], y2 = gt[p + 2 * HW];
      // torch.norm(gt, dim=0) > 0 (metric.py:205-211), ANDed with the caller's mask
      const float ny = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(y0, y0), __fmul_rn(y1, y1)), __fmul_rn(y2, y2)));
      valid = ny > 0.f && (!mask || mask[p]);
      float e = __int_as_float(0x7fffffff);
      if (valid) {
        e = angular_error(pred[p], pred[p + HW], pred[p + 2 * HW], y0, y1, y2, ny);
        bits = e == e ? __float_as_uint(e) : 0x7fffffffu;
        const double d = e;
        v[0] += 1.0; v[1] += d; v[2] += d * d;
        v[3] += e < 5.0f ? 1.0 : 0.0;
        v[4] += e < 7.5f ? 1.0 : 0.0;
        v[5] += e < 11.25f ? 1.0 : 0.0;
        v[6] += e < 22.5f ? 1.0 : 0.0;
        v[7] += e < 30.0f ? 1.0 : 0.0;
      }
      err_bits[p] = bits;
      if (err_out) err_out[p] = e;
    }
    warp_agg_add(sh_hist, nr_bin(bits), valid);
  }
  block_reduce_store(v, 8, part);
  __syncthreads();
  for (int i = threadIdx.x; i < kNrHiBins; i += blockDim.x)
    if (sh_hist[i]) atomicAdd(hist_hi + i, sh_hist[i]);
}

// Exclusive prefix sum over a block of kNrSelThreads threads; *total = the sum of all.
__device__ __forceinline__ unsigned block_exclusive_scan(unsigned x, unsigned* total) {
  __shared__ unsigned sh[kNrSelThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  __syncthreads();                     // sh may still be read by a previous call
  if (lane == 31) sh[warp] = inc;
  __syncthreads();
  unsigned before = 0, all = 0;
  for (int w = 0; w < kNrSelThreads / 32; ++w) {
    if (w < warp) before += sh[w];
    all += sh[w];
  }
  *total = all;
  return before + inc - x;
}

// Thread t owns bins [t * per, (t + 1) * per): finds the bin holding rank k and the rank inside it.
__device__ __forceinline__ void find_rank(const unsigned* __restrict__ hist, int nbins, unsigned k, unsigned* bin_out,
                                          unsigned* rank_out) {
  const int per = (nbins + kNrSelThreads - 1) / kNrSelThreads;
  const int b0 = threadIdx.x * per, b1 = min(b0 + per, nbins);
  unsigned local = 0;
  for (int b = b0; b < b1; ++b) local += hist[b];
  unsigned total;
  unsigned c = block_exclusive_scan(local, &total);
  if (k < c || k >= c + local) return;
  for (int b = b0; b < b1; ++b) {
    if (k < c + hist[b]) { *bin_out = b; *rank_out = k - c; return; }
    c += hist[b];
  }
}

// One block: n = the keys counted in hist_hi, and the bins and in-bin ranks of two order statistics. q < 0: the
// median's, (n-1)/2 and n/2 (np.median). Otherwise torch.quantile(q)'s, whose rank is float32: r = fl(q * (n-1)),
// order statistics floor(r) and ceil(r), weight r - floor(r).
__global__ void __launch_bounds__(kNrSelThreads)
    sel_locate_kernel(const unsigned* __restrict__ hist_hi, int nbins, float q, NrSel* sel) {
  unsigned local = 0;
  const int per = (nbins + kNrSelThreads - 1) / kNrSelThreads;
  for (int b = threadIdx.x * per; b < min((int(threadIdx.x) + 1) * per, nbins); ++b) local += hist_hi[b];
  unsigned n;
  block_exclusive_scan(local, &n);
  unsigned k0 = (n - 1) / 2, k1 = n / 2;
  float frac = 0.f;
  if (q >= 0.f && n > 0) {
    const float r = __fmul_rn(q, float(n - 1)), f = floorf(r);
    k0 = unsigned(f);
    k1 = min(unsigned(ceilf(r)), n - 1);
    frac = __fsub_rn(r, f);
  }
  if (threadIdx.x == 0) {
    sel->n = n;
    sel->bin[0] = sel->bin[1] = kNrInvalid;
    sel->frac = frac;
  }
  __syncthreads();
  if (n == 0) return;
  find_rank(hist_hi, nbins, k0, &sel->bin[0], &sel->rank[0]);
  find_rank(hist_hi, nbins, k1, &sel->bin[1], &sel->rank[1]);
}

// Histograms of the low 16 bits of the keys in the two located bins (top: the highest bin, as in sel_bin).
__global__ void __launch_bounds__(kEvThreads)
    sel_refine_kernel(const unsigned* __restrict__ keys, long long HW, unsigned top, const NrSel* __restrict__ sel,
                      unsigned* __restrict__ hist_lo) {
  const unsigned b0 = sel->bin[0], b1 = sel->bin[1];
  for (long long base = (long long)blockIdx.x * blockDim.x; base < HW; base += (long long)gridDim.x * blockDim.x) {
    const long long p = base + threadIdx.x;
    const unsigned bits = p < HW ? keys[p] : kNrInvalid;
    const unsigned bin = bits == kNrInvalid ? kNrInvalid : sel_bin(bits, top);
    const unsigned which = bin == b0 ? 0u : 1u;     // both ranks in one bin: one histogram serves both
    warp_agg_add(hist_lo, which * kNrLoBins + (bits & 0xFFFFu), bin == b0 || bin == b1);
  }
}

// The low 16 bits of both order statistics (block-wide; sel->n > 0).
__device__ __forceinline__ void sel_find_low(const NrSel* sel, const unsigned* __restrict__ hist_lo, unsigned* lo) {
  __shared__ unsigned rank_unused;
  find_rank(hist_lo, kNrLoBins, sel->rank[0], &lo[0], &rank_unused);
  find_rank(hist_lo + (sel->bin[1] == sel->bin[0] ? 0 : kNrLoBins), kNrLoBins, sel->rank[1], &lo[1], &rank_unused);
}

// out: {n_valid, mean, median, rmse, sub5, sub7.5, sub11.25, sub22.5, sub30}
__global__ void __launch_bounds__(kNrSelThreads)
    eval_normals_final_kernel(const double* __restrict__ part, int nblocks, NrSel* sel, const unsigned* __restrict__ hist_lo,
                              double* __restrict__ out) {
  __shared__ unsigned lo[2];
  const unsigned n = sel->n;
  if (n > 0) sel_find_low(sel, hist_lo, lo);
  __shared__ double s[8];
  if (threadIdx.x < 32)
    for (int k = 0; k < 8; ++k) {
      const double t = warp_sum_partials(part, nblocks, k);
      if (threadIdx.x == 0) s[k] = t;
    }
  __syncthreads();
  if (threadIdx.x != 0) return;
  out[0] = s[0];
  if (n == 0) {                        // numpy's statistics of an empty array
#pragma unroll
    for (int k = 1; k < 9; ++k) out[k] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  const unsigned nan_bits = 0x7fffffffu, top = kNrHiBins - 1;
  const float v0 = __uint_as_float(sel->bin[0] == top ? nan_bits : (sel->bin[0] << 16) | lo[0]);
  const float v1 = __uint_as_float(sel->bin[1] == top ? nan_bits : (sel->bin[1] << 16) | lo[1]);
  out[1] = s[1] / s[0];
  out[2] = __fdiv_rn(__fadd_rn(v0, v1), 2.0f);       // np.median: float32 mean of the two middle values
  out[3] = sqrt(s[2] / s[0]);
#pragma unroll
  for (int k = 0; k < 5; ++k) out[4 + k] = 100.0 * (s[3 + k] / s[0]);
}

// Workspace: partials | 16 doubles of results | NrSel | high and low histograms | the error map (4 B per pixel).
constexpr size_t kNrOutOff = size_t(kEvBlocks) * kEvSums * sizeof(double);
constexpr size_t kNrSelOff = kNrOutOff + 16 * sizeof(double);
constexpr size_t kNrHistOff = kNrSelOff + 64;
constexpr size_t kNrHistBytes = (size_t(kNrHiBins + 3) / 4 * 4 + 2 * kNrLoBins) * sizeof(unsigned);
constexpr size_t kNrErrOff = kNrHistOff + kNrHistBytes;

size_t eval_normals_ws_bytes(long long HW) { return kNrErrOff + size_t(HW) * sizeof(unsigned); }
double* eval_normals_out(void* ws) { return reinterpret_cast<double*>(static_cast<char*>(ws) + kNrOutOff); }

int launch_eval_normals(const float* pred, const float* gt, const uint8_t* mask, long long HW, float* err_out, void* ws,
                        cudaStream_t stream) {
  char* w = static_cast<char*>(ws);
  double* part = reinterpret_cast<double*>(w);
  NrSel* sel = reinterpret_cast<NrSel*>(w + kNrSelOff);
  unsigned* hist_hi = reinterpret_cast<unsigned*>(w + kNrHistOff);
  unsigned* hist_lo = hist_hi + (kNrHiBins + 3) / 4 * 4;
  unsigned* err_bits = reinterpret_cast<unsigned*>(w + kNrErrOff);
  constexpr size_t smem = kNrHiBins * sizeof(unsigned);
  TRY(raise_smem_limit_once<eval_normals_error_kernel>("eval_normals", int(smem)));
  const int blocks = int(std::min<long long>((HW + kEvThreads - 1) / kEvThreads, kEvBlocks));
  cudaError_t e = cudaMemsetAsync(hist_hi, 0, kNrHistBytes, stream);
  if (e != cudaSuccess) { set_error("eval_normals memset: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  TRY(launch_plain("eval_normals_error", eval_normals_error_kernel, blocks, kEvThreads, smem, stream, pred, gt, mask, HW,
                   err_bits, err_out, hist_hi, part));
  TRY(launch_plain("eval_normals_locate", sel_locate_kernel, 1, kNrSelThreads, 0, stream, hist_hi, kNrHiBins, -1.0f, sel));
  TRY(launch_plain("eval_normals_refine", sel_refine_kernel, blocks, kEvThreads, 0, stream, err_bits, HW,
                   unsigned(kNrHiBins - 1), sel, hist_lo));
  return launch_plain("eval_normals_final", eval_normals_final_kernel, 1, kNrSelThreads, 0, stream, part, blocks, sel,
                      hist_lo, eval_normals_out(ws));
}

// ---------------------------------------------------------------------------------------------------------------------
// Intrinsic-image evaluation of one (sample, target) pair (script/iid/eval.py:182-213 -> compute_iid_metric,
// src/util/metric.py:263-338): PSNR and SSIM (torchmetrics, data_range 1) of the optionally colour-transformed maps and,
// for the up-to-scale targets, after the least-squares scale and the quantile map. ONE synchronisation per call.
//   stats   (up-to-scale) fixed-order double sums of p g and p^2 over the masked elements -> s = sum pg / sum p^2 (the
//           1 x 1 lstsq); the brightness 0.3 g0 + 0.59 g1 + 0.11 g2 of every pixel valid in mask channel 0 as an
//           order-preserving key, and a global histogram of the keys' high 16 bits
//   locate, refine (sel_*), select   the order statistics floor(r), ceil(r) of torch.quantile(0.9) exactly; q, k
//   ssim    tiles of 32 x 32 outputs per channel: the mapped maps in shared memory with a 5-pixel halo, the separable
//           11-tap Gaussian over the five moment maps, SSIM of every window that lies inside the image (torchmetrics'
//           reflect padding touches only the outputs it crops), the squared error of the masked elements the tile owns
//   final   PSNR = 10 log10(1 / (SSE / n)), SSIM = the mean over the 3 (H-10)(W-10) windows
// The non-scale targets run ssim and final only. Atomics add integer counts only: equal inputs give equal bits.
constexpr int kIidHiBins = 1 << 16;              // brightness keys span every float: the whole high half
constexpr unsigned kIidNanKey = 0xFFFFFFFEu;     // every NaN: above +inf (0xFF800000), alone in the top bin
constexpr int kSsTile = 32, kSsHalo = 5, kSsIn = kSsTile + 2 * kSsHalo, kSsTaps = 2 * kSsHalo + 1;

// image_util.py:144-149 as torch evaluates x ** 2.2 and x ** (1 / 2.2) on a float32 tensor: powf, float32 exponent
__device__ __forceinline__ float iid_transform(float x, int t) {
  return t == 1 ? powf(x, 2.2f) : t == 2 ? powf(x, float(1.0 / 2.2)) : x;
}

__device__ __forceinline__ unsigned iid_key(float b) {
  if (b != b) return kIidNanKey;
  const unsigned u = __float_as_uint(b);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float iid_key_value(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// torch.clamp(x, 0, 1): NaN stays NaN
__device__ __forceinline__ float clamp01(float x) { return x != x ? x : fminf(fmaxf(x, 0.f), 1.f); }

__global__ void __launch_bounds__(kEvThreads)
    eval_iid_stats_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                          long long HW, int transform, unsigned* __restrict__ keys, unsigned* __restrict__ hist_hi,
                          double* __restrict__ part) {
  double v[kEvSums] = {0};
  for (long long base = (long long)blockIdx.x * blockDim.x; base < HW; base += (long long)gridDim.x * blockDim.x) {
    const long long p = base + threadIdx.x;
    bool take = false;
    unsigned key = kNrInvalid;
    if (p < HW) {
      float g[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        g[c] = iid_transform(gt[p + c * HW], transform);
        if (mask && !mask[p + c * HW]) continue;
        const double a = iid_transform(pred[p + c * HW], transform), b = g[c];
        v[0] += a * b; v[1] += a * a;                    // exact products of float32 values
      }
      take = !mask || mask[p];                           // quantile_map: brightness[valid_mask[0]]
      if (take) key = iid_key(__fadd_rn(__fadd_rn(__fmul_rn(0.3f, g[0]), __fmul_rn(0.59f, g[1])), __fmul_rn(0.11f, g[2])));
      keys[p] = key;
    }
    warp_agg_add(hist_hi, key >> 16, take);
  }
  block_reduce_store(v, 2, part);
}

// One block. sk = {s, k} for the ssim pass; out[3..6] = {s, q, k, pixels in the quantile}.
__global__ void __launch_bounds__(kNrSelThreads)
    eval_iid_select_kernel(const double* __restrict__ part, int nblocks, const NrSel* sel, const unsigned* __restrict__ hist_hi,
                           const unsigned* __restrict__ hist_lo, float* __restrict__ sk, double* __restrict__ out) {
  __shared__ unsigned lo[2];
  __shared__ double sums[2];
  const unsigned n = sel->n;
  if (n > 0) sel_find_low(sel, hist_lo, lo);
  if (threadIdx.x < 32)
    for (int k = 0; k < 2; ++k) {
      const double t = warp_sum_partials(part, nblocks, k);
      if (threadIdx.x == 0) sums[k] = t;
    }
  __syncthreads();
  if (threadIdx.x != 0) return;
  // lstsq of the masked elements: sum pg / sum p^2, and 0 (the minimum-norm solution) when every p is 0
  const float s = sums[1] == 0.0 ? 0.f : float(sums[0] / sums[1]);
  float q = __int_as_float(0x7fffffff);
  if (n > 0 && hist_hi[kIidHiBins - 1] == 0) {            // a NaN brightness makes torch.quantile NaN
    const float v0 = iid_key_value((sel->bin[0] << 16) | lo[0]), v1 = iid_key_value((sel->bin[1] << 16) | lo[1]);
    const float w = sel->frac, d = __fsub_rn(v1, v0);      // torch's lerp, un-fused
    q = w < 0.5f ? __fadd_rn(v0, __fmul_rn(w, d)) : __fsub_rn(v1, __fmul_rn(d, __fsub_rn(1.f, w)));
  }
  // quantile_map: 0 below 1e-4, else float(0.8 / q), which torch evaluates as q.reciprocal() * 0.8 in float32
  const float k = q < 1e-4f ? 0.f : __fmul_rn(__frcp_rn(q), 0.8f);
  sk[0] = s; sk[1] = k;
  out[3] = s; out[4] = q; out[5] = k; out[6] = n;
}

// The Gaussian of torchmetrics' SSIM (sigma 1.5, 11 taps): exp(-(d / 1.5)^2 / 2) over d = -5..5, over its float32 sum
__device__ __forceinline__ void ssim_gauss(float (&w)[kSsTaps]) {
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kSsTaps; ++i) {
    const float t = __fdiv_rn(float(i - kSsHalo), 1.5f);
    w[i] = expf(__fdiv_rn(-__fmul_rn(t, t), 2.f));
    sum = __fadd_rn(sum, w[i]);
  }
#pragma unroll
  for (int i = 0; i < kSsTaps; ++i) w[i] = __fdiv_rn(w[i], sum);
}

// One CTA per (channel, 32 x 32 tile). sk: {s, k} of the up-to-scale targets, or nullptr (maps used as they are).
// Partials: {sum of SSIM over the tile's interior windows, SSE and count of the masked elements the tile owns}.
__global__ void __launch_bounds__(kEvThreads)
    eval_iid_ssim_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                         int H, int W, int transform, const float* __restrict__ sk, int tiles_x, int tiles_y,
                         double* __restrict__ part) {
  __shared__ float sp[kSsIn][kSsIn + 1], sg[kSsIn][kSsIn + 1];
  __shared__ float sh[5][kSsIn][kSsTile + 1];                  // the row pass: five moment maps
  const int c = blockIdx.x / (tiles_x * tiles_y), t = blockIdx.x % (tiles_x * tiles_y);
  const int y0 = (t / tiles_x) * kSsTile, x0 = (t % tiles_x) * kSsTile;
  const long long plane = (long long)c * H * W;
  const float s = sk ? sk[0] : 1.f, k = sk ? sk[1] : 1.f;
  double v[kEvSums] = {0};
  for (int i = threadIdx.x; i < kSsIn * kSsIn; i += blockDim.x) {
    const int r = i / kSsIn, q = i % kSsIn, y = y0 - kSsHalo + r, x = x0 - kSsHalo + q;
    float pv = 0.f, gv = 0.f;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      const long long e = plane + (long long)y * W + x;
      pv = iid_transform(pred[e], transform);
      gv = iid_transform(gt[e], transform);
      if (sk) {                                             // pred = s * pred, then quantile_map's clamp(k * .)
        pv = clamp01(__fmul_rn(k, __fmul_rn(s, pv)));
        gv = clamp01(__fmul_rn(k, gv));
      }
      const bool valid = !mask || mask[e];
      const bool own = r >= kSsHalo && r < kSsHalo + kSsTile && q >= kSsHalo && q < kSsHalo + kSsTile;
      if (valid && own) {                                   // PSNR of pred[mask], gt[mask]
        const double d = double(pv) - double(gv);
        v[1] += d * d; v[2] += 1.0;
      }
      if (!valid) pv = gv = 0.f;                            // SSIM: pred[~mask] = gt[~mask] = 0
    }
    sp[r][q] = pv; sg[r][q] = gv;
  }
  __syncthreads();
  float w[kSsTaps];
  ssim_gauss(w);
  for (int i = threadIdx.x; i < kSsIn * kSsTile; i += blockDim.x) {
    const int r = i / kSsTile, j = i % kSsTile;
    float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int a = 0; a < kSsTaps; ++a) {
      const float pv = sp[r][j + a], gv = sg[r][j + a];
      m[0] = fmaf(w[a], pv, m[0]);
      m[1] = fmaf(w[a], gv, m[1]);
      m[2] = fmaf(w[a], __fmul_rn(pv, pv), m[2]);
      m[3] = fmaf(w[a], __fmul_rn(gv, gv), m[3]);
      m[4] = fmaf(w[a], __fmul_rn(pv, gv), m[4]);
    }
#pragma unroll
    for (int u = 0; u < 5; ++u) sh[u][r][j] = m[u];
  }
  __syncthreads();
  const float c1 = float(0.01 * 0.01), c2 = float(0.03 * 0.03);
  for (int i = threadIdx.x; i < kSsTile * kSsTile; i += blockDim.x) {
    const int a0 = i / kSsTile, j = i % kSsTile, y = y0 + a0, x = x0 + j;
    if (y < kSsHalo || y >= H - kSsHalo || x < kSsHalo || x >= W - kSsHalo) continue;
    float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int a = 0; a < kSsTaps; ++a)
#pragma unroll
      for (int u = 0; u < 5; ++u) m[u] = fmaf(w[a], sh[u][a0 + a][j], m[u]);
    // torchmetrics _ssim_update, in its order
    const float mu_pp = __fmul_rn(m[0], m[0]), mu_gg = __fmul_rn(m[1], m[1]), mu_pg = __fmul_rn(m[0], m[1]);
    float s_pp = __fsub_rn(m[2], mu_pp), s_gg = __fsub_rn(m[3], mu_gg);
    s_pp = s_pp < 0.f ? 0.f : s_pp;                         // clamp(min=0); NaN stays NaN
    s_gg = s_gg < 0.f ? 0.f : s_gg;
    const float s_pg = __fsub_rn(m[4], mu_pg);
    const float upper = __fadd_rn(__fmul_rn(2.f, s_pg), c2), lower = __fadd_rn(__fadd_rn(s_pp, s_gg), c2);
    const float num = __fmul_rn(__fadd_rn(__fmul_rn(2.f, mu_pg), c1), upper);
    const float den = __fmul_rn(__fadd_rn(__fadd_rn(mu_pp, mu_gg), c1), lower);
    v[0] += double(__fdiv_rn(num, den));
  }
  block_reduce_store(v, 3, part);
}

// out[0..2] = {n_valid, psnr, ssim}; without the up-to-scale passes also out[3..6] = {1, NaN, 1, 0}.
__global__ void eval_iid_final_kernel(const double* __restrict__ part, int nblocks, double windows, int up_to_scale,
                                      double* __restrict__ out) {
  double s[3];
  for (int k = 0; k < 3; ++k) s[k] = warp_sum_partials(part, nblocks, k);
  if (threadIdx.x != 0) return;
  out[0] = s[2];
  out[1] = 10.0 * log10(1.0 / (s[1] / s[2]));              // SSE 0: +inf; no element: NaN
  out[2] = s[0] / windows;
  if (!up_to_scale) {
    out[3] = 1.0; out[4] = __longlong_as_double(0x7ff8000000000000ll); out[5] = 1.0; out[6] = 0.0;
  }
}

// Workspace: partials | 16 doubles of results | NrSel | {s, k} | high and low histograms | the keys (4 B per pixel).
struct IidLayout {
  size_t out, sel, sk, hist, keys, total;
  int tiles_x, tiles_y;
};
static IidLayout iid_layout(long long H, long long W) {
  IidLayout l;
  l.tiles_x = int((W + kSsTile - 1) / kSsTile);
  l.tiles_y = int((H + kSsTile - 1) / kSsTile);
  const size_t blocks = std::max<size_t>(kEvBlocks, size_t(3) * l.tiles_x * l.tiles_y);
  l.out = blocks * kEvSums * sizeof(double);
  l.sel = l.out + 16 * sizeof(double);
  l.sk = l.sel + 64;
  l.hist = l.sk + 64;
  l.keys = l.hist + size_t(kIidHiBins + 2 * kNrLoBins) * sizeof(unsigned);
  l.total = l.keys + size_t(H * W) * sizeof(unsigned);
  return l;
}

size_t eval_iid_ws_bytes(long long H, long long W) { return iid_layout(H, W).total; }
double* eval_iid_out(void* ws, long long H, long long W) {
  return reinterpret_cast<double*>(static_cast<char*>(ws) + iid_layout(H, W).out);
}

int launch_eval_iid(const float* pred, const float* gt, const uint8_t* mask, long long H, long long W, int up_to_scale,
                    int transform, void* ws, cudaStream_t stream) {
  const IidLayout l = iid_layout(H, W);
  char* w = static_cast<char*>(ws);
  double* part = reinterpret_cast<double*>(w);
  double* out = reinterpret_cast<double*>(w + l.out);
  const long long HW = H * W;
  float* sk = nullptr;
  if (up_to_scale) {
    NrSel* sel = reinterpret_cast<NrSel*>(w + l.sel);
    sk = reinterpret_cast<float*>(w + l.sk);
    unsigned* hist_hi = reinterpret_cast<unsigned*>(w + l.hist);
    unsigned* hist_lo = hist_hi + kIidHiBins;
    unsigned* keys = reinterpret_cast<unsigned*>(w + l.keys);
    const int blocks = int(std::min<long long>((HW + kEvThreads - 1) / kEvThreads, kEvBlocks));
    cudaError_t e = cudaMemsetAsync(hist_hi, 0, size_t(kIidHiBins + 2 * kNrLoBins) * sizeof(unsigned), stream);
    if (e != cudaSuccess) { set_error("eval_iid memset: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
    TRY(launch_plain("eval_iid_stats", eval_iid_stats_kernel, blocks, kEvThreads, 0, stream, pred, gt, mask, HW, transform,
                     keys, hist_hi, part));
    TRY(launch_plain("eval_iid_locate", sel_locate_kernel, 1, kNrSelThreads, 0, stream, hist_hi, kIidHiBins, 0.9f, sel));
    TRY(launch_plain("eval_iid_refine", sel_refine_kernel, blocks, kEvThreads, 0, stream, keys, HW,
                     unsigned(kIidHiBins - 1), sel, hist_lo));
    TRY(launch_plain("eval_iid_select", eval_iid_select_kernel, 1, kNrSelThreads, 0, stream, part, blocks, sel, hist_hi,
                     hist_lo, sk, out));
  }
  const int tiles = 3 * l.tiles_x * l.tiles_y;
  TRY(launch_plain("eval_iid_ssim", eval_iid_ssim_kernel, tiles, kEvThreads, 0, stream, pred, gt, mask, int(H), int(W),
                   transform, sk, l.tiles_x, l.tiles_y, part));
  return launch_plain("eval_iid_final", eval_iid_final_kernel, 1, 32, 0, stream, part, tiles,
                      3.0 * double(H - 2 * kSsHalo) * double(W - 2 * kSsHalo), up_to_scale, out);
}

}  // namespace mgb
