// Device-side evaluation step that follows the hot path in dataset evaluation (SURVEY.md 8f-4): least-squares
// scale / shift alignment of a prediction to the ground truth over the valid pixels (reference
// src/util/alignment.py:35-82) and the masked depth metrics (src/util/metric.py:64-191) in two streaming passes and ONE
// host synchronisation per sample (the reference does a numpy lstsq on the host and one `.item()` per metric).
//   pass 1  sums n, sum p, sum p^2, sum g, sum p g over the mask (double) -> scale, shift from the 2 x 2 normal equations
//   pass 2  aligned = clip(clip(p * scale + shift, dmin, dmax), 1e-6) (script/depth/eval.py:201-207) and the sums of every
//           metric; a last block turns them into the metric values.
// HBM-bound: 9 bytes / pixel / pass (pred f32, gt f32, mask u8).
#include <cfloat>

#include "common.cuh"
#include "kernels.h"

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

__global__ void __launch_bounds__(kEvThreads)
    eval_align_sums_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const uint8_t* __restrict__ mask,
                           long long HW, double* __restrict__ part) {
  double v[kEvSums] = {0};
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    if (mask && !mask[p]) continue;
    const double a = pred[p], g = gt[p];
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
                            long long HW, const double* __restrict__ st, float dmin, float dmax, float* __restrict__ aligned_out,
                            double* __restrict__ part) {
  // numpy: float32 pred * float64 scale + float64 shift is float64, and torch promotes the float64 prediction against the
  // float32 ground truth (script/depth/eval.py:177-213), so the reference's metric arithmetic is double: so is this
  const double scale = st[0], shift = st[1];
  double v[kEvSums] = {0};
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    double a = double(pred[p]) * scale + shift;
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
int launch_eval_depth(const float* pred, const float* gt, const uint8_t* mask, long long HW, int do_align, float dmin, float dmax,
                      float* aligned_out, void* ws, double* out_dev, cudaStream_t stream) {
  double* part = static_cast<double*>(ws);
  double* st = part + size_t(kEvBlocks) * kEvSums;
  const int blocks = int(std::min<long long>((HW + kEvThreads - 1) / kEvThreads, kEvBlocks));
  eval_align_sums_kernel<<<blocks, kEvThreads, 0, stream>>>(pred, gt, mask, HW, part);
  eval_align_solve_kernel<<<1, 32, 0, stream>>>(part, blocks, do_align, st);
  eval_metric_sums_kernel<<<blocks, kEvThreads, 0, stream>>>(pred, gt, mask, HW, st, dmin, dmax, aligned_out, part);
  eval_metric_final_kernel<<<1, 32, 0, stream>>>(part, blocks, st, out_dev);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error("eval_depth launch: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  return MGB_OK;
}

}  // namespace mgb
