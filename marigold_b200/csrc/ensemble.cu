// Test-time ensembling on the device (reference marigold/util/ensemble.py).
//
//  * ens_depth_cost   : the BFGS objective of ensemble_depth (ensemble.py:138-152) at a base point and, optionally,
//                       the 2E forward-difference points of one scipy gradient, in ONE host synchronisation (the
//                       reference does C(E,2)+2 `.item()` syncs per point). E <= 16: a base pass and a pass that
//                       only updates what one perturbed coordinate changes; E > 16: one generic pass per point
//                       (grid.y). The E maps are L2-resident (E x 2.4 MB at 768 px), so re-reading them per point
//                       costs L2 bandwidth only. Every value is bit-identical to the point evaluated alone.
//  * ens_depth_reduce : align (ensemble.py:107-118) + median/mean (+MAD/std) (:120-136) + min-max
//                       renormalisation (:184-194), plus the index of the member the lower median picks.
//  * ens_normals      : ensemble_normals (:199-249): mean -> normalise -> cosine -> clamp -> argmax -> gather.
//
// These are HBM-bound streaming kernels: each reads the E maps exactly once (E*4 bytes / pixel).
// Arithmetic that decides an index (median / argmax) uses explicitly un-fused fp32 ops
// (__fmul_rn/__fadd_rn) in the reference's operation order so that ties break identically.
#include <algorithm>
#include <cfloat>
#include <type_traits>

#include "common.cuh"
#include "kernels.h"
#include "launch.h"

namespace mgb {

constexpr int kEnsThreads = 256;
constexpr int kEnsMaxBlocks = kNumSMs * 4;    // reduce / normals kernels
constexpr int kEnsCostBlocks = kNumSMs * 2;   // register-resident cost kernels: blocks per pass
constexpr int kEnsDynMaxE = 64;
constexpr int kEnsMaxP = 2 * kEnsDynMaxE + 1;   // points per cost call: a base point and its forward-difference points
constexpr int kDynPairs = 32;              // pairs per blockIdx.z chunk of the generic cost kernel
constexpr int kDynBlocks = 48;
constexpr size_t kDynPartialBytes = size_t(16) << 20;

__device__ __forceinline__ float align1(float d, float s, float t, int shift) {
  // torch: depth * s + t  (two roundings; no FMA)
  const float m = __fmul_rn(d, s);
  return shift ? __fadd_rn(m, t) : m;
}

template <int E>
__device__ __forceinline__ void sort_small(float (&v)[E], int (&idx)[E]) {
#pragma unroll
  for (int i = 1; i < E; ++i) {
#pragma unroll
    for (int j = i; j > 0; --j) {
      // stable: only swap on strict greater, so equal values keep ascending member index
      if (v[j - 1] > v[j]) {
        const float tv = v[j]; v[j] = v[j - 1]; v[j - 1] = tv;
        const int ti = idx[j]; idx[j] = idx[j - 1]; idx[j - 1] = ti;
      }
    }
  }
}

struct CostPartial {
  double pair_sum[kEnsMaxE * (kEnsMaxE - 1) / 2];
  float pmin, pmax;
};

// Block-level reduction of one fp32 accumulator to a double (fixed order: xor tree inside a warp, warps in index order)
__device__ __forceinline__ double block_sum_double(float v, double* sh /* [kEnsThreads / 32] */) {
  double d = double(v);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = d;
  __syncthreads();
  double tot = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kEnsThreads / 32; ++w) tot += sh[w];
  __syncthreads();
  return tot;   // valid in thread 0
}
__device__ __forceinline__ void block_minmax(float& pmin, float& pmax, float (*shf)[kEnsThreads / 32]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    pmin = fminf(pmin, __shfl_xor_sync(0xffffffffu, pmin, o));
    pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, o));
  }
  if ((threadIdx.x & 31) == 0) { shf[0][threadIdx.x >> 5] = pmin; shf[1][threadIdx.x >> 5] = pmax; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < kEnsThreads / 32; ++w) { pmin = fminf(pmin, shf[0][w]); pmax = fmaxf(pmax, shf[1][w]); }
  __syncthreads();
}

// One block's share of the objective for ONE parameter set: E (E - 1) / 2 pair sums + min / max of the ensembled map.
// v3_out (optional, median only): per pixel the order statistics v[R-1], v[R], v[R+1] of the aligned values around the
// lower-median rank R (-FLT_MAX / FLT_MAX where they do not exist), for the forward-difference rows.
template <int E>
__device__ __forceinline__ void cost_block(const float* __restrict__ depth, const float* __restrict__ st, long long HW,
                                           int shift, int median, CostPartial* __restrict__ out,
                                           float* __restrict__ v3_out = nullptr) {
  constexpr int NP = E * (E - 1) / 2;
  float s[E], t[E];
#pragma unroll
  for (int e = 0; e < E; ++e) { s[e] = st[e]; t[e] = st[E + e]; }
  float acc[NP];
#pragma unroll
  for (int k = 0; k < NP; ++k) acc[k] = 0.f;
  float pmin = FLT_MAX, pmax = -FLT_MAX;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    float a[E];
#pragma unroll
    for (int e = 0; e < E; ++e) a[e] = align1(__ldg(depth + (long long)e * HW + p), s[e], t[e], shift);
    int k = 0;
#pragma unroll
    for (int i = 0; i < E; ++i)
#pragma unroll
      for (int j = i + 1; j < E; ++j) {
        const float d = a[i] - a[j];
        acc[k] = fmaf(d, d, acc[k]);
        ++k;
      }
    float pred;
    if (median) {
      int idx[E];
#pragma unroll
      for (int e = 0; e < E; ++e) idx[e] = e;
      sort_small<E>(a, idx);
      constexpr int R = (E - 1) / 2;
      pred = a[R];
      if (v3_out) {
        v3_out[3 * p + 0] = R > 0 ? a[R > 0 ? R - 1 : 0] : -FLT_MAX;
        v3_out[3 * p + 1] = a[R];
        v3_out[3 * p + 2] = R + 1 < E ? a[R + 1 < E ? R + 1 : R] : FLT_MAX;
      }
    } else {
      float sm = 0.f;
#pragma unroll
      for (int e = 0; e < E; ++e) sm += a[e];
      pred = sm / float(E);
    }
    pmin = fminf(pmin, pred);
    pmax = fmaxf(pmax, pred);
  }
  __shared__ double sh[kEnsThreads / 32];
  __shared__ float shf[2][kEnsThreads / 32];
#pragma unroll 1
  for (int k = 0; k < NP; ++k) {
    const double tot = block_sum_double(acc[k], sh);
    if (threadIdx.x == 0) out->pair_sum[k] = tot;
  }
  block_minmax(pmin, pmax, shf);
  if (threadIdx.x == 0) { out->pmin = pmin; out->pmax = pmax; }
}

// ---- E <= 16: the objective and one forward-difference gradient in ONE round trip: the base point plus the n = 2E (or
// E) single-coordinate perturbations scipy's approx_derivative evaluates. Perturbing member m only changes the E - 1
// pairs (m, j) and moves one element of the per-pixel order statistics, so after the base pass (which also stores three
// order statistics per pixel) block row m of the perturbation pass recomputes just those, without sorting: ~5x less
// arithmetic than 2E + 1 independent evaluations. Every sum is formed exactly as cost_block forms it (same
// pixel-to-thread map, same reduction order), and the final kernel assembles each perturbed objective from base +
// perturbed pair sums in pair order, so each value equals the base pass run at that point, bit for bit
// (tests/test_ensemble_gpu.py).
struct PertPartial {
  double pair_sum[2][kEnsMaxE];   // [s' | t'][other member j]
  float pmin[2], pmax[2];
};

// v3 (median only; null for a point without perturbations): the order statistics the perturbation pass reads
template <int E>
__global__ void __launch_bounds__(kEnsThreads)
    ens_cost_base_kernel(const float* __restrict__ depth, const float* __restrict__ st, long long HW, int shift, int median,
                         CostPartial* __restrict__ base_part, float* __restrict__ v3) {
  cost_block<E>(depth, st, HW, shift, median, base_part + blockIdx.x, median ? v3 : nullptr);
}

// block row m: member m perturbed (s_m -> s', and t_m -> t' when shift): the E - 1 pair sums with the other members, and
// min / max of the re-ensembled map. No sort here: with v = the sorted base values (from ens_cost_base_kernel) and w = v
// without one instance of a_m, the perturbed lower median is clamp(x', w[R-1], w[R]), where
//   a_m <= v[R-1]          : w[R-1] = v[R],   w[R] = v[R+1]
//   v[R-1] < a_m <= v[R]   : w[R-1] = v[R-1], w[R] = v[R+1]      (a_m is v[R])
//   a_m > v[R]             : w[R-1] = v[R-1], w[R] = v[R]
template <int E>
__global__ void __launch_bounds__(kEnsThreads)
    ens_cost_pert_kernel(const float* __restrict__ depth, const float* __restrict__ st /* [2E] base */,
                         const float* __restrict__ pert /* [2E]: s'_0..s'_{E-1} | t'_0..t'_{E-1} */, long long HW, int shift,
                         int median, const float* __restrict__ v3, PertPartial* __restrict__ pert_part) {
  const int m = blockIdx.y;
  const int nk = shift ? 2 : 1;
  float s[E], t[E];
#pragma unroll
  for (int e = 0; e < E; ++e) { s[e] = st[e]; t[e] = st[E + e]; }
  const float sp = pert[m], tp = pert[E + m];
  const float sm_base = st[m], tm_base = st[E + m];
  float acc0[E], acc1[E];
#pragma unroll
  for (int e = 0; e < E; ++e) { acc0[e] = 0.f; acc1[e] = 0.f; }
  float mn0 = FLT_MAX, mx0 = -FLT_MAX, mn1 = FLT_MAX, mx1 = -FLT_MAX;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    float a[E];
#pragma unroll
    for (int e = 0; e < E; ++e) a[e] = align1(__ldg(depth + (long long)e * HW + p), s[e], t[e], shift);
    const float dm = __ldg(depth + (long long)m * HW + p);
    const float am = align1(dm, sm_base, tm_base, shift);
    const float x0 = align1(dm, sp, tm_base, shift);      // s_m perturbed
    const float x1 = align1(dm, sm_base, tp, shift);      // t_m perturbed
#pragma unroll
    for (int j = 0; j < E; ++j) {
      // (the j == m slot accumulates (x' - a_m)^2 and is never read)
      const float d0 = x0 - a[j], d1 = x1 - a[j];
      acc0[j] = fmaf(d0, d0, acc0[j]);
      acc1[j] = fmaf(d1, d1, acc1[j]);
    }
    float p0, p1;
    if (median) {
      const float vlo = __ldg(v3 + 3 * p), vmid = __ldg(v3 + 3 * p + 1), vhi = __ldg(v3 + 3 * p + 2);
      float lo, hi;
      if (am <= vlo) { lo = vmid; hi = vhi; }
      else if (am <= vmid) { lo = vlo; hi = vhi; }
      else { lo = vlo; hi = vmid; }
      p0 = fminf(fmaxf(x0, lo), hi);
      p1 = fminf(fmaxf(x1, lo), hi);
    } else {
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int e = 0; e < E; ++e) { s0 += (e == m ? x0 : a[e]); s1 += (e == m ? x1 : a[e]); }
      p0 = s0 / float(E); p1 = s1 / float(E);
    }
    mn0 = fminf(mn0, p0); mx0 = fmaxf(mx0, p0);
    mn1 = fminf(mn1, p1); mx1 = fmaxf(mx1, p1);
  }
  __shared__ double sh[kEnsThreads / 32];
  __shared__ float shf[2][kEnsThreads / 32];
  PertPartial* out = pert_part + size_t(m) * gridDim.x + blockIdx.x;
#pragma unroll
  for (int j = 0; j < E; ++j) {
    const double t0 = block_sum_double(acc0[j], sh);
    const double t1 = nk == 2 ? block_sum_double(acc1[j], sh) : 0.0;
    if (threadIdx.x == 0) { out->pair_sum[0][j] = t0; out->pair_sum[1][j] = t1; }
  }
  block_minmax(mn0, mx0, shf);
  block_minmax(mn1, mx1, shf);
  if (threadIdx.x == 0) { out->pmin[0] = mn0; out->pmax[0] = mx0; out->pmin[1] = mn1; out->pmax[1] = mx1; }
}

// Sum over the blocks' partials of one pair, one warp per call: lane l takes blocks l, l + 32, ...; xor tree. Base and
// perturbed pair sums are combined the same way, so a pair total has ONE value no matter which pass produced it.
template <typename F>
__device__ __forceinline__ double warp_total(int nblocks, F&& get) {
  double tot = 0.0;
  for (int b = threadIdx.x & 31; b < nblocks; b += 32) tot += get(b);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
  return tot;
}

// {cost, min, max} of one point from its summed pair RMSEs and the range of its ensembled map (ensemble.py:147-152)
__device__ __forceinline__ void store_cost(double cost, float pmin, float pmax, double reg, double* out) {
  if (reg > 0.0) cost += (double(fabsf(0.0f - pmin)) + double(fabsf(1.0f - pmax))) * reg;
  out[0] = cost;
  out[1] = double(pmin);
  out[2] = double(pmax);
}

// one block per point q: 0 = the base point; q >= 1: coordinate i = q - 1 perturbed (i < E: s_i, else t_{i-E});
// one warp per pair (warps stride over the pairs)
__global__ void __launch_bounds__(256) ens_cost_final_kernel(const CostPartial* __restrict__ base_part,
                                                             const PertPartial* __restrict__ pert_part, int nblocks, int E,
                                                             long long HW, double reg, double* __restrict__ out_all) {
  const int q = blockIdx.x;
  const int m = q == 0 ? -1 : (q - 1) % E, kk = q == 0 ? 0 : (q - 1) / E;
  const PertPartial* fp = q == 0 ? nullptr : pert_part + size_t(m) * nblocks;
  const int NP = E * (E - 1) / 2;
  __shared__ double c[kEnsMaxE * (kEnsMaxE - 1) / 2];
  for (int k = threadIdx.x >> 5; k < NP; k += blockDim.x >> 5) {
    int i = 0, r = k;                                       // pair index -> (i, j), torch.combinations order
    while (r >= E - 1 - i) { r -= E - 1 - i; ++i; }
    const int j = i + 1 + r;
    double tot;
    if (i == m) tot = warp_total(nblocks, [&](int b) { return fp[b].pair_sum[kk][j]; });
    else if (j == m) tot = warp_total(nblocks, [&](int b) { return fp[b].pair_sum[kk][i]; });
    else tot = warp_total(nblocks, [&](int b) { return base_part[b].pair_sum[k]; });
    // reference: (diff**2).mean().sqrt() evaluated in fp32
    if ((threadIdx.x & 31) == 0) c[k] = double(sqrtf(float(tot / double(HW))));
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    float pmin = FLT_MAX, pmax = -FLT_MAX;
    for (int b = threadIdx.x; b < nblocks; b += 32) {
      pmin = fminf(pmin, q == 0 ? base_part[b].pmin : fp[b].pmin[kk]);
      pmax = fmaxf(pmax, q == 0 ? base_part[b].pmax : fp[b].pmax[kk]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      pmin = fminf(pmin, __shfl_xor_sync(0xffffffffu, pmin, o));
      pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, o));
    }
    if (threadIdx.x == 0) {
      double cost = 0.0;
      for (int k = 0; k < NP; ++k) cost += c[k];          // pair order, like the reference's Python loop
      store_cost(cost, pmin, pmax, reg, out_all + 3 * q);
    }
  }
}

// ---- generic ensemble size (E > 16): values in local memory, pairs in chunks of 32 over blockIdx.z ------------------
// lower median with torch's stable tie order = the element whose rank (count of smaller values, plus equal values with
// a smaller member index) is (E-1)/2
__device__ __forceinline__ float select_lower_median(const float* a, int E, int* pick) {
  const int r = (E - 1) / 2;
  for (int e = 0; e < E; ++e) {
    int rank = 0;
    const float v = a[e];
    for (int j = 0; j < E; ++j) rank += (a[j] < v) || (a[j] == v && j < e);
    if (rank == r) { if (pick) *pick = e; return v; }
  }
  if (pick) *pick = 0;
  return a[0];   // unreachable for finite inputs
}

__global__ void __launch_bounds__(kEnsThreads)
    ens_cost_dyn_kernel(const float* __restrict__ depth, const float* __restrict__ st_all, int E, long long HW, int shift,
                        int median, double* __restrict__ pair_part /* [P][NP][gridDim.x] */,
                        float* __restrict__ mm_part /* [P][gridDim.x][2] */) {
  const int NP = E * (E - 1) / 2;
  const int ps = blockIdx.y, k0 = blockIdx.z * kDynPairs, nk = min(kDynPairs, NP - k0);
  __shared__ float s_s[kEnsDynMaxE], s_t[kEnsDynMaxE];
  __shared__ unsigned char s_pi[kDynPairs], s_pj[kDynPairs];
  __shared__ double sh[kEnsThreads / 32];
  __shared__ float shf[2][kEnsThreads / 32];
  if (threadIdx.x < E) { s_s[threadIdx.x] = st_all[size_t(ps) * 2 * E + threadIdx.x]; s_t[threadIdx.x] = st_all[size_t(ps) * 2 * E + E + threadIdx.x]; }
  if (threadIdx.x < kDynPairs) {
    // pair index k0 + threadIdx.x in torch.combinations order: (0,1), (0,2), ..., (1,2), ...
    int k = k0 + threadIdx.x, i = 0;
    while (i < E - 1 && k >= E - 1 - i) { k -= E - 1 - i; ++i; }
    s_pi[threadIdx.x] = (unsigned char)min(i, E - 1);
    s_pj[threadIdx.x] = (unsigned char)min(i + 1 + k, E - 1);
  }
  __syncthreads();
  float acc[kDynPairs];
#pragma unroll
  for (int k = 0; k < kDynPairs; ++k) acc[k] = 0.f;
  float pmin = FLT_MAX, pmax = -FLT_MAX;
  float a[kEnsDynMaxE];
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    for (int e = 0; e < E; ++e) a[e] = align1(__ldg(depth + (long long)e * HW + p), s_s[e], s_t[e], shift);
#pragma unroll
    for (int k = 0; k < kDynPairs; ++k) {
      if (k < nk) {
        const float d = a[s_pi[k]] - a[s_pj[k]];
        acc[k] = fmaf(d, d, acc[k]);
      }
    }
    if (blockIdx.z == 0) {
      float pred;
      if (median) {
        pred = select_lower_median(a, E, nullptr);
      } else {
        float sm = 0.f;
        for (int e = 0; e < E; ++e) sm += a[e];
        pred = sm / float(E);
      }
      pmin = fminf(pmin, pred);
      pmax = fmaxf(pmax, pred);
    }
  }
#pragma unroll
  for (int k = 0; k < kDynPairs; ++k) {
    if (k >= nk) break;
    const double tot = block_sum_double(acc[k], sh);
    if (threadIdx.x == 0) pair_part[(size_t(ps) * NP + k0 + k) * gridDim.x + blockIdx.x] = tot;
  }
  if (blockIdx.z == 0) {
    block_minmax(pmin, pmax, shf);
    if (threadIdx.x == 0) {
      mm_part[(size_t(ps) * gridDim.x + blockIdx.x) * 2] = pmin;
      mm_part[(size_t(ps) * gridDim.x + blockIdx.x) * 2 + 1] = pmax;
    }
  }
}

__global__ void ens_cost_dyn_final_kernel(const double* __restrict__ pair_part, const float* __restrict__ mm_part, int nblocks,
                                          int E, long long HW, double reg, double* __restrict__ out_all) {
  const int NP = E * (E - 1) / 2, ps = blockIdx.x;
  __shared__ double sh[128];
  double c = 0.0;
  for (int k = threadIdx.x; k < NP; k += blockDim.x) {
    double tot = 0.0;
    for (int b = 0; b < nblocks; ++b) tot += pair_part[(size_t(ps) * NP + k) * nblocks + b];
    c += double(sqrtf(float(tot / double(HW))));
  }
  sh[threadIdx.x] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    double cost = 0.0;
    for (int i = 0; i < int(blockDim.x); ++i) cost += sh[i];
    float pmin = FLT_MAX, pmax = -FLT_MAX;
    for (int b = 0; b < nblocks; ++b) {
      pmin = fminf(pmin, mm_part[(size_t(ps) * nblocks + b) * 2]);
      pmax = fmaxf(pmax, mm_part[(size_t(ps) * nblocks + b) * 2 + 1]);
    }
    store_cost(cost, pmin, pmax, reg, out_all + 3 * ps);
  }
}

// ws layout: [partials: max(register-resident: base + E perturbation rows per block, generic: kDynPartialBytes + min/max)]
//            [st: kEnsMaxP x 2 kEnsDynMaxE floats][out: kEnsMaxP x 3 doubles]
static size_t ens_partial_bytes() {
  const size_t t = (sizeof(CostPartial) + sizeof(PertPartial) * kEnsMaxE) * kEnsCostBlocks;
  const size_t d = kDynPartialBytes + size_t(kEnsMaxP) * kDynBlocks * 2 * sizeof(float);
  return (std::max(t, d) + 255) & ~size_t(255);
}
size_t ens_ws_bytes() {
  return ens_partial_bytes() + size_t(kEnsMaxP) * 2 * kEnsDynMaxE * sizeof(float) + size_t(kEnsMaxP) * 3 * sizeof(double) + 256;
}
static float* ens_ws_st(void* ws) { return reinterpret_cast<float*>(static_cast<char*>(ws) + ens_partial_bytes()); }
static double* ens_ws_out(void* ws) { return reinterpret_cast<double*>(ens_ws_st(ws) + size_t(kEnsMaxP) * 2 * kEnsDynMaxE); }
int ens_max_batch() { return kEnsMaxP; }
int ens_max_members() { return kEnsDynMaxE; }

// f(std::integral_constant<int, E>()) for the register-resident sizes E <= kEnsMaxE, f(std::integral_constant<int, 0>())
// for the larger ones; returns what f returns
template <typename F>
static int dispatch_members(int E, F&& f) {
  switch (E) {
#define CASE(n) case n: return f(std::integral_constant<int, n>());
    CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8) CASE(9) CASE(10) CASE(11) CASE(12) CASE(13) CASE(14)
    CASE(15) CASE(16)
#undef CASE
  }
  return f(std::integral_constant<int, 0>());
}

int launch_ens_depth_cost(const float* depth, float* st_host, int n, int E, long long HW, int shift, int median,
                          double reg, void* ws, float* v3, double* out_host_pinned, cudaStream_t stream) {
  if (E < 1 || E > kEnsDynMaxE) { set_error("ensemble size %d outside [1, %d]", E, kEnsDynMaxE); return MGB_ERR_UNSUPPORTED; }
  const int P = 1 + n;
  int rows = n > 0 ? 2 : 1;
  if (!ens_register_resident(E) && n > 0) {
    // the generic kernels evaluate whole points: row 1 + i = the base with coordinate i moved (each coordinate was
    // converted to float on its own, so these are the rows of the moved double vectors)
    float moved[2 * kEnsDynMaxE];
    std::copy(st_host + 2 * E, st_host + 4 * E, moved);
    for (int i = 0; i < n; ++i) {
      float* row = st_host + size_t(1 + i) * 2 * E;
      std::copy(st_host, st_host + 2 * E, row);
      row[i] = moved[i];
    }
    rows = P;
  }
  float* st = ens_ws_st(ws);
  double* out = ens_ws_out(ws);
  cudaError_t e = cudaMemcpyAsync(st, st_host, sizeof(float) * 2 * E * rows, cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) { set_error("ens cost H2D: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  TRY(dispatch_members(E, [&](auto members) -> int {
    constexpr int kE = decltype(members)::value;
    if constexpr (kE > 0) {
      CostPartial* base_part = reinterpret_cast<CostPartial*>(ws);
      PertPartial* pert_part = reinterpret_cast<PertPartial*>(base_part + kEnsCostBlocks);
      const int blocks = int(std::min<long long>((HW + kEnsThreads - 1) / kEnsThreads, kEnsCostBlocks));
      TRY(launch_plain("ens cost", ens_cost_base_kernel<kE>, blocks, kEnsThreads, 0, stream, depth, st, HW, shift, median,
                       base_part, n > 0 ? v3 : nullptr));
      if (n > 0)
        TRY(launch_plain("ens cost", ens_cost_pert_kernel<kE>, dim3(blocks, E), kEnsThreads, 0, stream, depth, st,
                         st + 2 * E, HW, shift, median, v3, pert_part));
      return launch_plain("ens cost", ens_cost_final_kernel, P, 256, 0, stream, base_part, pert_part, blocks, E, HW, reg,
                          out);
    } else {
      // one member (no pairs: the objective is the regulariser alone) still takes one z-slice for the min / max
      const int NP = E * (E - 1) / 2, chunks = std::max(1, (NP + kDynPairs - 1) / kDynPairs);
      const int blocks = int(std::min<long long>((HW + kEnsThreads - 1) / kEnsThreads, kDynBlocks));
      double* pair_part = reinterpret_cast<double*>(ws);
      float* mm_part = reinterpret_cast<float*>(static_cast<char*>(ws) + kDynPartialBytes);
      const int p_max = std::max<int>(1, int(kDynPartialBytes / (size_t(std::max(NP, 1)) * blocks * sizeof(double))));
      for (int p0 = 0; p0 < P; p0 += p_max) {
        const int pn = std::min(p_max, P - p0);
        TRY(launch_plain("ens cost", ens_cost_dyn_kernel, dim3(blocks, pn, chunks), kEnsThreads, 0, stream, depth,
                         st + size_t(p0) * 2 * E, E, HW, shift, median, pair_part, mm_part));
        TRY(launch_plain("ens cost", ens_cost_dyn_final_kernel, pn, 128, 0, stream, pair_part, mm_part, blocks, E, HW, reg,
                         out + 3 * p0));
      }
      return MGB_OK;
    }
  }));
  e = cudaMemcpyAsync(out_host_pinned, out, size_t(P) * 3 * sizeof(double), cudaMemcpyDeviceToHost, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e != cudaSuccess) { set_error("ens cost: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  return MGB_OK;
}

// ---- per-member min / max (init_param, ensemble.py:91-105) ----------------------------------------
__global__ void __launch_bounds__(kEnsThreads) ens_minmax_kernel(const float* __restrict__ depth, long long HW,
                                                                 float* __restrict__ out /* [E, gridDim.x, 2] */) {
  const int e = blockIdx.y;
  float mn = FLT_MAX, mx = -FLT_MAX;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    const float v = __ldg(depth + (long long)e * HW + p);
    mn = fminf(mn, v); mx = fmaxf(mx, v);
  }
  __shared__ float sh[2][kEnsThreads / 32];
  block_minmax(mn, mx, sh);
  if (threadIdx.x == 0) {
    out[((long long)e * gridDim.x + blockIdx.x) * 2 + 0] = mn;
    out[((long long)e * gridDim.x + blockIdx.x) * 2 + 1] = mx;
  }
}

int launch_ens_minmax(const float* depth, int E, long long HW, float* ws, float* host_pinned, int* blocks_out,
                      cudaStream_t stream) {
  const int blocks = int(std::min<long long>((HW + kEnsThreads - 1) / kEnsThreads, 64));
  dim3 grid(blocks, E);
  TRY(launch_plain("ens minmax", ens_minmax_kernel, grid, kEnsThreads, 0, stream, depth, HW, ws));
  cudaError_t e = cudaMemcpyAsync(host_pinned, ws, sizeof(float) * 2 * blocks * E, cudaMemcpyDeviceToHost, stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  if (e != cudaSuccess) { set_error("ens minmax: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  *blocks_out = blocks;
  return MGB_OK;
}

// ---- reduce: align + (median | mean) (+ uncertainty) ; then global min-max renormalisation ------
// lower median with torch's stable tie order: its value, and in *pick (when given) the member it comes from. kE > 0:
// sorting network over kE register values; kE = 0: rank counting over E values (the same value and member).
template <int kE, int N>
__device__ __forceinline__ float lower_median(const float (&a)[N], int E, int* pick) {
  if constexpr (kE > 0) {
    float v[kE]; int idx[kE];
#pragma unroll
    for (int e = 0; e < kE; ++e) { v[e] = a[e]; idx[e] = e; }
    sort_small<kE>(v, idx);
    if (pick) *pick = idx[(kE - 1) / 2];
    return v[(kE - 1) / 2];
  } else {
    return select_lower_median(a, E, pick);
  }
}

// kE > 0: exactly kE members, values in registers; kE = 0: any E <= kEnsDynMaxE members, values in local memory
template <int kE>
__global__ void __launch_bounds__(kEnsThreads)
    ens_reduce_kernel(const float* __restrict__ depth, const float* __restrict__ st, int n_members, long long HW, int shift,
                      int median, float* __restrict__ pred_out, float* __restrict__ unc_out,
                      int* __restrict__ idx_out, float* __restrict__ bmm) {
  constexpr int N = kE > 0 ? kE : kEnsDynMaxE;
  const int E = kE > 0 ? kE : n_members;
  __shared__ float s_s[N], s_t[N];
  if (threadIdx.x < E) { s_s[threadIdx.x] = st[threadIdx.x]; s_t[threadIdx.x] = st[E + threadIdx.x]; }
  __syncthreads();
  float pmin = FLT_MAX, pmax = -FLT_MAX;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    float a[N];
#pragma unroll
    for (int e = 0; e < E; ++e) a[e] = align1(__ldg(depth + (long long)e * HW + p), s_s[e], s_t[e], shift);
    float pred, unc = 0.f;
    int pick = -1;
    if (median) {
      pred = lower_median<kE>(a, E, &pick);        // torch.median: LOWER median for even E
      if (unc_out) {
        float dv[N];
#pragma unroll
        for (int e = 0; e < E; ++e) dv[e] = fabsf(a[e] - pred);
        unc = lower_median<kE>(dv, E, nullptr);    // MAD
      }
    } else {
      float sm = 0.f;
#pragma unroll
      for (int e = 0; e < E; ++e) sm += a[e];
      pred = sm / float(E);
      if (unc_out) {                    // torch.std: unbiased
        float q = 0.f;
#pragma unroll
        for (int e = 0; e < E; ++e) { const float d = a[e] - pred; q += d * d; }
        unc = sqrtf(q / float(E - 1));
      }
    }
    pred_out[p] = pred;
    if (unc_out) unc_out[p] = unc;
    if (idx_out) idx_out[p] = pick;
    pmin = fminf(pmin, pred); pmax = fmaxf(pmax, pred);
  }
  __shared__ float shf[2][kEnsThreads / 32];
  block_minmax(pmin, pmax, shf);
  if (threadIdx.x == 0) { bmm[2 * blockIdx.x] = pmin; bmm[2 * blockIdx.x + 1] = pmax; }
}

__global__ void __launch_bounds__(kEnsThreads)
    ens_renorm_kernel(float* __restrict__ pred, float* __restrict__ unc, long long HW, const float* __restrict__ bmm,
                      int nblocks, int use_min) {
  __shared__ float s_min, s_rng;
  __shared__ float shf[2][kEnsThreads / 32];
  {
    float mn = FLT_MAX, mx = -FLT_MAX;
    for (int b = threadIdx.x; b < nblocks; b += blockDim.x) { mn = fminf(mn, bmm[2 * b]); mx = fmaxf(mx, bmm[2 * b + 1]); }
    block_minmax(mn, mx, shf);
    if (threadIdx.x == 0) {
      if (!use_min) mn = 0.f;                     // scale-only alignment: depth_min = 0 (ensemble.py:187-188)
      s_min = mn;
      s_rng = fmaxf(mx - mn, 1e-6f);              // .clamp(min=1e-6)
    }
  }
  __syncthreads();
  const float mn = s_min, rng = s_rng;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    pred[p] = (pred[p] - mn) / rng;
    if (unc) unc[p] = unc[p] / rng;
  }
}

int launch_ens_depth_reduce(const float* depth, const float* st_host, int E, long long HW, int shift, int median,
                            int use_min, float* pred, float* unc, int* idx, void* ws, cudaStream_t stream) {
  if (E < 1 || E > kEnsDynMaxE) { set_error("ensemble size %d outside [1, %d]", E, kEnsDynMaxE); return MGB_ERR_UNSUPPORTED; }
  float* st = ens_ws_st(ws);
  float* bmm = reinterpret_cast<float*>(ws);  // reuse the partial area for block min/max
  cudaError_t e = cudaMemcpyAsync(st, st_host, sizeof(float) * 2 * E, cudaMemcpyHostToDevice, stream);
  if (e != cudaSuccess) { set_error("ens reduce H2D: %s", cudaGetErrorString(e)); return MGB_ERR_CUDA; }
  const int blocks = int(std::min<long long>((HW + kEnsThreads - 1) / kEnsThreads, kEnsMaxBlocks));
  TRY(dispatch_members(E, [&](auto members) -> int {
    return launch_plain("ens reduce", ens_reduce_kernel<decltype(members)::value>, blocks, kEnsThreads, 0, stream, depth, st,
                        E, HW, shift, median, pred, unc, idx, bmm);
  }));
  return launch_plain("ens renorm", ens_renorm_kernel, blocks, kEnsThreads, 0, stream, pred, unc, HW, bmm, blocks, use_min);
}

// ---- ensemble_iid (ensemble.py:252-270): per element, plain median (+ MAD) or mean (+ unbiased std) over E ------------
__global__ void __launch_bounds__(kEnsThreads)
    ens_iid_kernel(const float* __restrict__ x, int E, long long N, int median, float* __restrict__ pred,
                   float* __restrict__ unc) {
  float a[kEnsDynMaxE], dv[kEnsDynMaxE];
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (long long)gridDim.x * blockDim.x) {
    for (int e = 0; e < E; ++e) a[e] = __ldg(x + (long long)e * N + p);
    float pr, u = 0.f;
    if (median) {
      pr = select_lower_median(a, E, nullptr);            // torch.median: lower median for even E
      if (unc) {
        for (int e = 0; e < E; ++e) dv[e] = fabsf(a[e] - pr);
        u = select_lower_median(dv, E, nullptr);
      }
    } else {
      float sm = 0.f;
      for (int e = 0; e < E; ++e) sm += a[e];
      pr = sm / float(E);
      if (unc) {
        float q = 0.f;
        for (int e = 0; e < E; ++e) { const float d = a[e] - pr; q += d * d; }
        u = sqrtf(q / float(E - 1));
      }
    }
    pred[p] = pr;
    if (unc) unc[p] = u;
  }
}

int launch_ens_iid(const float* x, int E, long long N, int median, float* pred, float* unc, cudaStream_t stream) {
  if (E < 1 || E > kEnsDynMaxE) { set_error("ensemble size %d outside [1, %d]", E, kEnsDynMaxE); return MGB_ERR_UNSUPPORTED; }
  const int blocks = int(std::min<long long>((N + kEnsThreads - 1) / kEnsThreads, kEnsMaxBlocks * 4));
  return launch_plain("ens iid", ens_iid_kernel, blocks, kEnsThreads, 0, stream, x, E, N, median, pred, unc);
}

// ---- ensemble_normals -------------------------------------------------------------------------------
__global__ void __launch_bounds__(kEnsThreads)
    ens_normals_kernel(const float* __restrict__ nrm, int E, long long HW, int closest, float* __restrict__ out,
                       float* __restrict__ unc, int* __restrict__ idx_out) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (long long)gridDim.x * blockDim.x) {
    // mean over members: sequential fp32 sum in member order, then one division (torch CPU mean)
    float mx = 0.f, my = 0.f, mz = 0.f;
    for (int e = 0; e < E; ++e) {
      const float* q = nrm + ((long long)e * 3) * HW + p;
      mx = __fadd_rn(mx, __ldg(q)); my = __fadd_rn(my, __ldg(q + HW)); mz = __fadd_rn(mz, __ldg(q + 2 * HW));
    }
    mx = __fdiv_rn(mx, float(E)); my = __fdiv_rn(my, float(E)); mz = __fdiv_rn(mz, float(E));
    const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), __fmul_rn(mz, mz));
    const float nn = fmaxf(__fsqrt_rn(n2), 1e-6f);
    mx = __fdiv_rn(mx, nn); my = __fdiv_rn(my, nn); mz = __fdiv_rn(mz, nn);
    float best = -FLT_MAX, acc_unc = 0.f;
    int bi = 0;
    for (int e = 0; e < E; ++e) {
      const float* q = nrm + ((long long)e * 3) * HW + p;
      float sim = __fadd_rn(__fadd_rn(__fmul_rn(mx, __ldg(q)), __fmul_rn(my, __ldg(q + HW))),
                            __fmul_rn(mz, __ldg(q + 2 * HW)));
      sim = fminf(fmaxf(sim, -1.f), 1.f);
      if (sim > best) { best = sim; bi = e; }      // first maximum wins (torch.argmax)
      if (unc) acc_unc += acosf(sim);
    }
    if (unc) unc[p] = (acc_unc / float(E)) / 3.14159265358979323846f;
    if (closest) {
      const float* q = nrm + ((long long)bi * 3) * HW + p;
      out[p] = __ldg(q); out[HW + p] = __ldg(q + HW); out[2 * HW + p] = __ldg(q + 2 * HW);
    } else {
      out[p] = mx; out[HW + p] = my; out[2 * HW + p] = mz;
    }
    if (idx_out) idx_out[p] = bi;
  }
}

int launch_ens_normals(const float* nrm, int E, long long HW, int closest, float* out, float* unc, int* idx,
                       cudaStream_t stream) {
  if (E < 1) { set_error("ensemble size %d", E); return MGB_ERR_INVALID; }
  const int blocks = int(std::min<long long>((HW + kEnsThreads - 1) / kEnsThreads, kEnsMaxBlocks));
  return launch_plain("ens normals", ens_normals_kernel, blocks, kEnsThreads, 0, stream, nrm, E, HW, closest, out, unc, idx);
}

}  // namespace mgb
