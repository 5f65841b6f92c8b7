// C ABI, ensembling part (reference marigold/util/ensemble.py).
#include <algorithm>
#include <cfloat>
#include <vector>

#include "net.h"

using namespace mgb;

// pinned staging: [out: kMaxP x 3 doubles][st: kMaxP x 2 x maxE floats][min/max: maxE x 64 x 2 floats]
static size_t pinned_out_doubles() { return size_t(ens_max_batch()) * 3; }
static size_t pinned_bytes() {
  return pinned_out_doubles() * sizeof(double) + size_t(ens_max_batch()) * 2 * ens_max_members() * sizeof(float) +
         size_t(ens_max_members()) * 64 * 2 * sizeof(float);
}
static float* pinned_st(mgb_handle* h) { return reinterpret_cast<float*>(h->ens_pinned.get() + pinned_out_doubles()); }

// The device workspace and the pinned staging, allocated by the first call: the handle holds both or neither.
static int ens_prepare(mgb_handle* h) {
  if (!h) { set_error("null handle"); return MGB_ERR_INVALID; }
  int rc = h->ens_ws.grow(std::max(ens_ws_bytes(), size_t(ens_max_members()) * 64 * 2 * 4));
  if (!rc) rc = h->ens_pinned.grow(pinned_bytes());
  if (rc) h->ens_ws.reset();
  return rc;
}

static int make_st(const double* param, int E, int scale_inv, int shift_inv, float* st) {
  if (!scale_inv) {
    // reference: "Pure shift-invariant ensembling is not supported" (ensemble.py:88-89) / "Unrecognized alignment"
    set_error("ensemble_depth: alignment requires scale_invariant");
    return MGB_ERR_INVALID;
  }
  for (int e = 0; e < E; ++e) {
    st[e] = float(param[e]);                       // torch.from_numpy(s).to(depth): float64 -> float32
    st[E + e] = shift_inv ? float(param[E + e]) : 0.f;
  }
  return MGB_OK;
}

// The objective at base and, when pert is given, at the n points that each move one coordinate of base to its value
// in pert: costs_out [1 + n].
static int ens_depth_cost(mgb_handle* h, const float* depth, const double* base, const double* pert, int32_t E, int64_t HW,
                          int32_t scale_inv, int32_t shift_inv, int32_t median, double reg, double* costs_out,
                          void* stream) {
  int rc = ens_prepare(h);
  if (rc) return rc;
  if (!depth || !base || !costs_out || HW <= 0) { set_error("ens_depth_cost: bad argument"); return MGB_ERR_INVALID; }
  if (E < 1 || E > ens_max_members()) { set_error("ensemble size %d outside [1,%d]", E, ens_max_members()); return MGB_ERR_UNSUPPORTED; }
  const int n = pert ? (shift_inv ? 2 * E : E) : 0;
  // the staging area is reused by every call: wait for earlier users of this stream (each cost call ends with a
  // synchronisation, so this is only ever non-trivial after an asynchronous reduce)
  CUDA_TRY(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream)));
  float* st = pinned_st(h);
  rc = make_st(base, E, scale_inv, shift_inv, st);
  if (!rc && pert) rc = make_st(pert, E, scale_inv, shift_inv, st + 2 * E);
  if (rc) return rc;
  // per-pixel order statistics of the base point for the register-resident perturbation pass
  if (pert && ens_register_resident(E)) {
    rc = h->ens_v3.grow(size_t(HW) * 3 * sizeof(float));
    if (rc) return rc;
  }
  rc = launch_ens_depth_cost(depth, st, n, E, HW, shift_inv, median, reg, h->ens_ws, h->ens_v3, h->ens_pinned,
                             reinterpret_cast<cudaStream_t>(stream));
  if (rc) return rc;
  for (int i = 0; i <= n; ++i) costs_out[i] = h->ens_pinned[3 * i];
  return MGB_OK;
}

extern "C" {

int mgb_ens_depth_cost_fd(mgb_handle* h, const float* depth, const double* base, const double* pert, int32_t E, int64_t HW,
                          int32_t scale_inv, int32_t shift_inv, int32_t median, double reg, double* costs_out, void* stream) {
  if (!pert) { set_error("ens_depth_cost_fd: bad argument"); return MGB_ERR_INVALID; }
  return ens_depth_cost(h, depth, base, pert, E, HW, scale_inv, shift_inv, median, reg, costs_out, stream);
}

int mgb_ens_depth_cost(mgb_handle* h, const float* depth, const double* param, int32_t E, int64_t HW,
                       int32_t scale_inv, int32_t shift_inv, int32_t median, double reg, double* cost_out,
                       void* stream) {
  return ens_depth_cost(h, depth, param, nullptr, E, HW, scale_inv, shift_inv, median, reg, cost_out, stream);
}

int mgb_ens_max_members(void) { return ens_max_members(); }

int mgb_ens_minmax(mgb_handle* h, const float* depth, int32_t E, int64_t HW, float* min_host, float* max_host,
                   void* stream) {
  int rc = ens_prepare(h);
  if (rc) return rc;
  if (!depth || !min_host || !max_host || HW <= 0) { set_error("ens_minmax: bad argument"); return MGB_ERR_INVALID; }
  if (E < 1 || E > ens_max_members()) { set_error("ensemble size %d outside [1,%d]", E, ens_max_members()); return MGB_ERR_UNSUPPORTED; }
  int blocks = 0;
  CUDA_TRY(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream)));
  float* hp = pinned_st(h) + size_t(ens_max_batch()) * 2 * ens_max_members();
  rc = launch_ens_minmax(depth, E, HW, h->ens_ws, hp, &blocks,
                         reinterpret_cast<cudaStream_t>(stream));
  if (rc) return rc;
  for (int e = 0; e < E; ++e) {
    float mn = FLT_MAX, mx = -FLT_MAX;
    for (int b = 0; b < blocks; ++b) { mn = std::min(mn, hp[(e * blocks + b) * 2]); mx = std::max(mx, hp[(e * blocks + b) * 2 + 1]); }
    min_host[e] = mn; max_host[e] = mx;
  }
  return MGB_OK;
}

int mgb_ens_depth_reduce(mgb_handle* h, const float* depth, const double* param, int32_t E, int64_t HW,
                         int32_t scale_inv, int32_t shift_inv, int32_t median, float* pred, float* unc,
                         int32_t* member_idx, void* stream) {
  int rc = ens_prepare(h);
  if (rc) return rc;
  if (!depth || !param || !pred || HW <= 0) { set_error("ens_depth_reduce: bad argument"); return MGB_ERR_INVALID; }
  if (E < 1 || E > ens_max_members()) { set_error("ensemble size %d outside [1,%d]", E, ens_max_members()); return MGB_ERR_UNSUPPORTED; }
  CUDA_TRY(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream)));  // previous user of the staging area
  float* st_pinned = pinned_st(h);
  rc = make_st(param, E, scale_inv, shift_inv, st_pinned);
  if (rc) return rc;
  return launch_ens_depth_reduce(depth, st_pinned, E, HW, shift_inv, median, shift_inv ? 1 : 0, pred, unc, member_idx,
                                 h->ens_ws, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_ens_iid(mgb_handle* h, const float* targets, int32_t E, int64_t N, int32_t median, float* pred, float* unc,
                void* stream) {
  if (!h || !targets || !pred || N <= 0) { set_error("ens_iid: bad argument"); return MGB_ERR_INVALID; }
  return launch_ens_iid(targets, E, N, median, pred, unc, reinterpret_cast<cudaStream_t>(stream));
}

int mgb_ens_normals(mgb_handle* h, const float* normals, int32_t E, int64_t HW, int32_t closest, float* out,
                    float* unc, int32_t* member_idx, void* stream) {
  if (!h || !normals || !out || HW <= 0) { set_error("ens_normals: bad argument"); return MGB_ERR_INVALID; }
  return launch_ens_normals(normals, E, HW, closest, out, unc, member_idx, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
