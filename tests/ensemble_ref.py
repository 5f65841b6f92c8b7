"""Restatements of the ensembling kernels (csrc/ensemble.cu) for the tests, in plain torch on whatever device the inputs
live on. Nothing here calls the library.

Exact restatements. Wherever a kernel's arithmetic order is fixed, it is restated in float32 in that order, and the
device must return the same bits:
  * the alignment a = fl(fl(d * s) + t), un-fused, with s and t rounded from float64 as make_st does (`align`);
  * per-member min / max and the init_param built from them (`init_param`);
  * the lower median with torch's stable tie order, the member at position (E - 1) // 2 of a stable sort, and the
    MAD, the lower median of |a - med| (`lower_median`, `mad`);
  * the mean, a sequential fp32 sum in member order followed by one IEEE division (`seq_mean`);
  * the min-max renormalisation of an ensembled map and of its uncertainty (`renorm`);
  * ensemble_normals: sequential fp32 sums, the un-fused norm and dot product in x, y, z order, the clamps and the
    first maximum (`normals`), so the mean normals, the argmax and the gathered output.

Float64 restatements with a bound, for what the kernels sum in an order not restated here. u = 2^-24 and
gamma(n) = n u / (1 - n u):
  * Objective (`cost`). Pair k's sum S_k = sum_p fl(a_i - a_j)^2 is formed in float64 from the fp32 differences. The
    device accumulates each thread's pixels with an fp32 FMA chain: the square is exact inside the FMA and each step
    rounds once, so a thread's partial of n non-negative terms is within gamma(n) of its exact value. The partials
    are then summed in double (relative error ~1e-16 per block). The RMSE is sqrtf(float(S / HW)): the float cast adds
    u, the sqrt halves the relative error of its argument and rounds once more. Per pair,
        |rmse_dev - rmse| <= (gamma(n) / 2 + 2 u) rmse,   n = ceil(HW / (blocks * 256)),
    that is (n/2 + 2) u rmse up to O(n^2 u^2). The pair RMSEs are summed in double in pair
    order (relative 2^-53 per term). The regulariser is exact: min / max of the exactly restated median or mean map.
    `blocks` is restated from the launch constants in `cost_blocks`.
    One dropped pixel p moves pair k's RMSE by about d_pk^2 / (2 HW rmse_k), relative d_pk^2 / (2 S_k), typically
    1 / (2 HW): 8.5e-7 at 768 x 768, 4.1e-5 at 96 x 128. The register-resident kernels (2 <= E <= 16) run 264 blocks,
    so n = 9 at 768 x 768 and the bound is 6.5 u = 3.9e-7, below that. The generic kernels (E = 1 and E > 16) run 48
    blocks, n = 48 at 768 x 768 and the bound is 26 u = 1.55e-6: there the float64 check cannot see one dropped
    pixel, and the bit-level checks of the forward-difference rows against the point evaluated alone carry the weight.
    At 96 x 128 every thread has one pixel and the bound (2.5 u) is far below the effect of one pixel.
  * Mean (`mean_bound`). A sequential fp32 sum of E terms is within gamma(E - 1) sum |a| of the exact sum; the division
    adds u |mean|. Bound gamma(E + 1) sum |a| / E.
  * Unbiased std (`std64`). With x_e = a_e - m (float64 m) and dm the mean bound, the device's fl(a_e - mean_dev) is
    within u |x_e| + dm of x_e, so its square is within (u |x_e| + dm)(2 |x_e| + u |x_e| + dm); the FMA chain adds
    gamma(E) times the sum of squares. q' = q / (E - 1) rounds once and sqrtf once more, and
    |sqrt(q'_dev) - sqrt(q')| <= min(dq / sqrt(q'), sqrt(dq)).
  * Normals uncertainty (`normals`). The cosines are exact; CUDA's acosf is within 2 ulp <= 4 u |acos|, the sum of E
    non-negative terms adds gamma(E - 1), the two divisions 2 u, and pi rounded to fp32 its relative error.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
THREADS = 256
NUM_SMS = 132                  # kernels.h kNumSMs
COST_BLOCKS = 2 * NUM_SMS      # kEnsCostBlocks: register-resident cost kernels
DYN_BLOCKS = 48                # kDynBlocks: generic cost kernel
DYN_PARTIAL_BYTES = 16 << 20   # kDynPartialBytes
MAX_REG_E = 16                 # kEnsMaxE
PI_F32 = float(torch.tensor(math.pi, dtype=torch.float32))


def gamma(n: int) -> float:
    return n * U / (1 - n * U)


def register_resident(E: int) -> bool:
    return 2 <= E <= MAX_REG_E


# ---- launch constants ------------------------------------------------------------------------------------------------
def cost_blocks(E: int, HW: int) -> int:
    """Blocks of one cost pass (launch_ens_depth_cost)."""
    return min(-(-HW // THREADS), COST_BLOCKS if register_resident(E) else DYN_BLOCKS)


def pixels_per_thread(E: int, HW: int) -> int:
    return -(-HW // (cost_blocks(E, HW) * THREADS))


def cost_launches(E: int, HW: int, n_points: int) -> int:
    """Kernel launches of one cost call over n_points points (1, or 1 + n forward-difference points): 2 or 3 for the
    register-resident kernels, and 2 per chunk of p_max points for the generic ones."""
    if register_resident(E):
        return 3 if n_points > 1 else 2
    NP = E * (E - 1) // 2
    p_max = max(1, DYN_PARTIAL_BYTES // (max(NP, 1) * cost_blocks(E, HW) * 8))
    return 2 * -(-n_points // p_max)


# ---- exact restatements --------------------------------------------------------------------------------------------
def make_st(param, E: int, shift: bool):
    """s, t as float32 [E] tensors, each coordinate rounded from float64 on its own (t = None without shift)."""
    p = torch.as_tensor(param, dtype=torch.float64)
    s = p[:E].to(torch.float32)
    t = p[E:2 * E].to(torch.float32) if shift else None
    return s, t


def align(d: torch.Tensor, param, shift: bool) -> torch.Tensor:
    """d [E, ...] float32 -> fl(fl(d * s) + t) per member, two roundings (torch's d * s + t)."""
    E = d.shape[0]
    s, t = make_st(param, E, shift)
    view = (E,) + (1,) * (d.dim() - 1)
    a = d * s.to(d.device).view(view)
    return a + t.to(d.device).view(view) if shift else a


def member_minmax(d: torch.Tensor):
    """Per-member min and max over all pixels: float32 [E] each."""
    f = d.reshape(d.shape[0], -1)
    return f.min(dim=1).values, f.max(dim=1).values


def init_param(d: torch.Tensor, shift: bool):
    """init_param (ensemble.py:91-105) from the exact per-member min / max, as float64 numpy."""
    mn, mx = member_minmax(d)
    if shift:
        s = 1.0 / (mx - mn).clamp(min=1e-6)
        return torch.cat([s, -s * mn]).cpu().double().numpy()
    return (1.0 / mx.clamp(min=1e-6)).cpu().double().numpy()


def lower_median(a: torch.Tensor):
    """torch.median's lower median over dim 0 and the member it picks: position (E - 1) // 2 of a STABLE sort, so among
    equal values the lower member index ranks first."""
    v, i = torch.sort(a, dim=0, stable=True)
    r = (a.shape[0] - 1) // 2
    return v[r], i[r].to(torch.int32)


def mad(a: torch.Tensor, med: torch.Tensor) -> torch.Tensor:
    return torch.sort((a - med).abs(), dim=0).values[(a.shape[0] - 1) // 2]


def _divisor(like: torch.Tensor, E: int) -> torch.Tensor:
    """E as a tensor on like's device: torch's CUDA division by a host scalar multiplies by its reciprocal, which is not
    the kernels' IEEE division unless E is a power of two."""
    return torch.full_like(like, float(E))


def seq_mean(a: torch.Tensor) -> torch.Tensor:
    """Sequential fp32 sum in member order, then one division by E."""
    sm = torch.zeros_like(a[0])
    for e in range(a.shape[0]):
        sm = sm + a[e]
    return sm / _divisor(sm, a.shape[0])


def renorm(pred: torch.Tensor, unc, use_min: bool):
    """Min-max renormalisation (ensemble.py:184-194) in float32: (pred - min) / max(max - min, 1e-6), unc / range."""
    mn = pred.min() if use_min else torch.zeros((), dtype=torch.float32, device=pred.device)
    rng = torch.clamp(pred.max() - mn, min=1e-6)
    return (pred - mn) / rng, (None if unc is None else unc / rng), rng


# ---- float64 restatements with bounds ------------------------------------------------------------------------------
def mean_bound(a: torch.Tensor) -> torch.Tensor:
    E = a.shape[0]
    return gamma(E + 1) * a.double().abs().sum(0) / E


def std64(a: torch.Tensor):
    """Unbiased std over dim 0 in float64 and the bound on the device's fp32 value (NaN for one member, as torch)."""
    E = a.shape[0]
    a64 = a.double()
    m = a64.mean(0)
    x = (a64 - m).abs()
    if E == 1:
        nan = torch.full_like(m, math.nan)
        return nan, nan
    dm = mean_bound(a) * (1 + 2 * U)
    sq = ((x + dm) ** 2).sum(0)
    dq = ((U * x + dm) * ((2 + U) * x + dm)).sum(0) + gamma(E) * sq
    q = (x * x).sum(0) / (E - 1)
    dq = dq / (E - 1) * (1 + U) + U * q
    s = q.sqrt()
    ds = torch.minimum(dq / s.clamp(min=1e-300), dq.sqrt())
    return s, ds + U * (s + dq.sqrt()) + 1e-45


def cost(d: torch.Tensor, param, shift: bool, median: bool, reg: float):
    """The objective (ensemble.py:138-152) in float64 from the exactly aligned fp32 values, with the bound derived in the
    module docstring. d [E, HW] float32. Returns (value, bound, pmin, pmax)."""
    E, HW = d.shape[0], d[0].numel()
    a = align(d.reshape(E, -1), param, shift)
    n = pixels_per_thread(E, HW)
    per_pair = (gamma(n) / 2 + 2 * U)
    total, bound = 0.0, 0.0
    for i in range(E - 1):
        diff = (a[i + 1:] - a[i]).double()          # fp32 differences, squared and summed in float64
        rmse = ((diff * diff).sum(1) / HW).sqrt()
        total += float(rmse.sum())
        bound += float(rmse.sum()) * per_pair
    NP = E * (E - 1) // 2
    pred = lower_median(a)[0] if median else seq_mean(a)
    pmin, pmax = float(pred.min()), float(pred.max())
    if reg > 0:
        total += (abs(0.0 - pmin) + abs(1.0 - pmax)) * reg
    bound += (NP + 2) * 2.0 ** -52 * abs(total)
    return total, bound, pmin, pmax


def pixel_effect(d: torch.Tensor, param, shift: bool) -> float:
    """Median over pixels of what dropping that one pixel from every pair sum moves the pair-RMSE sum by, relative to it
    (module docstring). 0 for one member."""
    E, HW = d.shape[0], d[0].numel()
    if E < 2:
        return 0.0
    a = align(d.reshape(E, -1), param, shift)
    eff = torch.zeros(HW, dtype=torch.float64, device=d.device)
    tot = 0.0
    for i in range(E - 1):
        diff = (a[i + 1:] - a[i]).double()
        sq = diff * diff
        rmse = (sq.sum(1) / HW).sqrt()
        tot += float(rmse.sum())
        eff += (sq / (2 * HW * rmse.clamp(min=1e-300)[:, None])).sum(0)
    return float(eff.median()) / tot


def clamp_cases(d: torch.Tensor, param, pert, shift: bool):
    """For the register-resident median perturbation pass: which case of the lower-median update each (member, pixel)
    takes, and whether the moved value lands outside [lo, hi] (a member moved across the median). Returns
    (case counts [3], crossings) summed over the members and pixels of every moved coordinate."""
    E = d.shape[0]
    a = align(d.reshape(E, -1), param, shift)
    v = torch.sort(a, dim=0).values
    R = (E - 1) // 2
    big = torch.finfo(torch.float32).max
    vlo = v[R - 1] if R > 0 else torch.full_like(v[0], -big)
    vmid = v[R]
    vhi = v[R + 1] if R + 1 < E else torch.full_like(v[0], big)
    counts = [0, 0, 0]
    crossings = 0
    n = 2 * E if shift else E
    for c in range(n):
        m = c % E
        moved = torch.as_tensor(param, dtype=torch.float64).clone()
        moved[c] = float(pert[c])
        x = align(d[m:m + 1].reshape(1, -1), moved[[m, E + m]] if shift else moved[[m]], shift)[0]
        am = a[m]
        c1 = am <= vlo
        c2 = (~c1) & (am <= vmid)
        c3 = ~(c1 | c2)
        counts[0] += int(c1.sum())
        counts[1] += int(c2.sum())
        counts[2] += int(c3.sum())
        lo = torch.where(c1, vmid, vlo)
        hi = torch.where(c3, vmid, vhi)
        crossings += int(((x < lo) | (x > hi)).sum())
    return counts, crossings


def normals(n: torch.Tensor, closest: bool):
    """ensemble_normals as ens_normals_kernel computes it. n [E, 3, ...] float32. Returns (out, member_idx, unc64,
    unc_bound, cosines): out exact, member_idx exact (first maximum), the uncertainty in float64 from the exact clamped
    cosines [E, ...]."""
    E = n.shape[0]
    m = [torch.zeros_like(n[0, 0]) for _ in range(3)]
    for e in range(E):
        for c in range(3):
            m[c] = m[c] + n[e, c]
    m = [mc / _divisor(mc, E) for mc in m]
    n2 = (m[0] * m[0] + m[1] * m[1]) + m[2] * m[2]
    nn = torch.clamp(torch.sqrt(n2), min=1e-6)
    m = [mc / nn for mc in m]
    sims = []
    for e in range(E):
        s = (m[0] * n[e, 0] + m[1] * n[e, 1]) + m[2] * n[e, 2]
        sims.append(s.clamp(-1.0, 1.0))
    sim = torch.stack(sims)
    best = sim[0].clone()
    idx = torch.zeros_like(sim[0], dtype=torch.int64)
    for e in range(1, E):
        take = sim[e] > best                        # first maximum wins
        best = torch.where(take, sim[e], best)
        idx = torch.where(take, torch.full_like(idx, e), idx)
    if closest:
        out = torch.gather(n, 0, idx[None, None].expand((1, 3) + tuple(idx.shape)))[0]
    else:
        out = torch.stack(m)
    ac = torch.arccos(sim.double())
    unc = ac.sum(0) / E / math.pi
    rel_pi = abs(PI_F32 - math.pi) / math.pi
    bound = unc * (4 * U + gamma(E + 1) + 2 * U + rel_pi) * (1 + 1e-6) + 1e-45
    return out, idx.to(torch.int32), unc, bound, sim
