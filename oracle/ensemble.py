"""ORACLE (test infrastructure only — never imported by the product path).

CPU restatement of the reference's test-time ensembling, marigold/util/ensemble.py:
  ensemble_depth    :39-196  (init_param :91-105, align :107-118, ensemble :120-136, cost_fn :138-152,
                              compute_param :154-173, final min-max renormalisation :184-194)
  ensemble_normals  :199-249

PARITY PINNED: tests/golden/ensemble_*.npz were produced by running the reference's own functions in
tests/golden/make_golden.py (it imports the reference checkout's marigold/util/ensemble.py
through a package shim); tests/test_oracle.py checks this restatement against them, including the
member index picked by the lower median / argmax.
"""
from __future__ import annotations

from functools import partial
from typing import Optional, Tuple

import numpy as np
import torch


def _resize_max_res_nearest_exact(img: torch.Tensor, max_edge: int) -> torch.Tensor:
    """resize_max_res (marigold/util/image_util.py:90-120) specialised to NEAREST_EXACT."""
    h, w = img.shape[-2:]
    f = min(max_edge / w, max_edge / h)
    nw, nh = int(w * f), int(h * f)
    return torch.nn.functional.interpolate(img, size=(nh, nw), mode="nearest-exact")


def ensemble_depth(depth: torch.Tensor, scale_invariant: bool = True, shift_invariant: bool = True,
                   output_uncertainty: bool = False, reduction: str = "median", regularizer_strength: float = 0.02,
                   max_iter: int = 50, tol: float = 1e-6, max_res: int = 1024,
                   return_param: bool = False):
    if depth.dim() != 4 or depth.shape[1] != 1:
        raise ValueError(f"Expecting 4D tensor of shape [B,1,H,W]; got {depth.shape}.")
    if reduction not in ("mean", "median"):
        raise ValueError(f"Unrecognized reduction method: {reduction}.")
    if not scale_invariant and shift_invariant:
        raise ValueError("Pure shift-invariant ensembling is not supported.")
    E = depth.shape[0]

    def init_param(d):
        mn = d.reshape(E, -1).min(dim=1).values
        mx = d.reshape(E, -1).max(dim=1).values
        if scale_invariant and shift_invariant:
            s = 1.0 / (mx - mn).clamp(min=1e-6)
            t = -s * mn
            p = torch.cat((s, t)).cpu().numpy()
        elif scale_invariant:
            p = (1.0 / mx.clamp(min=1e-6)).cpu().numpy()
        else:
            raise ValueError("Unrecognized alignment.")
        return p.astype(np.float64)

    def align(d, p):
        if scale_invariant and shift_invariant:
            s, t = np.split(p, 2)
            s = torch.from_numpy(s).to(d).view(E, 1, 1, 1)
            t = torch.from_numpy(t).to(d).view(E, 1, 1, 1)
            return d * s + t
        s = torch.from_numpy(p).to(d).view(E, 1, 1, 1)
        return d * s

    def ensemble(d, return_uncertainty=False):
        unc = None
        if reduction == "mean":
            pred = torch.mean(d, dim=0, keepdim=True)
            if return_uncertainty:
                unc = torch.std(d, dim=0, keepdim=True)
        else:
            pred = torch.median(d, dim=0, keepdim=True).values  # LOWER median for even E
            if return_uncertainty:
                unc = torch.median(torch.abs(d - pred), dim=0, keepdim=True).values
        return pred, unc

    def cost_fn(p, d):
        cost = 0.0
        a = align(d, p)
        for i in range(E):
            for j in range(i + 1, E):
                diff = a[i] - a[j]
                cost += (diff ** 2).mean().sqrt().item()
        if regularizer_strength > 0:
            pred, _ = ensemble(a)
            cost += ((0.0 - pred.min()).abs().item() + (1.0 - pred.max()).abs().item()) * regularizer_strength
        return cost

    param = None
    if scale_invariant or shift_invariant:
        import scipy.optimize

        d32 = depth.to(torch.float32)
        if max_res is not None and max(d32.shape[2:]) > max_res:
            d32 = _resize_max_res_nearest_exact(d32, max_res)
        p0 = init_param(d32)
        res = scipy.optimize.minimize(partial(cost_fn, d=d32), p0, method="BFGS", tol=tol,
                                      options={"maxiter": max_iter, "disp": False})
        param = res.x
        depth = align(depth, param)

    depth, unc = ensemble(depth, return_uncertainty=output_uncertainty)
    dmax = depth.max()
    dmin = depth.min() if (scale_invariant and shift_invariant) else 0
    rng = (dmax - dmin).clamp(min=1e-6)
    depth = (depth - dmin) / rng
    if output_uncertainty:
        unc = unc / rng
    if return_param:
        return depth, unc, param
    return depth, unc


def ensemble_normals(normals: torch.Tensor, output_uncertainty: bool = False, reduction: str = "closest"
                     ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    if normals.dim() != 4 or normals.shape[1] != 3:
        raise ValueError(f"Expecting 4D tensor of shape [B,3,H,W]; got {normals.shape}.")
    if reduction not in ("closest", "mean"):
        raise ValueError(f"Unrecognized reduction method: {reduction}.")
    mean_normals = normals.mean(dim=0, keepdim=True)
    norm = torch.norm(mean_normals, dim=1, keepdim=True)
    mean_normals = mean_normals / norm.clamp(min=1e-6)
    sim_cos = None
    if output_uncertainty or reduction != "mean":
        sim_cos = (mean_normals * normals).sum(dim=1, keepdim=True).clamp(-1, 1)
    unc = None
    if output_uncertainty:
        unc = sim_cos.arccos().mean(dim=0, keepdim=True) / np.pi
    if reduction == "mean":
        return mean_normals, unc
    idx = sim_cos.argmax(dim=0, keepdim=True).repeat(1, 3, 1, 1)
    return torch.gather(normals, 0, idx), unc


def ensemble_iid(targets: torch.Tensor, output_uncertainty: bool = False, reduction: str = "median"
                 ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """marigold/util/ensemble.py:250-270 (SURVEY.md §8f rank 1): per-pixel statistic over the members of an
    [E, C, H, W] stack of intrinsic-image targets. "median" is torch's LOWER median (no affine alignment and no
    renormalisation, unlike ensemble_depth), uncertainty = median absolute deviation; "mean" pairs with the
    (unbiased) standard deviation."""
    unc = None
    if reduction == "mean":
        pred = targets.mean(dim=0, keepdim=True)
        if output_uncertainty:
            unc = targets.std(dim=0, keepdim=True)
    elif reduction == "median":
        pred = targets.median(dim=0, keepdim=True).values
        if output_uncertainty:
            unc = (targets - pred).abs().median(dim=0, keepdim=True).values
    else:
        raise ValueError(f"Unrecognized reduction method: {reduction}.")
    return pred, unc
