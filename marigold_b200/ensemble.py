"""Drop-in `ensemble_depth` / `ensemble_normals` / `ensemble_iid` (reference marigold/util/ensemble.py:39-196, 199-249,
252-270) backed by the CUDA kernels in csrc/ensemble.cu.

Same signatures, defaults, error behaviour and return shapes as the reference. The scipy BFGS driver
stays on the host as in the reference (ensemble.py:165-171); what changes is the objective: f(x) and
the 2E forward-difference points of its gradient are ONE device round trip (`mgb_ens_depth_cost_fd`)
instead of C(E,2)+2 `.item()` syncs per point. The gradient is formed from those points with scipy's
own step and arithmetic, so the trajectory is the one scipy's default (jac=None) takes.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr

_util_engine = None


def _handle(engine=None):
    """Any handle works for the ensemble entry points (they only use its scratch buffers)."""
    global _util_engine
    if engine is not None:
        return engine
    if _util_engine is None:
        from .engine import Engine, EngineConfig

        _util_engine = Engine(EngineConfig.tiny())
    return _util_engine


def _resize_max_res_nearest_exact(img: torch.Tensor, max_edge: int) -> torch.Tensor:
    # reference resize_max_res (image_util.py:90-120) with NEAREST_EXACT (ensemble.py:158-161)
    h, w = img.shape[-2:]
    f = min(max_edge / w, max_edge / h)
    return torch.nn.functional.interpolate(img, size=(int(h * f), int(w * f)), mode="nearest-exact")


_EPS = float(np.sqrt(np.finfo(np.float64).eps))   # scipy.optimize._optimize._epsilon (BFGS default `eps`)


def _scipy_fd_points(x: np.ndarray) -> np.ndarray:
    """x + h with scipy's forward-difference step for BFGS(jac=None): approx_derivative(..., abs_step=eps): h = eps, or
    eps * sign(x) * max(1, |x|) where x + eps == x."""
    h = np.full_like(x, _EPS)
    dx = (x + h) - x
    sign = (x >= 0).astype(np.float64) * 2 - 1
    h = np.where(dx == 0, _EPS * sign * np.maximum(1.0, np.abs(x)), h)
    return x + h


def _fd_grad(x: np.ndarray, f0: float, costs: np.ndarray, pert: np.ndarray) -> np.ndarray:
    """scipy's 2-point forward difference (approx_derivative as BFGS calls it with jac=None: f0 = f(x),
    df_i = f(x + h_i e_i) - f0 over dx_i = (x_i + h_i) - x_i), from costs already evaluated at `pert = x + h`."""
    return (np.asarray(costs, dtype=np.float64) - f0) / (pert - x)


def _bfgs(fun, param0, tol, max_iter):
    """scipy.optimize.minimize(..., method="BFGS", tol=tol, options={"maxiter": max_iter}) as the reference calls it
    (ensemble.py:165-171). The reference leaves jac=None, i.e. scipy's forward differences; `fun(x) -> (f, grad)`
    restates exactly those (`_scipy_fd_points`, `_fd_grad`: same points, same arithmetic, hence the same trajectory bit
    for bit) from one device pass, and jac=True keeps approx_derivative's per-call Python overhead (~2x the device time
    of a cost pass) out of the loop. scipy keeps the gradient of the last point it evaluated, so every new point is one
    call of `fun`."""
    import scipy.optimize

    res = scipy.optimize.minimize(fun, param0, jac=True, method="BFGS", tol=tol,
                                  options={"maxiter": max_iter, "disp": False})
    return res.x, res.nit


def ensemble_depth(
    depth: torch.Tensor,
    scale_invariant: bool = True,
    shift_invariant: bool = True,
    output_uncertainty: bool = False,
    reduction: str = "median",
    regularizer_strength: float = 0.02,
    max_iter: int = 50,
    tol: float = 1e-6,
    max_res: int = 1024,
    engine=None,
    return_aux: bool = False,
    param: Optional[np.ndarray] = None,
) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    if depth.dim() != 4 or depth.shape[1] != 1:
        raise ValueError(f"Expecting 4D tensor of shape [B,1,H,W]; got {depth.shape}.")
    if reduction not in ("mean", "median"):
        raise ValueError(f"Unrecognized reduction method: {reduction}.")
    if not scale_invariant and shift_invariant:
        raise ValueError("Pure shift-invariant ensembling is not supported.")
    if not scale_invariant:
        raise ValueError("Unrecognized alignment.")  # reference raises this at ensemble.py:190
    if not depth.is_cuda:
        raise _lib.MgbError("marigold_b200.ensemble_depth needs a CUDA tensor (no CPU fallback)")
    eng = _handle(engine)
    lib, h = eng.lib, eng._h
    E = depth.shape[0]
    H, W = depth.shape[2:]
    median = 1 if reduction == "median" else 0
    sc, sh = int(scale_invariant), int(shift_invariant)

    with torch.cuda.device(depth.device):
        d_full = depth.to(torch.float32).contiguous()
        d_align = d_full
        if max_res is not None and max(H, W) > max_res:
            d_align = _resize_max_res_nearest_exact(d_full, max_res).contiguous()
        hw_a = d_align.shape[2] * d_align.shape[3]

        # init_param (ensemble.py:91-105)
        mn = np.zeros(E, dtype=np.float32)
        mx = np.zeros(E, dtype=np.float32)
        check(lib.mgb_ens_minmax(h, ptr(d_align), E, hw_a, mn.ctypes.data_as(C.c_void_p),
                                 mx.ctypes.data_as(C.c_void_p), stream_ptr()), "mgb_ens_minmax")
        if shift_invariant:
            init_s = (np.float32(1.0) / np.maximum(mx - mn, np.float32(1e-6))).astype(np.float32)
            init_t = (-init_s * mn).astype(np.float32)
            param0 = np.concatenate([init_s, init_t]).astype(np.float64)
        else:
            param0 = (np.float32(1.0) / np.maximum(mx, np.float32(1e-6))).astype(np.float64)

        n_eval = [0, 0]   # objective evaluations, device round trips
        n_param = 2 * E if shift_invariant else E
        reg = float(regularizer_strength)

        def cost_fn(param: np.ndarray) -> float:
            """cost_fn (ensemble.py:138-152) at one point (`mgb_ens_depth_cost`)."""
            x = np.ascontiguousarray(param, dtype=np.float64)
            out = C.c_double()
            check(lib.mgb_ens_depth_cost(h, ptr(d_align), x.ctypes.data_as(C.c_void_p), E, hw_a, sc, sh, median, reg,
                                         C.byref(out), stream_ptr()), "mgb_ens_depth_cost")
            return out.value

        def cost_fd(base: np.ndarray, pert: np.ndarray) -> np.ndarray:
            """[1 + n]: the objective at `base`, then at `base` with coordinate i moved to pert[i], for each i. One
            device round trip (`mgb_ens_depth_cost_fd`)."""
            base = np.ascontiguousarray(base, dtype=np.float64)
            pert = np.ascontiguousarray(pert, dtype=np.float64)
            if base.shape != (n_param,) or pert.shape != (n_param,):
                raise ValueError(f"cost_fd expects two vectors of {n_param} parameters; got {base.shape}, {pert.shape}")
            out = np.empty(1 + n_param, dtype=np.float64)
            # plain integer addresses: this runs once per BFGS evaluation, and each data_as() costs ~2 us of host time
            check(lib.mgb_ens_depth_cost_fd(h, ptr(d_align), base.ctypes.data, pert.ctypes.data, E, hw_a, sc, sh,
                                            median, reg, out.ctypes.data, stream_ptr()), "mgb_ens_depth_cost_fd")
            n_eval[0] += out.size
            n_eval[1] += 1
            return out

        def fun(param: np.ndarray) -> Tuple[float, np.ndarray]:
            """f(param) and scipy's forward-difference gradient of it, from one `cost_fd` round trip."""
            x = np.ascontiguousarray(param, dtype=np.float64)
            pert = _scipy_fd_points(x)
            out = cost_fd(x, pert)
            f = float(out[0])
            return f, _fd_grad(x, f, out[1:], pert)

        nit = 0
        if param is None:
            param, nit = _bfgs(fun, param0, tol, max_iter)
        param = np.ascontiguousarray(param, dtype=np.float64)   # (tests may inject the alignment)

        pred = torch.empty(1, 1, H, W, dtype=torch.float32, device=depth.device)
        unc = torch.empty_like(pred) if output_uncertainty else None
        idx = torch.empty(1, 1, H, W, dtype=torch.int32, device=depth.device) if return_aux else None
        check(lib.mgb_ens_depth_reduce(h, ptr(d_full), param.ctypes.data_as(C.c_void_p), E, H * W, sc, sh, median,
                                       ptr(pred), ptr(unc), ptr(idx), stream_ptr()), "mgb_ens_depth_reduce")
    pred = pred.to(depth.dtype)
    if unc is not None:
        unc = unc.to(depth.dtype)
    if return_aux:
        return pred, unc, {"param": param, "param0": param0, "member_idx": idx, "nit": nit, "nfev": n_eval[0],
                            "round_trips": n_eval[1], "cost_fn": cost_fn, "cost_fd": cost_fd}
    return pred, unc


def ensemble_normals(
    normals: torch.Tensor,
    output_uncertainty: bool = False,
    reduction: str = "closest",
    engine=None,
    return_aux: bool = False,
) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    if normals.dim() != 4 or normals.shape[1] != 3:
        raise ValueError(f"Expecting 4D tensor of shape [B,3,H,W]; got {normals.shape}.")
    if reduction not in ("closest", "mean"):
        raise ValueError(f"Unrecognized reduction method: {reduction}.")
    if not normals.is_cuda:
        raise _lib.MgbError("marigold_b200.ensemble_normals needs a CUDA tensor (no CPU fallback)")
    eng = _handle(engine)
    E, _, H, W = normals.shape
    with torch.cuda.device(normals.device):
        n32 = normals.to(torch.float32).contiguous()
        out = torch.empty(1, 3, H, W, dtype=torch.float32, device=normals.device)
        unc = torch.empty(1, 1, H, W, dtype=torch.float32, device=normals.device) if output_uncertainty else None
        idx = torch.empty(1, 1, H, W, dtype=torch.int32, device=normals.device) if return_aux else None
        check(eng.lib.mgb_ens_normals(eng._h, ptr(n32), E, H * W, 1 if reduction == "closest" else 0, ptr(out),
                                      ptr(unc), ptr(idx), stream_ptr()), "mgb_ens_normals")
    out = out.to(normals.dtype)
    if unc is not None:
        unc = unc.to(normals.dtype)
    if return_aux:
        return out, unc, {"member_idx": idx}
    return out, unc


def ensemble_iid(
    targets: torch.Tensor,
    output_uncertainty: bool = False,
    reduction: str = "median",
    engine=None,
) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """reference ensemble.py:252-270: per-element (lower) median + MAD, or mean + unbiased std, over the members;
    no alignment and no renormalisation. targets [E, 3n, H, W] -> ([1, 3n, H, W], uncertainty or None)."""
    if reduction not in ("mean", "median"):
        raise ValueError(f"Unrecognized reduction method: {reduction}.")
    if not targets.is_cuda:
        raise _lib.MgbError("marigold_b200.ensemble_iid needs a CUDA tensor (no CPU fallback)")
    eng = _handle(engine)
    E = targets.shape[0]
    with torch.cuda.device(targets.device):
        x = targets.to(torch.float32).contiguous()
        n = x[0].numel()
        pred = torch.empty((1,) + tuple(x.shape[1:]), dtype=torch.float32, device=x.device)
        unc = torch.empty_like(pred) if output_uncertainty else None
        check(eng.lib.mgb_ens_iid(eng._h, ptr(x), E, n, 1 if reduction == "median" else 0, ptr(pred), ptr(unc),
                                  stream_ptr()), "mgb_ens_iid")
    pred = pred.to(targets.dtype)
    if unc is not None:
        unc = unc.to(targets.dtype)
    return pred, unc
