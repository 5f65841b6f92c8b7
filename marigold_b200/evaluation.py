"""Device-side evaluation step that follows the hot path in dataset evaluation (csrc/eval.cu).

Depth: least-squares scale / shift alignment in depth or disparity space (reference src/util/alignment.py:35-82,
script/depth/eval.py:171-207), the dataset clips and the masked depth metrics of src/util/metric.py:64-191 — two
streaming passes and one host synchronisation per sample.
Surface normals: the angular error of compute_cosine_error(masked=True) and the metrics of src/util/metric.py:194-257,
including the exact median — four launches and one host synchronisation per sample.
Intrinsic images: PSNR and SSIM of compute_iid_metric (src/util/metric.py:263-338) with the up-to-scale targets' lstsq
scale and quantile map — two launches (six for shading and residual) and one host synchronisation per target."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr

METRIC_NAMES = ("abs_relative_difference", "squared_relative_difference", "rmse_linear", "rmse_log", "log10", "delta1_acc",
                "delta2_acc", "delta3_acc", "i_rmse", "silog_rmse")
NORMALS_METRIC_NAMES = ("mean_angular_error", "median_angular_error", "rmse_angular_error", "sub5_error", "sub7_5_error",
                        "sub11_25_error", "sub22_5_error", "sub30_error")
IID_METRIC_NAMES = ("psnr", "ssim")
IID_TRANSFORMS = (None, "srgb2linear", "linear2srgb")
ALIGNMENTS = (None, "least_square", "least_square_disparity")
_ERR_INVALID = -1     # MGB_ERR_INVALID
_ws = {}
_normals_ws = {}
_iid_ws = {}


def _inputs(pred, gt, mask):
    if not (pred.is_cuda and gt.is_cuda):
        raise _lib.MgbError("marigold_b200.evaluation needs CUDA tensors (no CPU fallback)")
    p = pred.to(torch.float32).contiguous().reshape(-1)
    g = gt.to(torch.float32).contiguous().reshape(-1)
    assert p.numel() == g.numel(), f"{tuple(pred.shape)} vs {tuple(gt.shape)}"
    m = None
    if mask is not None:
        m = mask.to(device=p.device).to(torch.uint8).contiguous().reshape(-1)
    return p, g, m


def _depth_ws(lib, device):
    ws = _ws.get(device)
    if ws is None:
        ws = torch.empty(int(lib.mgb_eval_ws_bytes()), dtype=torch.uint8, device=device)
        _ws[device] = ws
    return ws


def _run(pred, gt, mask, least_squares: bool, dmin: float, dmax: float, want_aligned: bool):
    p, g, m = _inputs(pred, gt, mask)
    assert m is None or m.numel() == p.numel()
    lib = _lib.load()
    with torch.cuda.device(p.device):
        ws = _depth_ws(lib, p.device)
        aligned = torch.empty_like(p) if want_aligned else None
        out = np.zeros(13, dtype=np.float64)
        check(lib.mgb_eval_depth(ptr(p), ptr(g), ptr(m), p.numel(), int(least_squares), float(dmin), float(dmax), ptr(aligned),
                                 ptr(ws), out.ctypes.data_as(C.c_void_p), stream_ptr()), "mgb_eval_depth")
    return out, (aligned.reshape(pred.shape) if aligned is not None else None)


def fit_index_tables(H: int, W: int, max_resolution: Optional[int]):
    """Source rows and columns of the maps align_depth_least_square fits when given max_resolution (alignment.py:48-59),
    or None when the fit uses the full maps. The reference hands torch.nn.Upsample a [1, H, W] tensor (the squeezed map
    with one leading dimension), which Upsample reads as a batch of H one-dimensional signals of length W: only the width
    is downsampled. The tables are that same Upsample applied to the indices themselves, so its rounding is torch's."""
    if max_resolution is None:
        return None
    sf = np.min(max_resolution / np.array((H, W)))
    if not sf < 1:
        return None
    down = torch.nn.Upsample(scale_factor=sf, mode="nearest")
    cols = down(torch.arange(W, dtype=torch.float64).reshape(1, 1, W)).reshape(-1)
    rows = torch.arange(H, dtype=torch.float64)
    return rows.to(torch.int32), cols.to(torch.int32)


def _run_ex(pred, gt, mask, mode: int, max_resolution, dmin: float, dmax: float):
    H, W = pred.shape[-2:]
    p, g, m = _inputs(pred, gt, mask)
    lib = _lib.load()
    assert p.numel() == H * W and (m is None or m.numel() == p.numel()), "depth maps must be [H, W] (or squeeze to it)"
    tables = fit_index_tables(H, W, max_resolution) if mode else None
    with torch.cuda.device(p.device):
        ws = _depth_ws(lib, p.device)
        rows = cols = None
        if tables is not None:
            rows, cols = (t.to(p.device) for t in tables)
        out = np.zeros(13, dtype=np.float64)
        check(lib.mgb_eval_depth_ex(ptr(p), ptr(g), ptr(m), H, W, mode, ptr(rows), ptr(cols),
                                    0 if rows is None else rows.numel(), 0 if cols is None else cols.numel(), float(dmin),
                                    float(dmax), None, ptr(ws), out.ctypes.data_as(C.c_void_p), stream_ptr()),
              "mgb_eval_depth_ex")
    return out


def align_depth_least_square(gt: torch.Tensor, pred: torch.Tensor, valid_mask: Optional[torch.Tensor],
                             return_scale_shift: bool = True, max_resolution: Optional[int] = None):
    """src/util/alignment.py:35-82 on the device: (aligned_pred, scale, shift). `max_resolution` downsamples the three
    maps with the reference's nearest Upsample before the fit; the fitted map is always the full-resolution prediction."""
    fit_p, fit_g, fit_m = pred, gt, valid_mask
    if max_resolution is not None:
        sf = float(np.min(max_resolution / np.array(pred.shape[-2:])))
        if sf < 1:
            down = torch.nn.Upsample(scale_factor=sf, mode="nearest")
            fit_g = down(gt.reshape(1, 1, *gt.shape[-2:]).float())
            fit_p = down(pred.reshape(1, 1, *pred.shape[-2:]).float())
            fit_m = down(valid_mask.reshape(1, 1, *valid_mask.shape[-2:]).float()).bool() if valid_mask is not None else None
    out, _ = _run(fit_p, fit_g, fit_m, True, -3.0e38, 3.0e38, False)      # only the fit is used from this call
    scale, shift = out[0], out[1]
    aligned = pred.to(torch.float64) * scale + shift
    return (aligned, scale, shift) if return_scale_shift else aligned


def evaluate_depth(pred: torch.Tensor, gt: torch.Tensor, valid_mask: Optional[torch.Tensor] = None,
                   alignment: Optional[str] = "least_square", min_depth: float = 1e-6, max_depth: float = 3.0e38,
                   alignment_max_res: Optional[int] = None) -> Tuple[Dict[str, float], Dict[str, float]]:
    """One sample of script/depth/eval.py:171-217: align (or not), clip to the dataset range and to d > 1e-6, all metrics.

    alignment: None, "least_square" (fit pred to gt) or "least_square_disparity" (fit pred to 1 / gt over the valid
    pixels where gt > 0 and pred > 0, clip the aligned disparity to >= 1e-3 and take its reciprocal). The metrics always
    use `valid_mask`. alignment_max_res: fit on the maps downsampled as align_depth_least_square(max_resolution=...)
    downsamples them (see fit_index_tables); the metrics use the full-resolution maps.
    Returns (metrics by the reference's function names, {"scale", "shift", "n_valid"})."""
    if alignment not in ALIGNMENTS:
        raise ValueError(f"unsupported alignment {alignment!r}; expected one of {ALIGNMENTS}")
    if alignment in (None, "least_square") and alignment_max_res is None:
        out, _ = _run(pred, gt, valid_mask, alignment == "least_square", min_depth, max_depth, False)
    else:
        out = _run_ex(pred, gt, valid_mask, ALIGNMENTS.index(alignment), alignment_max_res, min_depth, max_depth)
    metrics = dict(zip(METRIC_NAMES, (float(v) for v in out[3:13])))
    return metrics, {"scale": float(out[0]), "shift": float(out[1]), "n_valid": int(out[2])}


def evaluate_normals(pred: torch.Tensor, gt: torch.Tensor, valid_mask: Optional[torch.Tensor] = None,
                     return_error_map: bool = False) -> Tuple[Dict[str, float], Dict[str, object]]:
    """One sample of script/normals/eval.py:145-157: the angular error in degrees of compute_cosine_error(pred, gt,
    masked=True) (src/util/metric.py:194-219) and the metrics of metric.py:222-257 over it.

    pred, gt: [3, H, W] or [1, 3, H, W] CUDA tensors, channel first. A pixel counts where ||gt|| > 0, as in the
    reference, and, when `valid_mask` ([H, W]) is given, where it is also true. The median is np.median's exactly: the
    middle error for odd n, the float32 mean of the two middle errors for even n. The values are NOT rounded; the
    reference rounds each to 4 decimals (round(x, 4)). With no valid pixel every metric is NaN, as numpy gives for an
    empty array. Returns (metrics by the reference's function names, {"n_valid"[, "error_map"]}), where "error_map" is
    the [H, W] float32 error, NaN where the pixel does not count."""
    if pred.dim() == 4:
        pred = pred.squeeze(0)
    if gt.dim() == 4:
        gt = gt.squeeze(0)
    assert pred.shape[0] == 3 and gt.shape == pred.shape, f"expected [3, H, W], got {tuple(pred.shape)} and {tuple(gt.shape)}"
    H, W = pred.shape[-2:]
    p, g, m = _inputs(pred, gt, valid_mask)
    assert m is None or m.numel() == H * W
    lib = _lib.load()
    with torch.cuda.device(p.device):
        need = int(lib.mgb_eval_normals_ws_bytes(H * W))
        ws = _normals_ws.get(p.device)
        if ws is None or ws.numel() < need:
            ws = torch.empty(need, dtype=torch.uint8, device=p.device)
            _normals_ws[p.device] = ws
        err = torch.empty(H, W, dtype=torch.float32, device=p.device) if return_error_map else None
        out = np.zeros(9, dtype=np.float64)
        check(lib.mgb_eval_normals(ptr(p), ptr(g), ptr(m), H, W, ptr(err), ptr(ws), out.ctypes.data_as(C.c_void_p),
                                   stream_ptr()), "mgb_eval_normals")
    info = {"n_valid": int(out[0])}
    if err is not None:
        info["error_map"] = err
    return dict(zip(NORMALS_METRIC_NAMES, (float(v) for v in out[1:]))), info


def _as_chw(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.dim() == 4 and t.shape[0] == 1:
        t = t.squeeze(0)
    if t.dim() != 3 or t.shape[0] != 3:
        raise ValueError(f"{what} must be [3, H, W] or [1, 3, H, W], got {tuple(t.shape)}")
    return t


def evaluate_iid(pred: torch.Tensor, gt: torch.Tensor, target_name: str, valid_mask: Optional[torch.Tensor] = None,
                 transform: Optional[str] = None) -> Tuple[Dict[str, float], Dict[str, object]]:
    """PSNR and SSIM of one intrinsic-image target of one sample: compute_iid_metric (src/util/metric.py:263-338) as
    script/iid/eval.py:182-213 calls it, with torchmetrics' PeakSignalNoiseRatio and StructuralSimilarityIndexMeasure
    (data_range=1.0). LPIPS is not computed.

    pred, gt: [3, H, W] or [1, 3, H, W] CUDA tensors, H and W >= 11. valid_mask: bool [3, H, W] (one mask per channel,
    as the datasets build it) or None. transform: None, "srgb2linear" or "linear2srgb", applied to both maps first (the
    caller decides it per dataset and target, as eval.py does). "shading" and "residual" are up to scale: the prediction
    is fitted to gt by least squares and both are mapped to [0, 1] by the brightness quantile of gt.
    Returns ({"psnr", "ssim"}, {"n_valid", "scale", "quantile", "quantile_scale"}); the last three are None for the
    other targets. Raises ValueError for malformed input and, for an up-to-scale target, when no pixel is valid in
    channel 0 of the mask (the reference's torch.quantile of an empty tensor)."""
    if transform not in IID_TRANSFORMS:
        raise ValueError(f"unsupported transform {transform!r}; expected one of {IID_TRANSFORMS}")
    pred, gt = _as_chw(pred, "pred"), _as_chw(gt, "gt")
    if gt.shape != pred.shape:
        raise ValueError(f"pred {tuple(pred.shape)} and gt {tuple(gt.shape)} differ")
    if valid_mask is not None:
        valid_mask = _as_chw(valid_mask, "valid_mask")
        if valid_mask.shape != pred.shape:
            raise ValueError(f"valid_mask {tuple(valid_mask.shape)} does not match {tuple(pred.shape)}")
    H, W = pred.shape[-2:]
    if H < 11 or W < 11:
        raise ValueError(f"SSIM's 11 x 11 window needs H, W >= 11, got {H} x {W}")
    up_to_scale = target_name in ("shading", "residual")
    p, g, m = _inputs(pred, gt, valid_mask)
    lib = _lib.load()
    with torch.cuda.device(p.device):
        need = int(lib.mgb_eval_iid_ws_bytes(H, W))
        ws = _iid_ws.get(p.device)
        if ws is None or ws.numel() < need:
            ws = torch.empty(need, dtype=torch.uint8, device=p.device)
            _iid_ws[p.device] = ws
        out = np.zeros(6, dtype=np.float64)
        rc = lib.mgb_eval_iid(ptr(p), ptr(g), ptr(m), H, W, int(up_to_scale), IID_TRANSFORMS.index(transform), ptr(ws),
                              out.ctypes.data_as(C.c_void_p), stream_ptr())
    if rc == _ERR_INVALID:
        raise ValueError(lib.mgb_last_error().decode("utf-8", "replace"))
    check(rc, "mgb_eval_iid")
    scaled = (float(out[3]), float(out[4]), float(out[5])) if up_to_scale else (None, None, None)
    info = {"n_valid": int(out[0]), **dict(zip(("scale", "quantile", "quantile_scale"), scaled))}
    return dict(zip(IID_METRIC_NAMES, (float(out[1]), float(out[2])))), info
