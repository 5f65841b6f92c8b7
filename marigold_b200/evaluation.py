"""Device-side evaluation step that follows the hot path in dataset evaluation (csrc/eval.cu).

Depth: least-squares scale / shift alignment in depth or disparity space (reference src/util/alignment.py:35-82,
script/depth/eval.py:171-207), the dataset clips and the masked depth metrics of src/util/metric.py:64-191 — two
streaming passes and one host synchronisation per sample.
Surface normals: the angular error of compute_cosine_error(masked=True) and the metrics of src/util/metric.py:194-257,
including the exact median — four launches and one host synchronisation per sample.
Intrinsic images: PSNR and SSIM of compute_iid_metric (src/util/metric.py:263-338) with the up-to-scale targets' lstsq
scale and quantile map — two launches (six for shading and residual) and one host synchronisation per target — and,
with LPIPS weights, the AlexNet, VGG16 or SqueezeNet 1.1 LPIPS of the same maps in the same synchronisation
(csrc/lpips.cu)."""
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
    """src/util/alignment.py:35-82 on the device: (aligned_pred, scale, shift). `max_resolution` fits the pixels the
    reference's nearest Upsample keeps (fit_index_tables: its [1, H, W] input downsamples the width only), as
    evaluate_depth(alignment_max_res=...) does; the fitted map is always the full-resolution prediction."""
    H, W = pred.shape[-2:]
    out = _run_ex(pred.reshape(H, W), gt.reshape(H, W), None if valid_mask is None else valid_mask.reshape(H, W), 1,
                  max_resolution, -3.0e38, 3.0e38)                          # only the fit is used from this call
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
    downsamples them (see fit_index_tables); the metrics use the full-resolution maps. The sums are taken in double;
    the delta accuracies count the reference's float32 decisions. With no valid pixel every metric is NaN (n_valid 0),
    as the reference's 0 / 0 gives; a fit over no pixel gives scale 0, shift 0, as np.linalg.lstsq does.
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


# torchvision alexnet().features: the index of each convolution and its weight shape
_ALEX_CONVS = ((0, (64, 3, 11, 11)), (3, (192, 64, 5, 5)), (6, (384, 192, 3, 3)), (8, (256, 384, 3, 3)),
               (10, (256, 256, 3, 3)))


def _vgg16_convs():
    """vgg16().features: (key prefix, weight shape) of the thirteen 3 x 3 convolutions."""
    idx = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
    cout = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
    return tuple((f"features.{i}", (co, ci, 3, 3)) for i, co, ci in zip(idx, cout, (3,) + cout[:-1]))


def _squeezenet1_1_convs():
    """squeezenet1_1().features: (key prefix, weight shape) of conv1 and each Fire module's squeeze, expand1x1 and
    expand3x3, in that order."""
    convs = [("features.0", (64, 3, 3, 3))]
    fires = ((3, 64, 16, 64), (4, 128, 16, 64), (6, 128, 32, 128), (7, 256, 32, 128), (9, 256, 48, 192),
             (10, 384, 48, 192), (11, 384, 64, 256), (12, 512, 64, 256))
    for i, cin, sq, e in fires:
        convs += [(f"features.{i}.squeeze", (sq, cin, 1, 1)), (f"features.{i}.expand1x1", (e, sq, 1, 1)),
                  (f"features.{i}.expand3x3", (e, sq, 3, 3))]
    return tuple(convs)


# net_type -> (C ABI net, name, convolutions, channels of each lin layer): torchmetrics' vendored lpips pretrained_networks
LPIPS_NETS = {
    "alex": (0, "AlexNet", tuple((f"features.{i}", shape) for i, shape in _ALEX_CONVS), (64, 192, 384, 256, 256)),
    "vgg": (1, "VGG16", _vgg16_convs(), (64, 128, 256, 512, 512)),
    "squeeze": (2, "SqueezeNet 1.1", _squeezenet1_1_convs(), (64, 128, 256, 384, 384, 512, 512)),
}


def lpips_min_size(net_type: str = "alex") -> int:
    """The smallest H (and W) evaluate_iid accepts with LPIPS weights of `net_type`: the smallest for which every tapped
    layer of the torchvision module is non-empty (31 alex, 16 vgg, 17 squeeze)."""
    if net_type not in LPIPS_NETS:
        raise ValueError(f"unsupported net_type {net_type!r}; expected one of {tuple(LPIPS_NETS)}")
    return int(_lib.load().mgb_lpips_min_size(LPIPS_NETS[net_type][0]))


class LPIPS:
    """The weights of torchmetrics' LearnedPerceptualImagePatchSimilarity(net_type=net_type) on the device, for
    evaluate_iid(..., lpips=...). net_state_dict: the torchvision state dict of the backbone (other keys are ignored):
      "alex" (default)  alexnet() keys features.{0,3,6,8,10}.{weight,bias}
      "vgg"             vgg16() keys features.{0,2,5,7,10,12,14,17,19,21,24,26,28}.{weight,bias}
      "squeeze"         squeezenet1_1() keys features.0.{weight,bias} and
                        features.{3,4,6,7,9,10,11,12}.{squeeze,expand1x1,expand3x3}.{weight,bias}
    lin_state_dict: lpips / torchmetrics keys lin{0..4}.model.1.weight (lin{0..6} for "squeeze"), each [1, C, 1, 1].
    Loading the files is the caller's (torch.load(path, weights_only=True)). The convolutions are held in bf16, lin in
    fp32. A missing key, a misshaped tensor or an unknown net_type raises ValueError."""

    def __init__(self, net_state_dict, lin_state_dict, device=None, *, net_type: str = "alex"):
        if net_type not in LPIPS_NETS:
            raise ValueError(f"unsupported net_type {net_type!r}; expected one of {tuple(LPIPS_NETS)}")
        net, self.net_name, convs, chans = LPIPS_NETS[net_type]

        def get(sd, key, shape, what):
            if key not in sd:
                raise ValueError(f"{what} has no {key!r}")
            t = sd[key].detach()
            if tuple(t.shape) != tuple(shape):
                raise ValueError(f"{what}[{key!r}] has shape {tuple(t.shape)}, expected {tuple(shape)}")
            return t.to("cpu", torch.float32).contiguous()

        what = "alexnet_state_dict" if net_type == "alex" else "net_state_dict"
        ws = [get(net_state_dict, f"{k}.weight", shape, what) for k, shape in convs]
        bs = [get(net_state_dict, f"{k}.bias", shape[:1], what) for k, shape in convs]
        lins = [get(lin_state_dict, f"lin{l}.model.1.weight", (1, c, 1, 1), "lin_state_dict") for l, c in enumerate(chans)]
        dev = torch.device("cuda" if device is None else device)
        self.device = dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())
        self.net_type = net_type
        vp = lambda ts: (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])  # noqa: E731
        shapes = (C.c_int32 * (4 * len(convs)))(*[s for _, shape in convs for s in shape])
        lin_c = (C.c_int32 * len(chans))(*chans)
        lib = _lib.load()
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            check(lib.mgb_lpips_create_net(net, len(convs), vp(ws), shapes, vp(bs), len(chans), vp(lins), lin_c, C.byref(h)),
                  "mgb_lpips_create_net")
        self._lib, self._h = lib, h
        self.min_size = int(lib.mgb_lpips_min_size(net))
        self._ws = None

    def _workspace(self, H: int, W: int) -> torch.Tensor:
        need = int(self._lib.mgb_lpips_ws_bytes_h(self._h, H, W))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def close(self) -> None:
        if self._h:
            torch.cuda.synchronize(self.device)      # a call may still be reading the weights
            self._lib.mgb_lpips_destroy(self._h)
            self._h = None
        self._ws = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001 (interpreter shutdown)
            pass


def evaluate_iid(pred: torch.Tensor, gt: torch.Tensor, target_name: str, valid_mask: Optional[torch.Tensor] = None,
                 transform: Optional[str] = None, lpips: Optional[LPIPS] = None) -> Tuple[Dict[str, float], Dict[str, object]]:
    """PSNR, SSIM and, given `lpips`, LPIPS of one intrinsic-image target of one sample: compute_iid_metric
    (src/util/metric.py:263-338) as script/iid/eval.py:182-213 calls it, with torchmetrics' PeakSignalNoiseRatio and
    StructuralSimilarityIndexMeasure (data_range=1.0) and LearnedPerceptualImagePatchSimilarity(net_type=lpips.net_type,
    normalize=True), one host synchronisation per call.

    pred, gt: [3, H, W] or [1, 3, H, W] CUDA tensors, H and W >= 11 and, with lpips, >= lpips.min_size (31 alex: its
    second pool needs a 3 x 3 input; 16 vgg; 17 squeeze). valid_mask: bool [3, H, W] (one mask per channel, as the datasets build it) or None. transform: None,
    "srgb2linear" or "linear2srgb", applied to both maps first (the caller decides it per dataset and target, as eval.py
    does). "shading" and "residual" are up to scale: the prediction is fitted to gt by least squares and both are mapped
    to [0, 1] by the brightness quantile of gt. LPIPS sees the maps SSIM sees (invalid elements 0), which must lie in
    [0, 1]; its convolutions run in bf16 with fp32 accumulation.
    Returns ({"psnr", "ssim"[, "lpips"]}, {"n_valid", "scale", "quantile", "quantile_scale"}); the last three are None
    for the other targets. Raises ValueError for malformed input, for an up-to-scale target when no pixel is valid in
    channel 0 of the mask (the reference's torch.quantile of an empty tensor) and, with lpips, when a map the metric sees
    holds a value outside [0, 1] or a NaN (torchmetrics' input check)."""
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
    if lpips is not None and (H < lpips.min_size or W < lpips.min_size):
        raise ValueError(f"LPIPS ({lpips.net_name}) needs H, W >= {lpips.min_size}, got {H} x {W}")
    up_to_scale = target_name in ("shading", "residual")
    p, g, m = _inputs(pred, gt, valid_mask)
    if lpips is not None and lpips._h is None:
        raise ValueError("the LPIPS weights were closed")
    if lpips is not None and p.device != lpips.device:
        raise ValueError(f"the LPIPS weights are on {lpips.device}, the maps on {p.device}")
    lib = _lib.load()
    with torch.cuda.device(p.device):
        out = np.zeros(6 if lpips is None else 7, dtype=np.float64)
        if lpips is None:
            need = int(lib.mgb_eval_iid_ws_bytes(H, W))
            ws = _iid_ws.get(p.device)
            if ws is None or ws.numel() < need:
                ws = torch.empty(need, dtype=torch.uint8, device=p.device)
                _iid_ws[p.device] = ws
            rc = lib.mgb_eval_iid(ptr(p), ptr(g), ptr(m), H, W, int(up_to_scale), IID_TRANSFORMS.index(transform), ptr(ws),
                                  out.ctypes.data_as(C.c_void_p), stream_ptr())
        else:
            rc = lib.mgb_eval_iid_lpips(ptr(p), ptr(g), ptr(m), H, W, int(up_to_scale), IID_TRANSFORMS.index(transform),
                                        lpips._h, ptr(lpips._workspace(H, W)), out.ctypes.data_as(C.c_void_p), stream_ptr())
    if rc == _ERR_INVALID:
        raise ValueError(lib.mgb_last_error().decode("utf-8", "replace"))
    check(rc, "mgb_eval_iid" if lpips is None else "mgb_eval_iid_lpips")
    scaled = (float(out[3]), float(out[4]), float(out[5])) if up_to_scale else (None, None, None)
    info = {"n_valid": int(out[0]), **dict(zip(("scale", "quantile", "quantile_scale"), scaled))}
    metrics = dict(zip(IID_METRIC_NAMES, (float(out[1]), float(out[2]))))
    if lpips is not None:
        metrics["lpips"] = float(out[6])
    return metrics, info
