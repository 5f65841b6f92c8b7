"""The reference's evaluation steps restated with torch / numpy, for the evaluation tests: compute_cosine_error and the
normals metrics (src/util/metric.py:194-257, as script/normals/eval.py:145-157 calls them) and one depth sample of
script/depth/eval.py:171-217 in every alignment mode (src/util/alignment.py:35-101). Each runs on the device its inputs
are on; the reference's normals evaluation runs on CUDA when one is available."""
import numpy as np
import torch

NORMALS_METRICS = ("mean_angular_error", "median_angular_error", "rmse_angular_error", "sub5_error", "sub7_5_error",
                   "sub11_25_error", "sub22_5_error", "sub30_error")
THRESHOLDS = {"sub5_error": 5.0, "sub7_5_error": 7.5, "sub11_25_error": 11.25, "sub22_5_error": 22.5, "sub30_error": 30.0}


def cosine_error(pred: torch.Tensor, gt: torch.Tensor):
    """compute_cosine_error(pred, gt, masked=True) for [3,H,W] tensors: (errors of the valid pixels in row-major order as
    float32 numpy, the [H,W] valid mask as numpy)."""
    mask = torch.norm(gt, dim=0) > 0
    e = torch.cosine_similarity(pred[:, mask], gt[:, mask], dim=0)
    e = torch.acos(torch.clamp(e, min=-1.0, max=1.0)) * 180.0 / np.pi
    return e.cpu().numpy(), mask.cpu().numpy()


def normals_metrics(err: np.ndarray, decimals=None):
    """metric.py:222-257 on a float32 error vector, unrounded unless `decimals` is given."""
    n = err.shape[0]
    out = {"mean_angular_error": np.average(err), "median_angular_error": np.median(err),
           "rmse_angular_error": np.sqrt(np.sum(err * err) / n)}
    for k, t in THRESHOLDS.items():
        out[k] = 100.0 * (np.sum(err < t) / n)
    return {k: float(round(v, decimals) if decimals is not None else v) for k, v in out.items()}


def normals_metrics_f64(err: np.ndarray):
    """The same statistics of the float32 errors computed in float64 (no float32 accumulation)."""
    e = err.astype(np.float64)
    out = {"mean_angular_error": e.mean(), "median_angular_error": np.median(e), "rmse_angular_error": np.sqrt((e * e).mean())}
    for k, t in THRESHOLDS.items():
        out[k] = 100.0 * (np.sum(err < t) / err.shape[0])
    return {k: float(v) for k, v in out.items()}


def fit_maps(pred, gt, mask, max_res):
    """align_depth_least_square's downsampling (alignment.py:48-59): a [1,H,W] tensor through a nearest Upsample."""
    if max_res is None:
        return pred, gt, mask
    sf = np.min(max_res / np.array(pred.shape[-2:]))
    if not sf < 1:
        return pred, gt, mask
    down = torch.nn.Upsample(scale_factor=sf, mode="nearest")
    return (down(torch.as_tensor(pred).unsqueeze(0)).numpy(), down(torch.as_tensor(gt).unsqueeze(0)).numpy(),
            down(torch.as_tensor(mask).unsqueeze(0).float()).bool().numpy())


def lstsq(pred, gt, mask):
    p, g = pred[mask].reshape(-1, 1), gt[mask].reshape(-1, 1)
    X = np.linalg.lstsq(np.concatenate([p, np.ones_like(p)], axis=-1), g, rcond=None)[0]
    return X[0], X[1]


def depth_eval(pred, gt, valid, alignment, max_res, dmin, dmax):
    """script/depth/eval.py:171-217 for one [H,W] float32 sample on the CPU: (metrics, scale, shift)."""
    scale, shift = np.float32(1.0), np.float32(0.0)
    if alignment == "least_square":
        scale, shift = lstsq(*fit_maps(pred, gt, valid, max_res))
        pred = pred * scale + shift
    elif alignment == "least_square_disparity":
        disp = np.zeros_like(gt)
        disp[gt > 0] = 1.0 / gt[gt > 0]
        scale, shift = lstsq(*fit_maps(pred, disp, valid & (gt > 0) & (pred > 0), max_res))
        d = np.clip(pred * scale + shift, 1e-3, None)
        pred = np.zeros_like(d)
        pred[d > 0] = 1.0 / d[d > 0]
    pred = np.clip(np.clip(pred, dmin, dmax), 1e-6, None)
    o, t, m = torch.from_numpy(pred), torch.from_numpy(gt), torch.from_numpy(valid)
    n = m.sum()
    z = lambda v: torch.where(m, v, torch.zeros_like(v))  # noqa: E731
    dl = torch.log(o) - torch.log(t)
    r = torch.max(o / t, t / o)
    out = {
        "abs_relative_difference": (z((o - t).abs() / t).sum() / n).item(),
        "squared_relative_difference": (z((o - t).abs() ** 2 / t).sum() / n).item(),
        "rmse_linear": torch.sqrt(z((o - t) ** 2).sum() / n).item(),
        "rmse_log": torch.sqrt(z(dl ** 2).sum() / n).item(),
        "log10": (torch.log10(o[m]) - torch.log10(t[m])).abs().mean().item(),
        "delta1_acc": (z((r < 1.25).double()).sum() / n).item(),
        "delta2_acc": (z((r < 1.25 ** 2).double()).sum() / n).item(),
        "delta3_acc": (z((r < 1.25 ** 3).double()).sum() / n).item(),
        "i_rmse": torch.sqrt(z((1.0 / o - 1.0 / t) ** 2).sum() / n).item(),
        "silog_rmse": (torch.sqrt(z(dl ** 2).sum() / n - z(dl).sum() ** 2 / n ** 2) * 100).item(),
    }
    return out, float(np.asarray(scale).reshape(-1)[0]), float(np.asarray(shift).reshape(-1)[0])
