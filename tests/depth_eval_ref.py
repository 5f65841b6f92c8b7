"""Restatements of one depth sample of script/depth/eval.py:171-217 for the depth-evaluation tests (csrc/eval.cu:
eval_align_sums, eval_align_solve, eval_metric_sums, eval_metric_final), and the bounds the device is held to.

Three things are restated, none of them with a GPU:

fit_pixels        the flat indices of the pixels align_depth_least_square(max_resolution=...) fits. The reference gives
                  torch.nn.Upsample a [1, H, W] tensor, which Upsample reads as H signals of length W, so only the width
                  is downsampled; here the same call is applied to a [1, H, W] map of float64 flat indices (exact below
                  2^53; float32 indices would fail at 4032 x 6048 > 2^24).
depth_eval_f64    everything in float64 from the definition: the judge of the sums. The fit is np.linalg.lstsq in float64
                  (its rank rule: singular values of [p 1] at or below eps * max(n, 2) * sigma_max are dropped and the
                  minimum-norm solution returned), the disparity path, the clips, the sums, the metrics, the aligned map.
                  dmin and dmax are rounded to float32 first, as the device receives them.
depth_eval_ref32  the reference's dtype flow, step by step. np.linalg.lstsq on float32 maps computes in double and returns
                  a FLOAT32 scale and shift, so pred * scale + shift is fl(fl(p s) + t), np.clip(., 1e-3) clips at
                  float32(1e-3), disparity2depth is a float32 reciprocal, both clips are float32, and the torch metrics are
                  float32: o / t, t / o, max and < of threshold_percentage decide the delta accuracies in float32.
                  Returns those per-pixel decisions and the float32 aligned map.

What the device is held to. The delta accuracies are counts: they must EQUAL depth_eval_ref32's. Every other output is
held to depth_eval_f64 within a bound derived here, not measured (u = 2^-53):

  sums     A double sum of n terms, in any order, is off by at most gamma = n u / (1 - n u) times the sum of the terms'
           magnitudes (Higham, Accuracy and Stability, 4.2). The device's order (strided per-thread sums, xor trees) has
           chains far shorter than n, so n u is conservative; each term's own few roundings are covered by GAMMA_TERM u.
  fit      The device solves the 2 x 2 normal equations from sums of d = p - c about a pivot c that is some fit pixel's
           prediction (exact in double), so the cancellation in n sum d^2 - (sum d)^2 and n sum d g - sum d sum g is
           governed by how far the pivot is from the mean, not by mean / std: the error scales with the condition number
           of the centred problem, not its square. With d_w = |p - mean| + max |p - mean| (an upper bound of |d| for any
           pivot among the data),
             |ds| <= gamma |s| [ (sum d_w |g| + sum d_w sum |g| / n) / |cov| + (sum d_w^2 + (sum d_w)^2 / n) / var ],
             |dt| <= |ds| (|mean| + max |p - mean|) + d0,  d0 = gamma (sum |g| / n + |s| sum d_w / n) + 8 u |s| max |p|,
           and, because the errors of s and t cancel at the mean, the fitted value at p moves by at most
           |ds| (|p - mean| + max |p - mean|) + d0 (this, not |ds| |p| + |dt|, is what reaches the metrics), with
           cov = sum (p - mean)(g - gmean), var = sum (p - mean)^2. (Uncentred sums would carry mean^2 / var: at
           mean / std = 10^4 that is 10^8 u n, at 10^6 no digit is left.) For a rank-deficient fit the solution is
           g_mean (m, 1) / (m^2 + 1), whose error is a few gamma of its size.
  metrics  The aligned value moves by at most e = (the fitted value's bound above) + 4 u |a|; the clips are 1-Lipschitz, and a pixel that
           stays more than e beyond a clip does not move at all (without this a pixel saturated at a min_depth of 1e-5
           would charge e / 1e-5 to the logs); the disparity reciprocal turns e into e a^2 (1 + 2 e a). Each metric's sum then moves by its derivative times e:
           1 / g (abs_rel), (2 |a - g| + e) / g (sq_rel), 1 / a for the logs, 1 / a^2 for i_rmse, the root-mean-squares by
           the triangle inequality in l2, and silog through V = mean dl^2 - (mean dl)^2: dV <= d(mean dl^2) +
           2 |mean dl| d(mean dl), silog moves by at most 100 (sqrt(V + dV) - sqrt(max(V - dV, 0))), which states the
           cancellation: when V is of the order of dV nothing better than 100 sqrt(2 dV) holds. log and log10 on the
           device are within 2 ulp: 4 u (|log a| + |log g|) per term.
"""
import numpy as np
import torch

METRICS = ("abs_relative_difference", "squared_relative_difference", "rmse_linear", "rmse_log", "log10", "delta1_acc",
           "delta2_acc", "delta3_acc", "i_rmse", "silog_rmse")
DELTAS = ("delta1_acc", "delta2_acc", "delta3_acc")
THRESHOLDS = (1.25, 1.25 ** 2, 1.25 ** 3)          # exact in float32
U = 2.0 ** -53
GAMMA_TERM = 16                                    # roundings inside one term of a sum


def fit_pixels(H, W, max_res):
    """Flat int64 indices (row-major) of the pixels the fit uses, in the downsampled map's order."""
    idx = torch.arange(H * W, dtype=torch.float64).reshape(H, W)
    if max_res is not None:
        sf = np.min(max_res / np.array((H, W)))
        if sf < 1:
            idx = torch.nn.Upsample(scale_factor=sf, mode="nearest")(idx.unsqueeze(0))
    return idx.reshape(-1).to(torch.int64).numpy()


def _fit_set(pred, gt, valid, alignment, max_res):
    """(p, g) float32 vectors of the fit: the kept pixels that are valid (and gt > 0, pred > 0 for disparity)."""
    q = fit_pixels(*pred.shape, max_res)
    p, g, m = pred.reshape(-1)[q], gt.reshape(-1)[q], valid.reshape(-1)[q].copy()
    if alignment == "least_square_disparity":
        m &= (g > 0) & (p > 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            g = np.where(g > 0, np.float32(1.0) / g, np.float32(0.0)).astype(np.float32)    # depth2disparity, float32
    return p[m], g[m]


def lstsq_f64(p, g):
    """(scale, shift) of min ||[p 1] x - g|| in float64 by numpy's SVD lstsq; (0, 0) for an empty fit, as lstsq gives."""
    if p.size == 0:
        return 0.0, 0.0
    p, g = p.astype(np.float64), g.astype(np.float64)
    x = np.linalg.lstsq(np.stack([p, np.ones_like(p)], axis=-1), g, rcond=None)[0]
    return float(x[0]), float(x[1])


def fit_bound(p, g, s):
    """(|ds|, |dt|, (mean, R, d0)) the device's fit may differ by from the float64 SVD (module docstring); the fitted
    value at p moves by at most |ds| (|p - mean| + R) + d0."""
    n = p.size
    if n == 0:
        return 0.0, 0.0, (0.0, 0.0, 0.0)
    p, g = p.astype(np.float64), g.astype(np.float64)
    gamma = (n + GAMMA_TERM) * U
    pm, gm = p.mean(), g.mean()
    dp = p - pm
    var, cov = float((dp * dp).sum()), float((dp * (g - gm)).sum())
    A = np.stack([p, np.ones_like(p)], axis=-1)
    sv = np.linalg.svd(A, compute_uv=False)
    if n < 2 or sv[-1] <= np.finfo(np.float64).eps * max(n, 2) * sv[0]:                   # rank 1: gm (m, 1) / (m^2 + 1)
        size = abs(gm) / np.sqrt(pm * pm + 1.0)
        return 8 * gamma * size + 1e-300, 8 * gamma * size + 1e-300, (0.0, 0.0, 8 * gamma * size + 1e-300)
    R = float(np.abs(dp).max())
    dw = np.abs(dp) + R
    ag = np.abs(g)
    num = (dw * ag).sum() + dw.sum() * ag.sum() / n
    den = (dw * dw).sum() + dw.sum() ** 2 / n
    ds = gamma * abs(s) * (num / max(abs(cov), 1e-300) + den / var) if cov != 0.0 else gamma * num / var
    d0 = gamma * (ag.sum() / n + abs(s) * dw.sum() / n) + 8 * U * abs(s) * float(np.abs(p).max())
    return float(ds), float(ds * (abs(pm) + R) + d0), (float(pm), R, float(d0))


def _metrics_f64(a, g):
    dl = np.log(a) - np.log(g)
    out = {"abs_relative_difference": np.mean(np.abs(a - g) / g), "squared_relative_difference": np.mean((a - g) ** 2 / g),
           "rmse_linear": np.sqrt(np.mean((a - g) ** 2)), "rmse_log": np.sqrt(np.mean(dl ** 2)),
           "log10": np.mean(np.abs(np.log10(a) - np.log10(g)))}
    r = np.maximum(a / g, g / a)
    for k, t in zip(DELTAS, THRESHOLDS):
        out[k] = np.mean(r < t)
    out["i_rmse"] = np.sqrt(np.mean((1.0 / a - 1.0 / g) ** 2))
    out["silog_rmse"] = 100.0 * np.sqrt(max(np.mean(dl ** 2) - np.mean(dl) ** 2, 0.0))
    return {k: float(v) for k, v in out.items()}


def align_f64(pred, scale, shift, alignment, dmin, dmax):
    """The aligned, clipped map in float64 from a given scale and shift."""
    a = pred.astype(np.float64) * scale + shift
    if alignment == "least_square_disparity":
        a = 1.0 / np.maximum(a, 1e-3)
    lo, hi = float(np.float32(dmin)), float(np.float32(dmax))
    return np.maximum(np.minimum(np.maximum(a, lo), hi), 1e-6)


def depth_eval_f64(pred, gt, valid, alignment, max_res, dmin, dmax):
    """(metrics, scale, shift, n_valid, aligned float64 map, bounds): the float64 judge and the bound of |device - it|
    for every metric that is bounded (the deltas are not: they are exact against depth_eval_ref32), "scale" and "shift"."""
    pred, gt, valid = np.asarray(pred, np.float32), np.asarray(gt, np.float32), np.asarray(valid, bool)
    scale, shift, ds, dt, (pm, rad, d0) = 1.0, 0.0, 0.0, 0.0, (0.0, 0.0, 0.0)
    if alignment is not None:
        fp, fg = _fit_set(pred, gt, valid, alignment, max_res)
        scale, shift = lstsq_f64(fp, fg)
        ds, dt, (pm, rad, d0) = fit_bound(fp, fg, scale)
    aligned = align_f64(pred, scale, shift, alignment, dmin, dmax)
    n = int(valid.sum())
    bounds = {"scale": ds, "shift": dt}
    if n == 0:
        return {k: float("nan") for k in METRICS}, scale, shift, 0, aligned, bounds
    a, g, p = aligned[valid], gt[valid].astype(np.float64), pred[valid].astype(np.float64)
    with np.errstate(all="ignore"):
        m = _metrics_f64(a, g)
        lo, hi = max(float(np.float32(dmin)), 1e-6), float(np.float32(dmax))
        raw = p * scale + shift
        e = ds * (np.abs(p - pm) + rad) + d0 + 4 * U * np.abs(raw)
        if alignment == "least_square_disparity":
            e = np.where(raw + e < 1e-3, 0.0, e)              # stays clipped to 1e-3 whatever the fit's error
            raw = 1.0 / np.maximum(raw, 1e-3)
            e = e * raw * raw * (1.0 + 2.0 * e * raw)
        e = np.where((raw + e < lo) | (raw - e > hi), 0.0, e) + 4 * U * a      # a saturated pixel does not move
        gamma = (n + GAMMA_TERM) * U
        d = np.abs(a - g)
        la = e / np.maximum(a - e, 1e-300) + 4 * U * (np.abs(np.log(a)) + np.abs(np.log(g)))     # of dl
        dl = np.log(a) - np.log(g)
        bounds["abs_relative_difference"] = np.mean(e / g) + gamma * m["abs_relative_difference"]
        bounds["squared_relative_difference"] = np.mean((2 * d + e) * e / g) + gamma * m["squared_relative_difference"]
        bounds["rmse_linear"] = np.sqrt(np.mean(e * e)) + gamma * m["rmse_linear"]
        bounds["rmse_log"] = np.sqrt(np.mean(la * la)) + gamma * m["rmse_log"]
        bounds["log10"] = np.mean(la) / np.log(10.0) + gamma * m["log10"]
        ie = e / np.maximum(a - e, 1e-300) ** 2 + 4 * U * (1.0 / a + 1.0 / g)
        bounds["i_rmse"] = np.sqrt(np.mean(ie * ie)) + gamma * m["i_rmse"]
        m2, m1 = np.mean(dl * dl), np.mean(dl)
        dV = np.mean((2 * np.abs(dl) + la) * la) + gamma * m2 + 2 * abs(m1) * (np.mean(la) + gamma * np.mean(np.abs(dl)))
        V = m2 - m1 * m1
        dV += 4 * U * (m2 + m1 * m1)                                                             # the subtraction's operands
        bounds["silog_rmse"] = 100.0 * (np.sqrt(max(V, 0.0) + dV) - np.sqrt(max(V - dV, 0.0)))
    return m, scale, shift, n, aligned, {k: float(v) for k, v in bounds.items()}


def lstsq_ref32(p, g):
    """The reference's call: float32 columns into np.linalg.lstsq, which returns float32."""
    p, g = p.reshape(-1, 1), g.reshape(-1, 1)
    x = np.linalg.lstsq(np.concatenate([p, np.ones_like(p)], axis=-1), g, rcond=None)[0]
    assert x.dtype == np.float32
    return x[0, 0], x[1, 0]


def align_ref32(pred, scale, shift, alignment, dmin, dmax):
    """fl(fl(p s) + t), the float32 disparity clip and reciprocal, the float32 clips: the reference's aligned map."""
    a = pred * np.float32(scale) + np.float32(shift)
    assert a.dtype == np.float32
    if alignment == "least_square_disparity":
        a = np.float32(1.0) / np.maximum(a, np.float32(1e-3))
    return np.maximum(np.minimum(np.maximum(a, np.float32(dmin)), np.float32(dmax)), np.float32(1e-6))


def delta_bits_ref32(aligned32, gt):
    """[3, H, W] bool: threshold_percentage's bit_mat for 1.25, 1.25^2, 1.25^3, in torch float32."""
    o, t = torch.from_numpy(np.ascontiguousarray(aligned32)), torch.from_numpy(np.ascontiguousarray(gt))
    r = torch.max(o / t, t / o)
    return np.stack([(r < thr).numpy() for thr in THRESHOLDS])


def depth_eval_ref32(pred, gt, valid, alignment, max_res, dmin, dmax, scale_shift=None):
    """(metrics, scale, shift, n_valid, float32 aligned map, [3, H, W] delta decisions). The metrics are torch float32
    sums as the reference takes them; the delta values are count / n. scale_shift: use this (scale, shift) instead of the
    fit (to restate the device's decisions from the device's own fit)."""
    pred, gt, valid = np.asarray(pred, np.float32), np.asarray(gt, np.float32), np.asarray(valid, bool)
    scale, shift = np.float32(1.0), np.float32(0.0)
    if scale_shift is not None:
        scale, shift = np.float32(scale_shift[0]), np.float32(scale_shift[1])
    elif alignment is not None:
        scale, shift = lstsq_ref32(*_fit_set(pred, gt, valid, alignment, max_res))      # an empty fit gives 0, 0
    with np.errstate(all="ignore"):
        aligned = align_ref32(pred, scale, shift, alignment, dmin, dmax)      # p * 1 + 0 is p: alignment None
        bits = delta_bits_ref32(aligned, gt)
        n = int(valid.sum())
        o, t, m = torch.from_numpy(aligned), torch.from_numpy(gt), torch.from_numpy(valid)
        z = lambda v: torch.where(m, v, torch.zeros_like(v))  # noqa: E731
        dl = torch.log(o) - torch.log(t)
        out = {
            "abs_relative_difference": (z((o - t).abs() / t).sum() / n).item(),
            "squared_relative_difference": (z((o - t).abs() ** 2 / t).sum() / n).item(),
            "rmse_linear": torch.sqrt(z((o - t) ** 2).sum() / n).item(),
            "rmse_log": torch.sqrt(z(dl ** 2).sum() / n).item(),
            "log10": (torch.log10(o[m]) - torch.log10(t[m])).abs().mean().item(),
            "i_rmse": torch.sqrt(z((1.0 / o - 1.0 / t) ** 2).sum() / n).item(),
            "silog_rmse": (torch.sqrt(z(dl ** 2).sum() / n - z(dl).sum() ** 2 / n ** 2) * 100).item(),
        } if n else {k: float("nan") for k in METRICS}
        for k, b in zip(DELTAS, bits):
            out[k] = float(np.count_nonzero(b & valid)) / n if n else float("nan")
    return out, float(scale), float(shift), n, aligned, bits
