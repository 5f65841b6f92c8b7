"""Seeded inputs of the intrinsic-image evaluation cases (script/iid/eval.py:182-213), shared by make_iid_eval_golden.py
(reference run) and the tests.

mask: "none"; "pixel" (one random pixel mask on all three channels, as the datasets build it); "split" (channel 0 differs
from channels 1-2, so the quantile's pixels are not the fit's); "single" (one valid pixel); "empty" (none valid).
kind: "noisy" (pred = a * gt + noise); "q255" (gt quantised to 1/255: heavy ties at the quantile); "dark" (brightness
below 1e-4 everywhere: quantile scale 0); "nan" (gt NaN where no channel is valid); "wide" (pred outside [0, 1])."""
import numpy as np

IID_EVAL_CASES = {
    "albedo_11x11": dict(H=11, W=11, seed=71, target="albedo", mask="none", transform=None, kind="noisy"),
    "shading_11x11": dict(H=11, W=11, seed=72, target="shading", mask="pixel", transform=None, kind="noisy"),
    "shading_37x53_pixel": dict(H=37, W=53, seed=73, target="shading", mask="pixel", transform=None, kind="noisy"),
    "residual_37x53_split_lin": dict(H=37, W=53, seed=74, target="residual", mask="split", transform="srgb2linear",
                                     kind="noisy"),
    "material_37x53_pixel_srgb": dict(H=37, W=53, seed=75, target="material", mask="pixel", transform="linear2srgb",
                                      kind="noisy"),
    "albedo_48x64_split_lin": dict(H=48, W=64, seed=76, target="albedo", mask="split", transform="srgb2linear", kind="noisy"),
    "shading_48x64_q255": dict(H=48, W=64, seed=77, target="shading", mask="none", transform=None, kind="q255"),
    "residual_48x64_q255_srgb": dict(H=48, W=64, seed=78, target="residual", mask="pixel", transform="linear2srgb",
                                     kind="q255"),
    "shading_40x40_dark": dict(H=40, W=40, seed=79, target="shading", mask="none", transform=None, kind="dark"),
    "shading_37x53_single": dict(H=37, W=53, seed=80, target="shading", mask="single", transform=None, kind="noisy"),
    "albedo_37x53_single": dict(H=37, W=53, seed=81, target="albedo", mask="single", transform=None, kind="noisy"),
    "albedo_24x24_empty": dict(H=24, W=24, seed=82, target="albedo", mask="empty", transform=None, kind="noisy"),
    "shading_24x24_empty": dict(H=24, W=24, seed=83, target="shading", mask="empty", transform=None, kind="noisy"),
    "residual_64x80_nan": dict(H=64, W=80, seed=84, target="residual", mask="pixel", transform=None, kind="nan"),
    "albedo_64x80_nan_lin": dict(H=64, W=80, seed=85, target="albedo", mask="split", transform="srgb2linear", kind="nan"),
    "material_37x53_wide": dict(H=37, W=53, seed=86, target="material", mask="pixel", transform=None, kind="wide"),
    "albedo_37x53_wide_nomask": dict(H=37, W=53, seed=87, target="albedo", mask="none", transform=None, kind="wide"),
}


def iid_eval_input(cfg):
    """(pred, gt, mask) for one target of one sample: fp32 [3,H,W] maps and a bool [3,H,W] mask or None."""
    rng = np.random.default_rng(cfg["seed"])
    H, W = cfg["H"], cfg["W"]
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    base = 0.5 + 0.35 * np.sin(4 * xx + 3 * yy + np.arange(3)[:, None, None])
    gt = np.clip(base + 0.08 * rng.standard_normal((3, H, W)), 0.0, 1.0)
    kind = cfg["kind"]
    if kind == "q255":
        gt = np.round(gt * 255) / 255
        gt[1:] = gt[0]               # grey: the brightness takes at most 256 values
    elif kind == "dark":
        gt = gt * 5e-5
    a = 0.6 if cfg["target"] in ("shading", "residual") else 1.0
    pred = a * gt + 0.04 * rng.standard_normal((3, H, W)) * (gt.max() if kind == "dark" else 1.0)
    if kind == "wide":
        pred = 1.6 * pred - 0.3
    pixel = rng.uniform(size=(H, W)) > 0.25
    m = cfg["mask"]
    if m == "none":
        mask = None
    elif m == "pixel":
        mask = np.broadcast_to(pixel, (3, H, W)).copy()
    elif m == "split":
        other = rng.uniform(size=(H, W)) > 0.4
        mask = np.stack([pixel, other, other])
    elif m == "single":
        mask = np.zeros((3, H, W), bool)
        mask[:, rng.integers(H), rng.integers(W)] = True
    else:
        assert m == "empty", m
        mask = np.zeros((3, H, W), bool)
    if kind == "nan":
        gt[:, ~mask.any(0)] = np.nan
    if cfg["transform"] is not None:
        pred = np.abs(pred)          # x ** 2.2 of a negative value is NaN
    return pred.astype(np.float32), gt.astype(np.float32), mask
