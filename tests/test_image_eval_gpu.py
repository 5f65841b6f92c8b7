"""Device-side bookends (`-m gpu`): antialiased resize, colourisation, least-squares alignment + depth metrics, each against
the reference's own code path restated with torch / numpy on the same inputs (reference marigold/util/image_util.py:38-120,
src/util/alignment.py:35-82, src/util/metric.py:64-191, script/depth/eval.py:171-217) and against the goldens the live
reference produced for resize_max_res (tests/golden/ensemble_golden.npz)."""
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.golden.cases import RESIZE_CASES, resize_input

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).resolve().parent / "golden" / "ensemble_golden.npz")


@pytest.mark.parametrize("name", list(RESIZE_CASES))
def test_resize_max_res_matches_reference_golden(name):
    from marigold_b200.pipeline import get_tv_resample_method, resize_max_res

    cfg = RESIZE_CASES[name]
    img = resize_input(cfg)                                              # uint8 [1,3,H,W]
    out = resize_max_res(img.cuda(), cfg["max_edge"], get_tv_resample_method(cfg["method"]))
    g = GOLD[f"resize/{name}"]
    assert out.dtype == torch.uint8 and tuple(out.shape) == g.shape
    d = np.abs(out.cpu().numpy().astype(np.int32) - g.astype(np.int32))
    assert d.max() == 0                                                  # the image is resized in torch CPU's arithmetic


@pytest.mark.parametrize("mode", ["bilinear", "bicubic", "nearest-exact"])
@pytest.mark.parametrize("size", [(768, 576), (100, 333), (37, 19)])
def test_resize_matches_torch_float_path(mode, size):
    from marigold_b200 import imageops

    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 3, 240, 320, generator=g).cuda() * 4 - 2
    out = imageops.resize(x, size, mode, arith="cuda")
    if mode == "nearest-exact":
        ref = F.interpolate(x, size=size, mode=mode)
    else:
        ref = F.interpolate(x, size=size, mode=mode, antialias=True, align_corners=False)
    assert torch.equal(out, ref) and torch.equal(out.view(torch.int32), ref.view(torch.int32))


def test_fused_normalisation_and_colorize():
    from marigold_b200 import imageops
    from marigold_b200.pipeline import colorize_depth_maps

    img = torch.randint(0, 256, (1, 3, 300, 500), dtype=torch.uint8, generator=torch.Generator().manual_seed(1)).cuda()
    a = imageops.resize(img, (230, 384), "bilinear", post=2)
    # the reference normalises on the HOST (true division; torch's CUDA div-by-scalar multiplies by the reciprocal instead)
    b = imageops.resize(img, (230, 384), "bilinear", post=1).cpu() / 255.0 * 2.0 - 1.0
    assert torch.equal(a.cpu(), b) and float(a.min()) >= -1 and float(a.max()) <= 1
    d = torch.rand(123, 77, generator=torch.Generator().manual_seed(2))
    d[0, 0], d[0, 1], d[0, 2] = 0.0, 1.0, 0.5
    got = imageops.colorize_u8(d.cuda(), 0, 1, imageops.spectral_lut_u8()).cpu().numpy()
    ref = np.moveaxis((colorize_depth_maps(d.numpy(), 0, 1).squeeze() * 255).astype(np.uint8), 0, -1)
    np.testing.assert_array_equal(got, ref)


def _ref_eval(pred, gt, mask, dmin, dmax, align):
    """script/depth/eval.py:171-217 with the reference's functions restated (numpy lstsq, torch metrics)."""
    p = pred.astype(np.float32)
    scale, shift = 1.0, 0.0
    if align:
        A = np.concatenate([p[mask].reshape(-1, 1), np.ones((int(mask.sum()), 1), np.float32)], axis=-1)
        X = np.linalg.lstsq(A, gt[mask].reshape(-1, 1), rcond=None)[0]
        scale, shift = float(X[0, 0]), float(X[1, 0])
        p = p * X[0] + X[1]                                             # lstsq returns float32: float32 throughout, as the reference
    p = np.clip(np.clip(p, dmin, dmax), 1e-6, None)
    o, t, m = torch.from_numpy(p), torch.from_numpy(gt), torch.from_numpy(mask)
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
    return out, scale, shift


@pytest.mark.parametrize("align", [True, False])
def test_alignment_and_metrics_match_reference_functions(align):
    from marigold_b200.evaluation import align_depth_least_square, evaluate_depth

    rng = np.random.default_rng(3)
    H, W = 480, 640
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    gt = (1.0 + 4.0 * (0.5 + 0.4 * np.sin(3 * xx + 2 * yy)) + 0.05 * rng.standard_normal((H, W))).astype(np.float32)
    pred = (((gt - 0.7) / 5.1) + 0.02 * rng.standard_normal((H, W))).astype(np.float32)     # affine-invariant prediction
    if not align:
        pred = (gt * (1 + 0.05 * rng.standard_normal((H, W)))).astype(np.float32)
    mask = rng.uniform(size=(H, W)) > 0.2
    ref, scale, shift = _ref_eval(pred, gt, mask, 0.5, 6.0, align)
    got, info = evaluate_depth(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(), torch.from_numpy(mask).cuda(),
                               alignment="least_square" if align else None, min_depth=0.5, max_depth=6.0)
    assert info["n_valid"] == int(mask.sum())
    if align:
        assert abs(info["scale"] - scale) <= 1e-5 * abs(scale) and abs(info["shift"] - shift) <= 1e-5 * max(1.0, abs(shift))
    tol = 2e-5 if align else 1e-6          # the fit differs in the 6th digit: normal equations in double vs float32 SVD lstsq
    for k, v in ref.items():
        assert abs(got[k] - v) <= tol * max(1.0, abs(v)), (k, got[k], v)
    if align:
        al, s2, t2 = align_depth_least_square(torch.from_numpy(gt).cuda(), torch.from_numpy(pred).cuda(),
                                              torch.from_numpy(mask).cuda())
        assert abs(s2 - scale) <= 1e-5 * abs(scale) and al.shape == (H, W)
        assert np.abs(al.cpu().numpy() - (pred * scale + shift)).max() < 1e-4
