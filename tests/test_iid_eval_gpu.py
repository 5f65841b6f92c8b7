"""Device intrinsic-image evaluation (`-m gpu`): evaluate_iid (csrc/eval.cu) against the float64 restatement of
compute_iid_metric (tests/iid_eval_ref.py), against torch's own float32 quantile on the same GPU, and against the
reference's results (tests/golden/iid_eval_golden.npz)."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import iid_eval_ref
from tests.golden.iid_eval_cases import IID_EVAL_CASES, iid_eval_input

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).resolve().parent / "golden" / "iid_eval_golden.npz")
LAUNCHES = {False: 2, True: 6}     # ssim, final; up to scale also stats, locate, refine, select (memsets not counted)
# Measured on an H100 80GB HBM3 (400 W power limit) over these cases: against the float64 restatement at most
# 7.3e-6 dB and 4.3e-7; against the reference's float32 results (the golden) at most 2.6e-5 dB (one valid pixel, where
# an ulp of the fitted scale shows) and 9.4e-7. The bounds leave a margin of 4x or more.
PSNR_TOL, SSIM_TOL = 5e-5, 3e-6                    # dB; against the float64 restatement
GOLD_PSNR_TOL, GOLD_SSIM_TOL = 1e-4, 5e-6          # dB; against the golden
SCALE_TOL = 1e-6                   # relative, against the float64 sum pg / sum p^2 and the reference's float32 lstsq
SIZES = [(11, 11), (37, 53), (480, 640), (768, 1024), (1080, 1920)]
# (target, mask, transform, kind): see tests/golden/iid_eval_cases.py
CONFIGS = [
    ("albedo", "none", None, "noisy"),
    ("material", "pixel", "srgb2linear", "noisy"),
    ("shading", "split", "linear2srgb", "noisy"),
    ("residual", "pixel", None, "q255"),
    ("shading", "none", "srgb2linear", "q255"),
    ("residual", "split", None, "nan"),
    ("albedo", "split", "linear2srgb", "nan"),
    ("material", "single", None, "wide"),
    ("albedo", "none", None, "wide"),
    ("shading", "single", None, "noisy"),
    ("residual", "none", None, "dark"),
    ("albedo", "empty", None, "noisy"),
]


def _dev(a):
    return torch.from_numpy(a).cuda() if a is not None else None


def _run(pred, gt, target, mask, transform):
    """evaluate_iid twice: the launch count of the first call, equal bits from the second."""
    from marigold_b200 import _lib
    from marigold_b200.evaluation import evaluate_iid

    lib = _lib.load()
    torch.cuda.synchronize()
    l0 = lib.mgb_launch_count()
    got, info = evaluate_iid(pred, gt, target, mask, transform)
    assert lib.mgb_launch_count() - l0 == LAUNCHES[target in iid_eval_ref.UP_TO_SCALE]
    got2, info2 = evaluate_iid(pred, gt, target, mask, transform)
    assert np.array([got[k] for k in got]).tobytes() == np.array([got2[k] for k in got2]).tobytes()
    assert repr(info) == repr(info2)
    return got, info


def _close(a, b, tol):
    if np.isnan(b) or np.isinf(b):
        return np.array_equal(a, b, equal_nan=True)
    return abs(a - b) <= tol


def _check(pred, gt, target, mask, transform, got, info):
    """Against the float64 restatement and torch's float32 quantile; returns (|dpsnr|, |dssim|)."""
    ref, r64 = iid_eval_ref.evaluate(pred, gt, target, mask, transform, dtype=torch.float64)
    assert info["n_valid"] == (pred.numel() if mask is None else int(mask.sum()))
    if target in iid_eval_ref.UP_TO_SCALE:
        assert abs(info["scale"] - r64["scale"]) <= SCALE_TOL * abs(r64["scale"]), (info["scale"], r64["scale"])
        lo, hi, w = iid_eval_ref.quantile_order_statistics(gt, mask, transform)
        q = np.float32(info["quantile"])
        assert q == iid_eval_ref.lerp_f32(lo, hi, w), (q, lo, hi, w)          # the order statistics exactly
        b = iid_eval_ref.brightness(iid_eval_ref.colour(gt.float(), transform))
        tq = np.float32(torch.quantile(b[mask[0]] if mask is not None else b.reshape(-1), 0.9).item())
        assert abs(q - tq) <= np.spacing(tq), (q, tq)                          # torch's lerp to 1 ulp
        k = np.float32(0) if q < np.float32(1e-4) else np.float32(np.float32(1) / q) * np.float32(0.8)
        assert np.float32(info["quantile_scale"]) == k
    else:
        assert info["scale"] is None and info["quantile"] is None and info["quantile_scale"] is None
    assert _close(got["psnr"], ref["psnr"], PSNR_TOL), (got["psnr"], ref["psnr"])
    assert _close(got["ssim"], ref["ssim"], SSIM_TOL), (got["ssim"], ref["ssim"])
    d = lambda a, b: 0.0 if not np.isfinite(b) else abs(a - b)  # noqa: E731
    return d(got["psnr"], ref["psnr"]), d(got["ssim"], ref["ssim"])


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("target,mask,transform,kind", CONFIGS)
def test_iid_matches_float64_restatement(H, W, target, mask, transform, kind):
    from marigold_b200.evaluation import evaluate_iid

    cfg = dict(H=H, W=W, seed=H * 31 + W + CONFIGS.index((target, mask, transform, kind)), target=target, mask=mask,
               transform=transform, kind=kind)
    pred, gt, m = (_dev(a) for a in iid_eval_input(cfg))
    if mask == "empty" and target in iid_eval_ref.UP_TO_SCALE:
        with pytest.raises(ValueError):
            evaluate_iid(pred, gt, target, m, transform)
        return
    got, info = _run(pred, gt, target, m, transform)
    dp, ds = _check(pred, gt, target, m, transform, got, info)
    if kind == "nan":
        assert np.isfinite(got["psnr"]) and np.isfinite(got["ssim"])
    if kind == "dark":
        assert info["quantile_scale"] == 0.0 and got["psnr"] == np.inf and got["ssim"] == 1.0
    if mask == "empty":
        assert np.isnan(got["psnr"]) and got["ssim"] == 1.0 and info["n_valid"] == 0
    print(f"{target} {mask} {transform} {kind} {H}x{W}: |dpsnr| {dp:.3e} dB |dssim| {ds:.3e}")


@pytest.mark.parametrize("name", list(IID_EVAL_CASES))
def test_iid_matches_reference_golden(name):
    from marigold_b200.evaluation import evaluate_iid

    cfg = IID_EVAL_CASES[name]
    pred, gt, mask = (_dev(a) for a in iid_eval_input(cfg))
    if f"{name}/raises" in GOLD:
        with pytest.raises(ValueError):
            evaluate_iid(pred[None], gt[None], cfg["target"], mask, cfg["transform"])
        return
    got, info = _run(pred[None], gt[None], cfg["target"], mask, cfg["transform"])        # [1,3,H,W] as eval.py has them
    dp, ds = _check(pred, gt, cfg["target"], mask, cfg["transform"], got, info)
    if cfg["target"] in iid_eval_ref.UP_TO_SCALE:
        s, q = GOLD[f"{name}/scale"].astype(np.float64), GOLD[f"{name}/quantile"]
        assert np.abs(info["scale"] - s).max() <= SCALE_TOL * abs(info["scale"]), (info["scale"], s)
        if cfg["transform"] is None:     # otherwise the CPU's pow, not the GPU's, made the golden's brightness
            assert np.abs(np.float32(info["quantile"]) - q).max() <= np.spacing(q).max(), (info["quantile"], q)
    for k, tol in (("psnr", GOLD_PSNR_TOL), ("ssim", GOLD_SSIM_TOL)):
        g = float(GOLD[f"{name}/{k}"])
        assert _close(got[k], g, tol), (k, got[k], g)
    print(f"{name}: psnr {got['psnr']!r} vs {float(GOLD[f'{name}/psnr'])!r}, ssim {got['ssim']!r} vs "
          f"{float(GOLD[f'{name}/ssim'])!r}; float64: |dpsnr| {dp:.3e} dB |dssim| {ds:.3e}")


def test_iid_quantile_takes_channel_0_of_the_mask_and_the_float32_rank():
    """n = 307200 valid pixels: torch's float32 rank is 276479.09375 (not 276479.1); the pixels of channel 0 only."""
    from marigold_b200.evaluation import evaluate_iid

    H, W = 480, 640
    g = torch.Generator().manual_seed(11)
    gt = torch.rand(3, H, W, generator=g).cuda()
    pred = (0.7 * gt + 0.05 * torch.rand(3, H, W, generator=g).cuda()).contiguous()
    mask = torch.ones(3, H, W, dtype=torch.bool, device="cuda")
    assert np.float32(0.9) * np.float32(H * W - 1) == np.float32(276479.09375)
    _, info = evaluate_iid(pred, gt, "shading", mask)
    lo, hi, w = iid_eval_ref.quantile_order_statistics(gt, mask)
    assert w == np.float32(0.09375) and np.float32(info["quantile"]) == iid_eval_ref.lerp_f32(lo, hi, w)
    mask[1, : H // 2] = False                                         # channels 1-2 do not select the quantile's pixels
    mask[0, H // 2:] = False
    _, info = evaluate_iid(pred, gt, "shading", mask)
    lo, hi, w = iid_eval_ref.quantile_order_statistics(gt, mask)
    assert np.float32(info["quantile"]) == iid_eval_ref.lerp_f32(lo, hi, w)
    b = iid_eval_ref.brightness(gt)
    assert torch.quantile(b[mask[1]], 0.9).item() != info["quantile"]


def test_iid_rejects_malformed_input():
    from marigold_b200 import _lib
    from marigold_b200.evaluation import evaluate_iid

    x = torch.rand(3, 16, 16, device="cuda")
    with pytest.raises(_lib.MgbError):
        evaluate_iid(x.cpu(), x.cpu(), "albedo")
    with pytest.raises(ValueError):
        evaluate_iid(x, x[:, :, :15], "albedo")
    with pytest.raises(ValueError):
        evaluate_iid(x[:2], x[:2], "albedo")
    with pytest.raises(ValueError):
        evaluate_iid(x[:, :10], x[:, :10], "albedo")                  # SSIM's window needs H, W >= 11
    with pytest.raises(ValueError):
        evaluate_iid(x, x, "albedo", transform="gamma")
    with pytest.raises(ValueError):
        evaluate_iid(x, x, "albedo", torch.ones(16, 16, dtype=torch.bool, device="cuda"))
    m = torch.ones(3, 16, 16, dtype=torch.bool, device="cuda")
    m[0] = False                                                      # no pixel for the quantile, elements for the fit
    with pytest.raises(ValueError):
        evaluate_iid(x, x, "residual", m)
    got, info = evaluate_iid(x, x, "albedo", m)                       # a non-scale target does not need channel 0
    assert info["n_valid"] == 2 * 256 and got["psnr"] == np.inf and got["ssim"] == 1.0


# ---- the device's own float32 arithmetic, emulated element for element ----

def _fma32(a, b, c):
    """float32 fma: the product of two float32 values is exact in float64, so one float64 sum rounded to float32."""
    return (np.float64(a) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _ssim_f32(p, g):
    """eval_iid_ssim_kernel's SSIM of mapped, zeroed [3, H, W] float32 maps: the 1-D weights normalised by their float32
    sum, the row pass and then the column pass as fma chains over the 11 taps, torchmetrics' formula in float32, the mean
    over the windows inside the image."""
    t = (np.arange(11, dtype=np.float32) - np.float32(5)) / np.float32(1.5)
    w = np.exp(-(t * t) / np.float32(2))
    total = np.float32(0)
    for v in w:
        total = np.float32(total + v)
    w = w / total
    H, W = p.shape[-2:]
    x = [p, g, p * p, g * g, p * g]
    rows = []
    for m in x:
        acc = np.zeros((3, H, W - 10), np.float32)
        for a in range(11):
            acc = _fma32(w[a], m[:, :, a:a + W - 10], acc)
        rows.append(acc)
    mom = []
    for m in rows:
        acc = np.zeros((3, H - 10, W - 10), np.float32)
        for a in range(11):
            acc = _fma32(w[a], m[:, a:a + H - 10], acc)
        mom.append(acc)
    mu_p, mu_g, e_pp, e_gg, e_pg = mom
    c1, c2 = np.float32(0.01 * 0.01), np.float32(0.03 * 0.03)
    mu_pp, mu_gg, mu_pg = mu_p * mu_p, mu_g * mu_g, mu_p * mu_g
    s_pp, s_gg, s_pg = np.maximum(e_pp - mu_pp, 0), np.maximum(e_gg - mu_gg, 0), e_pg - mu_pg
    num = (np.float32(2) * mu_pg + c1) * (np.float32(2) * s_pg + c2)
    den = (mu_pp + mu_gg + c1) * ((s_pp + s_gg) + c2)
    return float(np.mean((num / den).astype(np.float64))), int(((e_pp - mu_pp) < 0).sum() + ((e_gg - mu_gg) < 0).sum())


# The emulation's weights come from numpy's exp, the kernel's from CUDA's expf: their last bits can differ, which moves
# textured SSIM by at most 1.4e-7 (measured on an H100 80GB HBM3 over the golden cases). On flat maps those bits decide
# which windows cancel below zero, so there the emulation pins the size of the clamp's effect, not its bits.
SSIM_EMUL_TOL = 5e-7


@pytest.mark.parametrize("value", [0.3, 0.77])
def test_iid_ssim_clamps_negative_variances_of_flat_maps(value):
    """pred == gt == a constant: every window's moments are equal pairs, so without the clamp each window is exactly 1;
    float32 cancellation in E[x^2] - mu^2 makes variances negative, and torchmetrics' clamp(min=0) then gives SSIM < 1
    (float64 gives exactly 1: on flat maps the float32 SSIM departs from it by this much, here 1e-5 to 5e-5)."""
    from marigold_b200.evaluation import evaluate_iid

    H, W = 40, 48
    x = np.full((3, H, W), value, np.float32)
    x[:, :, W // 2:] = np.float32(value / 3)                        # two flat regions and the edge between them
    want, negative = _ssim_f32(x, x)
    assert negative > 0 and want < 1.0
    got, info = _run(_dev(x), _dev(x), "albedo", None, None)
    print(f"flat {value}: SSIM {got['ssim']!r}, float32 emulation {want!r} ({negative} negative variances)")
    assert got["ssim"] < 1.0 - 1e-6, got["ssim"]
    assert (1.0 - want) / 3 <= 1.0 - got["ssim"] <= 3 * (1.0 - want), (got["ssim"], want)
    assert got["psnr"] == np.inf


@pytest.mark.parametrize("name", [n for n, c in IID_EVAL_CASES.items() if c["transform"] is None and c["mask"] != "empty"])
def test_iid_metrics_follow_the_device_maps(name):
    """PSNR exactly and SSIM to SSIM_EMUL_TOL from the maps the kernel forms: fl(k * fl(s * p)) and fl(k * g) clamped to
    [0, 1] with the device's own s and k, then zeroed outside the mask for SSIM."""
    cfg = IID_EVAL_CASES[name]
    pred, gt, mask = iid_eval_input(cfg)
    got, info = _run(_dev(pred), _dev(gt), cfg["target"], _dev(mask), None)
    p, g = pred, gt
    if cfg["target"] in iid_eval_ref.UP_TO_SCALE:
        s, k = np.float32(info["scale"]), np.float32(info["quantile_scale"])
        p, g = np.clip(k * (s * p), 0, 1), np.clip(k * g, 0, 1)
    m = np.ones(p.shape, bool) if mask is None else mask
    d = p[m].astype(np.float64) - g[m].astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        psnr = 10.0 * np.log10(1.0 / (np.sum(d * d) / m.sum()))
    ssim, _ = _ssim_f32(np.where(m, p, 0).astype(np.float32), np.where(m, g, 0).astype(np.float32))
    print(f"{name}: psnr {got['psnr']!r} vs {psnr!r}; ssim {got['ssim']!r} vs {ssim!r}")
    assert _close(got["psnr"], psnr, 1e-10 * max(1.0, abs(psnr))), (got["psnr"], psnr)
    assert _close(got["ssim"], ssim, SSIM_EMUL_TOL), (got["ssim"], ssim)
