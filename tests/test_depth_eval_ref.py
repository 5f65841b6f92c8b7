"""The depth evaluation's restatements (tests/depth_eval_ref.py) against the reference's recorded results
(tests/golden/eval_golden.npz), against each other, and the host side of the alignment's pixel selection. No GPU."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import depth_eval_ref as R
from tests.golden.eval_cases import DEPTH_EVAL_CASES, depth_eval_input, depth_eval_range

GOLD = np.load(Path(__file__).resolve().parent / "golden" / "eval_golden.npz")
SIZES = [(37, 53, 16), (96, 128, 64), (128, 96, 64), (352, 1216, 1024), (1216, 352, 1024), (480, 640, 100),
         (768, 1024, 1024), (1080, 1920, 1024), (4032, 6048, 1024), (96, 128, 128), (96, 128, None)]


def _case(name):
    cfg = DEPTH_EVAL_CASES[name]
    return cfg, depth_eval_input(cfg), depth_eval_range(cfg)


@pytest.mark.parametrize("name", list(DEPTH_EVAL_CASES))
def test_ref32_reproduces_the_reference(name):
    """scale, shift, n_valid and the delta accuracies exactly; the float32-summed metrics to 1e-6."""
    cfg, (pred, gt, valid), rng = _case(name)
    m, scale, shift, n, _, bits = R.depth_eval_ref32(pred, gt, valid, cfg["alignment"], cfg["max_res"], *rng)
    g = lambda k: float(GOLD[f"depth/{name}/{k}"])  # noqa: E731
    assert (scale, shift, n) == (g("scale"), g("shift"), int(g("n_valid")))
    for k, b in zip(R.DELTAS, bits):
        assert float(np.float32(np.count_nonzero(b & valid)) / np.float32(n)) == g(k), k
    for k in R.METRICS:
        if k not in R.DELTAS:
            assert abs(m[k] - g(k)) <= 1e-6 * max(1.0, abs(g(k))), (k, m[k], g(k))
    key = f"depth/{name}/delta_bits"
    if key in GOLD:
        assert np.array_equal(np.packbits(bits), GOLD[key])


@pytest.mark.parametrize("name", list(DEPTH_EVAL_CASES))
def test_f64_judge_agrees_with_ref32_to_float32(name):
    """The un-rounded float64 evaluation and the reference's float32 one differ by float32 rounding only: 1e-4 relative
    on the metrics (float32 sums over up to 6e5 pixels of terms that each carry a few 6e-8), the fit to 2e-6."""
    cfg, (pred, gt, valid), rng = _case(name)
    m32, s32, t32, n32, a32, _ = R.depth_eval_ref32(pred, gt, valid, cfg["alignment"], cfg["max_res"], *rng)
    m64, s64, t64, n64, a64, bounds = R.depth_eval_f64(pred, gt, valid, cfg["alignment"], cfg["max_res"], *rng)
    assert n32 == n64
    assert abs(s32 - s64) <= 2e-6 * max(1.0, abs(s64)) and abs(t32 - t64) <= 2e-6 * max(1.0, abs(t64), abs(s64))
    for k in R.METRICS:
        tol = 2e-3 if k in R.DELTAS else 1e-4          # a delta moves by 1 / n per pixel that sits on a threshold
        if "planted" in name and k in R.DELTAS:
            continue
        assert abs(m32[k] - m64[k]) <= tol * max(1.0, abs(m64[k])), (k, m32[k], m64[k])
    # the bounds are finite and at most a tenth of the float32 allowance above: largest where a clip at 1e-3 or a
    # reciprocal of a small disparity multiplies the fit's error (i_rmse at NYU's range, sq_rel at DIODE's)
    for k, b in bounds.items():
        assert np.isfinite(b) and b <= 1e-5 * max(1.0, abs(m64.get(k, s64))), (k, b)


@pytest.mark.parametrize("name", ["planted_none_96x128", "planted_ls_96x128"])
def test_planted_pixels_separate_float32_from_double_decisions(name):
    """The planted cases hold pixels that r < T decides differently in the reference's float32 and in double, in both
    directions: without them the exact-delta tests would pass with double arithmetic."""
    cfg, (pred, gt, valid), rng = _case(name)
    _, s32, t32, n, a32, bits32 = R.depth_eval_ref32(pred, gt, valid, cfg["alignment"], cfg["max_res"], *rng)
    _, s64, t64, _, a64, _ = R.depth_eval_f64(pred, gt, valid, cfg["alignment"], cfg["max_res"], *rng)
    g = gt.astype(np.float64)
    with np.errstate(all="ignore"):
        r64 = np.maximum(a64 / g, g / a64)
    for thr, b32 in zip(R.THRESHOLDS, bits32):
        b64 = r64 < thr
        lost, gained = int((b64 & ~b32 & valid).sum()), int((~b64 & b32 & valid).sum())
        print(f"{name} T={thr}: double says inside and float32 outside for {lost} pixels, the reverse for {gained}")
        assert lost > 0, (thr, lost, gained)
        with np.errstate(all="ignore"):
            on = a32.astype(np.float64) / g == thr                    # float32 operands whose exact ratio is the threshold
        assert (a32[valid] / gt[valid] == np.float32(thr)).sum() > on[valid].sum()     # ... and ones that round onto it
    assert any(int((~(r64 < t) & b & valid).sum()) > 0 for t, b in zip(R.THRESHOLDS, bits32)) or cfg["alignment"] is None


@pytest.mark.parametrize("H,W,max_res", SIZES)
def test_fit_pixels_are_the_index_tables(H, W, max_res):
    from marigold_b200.evaluation import fit_index_tables

    q = R.fit_pixels(H, W, max_res)
    tables = fit_index_tables(H, W, max_res)
    if tables is None:
        assert np.array_equal(q, np.arange(H * W))
        return
    rows, cols = (t.numpy().astype(np.int64) for t in tables)
    assert rows.size == H and cols.size < W                        # the width only
    assert np.array_equal(q, (rows[:, None] * W + cols[None, :]).reshape(-1))


@pytest.mark.parametrize("H,W,max_res", [(96, 128, 64), (160, 120, 100), (120, 160, 77), (96, 128, 500)])
def test_align_depth_least_square_fits_the_reference_pixels(H, W, max_res, monkeypatch):
    """align_depth_least_square(max_resolution=...) hands the device the pixels the reference's Upsample keeps (the host
    side runs here: the device entry points are replaced by recorders)."""
    from marigold_b200 import evaluation

    pred = torch.arange(H * W, dtype=torch.float32).reshape(H, W)          # a pixel's value is its index
    fitted = []

    def run(p, g, m, *a):
        fitted.append(p.reshape(-1).long().numpy())
        return np.zeros(13), None

    def run_ex(p, g, m, mode, max_resolution, *a):
        t = evaluation.fit_index_tables(*p.shape[-2:], max_resolution)
        idx = np.arange(H * W) if t is None else (t[0].long()[:, None] * W + t[1].long()[None, :]).reshape(-1).numpy()
        fitted.append(p.reshape(-1).long().numpy()[idx])
        return np.zeros(13)

    monkeypatch.setattr(evaluation, "_run", run)
    monkeypatch.setattr(evaluation, "_run_ex", run_ex)
    evaluation.align_depth_least_square(pred + 1.0, pred, torch.ones(H, W, dtype=torch.bool), max_resolution=max_res)
    assert len(fitted) == 1 and np.array_equal(fitted[0], R.fit_pixels(H, W, max_res))


@pytest.mark.parametrize("c", [0.0, 0.3, 0.5, 0.7123])
@pytest.mark.parametrize("n", [1, 2, 12288])
def test_constant_prediction_has_the_minimum_norm_fit(c, n):
    """numpy's rank rule on a constant prediction: scale, shift = mean(g) (c, 1) / (c^2 + 1), in float64 and float32."""
    g = np.random.default_rng(n).uniform(1, 5, n).astype(np.float32)
    p = np.full(n, c, np.float32)
    gm, m = float(g.astype(np.float64).mean()), float(np.float32(c))
    s, t = R.lstsq_f64(p, g)
    assert abs(s - gm * m / (m * m + 1)) <= 1e-12 * gm and abs(t - gm / (m * m + 1)) <= 1e-12 * gm
    s32, t32 = R.lstsq_ref32(p, g)
    assert abs(s32 - s) <= 2e-7 * gm and abs(t32 - t) <= 2e-7 * gm
    ds, dt, _ = R.fit_bound(p, g, s)
    assert 0 < ds < 1e-9 and 0 < dt < 1e-9


def test_jittered_constant_keeps_full_rank_and_a_usable_bound():
    """pred = 0.3 + k 3e-8 (a few float32 ulps of jitter): full rank by numpy's rule, and the centred bound stays far
    below the 0.7 % an uncentred solve loses on it."""
    rng = np.random.default_rng(5)
    k = rng.integers(0, 4, 245760)
    p = (np.float32(0.3) + k.astype(np.float32) * np.float32(3e-8)).astype(np.float32)
    assert np.unique(p).size >= 3
    g = (2.0 + 1e6 * (p.astype(np.float64) - 0.3) + 0.01 * rng.standard_normal(p.size)).astype(np.float32)
    s, t = R.lstsq_f64(p, g)
    s32, _ = R.lstsq_ref32(p, g)
    ds, _, _ = R.fit_bound(p, g, s)
    assert abs(s32 - s) <= 1e-6 * abs(s) and ds <= 1e-8 * abs(s)
    pd, gd = p.astype(np.float64), g.astype(np.float64)
    n = p.size
    uncentred = (n * (pd * gd).sum() - pd.sum() * gd.sum()) / (n * (pd * pd).sum() - pd.sum() ** 2)
    d = pd - pd[0]
    centred = (n * (d * gd).sum() - d.sum() * gd.sum()) / (n * (d * d).sum() - d.sum() ** 2)
    print(f"scale {s!r}: uncentred normal equations off by {abs(uncentred - s) / abs(s):.2e}, centred by "
          f"{abs(centred - s) / abs(s):.2e}, bound {ds / abs(s):.2e}")
    assert abs(centred - s) <= ds < abs(uncentred - s)
