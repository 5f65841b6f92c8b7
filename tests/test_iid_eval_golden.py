"""The intrinsic-image evaluation's restatement (tests/iid_eval_ref.py, float32 variant) against what the reference's own
compute_iid_metric / compute_alignment_scale / quantile_map computed (tests/golden/iid_eval_golden.npz, written by
make_iid_eval_golden.py): the scale, the quantile, the mapped maps and both metrics, bit for bit. Runs on the CPU, where
the fixtures were made."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import iid_eval_ref
from tests.golden.iid_eval_cases import IID_EVAL_CASES, iid_eval_input

GOLD = np.load(Path(__file__).resolve().parent / "golden" / "iid_eval_golden.npz")


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize("name", list(IID_EVAL_CASES))
def test_iid_restatement_reproduces_reference(name):
    cfg = IID_EVAL_CASES[name]
    pred, gt, mask = (torch.from_numpy(a) if a is not None else None for a in iid_eval_input(cfg))
    if f"{name}/raises" in GOLD:
        with pytest.raises(RuntimeError):
            iid_eval_ref.evaluate(pred, gt, cfg["target"], mask, cfg["transform"])
        return
    if cfg["target"] not in iid_eval_ref.UP_TO_SCALE:
        got, _ = iid_eval_ref.evaluate(pred, gt, cfg["target"], mask, cfg["transform"])
        for k in ("psnr", "ssim"):
            assert _same(got[k], GOLD[f"{name}/{k}"]), (k, got[k], float(GOLD[f"{name}/{k}"]))
        return
    # torch's CPU lstsq returns slightly different floats for the same inputs from call to call (up to 5 ulp seen): the
    # restatement's own fit agrees to 1e-6, and everything after the fit is compared bit for bit from the scale each
    # reference call used
    scales, quantiles = GOLD[f"{name}/scale"], GOLD[f"{name}/quantile"]
    _, fit = iid_eval_ref.evaluate(pred, gt, cfg["target"], mask, cfg["transform"])
    assert np.abs(fit["scale"] - scales.astype(np.float64)).max() <= 1e-6 * abs(fit["scale"]), (fit["scale"], scales)
    for i, k in enumerate(("psnr", "ssim", None)):
        got, info = iid_eval_ref.evaluate(pred, gt, cfg["target"], mask, cfg["transform"], scale=scales[i])
        assert _same(np.float32(info["quantile"]), quantiles[i])
        if k is not None:
            assert _same(got[k], GOLD[f"{name}/{k}"]), (k, got[k], float(GOLD[f"{name}/{k}"]))
        elif f"{name}/pred" in GOLD:
            assert _same(info["pred"].numpy(), GOLD[f"{name}/pred"])
            assert _same(info["gt"].numpy(), GOLD[f"{name}/gt"])


def test_iid_golden_covers_the_edge_cases():
    """The fixtures hold the cases the device tests lean on: a quantile scale of 0 (PSNR +inf, SSIM 1), a non-scale
    target without a valid element (PSNR NaN), an up-to-scale target that raises, and ties at the quantile."""
    assert np.isposinf(GOLD["shading_40x40_dark/psnr"]) and float(GOLD["shading_40x40_dark/ssim"]) == 1.0
    assert float(GOLD["shading_40x40_dark/quantile"][0]) < 1e-4
    assert np.isnan(GOLD["albedo_24x24_empty/psnr"]) and float(GOLD["albedo_24x24_empty/ssim"]) == 1.0
    assert int(GOLD["shading_24x24_empty/raises"]) == 1
    pred, gt, _ = iid_eval_input(IID_EVAL_CASES["shading_48x64_q255"])
    lo, hi, _ = iid_eval_ref.quantile_order_statistics(torch.from_numpy(gt))
    b = iid_eval_ref.brightness(torch.from_numpy(gt)).reshape(-1).numpy()
    assert (b == lo).sum() > 1 and (b == hi).sum() > 1
