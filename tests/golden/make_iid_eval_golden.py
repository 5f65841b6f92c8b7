"""Generate tests/golden/iid_eval_golden.npz by running the REFERENCE's own intrinsic-image evaluation on the CPU:
compute_iid_metric, compute_alignment_scale and quantile_map (src/util/metric.py:263-338) and the colour transforms
srgb2linear / linear2srgb (marigold/util/image_util.py:144-149), in script/iid/eval.py:182-213's order. Needs a checkout
of the original Marigold repository (path in $MARIGOLD_REFERENCE) and pandas. torchmetrics is not available, so the
metric objects handed to compute_iid_metric are the float32 restatements of tests/iid_eval_ref.py. Inputs are
regenerated from seeds by tests/golden/iid_eval_cases.py.

    python tests/golden/make_iid_eval_golden.py

<case>/psnr, <case>/ssim: compute_iid_metric's values. Up-to-scale targets also store <case>/scale and
<case>/quantile: what torch.linalg.lstsq and torch.quantile returned inside the psnr call, the ssim call and a third
compute_alignment_scale + quantile_map call, and, for cases of at most 48 x 64, <case>/pred and <case>/gt: that third
call's mapped [3,H,W] maps. Each call's fit is kept because torch's CPU lstsq returns one of two neighbouring floats
for the same inputs from one call to the next. <case>/raises = 1 where the reference raised (no pixel valid in
mask channel 0 of an up-to-scale target).
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from tests import iid_eval_ref  # noqa: E402
from tests.golden._ref_eval_shim import load_reference_eval_utils  # noqa: E402
from tests.golden._ref_shim import load_reference_utils  # noqa: E402
from tests.golden.iid_eval_cases import IID_EVAL_CASES, iid_eval_input  # noqa: E402

metric = load_reference_eval_utils()["metric"]
image_util = load_reference_utils()["image_util"]
torch.set_num_threads(4)
METRICS = {"psnr": iid_eval_ref.psnr, "ssim": iid_eval_ref.ssim}
TRANSFORM = {None: None, "srgb2linear": image_util.srgb2linear, "linear2srgb": image_util.linear2srgb}

recorded = {"lstsq": [], "quantile": []}
_lstsq, _quantile = torch.linalg.lstsq, torch.quantile


def _recording_lstsq(*args, **kw):
    r = _lstsq(*args, **kw)
    recorded["lstsq"].append(float(r[0].reshape(-1)[0]))
    return r


def _recording_quantile(*args, **kw):
    q = _quantile(*args, **kw)
    recorded["quantile"].append(float(q))
    return q


torch.linalg.lstsq, torch.quantile = _recording_lstsq, _recording_quantile
store = {}
for name, cfg in IID_EVAL_CASES.items():
    pred, gt, mask = iid_eval_input(cfg)
    # script/iid/eval.py:178-196: [1,3,H,W] prediction, [1,3,H,W] ground truth and mask from the data loader
    target_pred, target_gt = torch.from_numpy(pred)[None], torch.from_numpy(gt)[None]
    valid_mask = torch.from_numpy(mask)[None] if mask is not None else None
    if cfg["transform"] is not None:
        target_gt = TRANSFORM[cfg["transform"]](target_gt)
        target_pred = TRANSFORM[cfg["transform"]](target_pred)
    target = cfg["target"]
    recorded["lstsq"].clear()
    recorded["quantile"].clear()
    try:
        for k, fn in METRICS.items():
            store[f"{name}/{k}"] = np.array(metric.compute_iid_metric(target_pred.clone(), target_gt.clone(), target, k, fn,
                                                                      valid_mask), np.float64)
    except RuntimeError as e:
        assert target in iid_eval_ref.UP_TO_SCALE and "non-empty" in str(e), e
        store[f"{name}/raises"] = np.array(1)
        print(name, "raises:", e)
        continue
    if target in iid_eval_ref.UP_TO_SCALE:
        s = metric.compute_alignment_scale(target_pred, target_gt, valid_mask)
        pm, gm = metric.quantile_map(s * target_pred, target_gt, valid_mask)
        # one fit and one quantile per call: the psnr call's, the ssim call's, the maps'
        store[f"{name}/scale"] = np.array(recorded["lstsq"], np.float32)
        store[f"{name}/quantile"] = np.array(recorded["quantile"], np.float32)
        assert store[f"{name}/scale"].shape == store[f"{name}/quantile"].shape == (3,)
        if cfg["H"] * cfg["W"] <= 48 * 64:
            store[f"{name}/pred"] = pm[0].numpy()
            store[f"{name}/gt"] = gm[0].numpy()
    print(name, {k: float(store[f"{name}/{k}"]) for k in METRICS},
          {k: store[f"{name}/{k}"].tolist() for k in ("scale", "quantile") if f"{name}/{k}" in store})

out = Path(__file__).resolve().parent / "iid_eval_golden.npz"
np.savez_compressed(out, **store)
print("wrote", out, out.stat().st_size / 1e3, "kB")
