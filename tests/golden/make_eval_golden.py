"""Generate tests/golden/eval_golden.npz by running the REFERENCE's own evaluation functions on the CPU (needs a
checkout of the original Marigold repository, path in $MARIGOLD_REFERENCE, and pandas). Inputs are regenerated from
seeds by tests/golden/eval_cases.py, so only the reference outputs are stored.

    python tests/golden/make_eval_golden.py

normals/<case>/: compute_cosine_error(pred, gt, masked=True) ("error", the valid pixels in row-major order; omitted for
the largest case), n_valid and every normals metric of src/util/metric.py:222-257 (rounded to 4 decimals, as the
reference returns them).
depth/<case>/: script/depth/eval.py:171-217 in the case's alignment mode: scale, shift, n_valid and the depth metrics;
for the threshold-planted cases also delta_bits, np.packbits of the [3, H, W] decisions max(o / t, t / o) < threshold on
the reference's aligned map (their masked count over n is asserted to be the reference's delta value).
Keys the file already holds must come out byte-identical; the run asserts it.
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from tests.golden._ref_eval_shim import load_reference_eval_utils  # noqa: E402
from tests.golden.eval_cases import (DELTA_THRESHOLDS, DEPTH_EVAL_CASES, NORMALS_EVAL_CASES, depth_eval_input,  # noqa: E402
                                depth_eval_range, normals_eval_input)

ref = load_reference_eval_utils()
metric, alignment = ref["metric"], ref["alignment"]
torch.set_num_threads(4)
NORMALS_METRICS = ("mean_angular_error", "median_angular_error", "rmse_angular_error", "sub5_error", "sub7_5_error",
                   "sub11_25_error", "sub22_5_error", "sub30_error")
DEPTH_METRICS = ("abs_relative_difference", "squared_relative_difference", "rmse_linear", "rmse_log", "log10", "delta1_acc",
                 "delta2_acc", "delta3_acc", "i_rmse", "silog_rmse")

store = {}
for name, cfg in NORMALS_EVAL_CASES.items():
    pred, gt = normals_eval_input(cfg)
    # script/normals/eval.py:138-150: [1,3,H,W] tensors
    err = metric.compute_cosine_error(torch.from_numpy(pred)[None], torch.from_numpy(gt)[None], masked=True)
    if cfg.get("store_map", True):
        store[f"normals/{name}/error"] = err
    store[f"normals/{name}/n_valid"] = np.array(err.shape[0])
    for k in NORMALS_METRICS:
        store[f"normals/{name}/{k}"] = np.array(float(getattr(metric, k)(err)), np.float64)
    print(name, "n", err.shape[0], {k: float(store[f"normals/{name}/{k}"]) for k in NORMALS_METRICS[:3]})

for name, cfg in DEPTH_EVAL_CASES.items():
    depth_pred, depth_raw, valid_mask = depth_eval_input(cfg)
    dmin, dmax = depth_eval_range(cfg)
    scale, shift = 1.0, 0.0
    # script/depth/eval.py:171-207, verbatim in order
    if cfg["alignment"] == "least_square":
        depth_pred, scale, shift = alignment.align_depth_least_square(
            gt_arr=depth_raw, pred_arr=depth_pred, valid_mask_arr=valid_mask, return_scale_shift=True,
            max_resolution=cfg["max_res"])
    elif cfg["alignment"] == "least_square_disparity":
        gt_disparity, gt_non_neg_mask = alignment.depth2disparity(depth=depth_raw, return_mask=True)
        pred_non_neg_mask = depth_pred > 0
        valid_nonnegative_mask = valid_mask & gt_non_neg_mask & pred_non_neg_mask
        disparity_pred, scale, shift = alignment.align_depth_least_square(
            gt_arr=gt_disparity, pred_arr=depth_pred, valid_mask_arr=valid_nonnegative_mask, return_scale_shift=True,
            max_resolution=cfg["max_res"])
        disparity_pred = np.clip(disparity_pred, a_min=1e-3, a_max=None)
        depth_pred = alignment.disparity2depth(disparity_pred)
    depth_pred = np.clip(depth_pred, a_min=dmin, a_max=dmax)
    depth_pred = np.clip(depth_pred, a_min=1e-6, a_max=None)
    assert depth_pred.dtype == np.float32 and np.asarray(scale).dtype in (np.float32, np.float64)
    # :209-216 on the CPU
    pred_ts, gt_ts, mask_ts = torch.from_numpy(depth_pred), torch.from_numpy(depth_raw), torch.from_numpy(valid_mask)
    store[f"depth/{name}/scale"] = np.array(float(np.asarray(scale).reshape(-1)[0]), np.float64)
    store[f"depth/{name}/shift"] = np.array(float(np.asarray(shift).reshape(-1)[0]), np.float64)
    store[f"depth/{name}/n_valid"] = np.array(int(valid_mask.sum()))
    for k in DEPTH_METRICS:
        store[f"depth/{name}/{k}"] = np.array(getattr(metric, k)(pred_ts, gt_ts, mask_ts).item(), np.float64)
    if cfg.get("scene") == "planted":
        r = torch.max(pred_ts / gt_ts, gt_ts / pred_ts)
        bits = np.stack([(r < t).numpy() for t in DELTA_THRESHOLDS])
        for b, k in zip(bits, ("delta1_acc", "delta2_acc", "delta3_acc")):
            n = np.float32(valid_mask.sum())
            assert float(np.float32((b & valid_mask).sum()) / n) == float(store[f"depth/{name}/{k}"]), (name, k)
        store[f"depth/{name}/delta_bits"] = np.packbits(bits)
    print(name, "scale", float(store[f"depth/{name}/scale"]), "shift", float(store[f"depth/{name}/shift"]),
          "abs_rel", float(store[f"depth/{name}/abs_relative_difference"]), "delta1",
          float(store[f"depth/{name}/delta1_acc"]), "dtype", depth_pred.dtype, np.asarray(scale).dtype)

out = Path(__file__).resolve().parent / "eval_golden.npz"
if out.exists():
    old = np.load(out)
    for k in old.files:
        assert k in store and old[k].dtype == store[k].dtype and old[k].tobytes() == np.asarray(store[k]).tobytes(), k
    print(len(old.files), "existing keys byte-identical;", len(store) - len(old.files), "new")
np.savez_compressed(out, **store)
print("wrote", out, out.stat().st_size / 1e3, "kB")
