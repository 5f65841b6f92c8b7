"""The evaluation tests' restatement of the reference (tests/eval_ref.py) against what the reference itself computed
(tests/golden/eval_golden.npz, written by make_eval_golden.py). Runs on the CPU, where the fixtures were made."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import eval_ref
from tests.golden.eval_cases import DEPTH_EVAL_CASES, DEPTH_EVAL_RANGE, NORMALS_EVAL_CASES, depth_eval_input, normals_eval_input

GOLD = np.load(Path(__file__).resolve().parent / "golden" / "eval_golden.npz")


@pytest.mark.parametrize("name", list(NORMALS_EVAL_CASES))
def test_normals_restatement_reproduces_reference(name):
    pred, gt = normals_eval_input(NORMALS_EVAL_CASES[name])
    err, mask = eval_ref.cosine_error(torch.from_numpy(pred), torch.from_numpy(gt))
    assert err.shape[0] == int(GOLD[f"normals/{name}/n_valid"]) == int(mask.sum())
    if f"normals/{name}/error" in GOLD:
        np.testing.assert_array_equal(err, GOLD[f"normals/{name}/error"])
    got = eval_ref.normals_metrics(err, decimals=4)
    for k in eval_ref.NORMALS_METRICS:
        assert got[k] == float(GOLD[f"normals/{name}/{k}"]), (k, got[k], float(GOLD[f"normals/{name}/{k}"]))


@pytest.mark.parametrize("name", list(DEPTH_EVAL_CASES))
def test_depth_restatement_reproduces_reference(name):
    cfg = DEPTH_EVAL_CASES[name]
    pred, gt, valid = depth_eval_input(cfg)
    got, scale, shift = eval_ref.depth_eval(pred, gt, valid, cfg["alignment"], cfg["max_res"], *DEPTH_EVAL_RANGE)
    assert scale == float(GOLD[f"depth/{name}/scale"]) and shift == float(GOLD[f"depth/{name}/shift"])
    assert int(valid.sum()) == int(GOLD[f"depth/{name}/n_valid"])
    for k, v in got.items():      # the reference's metrics of a float32 prediction accumulate in float32
        g = float(GOLD[f"depth/{name}/{k}"])
        assert abs(v - g) <= 1e-6 * max(1.0, abs(g)), (k, v, g)


def test_fit_index_tables_pick_the_reference_pixels():
    """The index tables evaluate_depth hands the fit kernel select exactly the pixels align_depth_least_square keeps."""
    from marigold_b200.evaluation import fit_index_tables

    for H, W, max_res in [(96, 128, 64), (120, 160, 100), (96, 128, 50), (120, 160, 77), (480, 640, 333), (30, 40, 64)]:
        idx = np.arange(H * W, dtype=np.float32).reshape(H, W)
        ref, _, _ = eval_ref.fit_maps(idx, idx, np.ones((H, W), bool), max_res)
        tables = fit_index_tables(H, W, max_res)
        if tables is None:
            assert ref is idx
            continue
        rows, cols = (t.numpy().astype(np.int64) for t in tables)
        np.testing.assert_array_equal(ref.reshape(len(rows), len(cols)), (rows[:, None] * W + cols[None, :]).astype(np.float32))
