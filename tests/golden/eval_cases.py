"""Seeded inputs of the evaluation cases (script/normals/eval.py, script/depth/eval.py), shared by make_eval_golden.py
(reference run) and the tests."""
import numpy as np

# parity: force an odd or even number of valid pixels.
NORMALS_EVAL_CASES = {
    "odd_480x640": dict(H=480, W=640, seed=51, parity=1, zero_gt=0.05, zero_pred=0.01, tie_block=64, store_map=False),
    "even_120x160": dict(H=120, W=160, seed=52, parity=0, zero_gt=0.1, zero_pred=0.02, tie_block=24),
    "odd_37x53": dict(H=37, W=53, seed=53, parity=1, zero_gt=0.2, zero_pred=0.05, tie_block=8),
    "even_ties_48x64": dict(H=48, W=64, seed=54, parity=0, zero_gt=0.0, zero_pred=0.0, tie_block=40),
    "n1": dict(H=16, W=16, seed=55, keep=1),
    "n2": dict(H=16, W=16, seed=56, keep=2),
}
DEPTH_EVAL_CASES = {
    "ls_96x128": dict(H=96, W=128, seed=61, alignment="least_square", max_res=None),
    "ls_maxres_96x128": dict(H=96, W=128, seed=62, alignment="least_square", max_res=64),
    "lsd_96x128": dict(H=96, W=128, seed=63, alignment="least_square_disparity", max_res=None),
    "lsd_maxres_120x160": dict(H=120, W=160, seed=64, alignment="least_square_disparity", max_res=100),
    "lsd_maxres_96x128": dict(H=96, W=128, seed=65, alignment="least_square_disparity", max_res=50),
    "ls_maxres_120x160": dict(H=120, W=160, seed=66, alignment="least_square", max_res=77),
}
DEPTH_EVAL_RANGE = (0.5, 8.0)   # dataset min / max depth of the depth cases


def normals_eval_input(cfg):
    """(pred, gt) fp32 [3,H,W]: noisy unit normals against unit ground truth, with zero ground-truth vectors (not
    valid), zero predictions (90 degrees), and a block where pred == gt == (0, 0, 1) (ties at exactly 0 degrees)."""
    rng = np.random.default_rng(cfg["seed"])
    H, W = cfg["H"], cfg["W"]
    gt = rng.normal(size=(3, H, W))
    gt[2] = np.abs(gt[2]) + 1.0
    gt /= np.linalg.norm(gt, axis=0, keepdims=True)
    pred = gt + rng.normal(0, 0.25, size=(3, H, W))
    pred /= np.linalg.norm(pred, axis=0, keepdims=True)
    gt, pred = gt.astype(np.float32), pred.astype(np.float32)
    if "keep" in cfg:
        valid = np.zeros(H * W, bool)
        valid[rng.choice(H * W, cfg["keep"], replace=False)] = True
        gt[:, ~valid.reshape(H, W)] = 0.0
        return pred, gt
    b = cfg["tie_block"]
    gt[:, :b, :b] = pred[:, :b, :b] = np.array([0, 0, 1], np.float32)[:, None, None]
    pred[:, rng.uniform(size=(H, W)) < cfg["zero_pred"]] = 0.0
    gt[:, rng.uniform(size=(H, W)) < cfg["zero_gt"]] = 0.0
    n = int((np.linalg.norm(gt, axis=0) > 0).sum())
    if n % 2 != cfg["parity"]:
        gt[:, H - 1, W - 1] = 0.0 if np.linalg.norm(gt[:, H - 1, W - 1]) > 0 else np.array([0, 1, 0], np.float32)
    return pred, gt


def depth_eval_input(cfg):
    """(pred, gt, valid) for one depth sample: a smooth scene with 0 outside the valid mask; the prediction is
    affine-invariant depth (least_square) or affine-invariant disparity with a few non-positive pixels
    (least_square_disparity)."""
    rng = np.random.default_rng(cfg["seed"])
    H, W = cfg["H"], cfg["W"]
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    gt = 1.0 + 5.0 * (0.5 + 0.4 * np.sin(3 * xx + 2 * yy)) + 0.05 * rng.standard_normal((H, W))
    valid = rng.uniform(size=(H, W)) > 0.2
    gt = np.where(valid, gt, 0.0).astype(np.float32)
    if cfg["alignment"] == "least_square":
        pred = (gt - 0.7) / 5.1 + 0.02 * rng.standard_normal((H, W))
    else:
        pred = 0.8 / np.maximum(gt, 0.5) - 0.05 + 0.01 * rng.standard_normal((H, W))
        pred[rng.uniform(size=(H, W)) < 0.02] = -0.1
    return pred.astype(np.float32), gt, valid
