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
    # portrait maps with max_res: the fit keeps every row and downsamples the width
    "ls_maxres_portrait_160x120": dict(H=160, W=120, seed=67, alignment="least_square", max_res=100),
    "lsd_maxres_portrait_160x120": dict(H=160, W=120, seed=68, alignment="least_square_disparity", max_res=100),
    # dataset-shaped (script/depth/eval/*.sh, src/dataset/*_dataset.py): sizes, ranges and masks
    "kitti_352x1216": dict(H=352, W=1216, seed=69, alignment="least_square", max_res=None, scene="steps", range=(1e-5, 80.0),
                           far=80.0, valid_frac=0.05),
    "nyu_480x640": dict(H=480, W=640, seed=70, alignment="least_square", max_res=None, scene="steps", range=(1e-3, 10.0),
                        far=10.0, valid_frac=0.9),
    "diode_768x1024": dict(H=768, W=1024, seed=71, alignment="least_square_disparity", max_res=None, scene="steps",
                           range=(0.6, 350.0), far=500.0, valid_frac=0.8),
    "inf_maxres_252x378": dict(H=252, W=378, seed=72, alignment="least_square", max_res=64, scene="steps",
                               range=(1e-5, float("inf")), far=60.0, valid_frac=0.7),
    # degenerate fits
    "const_0.3": dict(H=96, W=128, seed=73, alignment="least_square", max_res=None, scene="const", const=0.3),
    "const_0": dict(H=96, W=128, seed=74, alignment="least_square", max_res=None, scene="const", const=0.0),
    "n1": dict(H=32, W=48, seed=75, alignment="least_square", max_res=None, keep=1),
    "n2": dict(H=32, W=48, seed=76, alignment="least_square", max_res=None, keep=2),
    "lsd_no_positive_pred": dict(H=32, W=48, seed=77, alignment="least_square_disparity", max_res=None, scene="const",
                                 const=-0.25),
    # pixels whose float32 ratio sits on a delta threshold and one float32 ulp either side of it
    "planted_none_96x128": dict(H=96, W=128, seed=78, alignment=None, max_res=None, scene="planted"),
    "planted_ls_96x128": dict(H=96, W=128, seed=79, alignment="least_square", max_res=64, scene="planted"),
}
DEPTH_EVAL_RANGE = (0.5, 8.0)   # dataset min / max depth of the depth cases that name no range
# the smooth scene at DEPTH_EVAL_RANGE, which the float32 restatement of tests/eval_ref.py is held to at 1e-6
DEPTH_EVAL_SMOOTH_CASES = {n: c for n, c in DEPTH_EVAL_CASES.items() if "scene" not in c and "keep" not in c}
DELTA_THRESHOLDS = (1.25, 1.5625, 1.953125)


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


def depth_eval_range(cfg):
    return cfg.get("range", DEPTH_EVAL_RANGE)


def _steps_scene(cfg, rng):
    """Piecewise-planar depth with discontinuities up to `far`, a sparse or dense mask, and a prediction with a
    long-tailed (Student t, 2 degrees of freedom) error; in disparity mode the prediction overshoots both clips."""
    H, W = cfg["H"], cfg["W"]
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    lo = max(cfg["range"][0], 0.3)
    gt = np.full((H, W), lo)
    for _ in range(12):                                                   # planes pasted over each other
        y0, x0 = rng.uniform(0, 0.8, 2)
        box = (yy >= y0) & (yy < y0 + rng.uniform(0.1, 0.6)) & (xx >= x0) & (xx < x0 + rng.uniform(0.1, 0.6))
        z0 = lo + (cfg["far"] - lo) * rng.uniform() ** 2
        gt = np.where(box, np.maximum(z0 * (1.0 + 0.3 * (xx - x0) - 0.2 * (yy - y0)), lo), gt)
    valid = rng.uniform(size=(H, W)) < cfg["valid_frac"]
    gt = np.where(valid, gt, 0.0).astype(np.float32)
    tail = rng.standard_t(2, size=(H, W))
    if cfg["alignment"] == "least_square":
        pred = (gt - 0.2 * cfg["far"]) / (0.9 * cfg["far"]) + 0.004 * tail
    else:
        pred = 1.3 / np.maximum(gt, lo) - 0.02 + 0.003 * tail            # the tail crosses 0 and the far clip
    return pred.astype(np.float32), gt, valid


def _ulp_step(x, k):
    """float32 x moved k ulps (k in -1, 0, 1)."""
    return (x.view(np.int32) + np.int32(k)).view(np.float32)


def _planted_scene(cfg, rng):
    """Eighteen classes of pixels: for each threshold T, each direction (a / g or g / a is the larger ratio) and each of
    -1, 0, +1 float32 ulps, the value on one side is the float32 nearest to T times the other side, moved by that many
    ulps. Where T times the value is not a float32 the nearest one gives an exact quotient just off T whose float32
    rounding is T itself: float32 and double then decide r < T differently. With least_square the planted pixels sit in
    the columns the max_res fit does not keep, so they do not move the fit they were planted for; a is then the
    reference's fl(fl(p s) + t) with the float32 scale and shift np.linalg.lstsq returns for the kept columns."""
    import torch

    H, W = cfg["H"], cfg["W"]
    if cfg["alignment"] is None:
        planted = np.ones((H, W), bool)
        pred = rng.uniform(0.6, 4.0, (H, W)).astype(np.float32)
        a = pred.copy()
        gt = np.zeros((H, W), np.float32)
    else:
        pred, gt, valid = depth_eval_input(dict(cfg, scene=None))
        sf = np.min(cfg["max_res"] / np.array((H, W)))
        kept = torch.nn.Upsample(scale_factor=sf, mode="nearest")(torch.arange(W, dtype=torch.float64).reshape(1, 1, W))
        planted = np.ones((H, W), bool)
        planted[:, kept.reshape(-1).long().numpy()] = False
        fit = valid & ~planted
        A = np.stack([pred[fit], np.ones_like(pred[fit])], axis=-1)
        s, t = np.linalg.lstsq(A, gt[fit].reshape(-1, 1), rcond=None)[0].reshape(-1)          # float32, as the reference's
        assert s.dtype == np.float32
        pred = np.where(planted, rng.uniform(0.1, 0.6, (H, W)).astype(np.float32), pred)
        a = pred * s + t                                                                      # float32, two roundings
        assert a.dtype == np.float32 and a[planted].min() > 0.7 and a[planted].max() < 4.05
    cls = rng.integers(0, 18, (H, W))
    T = np.array(DELTA_THRESHOLDS)[cls // 6]
    a_over_g, k = (cls // 3) % 2 == 0, cls % 3 - 1
    if cfg["alignment"] is None:                      # the free side: the prediction itself
        g_free = a
        g = np.where(a_over_g, g_free, _ulp_step((g_free.astype(np.float64) * T).astype(np.float32), k))
        pred = np.where(a_over_g, _ulp_step((g_free.astype(np.float64) * T).astype(np.float32), k), a)
        return pred.astype(np.float32), g.astype(np.float32), planted
    g = np.where(a_over_g, _ulp_step((a.astype(np.float64) / T).astype(np.float32), k),
                 _ulp_step((a.astype(np.float64) * T).astype(np.float32), k))
    gt = np.where(planted, g, gt).astype(np.float32)
    return pred, gt, valid | planted


def depth_eval_input(cfg):
    """(pred, gt, valid) for one depth sample: a smooth scene with 0 outside the valid mask; the prediction is
    affine-invariant depth (least_square) or affine-invariant disparity with a few non-positive pixels
    (least_square_disparity). Cases that name a `scene` or `keep` vary it (see DEPTH_EVAL_CASES)."""
    rng = np.random.default_rng(cfg["seed"])
    H, W = cfg["H"], cfg["W"]
    if cfg.get("scene") == "steps":
        return _steps_scene(cfg, rng)
    if cfg.get("scene") == "planted":
        return _planted_scene(cfg, rng)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    gt = 1.0 + 5.0 * (0.5 + 0.4 * np.sin(3 * xx + 2 * yy)) + 0.05 * rng.standard_normal((H, W))
    valid = rng.uniform(size=(H, W)) > 0.2
    if "keep" in cfg:                                   # `keep` valid pixels only
        valid = np.zeros(H * W, bool)
        valid[rng.choice(H * W, cfg["keep"], replace=False)] = True
        valid = valid.reshape(H, W)
    gt = np.where(valid, gt, 0.0).astype(np.float32)
    if cfg.get("scene") == "const":                     # what a collapsed model predicts
        return np.full((H, W), cfg["const"], np.float32), gt, valid
    if cfg["alignment"] == "least_square":
        pred = (gt - 0.7) / 5.1 + 0.02 * rng.standard_normal((H, W))
    else:
        pred = 0.8 / np.maximum(gt, 0.5) - 0.05 + 0.01 * rng.standard_normal((H, W))
        pred[rng.uniform(size=(H, W)) < 0.02] = -0.1
    return pred.astype(np.float32), gt, valid
