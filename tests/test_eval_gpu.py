"""Device evaluation (`-m gpu`): surface-normals metrics (evaluate_normals, csrc/eval.cu) against the reference's
compute_cosine_error + metrics restated with torch on CUDA (tests/eval_ref.py) and against the reference's own results
(tests/golden/eval_golden.npz); the depth evaluation's least_square_disparity alignment and alignment_max_res against the
restated script/depth/eval.py:171-217 and the golden."""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import eval_ref
from tests.golden.eval_cases import DEPTH_EVAL_CASES, DEPTH_EVAL_RANGE, NORMALS_EVAL_CASES, depth_eval_input, normals_eval_input

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).resolve().parent / "golden" / "eval_golden.npz")
TOL = 1e-4            # degrees
LAUNCHES = 4          # error, locate, refine, final


def _angles(theta_deg, H, W):
    """(pred, gt) [3,H,W] on the GPU with pred at the given angle from gt = (0, 0, 1)."""
    t = torch.as_tensor(theta_deg, dtype=torch.float64).reshape(H, W) * (np.pi / 180.0)
    pred = torch.stack([torch.sin(t), torch.zeros_like(t), torch.cos(t)]).float()
    gt = torch.zeros(3, H, W)
    gt[2] = 1.0
    return pred.cuda(), gt.cuda()


def _random_normals(H, W, seed, odd, tie_frac=0.0):
    g = torch.Generator().manual_seed(seed)
    gt = torch.randn(3, H, W, generator=g)
    gt[2] = gt[2].abs() + 1.0
    gt = gt / gt.norm(dim=0, keepdim=True)
    pred = gt + 0.3 * torch.randn(3, H, W, generator=g)
    pred[:, torch.rand(H, W, generator=g) < 0.01] = 0.0                           # 90 degrees
    if tie_frac:
        tie = torch.rand(H, W, generator=g) < tie_frac
        pred[:, tie] = gt[:, tie]                                                  # pred == gt: heavy ties near 0
        pred[:, : H // 4, : W // 4] = gt[:, : H // 4, : W // 4] = torch.tensor([0.0, 0.0, 1.0])[:, None, None]
    gt[:, torch.rand(H, W, generator=g) < 0.05] = 0.0                               # not valid
    n = int((gt.norm(dim=0) > 0).sum())
    if n % 2 != odd:
        gt[:, H - 1, W - 1] = 0.0 if gt[:, H - 1, W - 1].norm() > 0 else torch.tensor([0.0, 1.0, 0.0])
    return pred.cuda(), gt.cuda()


def _check_against_torch(pred, gt, got, info):
    err_t, mask = eval_ref.cosine_error(pred, gt)                                  # torch on CUDA, as the reference runs
    n = err_t.shape[0]
    assert info["n_valid"] == n
    emap = info["error_map"].cpu().numpy()
    assert np.isnan(emap[~mask]).all() and not np.isnan(emap[mask]).any()
    mine = emap[mask]
    # exact median: np.median of the kernel's own error map
    assert got["median_angular_error"] == float(np.median(mine)), (got["median_angular_error"], float(np.median(mine)))
    ref = eval_ref.normals_metrics_f64(err_t)
    for k in ("mean_angular_error", "median_angular_error", "rmse_angular_error"):
        assert abs(got[k] - ref[k]) <= TOL, (k, got[k], ref[k])
    for k, t in eval_ref.THRESHOLDS.items():
        if np.abs(err_t.astype(np.float64) - t).min() > TOL:
            assert got[k] == ref[k], (k, got[k], ref[k])
        assert got[k] == 100.0 * (np.sum(mine < t) / n)
    assert np.abs(mine.astype(np.float64) - err_t).max() <= TOL
    return float(np.mean(mine.view(np.uint32) == err_t.view(np.uint32)))


@pytest.mark.parametrize("name", list(NORMALS_EVAL_CASES))
def test_normals_match_reference_golden(name):
    from marigold_b200 import evaluate_normals

    pred, gt = normals_eval_input(NORMALS_EVAL_CASES[name])
    got, info = evaluate_normals(torch.from_numpy(pred).cuda()[None], torch.from_numpy(gt).cuda()[None],
                                 return_error_map=True)
    assert info["n_valid"] == int(GOLD[f"normals/{name}/n_valid"])
    frac = _check_against_torch(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(), got, info)
    key = f"normals/{name}/error"
    if key in GOLD:               # the golden's errors were computed on the CPU, which divides by pi instead
        mine = info["error_map"].cpu().numpy()[np.linalg.norm(gt, axis=0) > 0]
        assert np.abs(mine.astype(np.float64) - GOLD[key]).max() <= TOL
    for k in eval_ref.NORMALS_METRICS:
        g = float(GOLD[f"normals/{name}/{k}"])            # rounded to 4 decimals by the reference
        assert abs(got[k] - g) <= TOL + 0.5e-4 + 1e-6 * abs(g), (k, got[k], g)
        if k.startswith("sub"):
            assert round(got[k], 4) == pytest.approx(g, abs=1e-6), (k, got[k], g)
    print(f"{name}: error bit-identical to torch CUDA for {frac:.4%} of the valid pixels")


@pytest.mark.parametrize("H,W", [(480, 640), (768, 1024), (1080, 1920)])
@pytest.mark.parametrize("odd", [0, 1])
@pytest.mark.parametrize("ties", [0.0, 0.6])
def test_normals_median_exact_and_metrics_match_torch(H, W, odd, ties):
    from marigold_b200 import _lib, evaluate_normals

    pred, gt = _random_normals(H, W, seed=H + 7 * odd + int(ties * 10), odd=odd, tie_frac=ties)
    mask = (torch.rand(H, W, generator=torch.Generator().manual_seed(3)) > 0.1).cuda() if odd else None
    lib = _lib.load()
    l0 = lib.mgb_launch_count()
    got, info = evaluate_normals(pred, gt, mask, return_error_map=True)
    assert lib.mgb_launch_count() - l0 == LAUNCHES
    assert info["n_valid"] % 2 == odd or mask is not None
    if mask is not None:            # the optional mask is ANDed into ||gt|| > 0
        gt = torch.where(mask[None], gt, torch.zeros_like(gt))
    frac = _check_against_torch(pred, gt, got, info)
    print(f"{H}x{W} odd={odd} ties={ties}: n={info['n_valid']} error bit-identical to torch CUDA for {frac:.4%}")


def test_normals_middle_ranks_in_different_radix_buckets():
    """Even n with the two middle errors far apart: order statistics (n-1)/2 and n/2 lie in different high-16 bins."""
    from marigold_b200 import evaluate_normals

    H, W = 64, 100
    theta = np.where(np.arange(H * W) % 2 == 0, 3.0, 40.0)
    pred, gt = _angles(theta, H, W)
    got, info = evaluate_normals(pred, gt, return_error_map=True)
    e = info["error_map"].cpu().numpy().reshape(-1)
    lo, hi = np.float32(e[theta == 3.0].max()), np.float32(e[theta == 40.0].min())
    assert lo.view(np.uint32) >> 16 != hi.view(np.uint32) >> 16
    assert got["median_angular_error"] == float(np.median(e)) == float((lo + hi) / np.float32(2))
    _check_against_torch(pred, gt, got, info)
    gt2 = gt.clone()                                                                # n odd: the middle value alone
    gt2[:, 0, 0] = 0.0
    got2, info2 = evaluate_normals(pred, gt2, return_error_map=True)
    e2 = info2["error_map"].cpu().numpy()
    assert info2["n_valid"] % 2 == 1 and got2["median_angular_error"] == float(np.median(e2[~np.isnan(e2)])) == float(hi)


def test_normals_all_ties_and_tiny_n():
    from marigold_b200 import evaluate_normals

    pred, gt = _angles(np.zeros(32 * 32), 32, 32)
    got, info = evaluate_normals(pred, gt)
    assert info["n_valid"] == 1024 and got["median_angular_error"] == 0.0 and got["mean_angular_error"] == 0.0
    assert all(got[k] == 100.0 for k in eval_ref.THRESHOLDS)
    for keep in (1, 2, 3):
        g2 = torch.zeros_like(gt)
        g2.view(3, -1)[:, :keep] = gt.view(3, -1)[:, :keep]
        p2 = pred.clone()
        p2.view(3, -1)[0, 1] = 1.0                                                  # a second, different error
        got, info = evaluate_normals(p2, g2, return_error_map=True)
        e = info["error_map"].cpu().numpy()
        assert info["n_valid"] == keep and got["median_angular_error"] == float(np.median(e[~np.isnan(e)]))


def test_normals_no_valid_pixel_gives_nan():
    from marigold_b200 import _lib, evaluate_normals

    pred, _ = _angles(np.full(16 * 24, 10.0), 16, 24)
    lib = _lib.load()
    l0 = lib.mgb_launch_count()
    got, info = evaluate_normals(pred, torch.zeros_like(pred), return_error_map=True)
    assert lib.mgb_launch_count() - l0 == LAUNCHES
    assert info["n_valid"] == 0 and all(np.isnan(v) for v in got.values())
    assert torch.isnan(info["error_map"]).all()
    got, info = evaluate_normals(pred, pred, torch.zeros(16, 24, dtype=torch.bool, device="cuda"))
    assert info["n_valid"] == 0 and all(np.isnan(v) for v in got.values())


def test_normals_deterministic():
    from marigold_b200 import evaluate_normals

    pred, gt = _random_normals(1080, 1920, seed=9, odd=1, tie_frac=0.3)
    a, ia = evaluate_normals(pred, gt, return_error_map=True)
    b, ib = evaluate_normals(pred, gt, return_error_map=True)
    assert np.array([a[k] for k in a]).tobytes() == np.array([b[k] for k in b]).tobytes()
    assert torch.equal(ia["error_map"].view(torch.int32), ib["error_map"].view(torch.int32))


def test_normals_rejects_cpu_tensors():
    from marigold_b200 import _lib, evaluate_normals

    with pytest.raises(_lib.MgbError):
        evaluate_normals(torch.zeros(3, 4, 4), torch.ones(3, 4, 4))


# ---- depth: least_square_disparity and alignment_max_res ----

# Relative metric difference against the restatement and the golden, both float32 as the reference is (numpy's float32
# SVD lstsq, a float32 aligned prediction and reciprocal): at most 6.1e-8 measured on an H100 over these cases, in both
# modes (the scale agrees to 5e-8). The bound leaves a 16x margin; the reciprocal of the disparity mode needed no more.
DEPTH_TOL = {"least_square": 1e-6, "least_square_disparity": 1e-6}
SCALE_TOL = 1e-6


def _depth_case(cfg):
    pred, gt, valid = depth_eval_input(cfg)
    return pred, gt, valid, (torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(), torch.from_numpy(valid).cuda())


@pytest.mark.parametrize("name", list(DEPTH_EVAL_CASES))
def test_depth_alignment_modes_match_reference(name):
    from marigold_b200 import _lib
    from marigold_b200.evaluation import evaluate_depth

    cfg = DEPTH_EVAL_CASES[name]
    pred, gt, valid, dev = _depth_case(cfg)
    lib = _lib.load()
    l0 = lib.mgb_launch_count()
    got, info = evaluate_depth(*dev, alignment=cfg["alignment"], min_depth=DEPTH_EVAL_RANGE[0],
                               max_depth=DEPTH_EVAL_RANGE[1], alignment_max_res=cfg["max_res"])
    assert lib.mgb_launch_count() - l0 == 4
    ref, scale, shift = eval_ref.depth_eval(pred, gt, valid, cfg["alignment"], cfg["max_res"], *DEPTH_EVAL_RANGE)
    assert info["n_valid"] == int(valid.sum()) == int(GOLD[f"depth/{name}/n_valid"])
    for s_ref, t_ref in ((scale, shift), (float(GOLD[f"depth/{name}/scale"]), float(GOLD[f"depth/{name}/shift"]))):
        assert abs(info["scale"] - s_ref) <= SCALE_TOL * abs(s_ref), (info["scale"], s_ref)
        assert abs(info["shift"] - t_ref) <= SCALE_TOL * max(1.0, abs(t_ref)), (info["shift"], t_ref)
    diffs = {(k, src): abs(got[k] - r) / max(1.0, abs(r))
             for k, v in ref.items() for src, r in (("restated", v), ("golden", float(GOLD[f"depth/{name}/{k}"])))}
    worst = max(diffs, key=diffs.get)
    print(f"{name}: scale {info['scale']!r} vs {scale!r}; worst relative metric difference {diffs[worst]:.3e} at {worst}")
    assert diffs[worst] <= DEPTH_TOL[cfg["alignment"]], (worst, diffs[worst])


def test_depth_least_square_new_entry_is_bit_identical_to_the_existing_one():
    """mgb_eval_depth_ex in mode 1 without index tables runs exactly what mgb_eval_depth runs."""
    import ctypes as C

    from marigold_b200 import _lib
    from marigold_b200._lib import ptr, stream_ptr
    from marigold_b200.evaluation import _depth_ws, _run, evaluate_depth

    pred, gt, valid, (p, g, m) = _depth_case(DEPTH_EVAL_CASES["ls_96x128"])
    H, W = gt.shape
    lib = _lib.load()
    for align in (0, 1):
        old, _ = _run(p, g, m, bool(align), 0.5, 8.0, False)
        new = np.zeros(13)
        _lib.check(lib.mgb_eval_depth_ex(ptr(p), ptr(g), ptr(m.to(torch.uint8)), H, W, align, None, None, 0, 0, 0.5, 8.0,
                                         None, ptr(_depth_ws(lib, p.device)), new.ctypes.data_as(C.c_void_p), stream_ptr()))
        assert old.tobytes() == new.tobytes()
    a, ia = evaluate_depth(p, g, m, alignment="least_square", min_depth=0.5, max_depth=8.0)
    b, ib = evaluate_depth(p, g, m, alignment="least_square", min_depth=0.5, max_depth=8.0, alignment_max_res=10 ** 6)
    assert a == b and ia == ib                                       # max_res above the size: the full-resolution fit


def test_depth_rejects_unknown_alignment():
    from marigold_b200.evaluation import evaluate_depth

    x = torch.ones(4, 4, device="cuda")
    with pytest.raises(ValueError):
        evaluate_depth(x, x, alignment="median")
