"""Depth evaluation on the device (`-m gpu`): evaluate_depth, align_depth_least_square, mgb_eval_depth and
mgb_eval_depth_ex (csrc/eval.cu) against the float64 judge and the float32 restatement of tests/depth_eval_ref.py and
the reference's recorded results. Every metric within its derived bound of the float64 value, the delta accuracies equal
to the reference's float32 counts, at the dataset sizes, the degenerate fits and the edges of the mask."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import depth_eval_ref as R
from tests.golden.eval_cases import DEPTH_EVAL_CASES, depth_eval_input, depth_eval_range

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).resolve().parent / "golden" / "eval_golden.npz")
ALIGN = (None, "least_square", "least_square_disparity")
BIG = 3.0e38


def _dev(*arrays):
    return tuple(None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays)


def _ex(pred, gt, valid, mode, tables=None, dmin=1e-6, dmax=BIG, want_aligned=False, H=None, W=None):
    """mgb_eval_depth_ex on device tensors: (13 doubles, aligned_out or None, status)."""
    from marigold_b200 import _lib
    from marigold_b200._lib import ptr, stream_ptr
    from marigold_b200.evaluation import _depth_ws

    lib = _lib.load()
    H, W = (H, W) if H is not None else pred.shape
    m = None if valid is None else valid.to(torch.uint8)
    rows, cols = tables if tables is not None else (None, None)
    aligned = torch.full_like(pred, -7.0) if want_aligned else None
    out = np.zeros(13)
    rc = lib.mgb_eval_depth_ex(ptr(pred), ptr(gt), ptr(m), H, W, mode, ptr(rows), ptr(cols),
                               0 if rows is None else rows.numel(), 0 if cols is None else cols.numel(), float(dmin),
                               float(dmax), ptr(aligned), ptr(_depth_ws(lib, pred.device)), out.ctypes.data_as(C.c_void_p),
                               stream_ptr())
    return out, aligned, rc


def _scene(H, W, seed, alignment, mask, lo=0.6, far=20.0):
    """A seeded scene: smooth depth with pasted planes (discontinuities), an affine-invariant prediction with a
    long-tailed error. mask: None, a valid fraction, "row" or "pixel"."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H, dtype=np.float32), np.linspace(0, 1, W, dtype=np.float32), indexing="ij")
    gt = lo + 0.3 * far * (0.55 + 0.4 * np.sin(3 * xx + 2 * yy))
    for _ in range(4):
        y0, x0, z0 = rng.uniform(0, 0.7), rng.uniform(0, 0.7), lo + (far - lo) * rng.uniform() ** 2
        gt = np.where((yy >= y0) & (yy < y0 + 0.3) & (xx >= x0) & (xx < x0 + 0.3), z0 * (1 + 0.2 * (xx - x0)), gt)
    gt = gt.astype(np.float32)
    tail = rng.standard_t(3, size=(H, W)).astype(np.float32)
    if alignment == "least_square_disparity":
        pred = 1.3 / gt - 0.02 + 0.004 * tail                           # some pred <= 0
    else:
        pred = (gt - 0.2 * far) / (0.9 * far) + 0.004 * tail
        if alignment is None:
            pred = gt * (1 + 0.1 * tail)
    if mask is None:
        valid = None
    elif mask == "row":
        valid = np.zeros((H, W), bool)
        valid[H // 2] = True
    elif mask == "pixel":
        valid = np.zeros((H, W), bool)
        valid[H // 3, W // 5] = True
    else:
        valid = rng.uniform(size=(H, W)) < mask
    if valid is not None:
        gt = np.where(valid, gt, 0.0).astype(np.float32)
    return pred.astype(np.float32), gt, valid


def _check(pred, gt, valid, alignment, max_res, dmin, dmax, label, golden=None):
    """One evaluate_depth call held to the judge; returns {metric: error / bound}."""
    from marigold_b200 import _lib
    from marigold_b200.evaluation import evaluate_depth

    lib = _lib.load()
    p, g, m = _dev(pred, gt, valid)
    l0 = lib.mgb_launch_count()
    got, info = evaluate_depth(p, g, m, alignment=alignment, min_depth=dmin, max_depth=dmax, alignment_max_res=max_res)
    assert lib.mgb_launch_count() - l0 == 4, label
    v = np.ones(pred.shape, bool) if valid is None else valid
    ref, scale, shift, n, _, bounds = R.depth_eval_f64(pred, gt, v, alignment, max_res, dmin, dmax)
    assert info["n_valid"] == n, label
    ratios = {}
    for k, mine, want in (("scale", info["scale"], scale), ("shift", info["shift"], shift)):
        ratios[k] = abs(mine - want) / bounds[k] if bounds[k] else float(mine != want)
        assert ratios[k] <= 1.0, (label, k, mine, want, bounds[k])
    for k in R.METRICS:
        if k in R.DELTAS:
            continue
        if n == 0:
            assert np.isnan(got[k]), (label, k, got[k])
            continue
        ratios[k] = abs(got[k] - ref[k]) / bounds[k]
        assert ratios[k] <= 1.0, (label, k, got[k], ref[k], bounds[k])
    # the delta accuracies: the reference's float32 decisions from the scale and shift the device found
    _, _, _, _, a32, bits = R.depth_eval_ref32(pred, gt, v, alignment, max_res, dmin, dmax,
                                               scale_shift=(info["scale"], info["shift"]))
    for k, b in zip(R.DELTAS, bits):
        if n == 0:
            assert np.isnan(got[k])
            continue
        count = int(np.count_nonzero(b & v))
        assert got[k] == count / n, (label, k, got[k] * n, count)
        if golden is not None:
            assert count == round(float(GOLD[f"depth/{golden}/{k}"]) * n), (label, k, "golden")
    worst = max((r, k) for k, r in ratios.items())
    print(f"{label}: n={n} scale={info['scale']!r} worst error / bound {worst[0]:.2e} ({worst[1]})")
    return got, info, ratios


# (H, W, alignment, max_res, mask, dmin, dmax)
CASES = [(H, W, a, None, mask, dmin, dmax)
         for (H, W, dmin, dmax), masks in (((37, 53, 1e-3, 10.0), (None, 0.8, "pixel")), ((96, 128, 0.5, 8.0), (0.8, "row", None)),
                                           ((352, 1216, 1e-5, 80.0), (0.05, None, 0.8)), ((480, 640, 1e-3, 10.0), (None, 0.8, 0.05)),
                                           ((768, 1024, 0.6, 350.0), (0.8, 0.05, "row")), ((1080, 1920, 1e-6, BIG), (0.05, 0.8, None)))
         for a, mask in zip(ALIGN, masks)]
CASES += [(37, 53, "least_square", 16, 0.8, 1e-3, 10.0), (96, 128, "least_square_disparity", 64, 0.8, 0.5, 8.0),
          (96, 128, "least_square", 64, "row", 0.5, 8.0), (1216, 352, "least_square", 1024, 0.05, 1e-5, 80.0),
          (1216, 352, "least_square_disparity", 1024, 0.8, 1e-5, 80.0), (1080, 1920, "least_square", 1024, 0.8, 1e-6, BIG),
          (4032, 6048, None, None, 0.8, 1e-5, float("inf")), (4032, 6048, "least_square", 1024, 0.8, 1e-5, float("inf")),
          (4032, 6048, "least_square_disparity", 1024, 0.05, 1e-5, float("inf"))]


@pytest.mark.parametrize("H,W,alignment,max_res,mask,dmin,dmax", CASES)
def test_every_size_and_mode_within_the_bound_of_float64(H, W, alignment, max_res, mask, dmin, dmax):
    pred, gt, valid = _scene(H, W, H + W + ALIGN.index(alignment), alignment, mask, lo=max(dmin, 0.3),
                             far=min(dmax, 60.0) * 1.2)
    _check(pred, gt, valid, alignment, max_res, dmin, dmax, f"{H}x{W} {alignment} max_res={max_res} mask={mask}")


@pytest.mark.parametrize("name", list(DEPTH_EVAL_CASES))
def test_reference_cases_deltas_exact_and_fit_to_float32(name):
    """Every recorded case of the reference: within the bound of float64, the delta counts equal to the reference's, the
    fit equal to its float32 scale and shift after rounding (or within 2e-7 where the last bit of the SVD decides)."""
    cfg = DEPTH_EVAL_CASES[name]
    pred, gt, valid = depth_eval_input(cfg)
    got, info, _ = _check(pred, gt, valid, cfg["alignment"], cfg["max_res"], *depth_eval_range(cfg), name, golden=name)
    gs, gt_ = float(GOLD[f"depth/{name}/scale"]), float(GOLD[f"depth/{name}/shift"])
    assert abs(info["scale"] - gs) <= 2e-7 * max(abs(gs), abs(gt_), 1e-30) and abs(info["shift"] - gt_) <= 2e-7 * max(abs(gs), abs(gt_), 1e-30)
    key = f"depth/{name}/delta_bits"
    if key in GOLD:                                        # planted: the device's fit must round to the reference's
        assert (np.float32(info["scale"]), np.float32(info["shift"])) == (np.float32(gs), np.float32(gt_))


def test_aligned_out_is_the_clipped_map_everywhere():
    for mode, (H, W) in ((0, (37, 53)), (1, (480, 640)), (2, (352, 1216))):
        alignment = ALIGN[mode]
        pred, gt, valid = _scene(H, W, 11 + mode, alignment, 0.5, lo=0.6, far=12.0)
        p, g, m = _dev(pred, gt, valid)
        plain, _, rc0 = _ex(p, g, m, mode, dmin=1.5, dmax=5.0)
        out, aligned, rc = _ex(p, g, m, mode, dmin=1.5, dmax=5.0, want_aligned=True)
        assert rc0 == rc == 0 and plain.tobytes() == out.tobytes()          # requesting the map changes no metric bit
        want = R.align_f64(pred, out[0], out[1], alignment, 1.5, 5.0).astype(np.float32)
        mine = aligned.cpu().numpy()
        ulps = np.abs(mine.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert ulps.max() <= 1, (alignment, int(ulps.max()))
        assert ulps[~valid].max() <= 1 and (mine[~valid] != -7.0).all()     # written outside the mask too
        assert (mine == 1.5).any() and (mine == 5.0).any()                  # both clips met


@pytest.mark.parametrize("ratio", [1.0, 1e2, 1e4, 1e6, "jitter"])
def test_conditioning_sweep_holds_the_centred_bound(ratio):
    """The same scene with the prediction offset to mean / std = 1 ... 10^6, and a constant with a few float32 ulps of
    jitter: the fit stays within the bound of the centred problem against the float64 SVD."""
    H, W = 480, 640
    rng = np.random.default_rng(3)
    if ratio == "jitter":
        pred = (np.float32(0.3) + rng.integers(0, 4, (H, W)).astype(np.float32) * np.float32(3e-8)).astype(np.float32)
        gt = (2.0 + 1e6 * (pred.astype(np.float64) - 0.3) + 0.01 * rng.standard_normal((H, W))).astype(np.float32)
    else:
        z = rng.standard_normal((H, W))
        pred = (ratio + z).astype(np.float32)
        gt = (3.0 + 0.5 * (pred.astype(np.float64) - ratio) + 0.01 * rng.standard_normal((H, W))).astype(np.float32)
    valid = rng.uniform(size=(H, W)) < 0.8
    _, info, ratios = _check(pred, gt, valid, "least_square", None, 1e-3, 10.0, f"mean/std={ratio}")
    s64, _ = R.lstsq_f64(pred[valid], gt[valid])
    s32, _ = R.lstsq_ref32(pred[valid], gt[valid])
    print(f"mean/std={ratio}: device scale off the float64 SVD by {abs(info['scale'] - s64) / abs(s64):.2e}, the "
          f"reference's float32 lstsq by {abs(float(s32) - s64) / abs(s64):.2e}")


@pytest.mark.parametrize("k", [1e-4, 1e4])
def test_fit_is_scale_equivariant(k):
    pred, gt, valid = _scene(480, 640, 21, "least_square", 0.8)
    a, ia, _ = _check(pred, gt, valid, "least_square", None, 1e-3, 30.0, "unscaled")
    b, ib, _ = _check((pred * np.float32(k)).astype(np.float32), gt, valid, "least_square", None, 1e-3, 30.0, f"pred x {k}")
    assert abs(ib["scale"] * k - ia["scale"]) <= 1e-6 * abs(ia["scale"])    # float32 rounding of pred * k
    for key in R.METRICS:
        assert abs(a[key] - b[key]) <= 1e-5 * max(1.0, abs(a[key])), key


@pytest.mark.parametrize("c", [0.0, 0.3, 0.5, 0.7123])
@pytest.mark.parametrize("n", [1, 2, 12288, 245760, 2073600])
def test_constant_prediction_gets_the_minimum_norm_fit(c, n):
    """What a collapsed model predicts: lstsq's minimum-norm solution mean(g) (c, 1) / (c^2 + 1), not noise over noise."""
    H, W = {1: (16, 24), 2: (16, 24), 12288: (96, 128), 245760: (384, 640), 2073600: (1080, 1920)}[n]
    rng = np.random.default_rng(n)
    gt = rng.uniform(1, 5, (H, W)).astype(np.float32)
    valid = np.zeros(H * W, bool)
    valid[rng.choice(H * W, n, replace=False)] = True
    valid = valid.reshape(H, W)
    pred = np.full((H, W), c, np.float32)
    _, info, _ = _check(pred, gt, valid, "least_square", None, 1e-3, 10.0, f"const {c} n={n}")
    gm, m = float(gt[valid].astype(np.float64).mean()), float(np.float32(c))
    assert abs(info["scale"] - gm * m / (m * m + 1)) <= 1e-9 and abs(info["shift"] - gm / (m * m + 1)) <= 1e-9


def test_two_one_and_no_valid_pixels():
    from marigold_b200.evaluation import evaluate_depth

    pred, gt, _ = _scene(32, 48, 5, "least_square", None)
    for eq in (False, True):                                # two pixels: the exact line, or the rank-1 system
        valid = np.zeros((32, 48), bool)
        valid[3, 4] = valid[20, 40] = True
        p2 = pred.copy()
        if eq:
            p2[20, 40] = p2[3, 4]
        _, info, _ = _check(p2, gt, valid, "least_square", None, 1e-3, 30.0, f"two pixels equal={eq}")
    valid = np.zeros((32, 48), bool)
    valid[7, 7] = True
    _check(pred, gt, valid, "least_square", None, 1e-3, 30.0, "one pixel")
    # no valid pixel: n_valid 0 and every metric NaN, as the reference's 0 / 0 (and evaluate_normals); the fit is 0, 0
    p, g, m = _dev(pred, gt, np.zeros((32, 48), bool))
    for alignment, fit in ((None, (1.0, 0.0)), ("least_square", (0.0, 0.0)), ("least_square_disparity", (0.0, 0.0))):
        got, info = evaluate_depth(p, g, m, alignment=alignment)
        assert info == {"scale": fit[0], "shift": fit[1], "n_valid": 0} and all(np.isnan(v) for v in got.values())
    # disparity with an empty fit (no pred > 0) over a non-empty mask: lstsq of no rows is 0, 0; the clips decide the map
    cfg = DEPTH_EVAL_CASES["lsd_no_positive_pred"]
    _, info, _ = _check(*depth_eval_input(cfg), cfg["alignment"], None, *depth_eval_range(cfg), "empty disparity fit")
    assert (info["scale"], info["shift"]) == (0.0, 0.0)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_poison_outside_the_mask_changes_no_bit(mode):
    H, W = 352, 1216
    pred, gt, valid = _scene(H, W, 31 + mode, ALIGN[mode], 0.3)
    rng = np.random.default_rng(4)
    poison = np.array([np.nan, np.inf, -np.inf, 0.0, -3.0], np.float32)
    clean_p, clean_g = np.where(valid, pred, 1.0).astype(np.float32), np.where(valid, gt, 1.0).astype(np.float32)
    bad_p = np.where(valid, pred, poison[rng.integers(0, 5, (H, W))]).astype(np.float32)
    bad_g = np.where(valid, gt, poison[rng.integers(0, 5, (H, W))]).astype(np.float32)
    _, _, m = _dev(None, None, valid)
    a, _, _ = _ex(*_dev(clean_p, clean_g), m, mode, dmin=1e-3, dmax=80.0)
    b, _, _ = _ex(*_dev(bad_p, bad_g), m, mode, dmin=1e-3, dmax=80.0)
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all()
    if mode == 2:            # inside the mask, pred <= 0 and gt <= 0 leave the fit whatever their value
        inside = valid & (rng.uniform(size=(H, W)) < 0.1)
        p1, p2 = np.where(inside, -1.0, pred).astype(np.float32), np.where(inside, 0.0, pred).astype(np.float32)
        g1, g2 = np.where(inside, 0.0, gt).astype(np.float32), np.where(inside, -2.0, gt).astype(np.float32)
        a, _, _ = _ex(*_dev(p1, g1), m, 2)
        b, _, _ = _ex(*_dev(p2, g2), m, 2)
        assert a[:2].tobytes() == b[:2].tobytes() and np.isfinite(a[:2]).all()


@pytest.mark.parametrize("H,W", [(37, 53), (96, 128), (352, 1216), (480, 640), (768, 1024), (1080, 1920), (4032, 6048)])
def test_entry_points_agree_bit_for_bit(H, W):
    from marigold_b200.evaluation import _run, align_depth_least_square, evaluate_depth

    pred, gt, valid = _scene(H, W, 41, "least_square", 0.8)
    p, g, m = _dev(pred, gt, valid)
    ident = (torch.arange(H, dtype=torch.int32, device="cuda"), torch.arange(W, dtype=torch.int32, device="cuda"))
    for mode in (0, 1):
        old, _ = _run(p, g, m, bool(mode), 0.5, 80.0, False)
        new, _, rc = _ex(p, g, m, mode, dmin=0.5, dmax=80.0)
        assert rc == 0 and old.tobytes() == new.tobytes()
    for mode in (1, 2):                                              # identity tables: the full-resolution fit
        a, _, _ = _ex(p, g, m, mode, dmin=0.5, dmax=80.0)
        b, _, _ = _ex(p, g, m, mode, tables=ident, dmin=0.5, dmax=80.0)
        assert a.tobytes() == b.tobytes()
    if H * W <= 1080 * 1920:
        a = evaluate_depth(p, g, m, alignment="least_square", min_depth=0.5, max_depth=80.0)
        assert a == evaluate_depth(p, g, m, alignment="least_square", min_depth=0.5, max_depth=80.0, alignment_max_res=max(H, W))
    for max_res in (None, max(16, max(H, W) // 3)):                 # the public alignment fits evaluate_depth's pixels
        _, info = evaluate_depth(p, g, m, alignment="least_square", alignment_max_res=max_res)
        aligned, scale, shift = align_depth_least_square(g, p, m, max_resolution=max_res)
        assert (float(scale), float(shift)) == (info["scale"], info["shift"]), max_res
        assert aligned.dtype == torch.float64 and aligned.shape == p.shape


def test_deterministic_at_4032x6048():
    pred, gt, valid = _scene(4032, 6048, 51, "least_square_disparity", 0.8)
    p, g, m = _dev(pred, gt, valid)
    from marigold_b200.evaluation import fit_index_tables

    tables = tuple(t.cuda() for t in fit_index_tables(4032, 6048, 1024))
    a, ma, _ = _ex(p, g, m, 2, tables=tables, dmin=1e-5, dmax=float("inf"), want_aligned=True)
    b, mb, _ = _ex(p, g, m, 2, tables=tables, dmin=1e-5, dmax=float("inf"), want_aligned=True)
    assert a.tobytes() == b.tobytes() and torch.equal(ma.view(torch.int32), mb.view(torch.int32))


def test_bad_arguments_are_refused_without_a_launch():
    from marigold_b200 import _lib

    lib = _lib.load()
    x = torch.ones(8, 8, device="cuda")
    t = torch.arange(8, dtype=torch.int32, device="cuda")
    l0 = lib.mgb_launch_count()
    assert _ex(x, x, None, 1, tables=(t, None))[2] == -1           # fit_rows without fit_cols
    assert _ex(x, x, None, 1, tables=(None, t))[2] == -1
    assert _ex(x, x, None, 1, tables=(t[:0], t))[2] == -1          # fit_h = 0
    assert _ex(x, x, None, 3)[2] == -1 and _ex(x, x, None, -1)[2] == -1
    assert _ex(x, x, None, 1, H=0, W=8)[2] == -1
    assert lib.mgb_launch_count() == l0
