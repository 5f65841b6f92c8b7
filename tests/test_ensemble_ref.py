"""The ensembling restatements (tests/ensemble_ref.py) against the reference-generated goldens and the float32 objective
restated from the reference with torch ops. CPU only."""
import numpy as np
import pytest
import torch

from tests import ensemble_ref as R
from tests.golden.cases import (DEPTH_CASES, IID_CASES, NORMALS_CASES, depth_input, iid_input, normals_input)
from tests.helpers import _ref_cost

_DIR = __file__.rsplit("/", 1)[0] + "/golden/"
GOLD = np.load(_DIR + "ensemble_golden.npz")
IID_GOLD = np.load(_DIR + "iid_golden.npz")


def _within(x, ref, bound, what):
    x, ref, bound = (torch.as_tensor(v).double() for v in (x, ref, bound))
    err = (x - ref).abs()
    assert bool((err <= bound).all()), f"{what}: max err / bound {float((err / bound).max()):.3g}"


@pytest.mark.parametrize("name", list(DEPTH_CASES))
def test_depth_reduce_reproduces_golden(name):
    """At the reference's final parameters: the median map and its MAD bit for bit, the mean map bit for bit (torch's
    CPU mean over E <= 17 members is a sequential fp32 sum), the std within its bound, and init_param exactly."""
    cfg = DEPTH_CASES[name]
    kw = cfg.get("kwargs", {})
    shift = kw.get("shift_invariant", True)
    median = kw.get("reduction", "median") == "median"
    d = depth_input(cfg)
    E = d.shape[0]
    a = R.align(d.reshape(E, -1), GOLD[f"depth/{name}/x"], shift)
    if median:
        pred, _ = R.lower_median(a)
        unc = R.mad(a, pred)
    else:
        pred = R.seq_mean(a)
        unc = R.std64(a)[0].float()
    pr, ur, rng = R.renorm(pred, unc, shift)
    np.testing.assert_array_equal(pr.reshape(GOLD[f"depth/{name}/pred"].shape).numpy(), GOLD[f"depth/{name}/pred"])
    if f"depth/{name}/unc" in GOLD:
        g = torch.from_numpy(GOLD[f"depth/{name}/unc"]).reshape(-1)
        if median:
            np.testing.assert_array_equal(ur.numpy(), g.numpy())
        else:
            s64, ds = R.std64(a)
            # the reference's own float32 std is held to the device's bound, plus the rounding of the division by rng
            _within(g, s64 / float(rng), ds / float(rng) * 1.001 + 2 * R.U * s64 / float(rng), f"{name} std")
    d_al = d
    mr = kw.get("max_res", 1024)
    if max(d.shape[2:]) > mr:
        from oracle.ensemble import _resize_max_res_nearest_exact

        d_al = _resize_max_res_nearest_exact(d, mr)
    np.testing.assert_array_equal(R.init_param(d_al, shift), GOLD[f"depth/{name}/x0"])


@pytest.mark.parametrize("name", list(DEPTH_CASES))
def test_objective_matches_float32_reference(name):
    """The float64 objective agrees with the reference's float32 arithmetic (torch CPU ops) to the float32 gap: each
    pair's torch mean is within (log2(HW) + 2) u of its exact value, halved by the sqrt."""
    cfg = DEPTH_CASES[name]
    kw = cfg.get("kwargs", {})
    shift = kw.get("shift_invariant", True)
    red = kw.get("reduction", "median")
    reg = kw.get("regularizer_strength", 0.02)
    d = depth_input(cfg)
    mr = kw.get("max_res", 1024)
    if max(d.shape[2:]) > mr:
        from oracle.ensemble import _resize_max_res_nearest_exact

        d = _resize_max_res_nearest_exact(d, mr)
    E, HW = d.shape[0], d[0].numel()
    for p in (GOLD[f"depth/{name}/x0"], GOLD[f"depth/{name}/x"]):
        val, bound, _, _ = R.cost(d, p, shift, red == "median", reg)
        pair_sum = R.cost(d, p, shift, red == "median", 0.0)[0]
        gap = pair_sum * ((np.log2(HW) + 2) / 2 + 1.5) * R.U + bound
        assert abs(val - _ref_cost(d, p, shift, red, reg)) <= gap


@pytest.mark.parametrize("name", list(NORMALS_CASES))
def test_normals_reproduce_golden(name):
    """The argmax and the gathered normals bit for bit; the mean normals to 2 ulp (torch's norm rounds in its own
    order); the uncertainty within the restatement's bound."""
    cfg = NORMALS_CASES[name]
    kw = cfg.get("kwargs", {})
    closest = kw.get("reduction", "closest") == "closest"
    n = normals_input(cfg)
    out, idx, unc, ub, sim = R.normals(n, closest)
    g = GOLD[f"normals/{name}/pred"][0]
    if closest:
        np.testing.assert_array_equal(idx.numpy(), GOLD[f"normals/{name}/argmax"].reshape(idx.shape))
        np.testing.assert_array_equal(out.numpy(), g)
    else:
        _within(out, torch.from_numpy(g), 4 * R.U * torch.from_numpy(g).abs() + 1e-12, f"{name} mean normals")
    if f"normals/{name}/unc" in GOLD:
        # torch forms each cosine in its own order (within 4 u of ours), and acos magnifies that near +-1:
        # |d acos| <= min(4 u / sqrt(1 - s^2), sqrt(8 u))
        s = sim.double()
        da = torch.minimum(4 * R.U / (1 - s * s).clamp(min=1e-300).sqrt(), torch.full_like(s, (8 * R.U) ** 0.5))
        g = torch.from_numpy(GOLD[f"normals/{name}/unc"]).reshape(unc.shape)
        _within(g, unc, ub + da.sum(0) / (n.shape[0] * np.pi), f"{name} unc")


@pytest.mark.parametrize("name", list(IID_CASES))
def test_iid_reproduces_golden(name):
    cfg = IID_CASES[name]
    kw = cfg.get("kwargs", {})
    x = iid_input(cfg)
    median = kw.get("reduction", "median") == "median"
    g = IID_GOLD[f"iid/{name}/pred"][0]
    if median:
        pred, _ = R.lower_median(x)
        np.testing.assert_array_equal(pred.numpy(), g)
        if f"iid/{name}/unc" in IID_GOLD:
            np.testing.assert_array_equal(R.mad(x, pred).numpy(), IID_GOLD[f"iid/{name}/unc"][0])
    else:
        np.testing.assert_array_equal(R.seq_mean(x).numpy(), g)
        s64, ds = R.std64(x)
        _within(torch.from_numpy(IID_GOLD[f"iid/{name}/unc"][0]), s64, ds, f"{name} std")


def test_iid_one_member_std_is_nan():
    x = iid_input(IID_CASES["e1"])
    assert torch.isnan(R.std64(x)[0]).all() and torch.isnan(x.std(dim=0)).all()


def test_stable_median_ties():
    """The lower median's member is position (E - 1) // 2 of a stable sort: with all members equal it is member
    (E - 1) // 2, and among equal values at the median the lowest index ranking there."""
    for E in (2, 3, 4, 17, 64):
        a = torch.full((E, 5), 0.25)
        v, i = R.lower_median(a)
        assert (i == (E - 1) // 2).all() and (v == 0.25).all()
    a = torch.tensor([[3.0], [1.0], [1.0], [2.0], [1.0]])       # sorted stably: 1(m1) 1(m2) 1(m4) 2(m3) 3(m0)
    assert int(R.lower_median(a)[1]) == 4
    a = torch.tensor([[2.0], [0.5], [2.0], [0.5]])              # 0.5(m1) 0.5(m3) 2(m0) 2(m2): lower median m3
    assert int(R.lower_median(a)[1]) == 3
    # the normals argmax keeps the first of equal cosines
    n = torch.nn.functional.normalize(torch.randn(1, 3, 4, 4, generator=torch.Generator().manual_seed(0)), dim=1)
    assert (R.normals(n.repeat(3, 1, 1, 1), True)[1] == 0).all()


def test_launch_constants():
    """The launch restatement: register-resident sizes make 2 / 3 launches; the generic kernel's chunked loop needs more
    than one launch first at E = 36 with shift and E = 45 scale-only (96 x 128 and larger: 48 blocks), and E = 64
    takes 7 chunks (14 launches) with shift."""
    HW = 96 * 128
    assert R.cost_blocks(10, HW) == 48 and R.pixels_per_thread(10, HW) == 1
    assert R.pixels_per_thread(10, 768 * 768) == 9 and R.pixels_per_thread(33, 768 * 768) == 48
    assert R.cost_launches(16, HW, 33) == 3 and R.cost_launches(16, HW, 1) == 2
    assert [R.cost_launches(E, HW, 2 * E + 1) for E in (1, 17, 35, 36, 64)] == [2, 2, 2, 4, 14]
    assert [R.cost_launches(E, HW, E + 1) for E in (44, 45, 64)] == [2, 4, 8]
