"""GPU parity of the ensembling kernels (through the C ABI) against the reference-generated goldens.

What can and cannot match: the reference's BFGS runs on finite-difference gradients of an fp32
objective with step 1.5e-8 — its trajectory is decided by rounding noise, so two mathematically
equal objectives that sum in a different order end ~1e-2 apart (measured on the CPU with the
reference itself, DESIGN.md §Ensemble). Hence: (1) the objective VALUE is checked at fixed
parameters, (2) the reduce step is checked at the reference's own final parameters — including the
index the lower median / argmax picks, bit-for-bit, (3) the end-to-end call must improve on the
initial alignment, reach an objective within 5 % of the reference's optimum, and stay within that band."""
import numpy as np
import pytest
import torch

from tests.golden.cases import DEPTH_CASES, NORMALS_CASES, depth_input, normals_input
from tests.helpers import _ref_cost

pytestmark = pytest.mark.gpu
GOLD = np.load(__file__.rsplit("/", 1)[0] + "/golden/ensemble_golden.npz")


@pytest.mark.parametrize("name", list(DEPTH_CASES))
def test_depth_cost_reduce_and_end_to_end(name):
    from marigold_b200.ensemble import ensemble_depth
    from oracle.ensemble import _resize_max_res_nearest_exact

    cfg = DEPTH_CASES[name]
    kw = dict(cfg.get("kwargs", {}))
    d = depth_input(cfg)
    shift = kw.get("shift_invariant", True)
    red = kw.get("reduction", "median")
    reg = kw.get("regularizer_strength", 0.02)
    x_ref, x0_ref = GOLD[f"depth/{name}/x"], GOLD[f"depth/{name}/x0"]

    # (2) reduce at the reference's final parameters
    pred, unc, aux = ensemble_depth(d.cuda(), return_aux=True, param=x_ref, **kw)
    g = GOLD[f"depth/{name}/pred"]
    assert np.abs(pred.cpu().numpy() - g).max() <= 2e-6
    if f"depth/{name}/unc" in GOLD:
        assert np.abs(unc.cpu().numpy() - GOLD[f"depth/{name}/unc"]).max() <= 2e-6
    np.testing.assert_allclose(aux["param0"], x0_ref, rtol=0, atol=0)           # init_param is exact
    # median index exactness: the member we report holds exactly torch.median's value
    if red == "median":
        E = d.shape[0]
        if shift:
            s, t = np.split(x_ref, 2)
            a = d * torch.from_numpy(s).float().view(E, 1, 1, 1) + torch.from_numpy(t).float().view(E, 1, 1, 1)
        else:
            a = d * torch.from_numpy(x_ref).float().view(E, 1, 1, 1)
        med = torch.median(a, dim=0, keepdim=True).values
        picked = torch.gather(a, 0, aux["member_idx"].cpu().long())
        assert torch.equal(picked, med)

    # (1) objective value at fixed parameters
    d_al = d
    mr = kw.get("max_res", 1024)
    if max(d.shape[2:]) > mr:
        d_al = _resize_max_res_nearest_exact(d, mr)
    for p in (x0_ref, x_ref):
        mine = aux["cost_fn"](p)
        ref = _ref_cost(d_al, p, shift, red, reg)
        assert abs(mine - ref) <= 2e-6 * max(1.0, abs(ref)), (mine, ref)

    # (3) end to end
    pred2, _, aux2 = ensemble_depth(d.cuda(), return_aux=True, **kw)
    if int(GOLD[f"depth/{name}/nit"]) == 0:
        assert np.abs(pred2.cpu().numpy() - g).max() <= 2e-6
    else:
        # BFGS here follows rounding noise (module docstring): require that our run improves on the
        # initial alignment and lands within 5 % of the objective value the reference's run reached
        c_mine = _ref_cost(d_al, aux2["param"], shift, red, reg)
        c_ref = _ref_cost(d_al, x_ref, shift, red, reg)
        c_init = _ref_cost(d_al, x0_ref, shift, red, reg)
        assert c_mine <= c_init + 1e-6, (c_mine, c_init)
        assert c_mine <= 1.05 * c_ref + 1e-4, (c_mine, c_ref)
        assert np.abs(pred2.cpu().numpy() - g).max() <= 5e-2


def test_depth_errors_match_reference():
    from marigold_b200.ensemble import ensemble_depth

    with pytest.raises(ValueError):
        ensemble_depth(torch.rand(2, 3, 4, 4).cuda())
    with pytest.raises(ValueError):
        ensemble_depth(torch.rand(2, 1, 4, 4).cuda(), reduction="mode")
    with pytest.raises(ValueError):
        ensemble_depth(torch.rand(2, 1, 4, 4).cuda(), scale_invariant=False, shift_invariant=True)


@pytest.mark.parametrize("name", list(NORMALS_CASES))
def test_normals_match_reference_golden(name):
    from marigold_b200.ensemble import ensemble_normals

    cfg = NORMALS_CASES[name]
    kw = dict(cfg.get("kwargs", {}))
    n = normals_input(cfg)
    pred, unc, aux = ensemble_normals(n.cuda(), return_aux=True, **kw)
    g = GOLD[f"normals/{name}/pred"]
    if kw.get("reduction", "closest") == "closest":
        np.testing.assert_array_equal(aux["member_idx"].cpu().numpy(), GOLD[f"normals/{name}/argmax"])  # bit-exact index
        np.testing.assert_array_equal(pred.cpu().numpy(), g)                                            # gather => exact
    else:
        assert np.abs(pred.cpu().numpy() - g).max() <= 1e-6
    if f"normals/{name}/unc" in GOLD:
        assert np.abs(unc.cpu().numpy() - GOLD[f"normals/{name}/unc"]).max() <= 2e-6


@pytest.mark.parametrize("E", [2, 3, 8, 10])
def test_median_and_argmax_index_properties_full_size(E):
    """Size-independent properties at the full 768x768 map: lower-median value equality and argmax
    equality against torch on the same device inputs."""
    from marigold_b200.ensemble import ensemble_depth, ensemble_normals

    g = torch.Generator().manual_seed(E)
    d = torch.rand(E, 1, 768, 768, generator=g)
    p = np.concatenate([np.ones(E), np.zeros(E)])
    pred, _, aux = ensemble_depth(d.cuda(), return_aux=True, param=p)
    med = torch.median(d, dim=0, keepdim=True).values
    assert torch.equal(torch.gather(d, 0, aux["member_idx"].cpu().long()), med)
    lo, hi = med.min(), med.max()
    assert torch.allclose(pred.cpu(), (med - lo) / (hi - lo), atol=1e-6)
    n = torch.nn.functional.normalize(torch.randn(E, 3, 256, 256, generator=g), dim=1)
    out, _, aux = ensemble_normals(n.cuda(), return_aux=True)
    m = n.mean(0, keepdim=True)
    m = m / torch.norm(m, dim=1, keepdim=True).clamp(min=1e-6)
    idx = (m * n).sum(1, keepdim=True).clamp(-1, 1).argmax(0, keepdim=True)
    assert torch.equal(aux["member_idx"].cpu().long(), idx)
    assert torch.equal(out.cpu(), torch.gather(n, 0, idx.repeat(1, 3, 1, 1)))


def test_cost_fd_is_one_round_trip_and_bit_identical():
    """f(x) and the forward-difference points of its gradient are ONE device round trip, and each of those values equals
    the objective evaluated alone at that point bit for bit (otherwise scipy's f(x+h) - f(x) would pick up summation
    noise), for the register-resident (E <= 16) and the generic kernels. The BFGS run built on it follows scipy's own
    default (jac=None, the reference's call) step for step."""
    import scipy.optimize

    from marigold_b200.ensemble import ensemble_depth

    rng = np.random.default_rng(0)
    for E in (10, 17, 33):
        g = torch.Generator().manual_seed(3)
        d = torch.rand(E, 1, 96, 128, generator=g).cuda()
        p0 = np.concatenate([np.ones(E), np.zeros(E)])
        for red, shift in (("median", True), ("mean", True), ("median", False)):
            kw = dict(reduction=red, shift_invariant=shift)
            n = 2 * E if shift else E
            b = p0[:n] + rng.normal(0, 1e-2, n)
            _, _, ax = ensemble_depth(d, return_aux=True, param=b, **kw)
            pert = b + rng.choice([1.5e-8, 1e-3], n)
            X = np.repeat(b[None], n, 0)
            X[np.arange(n), np.arange(n)] = pert
            fd = ax["cost_fd"](b, pert)
            assert fd.shape == (1 + n,)
            assert fd[0] == ax["cost_fn"](b)
            np.testing.assert_array_equal(fd[1:], np.array([ax["cost_fn"](x) for x in X]))
    # end to end: f(x) and the 2E points of its gradient share one round trip, and the trajectory is scipy's default one
    for E, max_iter in ((10, 50), (17, 8)):
        g = torch.Generator().manual_seed(3)
        d = torch.rand(E, 1, 96, 128, generator=g).cuda()
        _, _, aux = ensemble_depth(d, return_aux=True, max_iter=max_iter)
        assert aux["nit"] > 0
        assert aux["round_trips"] * 2 * E <= aux["nfev"]
        ref = scipy.optimize.minimize(aux["cost_fn"], aux["param0"], method="BFGS", tol=1e-6,
                                      options={"maxiter": max_iter, "disp": False})
        np.testing.assert_array_equal(aux["param"], ref.x)
        assert aux["nit"] == ref.nit


@pytest.mark.parametrize("E,reduction", [(20, "median"), (17, "mean"), (33, "median")])
def test_large_ensembles_generic_path(E, reduction):
    """ensemble_size > 16 (the reference accepts any size; 20 is a common setting) runs the generic kernels:
    objective, reduce, uncertainty and the lower-median index against torch on the same inputs."""
    from marigold_b200.ensemble import ensemble_depth

    g = torch.Generator().manual_seed(E)
    d = torch.rand(E, 1, 64, 80, generator=g)
    d[3] = d[5]                                  # exact ties across members
    rng = np.random.default_rng(E)
    p = np.concatenate([1 + 0.1 * rng.standard_normal(E), 0.05 * rng.standard_normal(E)])
    pred, unc, aux = ensemble_depth(d.cuda(), return_aux=True, param=p, reduction=reduction, output_uncertainty=True)
    s, t = np.split(p, 2)
    a = d * torch.from_numpy(s).float().view(E, 1, 1, 1) + torch.from_numpy(t).float().view(E, 1, 1, 1)
    if reduction == "median":
        med = torch.median(a, dim=0, keepdim=True).values
        assert torch.equal(torch.gather(a, 0, aux["member_idx"].cpu().long()), med)
        u = torch.median((a - med).abs(), dim=0, keepdim=True).values
    else:
        med = a.mean(0, keepdim=True)
        u = a.std(0, keepdim=True)
    lo, hi = med.min(), med.max()
    assert torch.allclose(pred.cpu(), (med - lo) / (hi - lo), atol=2e-6)
    assert torch.allclose(unc.cpu(), u / (hi - lo), atol=2e-6)
    ref = _ref_cost(d, p, True, reduction, 0.02)
    mine = aux["cost_fn"](p)
    assert abs(mine - ref) <= 2e-6 * max(1.0, abs(ref)), (mine, ref)
    # and the optimiser runs end to end
    pred2, _ = ensemble_depth(d.cuda(), reduction=reduction, max_iter=2)
    assert torch.isfinite(pred2).all() and float(pred2.min()) == 0.0 and abs(float(pred2.max()) - 1.0) < 1e-6
