"""The ensembling kernels at every ensemble size they compile or accept, against the restatements in
tests/ensemble_ref.py: selections, indices and fixed-order arithmetic bit for bit, sums within their float64 bounds.

Sizes: depth E = 1..17 (every register-resident instantiation, and one member through the generic kernels), 20, 33,
35, 36, 44, 45, 47 and 64 (the generic cost kernel's chunked launch loop first takes two launches at E = 36 with shift
and E = 45 scale-only; 64 is the largest size and fills the staging area). IID and normals E = 1, 2, 3, 16, 17, 33, 64;
normals also 65 and 100, which have no limit. Shapes: 37 x 53 (less than one wave, HW not a multiple of 256),
96 x 128 (one pixel per thread in every cost pass), 768 x 768 (9 to 48 pixels per thread), 1024 x 768 for a few
sizes, and 3024 x 4032 at the native-resolution pipelines' sizes (depth E = 10, IID and normals E = 2; about 90 pixels
per thread in the reduce passes, 180 in the register-resident cost passes). Inputs: the depth_input-style scene and a
map of five levels where several members are equal at the median at most pixels; from three members on, member 1 is a duplicate of member 0 in both."""
import numpy as np
import pytest
import torch

from tests import ensemble_ref as R
from tests.helpers import record

pytestmark = pytest.mark.gpu

DEPTH_E = list(range(1, 18)) + [20, 33, 35, 36, 44, 45, 47, 64]
SHAPES = [(37, 53), (96, 128), (768, 768)]
# 3024 x 4032: a phone photo at native resolution, with the native-resolution depth pipeline's ten members
NATIVE = (3024, 4032)
DEPTH_CASES = ([(E, s) for E in DEPTH_E for s in SHAPES] + [(E, (1024, 768)) for E in (2, 16, 17, 64)]
               + [(10, NATIVE)])
FD_CASES = [(E, s) for E in DEPTH_E for s in ((96, 128), (768, 768))]
IID_E = [1, 2, 3, 16, 17, 33, 64]
NORMALS_E = IID_E + [65, 100]
# (shape, E): every size at two shapes, and two members at native resolution
IID_CASES = [(s, E) for s in ((37, 53), (768, 768)) for E in IID_E] + [(NATIVE, 2)]
NORMALS_CASES = [(s, E) for s in ((37, 53), (768, 768)) for E in NORMALS_E] + [(NATIVE, 2)]
FD_STEPS = (1.5e-8, 1e-3, 0.3, -0.3)


def _id(case):
    E, (H, W) = case
    return f"E{E}-{H}x{W}"


def _shape_id(case):
    (H, W), E = case
    return f"{H}x{W}-{E}"


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _scene(E, H, W):
    """[E, 1, H, W] on the device: a smooth scene through per-member affine maps plus noise (tests/golden/cases.py's
    depth_input), from three members on member 1 an exact copy of member 0; and parameters near the identity, equal for
    members 0 and 1 so that the copy stays tied after alignment."""
    g = torch.Generator(device="cuda").manual_seed(1000 * E + H)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H, device="cuda", dtype=torch.float64),
                            torch.linspace(0, 1, W, device="cuda", dtype=torch.float64), indexing="ij")
    base = 0.5 + 0.25 * torch.sin(3 * xx + 2 * yy) + 0.2 * xx * yy
    base = (base - base.min()) / (base.max() - base.min())
    s = 0.4 + 0.5 * torch.rand(E, 1, 1, device="cuda", generator=g, dtype=torch.float64)
    t = 0.1 * torch.rand(E, 1, 1, device="cuda", generator=g, dtype=torch.float64)
    noise = 0.01 * torch.randn(E, H, W, device="cuda", generator=g, dtype=torch.float64)
    d = (base[None] * s + t + noise).clamp(0, 1).float()[:, None]
    rng = np.random.default_rng(E * 7 + H)
    p = np.concatenate([1 + 0.05 * rng.standard_normal(E), 0.02 * rng.standard_normal(E)])
    if E >= 3:
        d[1] = d[0]
        p[1], p[E + 1] = p[0], p[E]
    return d.contiguous(), p


def _ties(E, H, W):
    """Five levels per member and pixel, one parameter set for every member: exact ties everywhere, several members
    equal at the median at most pixels."""
    g = torch.Generator(device="cuda").manual_seed(2000 * E + H)
    d = torch.randint(0, 5, (E, 1, H, W), device="cuda", generator=g).float() / 4
    if E >= 3:
        d[1] = d[0]
    return d.contiguous(), np.concatenate([np.full(E, 0.9), np.full(E, 0.05)])


INPUTS = {"scene": _scene, "ties": _ties}


def _n_param(E, shift):
    return 2 * E if shift else E


def _call(d, p, shift, median, reg=0.02, unc=True, aux=True):
    """ensemble_depth with the alignment passes at full resolution (max_res=None): the restatements align the whole
    map. Up to 1024 x 1024 that is the default's behaviour; at 3024 x 4032 it holds the cost and min / max passes to
    the 12-megapixel map rather than the default's 768 x 1024 copy."""
    from marigold_b200.ensemble import ensemble_depth

    E = d.shape[0]
    return ensemble_depth(d, shift_invariant=shift, reduction="median" if median else "mean", param=p[:_n_param(E, shift)],
                          regularizer_strength=reg, output_uncertainty=unc, return_aux=aux, max_res=None)


def _launches(fn, *args):
    from marigold_b200 import _lib

    lib = _lib.load()
    torch.cuda.synchronize()
    l0 = lib.mgb_launch_count()
    r = fn(*args)
    torch.cuda.synchronize()
    return int(lib.mgb_launch_count() - l0), r


def _ratio(err, bound):
    return float((err.double() / bound.double()).max()) if err.numel() else 0.0


# ---- depth -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", DEPTH_CASES, ids=_id)
def test_depth_reduce_and_minmax(case):
    """The median map, its member and its MAD bit for bit against the stable restatement; the renormalised mean map bit
    for bit (sequential sum) and its std within the float64 bound (NaN for one member, as torch); init_param from the
    per-member min / max bit for bit; the same map without the uncertainty and the index."""
    E, (H, W) = case
    for kind, make in INPUTS.items():
        d, p = make(E, H, W)
        for shift in (True, False):
            for median in (True, False):
                pred, unc, aux = _call(d, p, shift, median)
                np.testing.assert_array_equal(aux["param0"], R.init_param(d, shift))
                a = R.align(d.reshape(E, -1), p[:_n_param(E, shift)], shift)
                if median:
                    med, idx = R.lower_median(a)
                    pr, ur, _ = R.renorm(med, R.mad(a, med), shift)
                    assert torch.equal(aux["member_idx"].reshape(-1), idx), (kind, shift)
                    assert torch.equal(unc.reshape(-1), ur), (kind, shift)
                else:
                    m = R.seq_mean(a)
                    assert bool(((m.double() - a.double().mean(0)).abs() <= R.mean_bound(a)).all())
                    pr, _, rng = R.renorm(m, None, shift)
                    s64, ds = R.std64(a)
                    u = unc.reshape(-1).double()
                    if E == 1:
                        assert torch.isnan(u).all()
                    else:
                        rng = float(rng)
                        b = ds / rng + R.U * (s64 + ds) / rng
                        r = record(f"ens_sizes/depth_std/E{E}", _ratio((u - s64 / rng).abs(), b))
                        assert r <= 1.0, (kind, shift, r)
                assert torch.equal(pred.reshape(-1), pr), (kind, shift, median)
                pred2, unc2 = _call(d, p, shift, median, unc=False, aux=False)
                assert unc2 is None and torch.equal(pred2, pred)


@pytest.mark.parametrize("case", DEPTH_CASES, ids=_id)
def test_depth_objective_within_float64_bound(case):
    """cost_fn against the float64 objective for median and mean, with and without shift, reg 0 and 0.02. For the
    register-resident kernels up to 1024 x 1024 the bound is also below what one dropped pixel moves the objective by."""
    E, (H, W) = case
    for kind, make in INPUTS.items():
        d, p = make(E, H, W)
        for shift in (True, False):
            q = p[:_n_param(E, shift)]
            for median in (True, False):
                for reg in (0.0, 0.02):
                    _, _, aux = _call(d, p, shift, median, reg=reg, unc=False)
                    n, cf = _launches(aux["cost_fn"], q)
                    assert n == R.cost_launches(E, H * W, 1)
                    val, bound, _, _ = R.cost(d, q, shift, median, reg)
                    r = record(f"ens_sizes/cost/E{E}", abs(cf - val) / bound if cf != val else 0.0)
                    assert r <= 1.0, (kind, shift, median, reg, cf, val, bound)
            # up to 1024 x 1024; at 3024 x 4032 one pixel moves the objective by less than the fp32 sums' bound
            if R.register_resident(E) and kind == "scene" and H * W <= 1024 * 1024:
                pair_sum = R.cost(d, q, shift, True, 0.0)[0]
                bound_rel = R.cost(d, q, shift, True, 0.0)[1] / pair_sum
                assert bound_rel < R.pixel_effect(d, q, shift), (bound_rel, shift)


@pytest.mark.parametrize("case", FD_CASES, ids=_id)
def test_cost_fd_rows_equal_points_alone(case):
    """cost_fd(b, pert)[1 + i] equals cost_fn(b with coordinate i moved) bit for bit, with steps of 1.5e-8, 1e-3 and
    +-0.3: the large steps move members across the median, so every case of the perturbation pass's clamp runs (checked
    on the restatement). The launch count shows how many chunks the generic kernels took."""
    E, (H, W) = case
    rng = np.random.default_rng(E + H)
    counts, crossings = [0, 0, 0], 0
    for kind, make in INPUTS.items():
        d, p = make(E, H, W)
        for median, shift in ((True, True), (False, True), (True, False)):
            n = _n_param(E, shift)
            b = p[:n]
            pert = b + rng.choice(FD_STEPS, n)
            _, _, aux = _call(d, p, shift, median, unc=False)
            launches, fd = _launches(aux["cost_fd"], b, pert)
            assert launches == R.cost_launches(E, H * W, 1 + n), launches
            X = np.repeat(b[None], n, 0)
            X[np.arange(n), np.arange(n)] = pert
            assert fd[0] == aux["cost_fn"](b)
            np.testing.assert_array_equal(fd[1:], np.array([aux["cost_fn"](x) for x in X]), err_msg=f"{kind} {shift}")
            if median and R.register_resident(E):
                c, x = R.clamp_cases(d, b, pert, shift)
                counts = [i + j for i, j in zip(counts, c)]
                crossings += x
    if R.register_resident(E):
        assert counts[1] > 0 and counts[2] > 0 and (E < 3 or counts[0] > 0), counts
        assert crossings > 0


def test_one_member_matches_reference_bit_for_bit():
    """One member: no pairs, the objective is the regulariser alone, and the reference's float32 objective is then
    the device's (exact min / max). The BFGS parameters and the map equal the reference's."""
    from marigold_b200.ensemble import ensemble_depth
    from oracle.ensemble import ensemble_depth as ref_ensemble_depth
    from tests.golden.cases import DEPTH_CASES as GOLDEN_CASES, depth_input

    d = depth_input(GOLDEN_CASES["e3_default"])[:1]
    for kw in (dict(), dict(reduction="mean", output_uncertainty=True), dict(shift_invariant=False),
               dict(output_uncertainty=True, regularizer_strength=0.1)):
        pred, unc, aux = ensemble_depth(d.cuda(), return_aux=True, **kw)
        rp, ru, rparam = ref_ensemble_depth(d, return_param=True, **kw)
        np.testing.assert_array_equal(aux["param"], rparam)
        assert torch.equal(pred.cpu(), rp)
        if ru is not None:
            np.testing.assert_array_equal(unc.cpu().numpy(), ru.numpy())


# ---- IID and normals ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,E", IID_CASES, ids=[_shape_id(c) for c in IID_CASES])
def test_iid_sizes(shape, E):
    """Median and MAD bit for bit (the generic rank-count selection); the mean bit for bit and within its float64
    bound; the std within its bound, NaN for one member as torch."""
    from marigold_b200.ensemble import ensemble_iid

    H, W = shape
    g = torch.Generator(device="cuda").manual_seed(E * 31 + H)
    x = torch.rand(E, 3, H, W, device="cuda", generator=g)
    x[:, :, : H // 2] = torch.randint(0, 5, (E, 3, H // 2, W), device="cuda", generator=g).float() / 4
    if E >= 2:
        x[1] = x[0]
    for median in (True, False):
        red = "median" if median else "mean"
        pred, unc = ensemble_iid(x, True, red)
        pred2, unc2 = ensemble_iid(x, False, red)
        assert unc2 is None and torch.equal(pred2, pred)
        if median:
            med, _ = R.lower_median(x)
            assert torch.equal(pred[0], med)
            assert torch.equal(unc[0], R.mad(x, med))
        else:
            m = R.seq_mean(x)
            assert torch.equal(pred[0], m)
            assert bool(((m.double() - x.double().mean(0)).abs() <= R.mean_bound(x)).all())
            s64, ds = R.std64(x)
            if E == 1:
                assert torch.isnan(unc).all()
            else:
                r = record(f"ens_sizes/iid_std/E{E}", _ratio((unc[0].double() - s64).abs(), ds))
                assert r <= 1.0, r


def _normals_input(E, H, W):
    """Unit normals with degenerate rows: members that cancel exactly (pairs n, -n; the odd one out zero) and nearly
    (mean norm below the 1e-6 clamp), an antiparallel pair among random members, and exact duplicates."""
    g = torch.Generator(device="cuda").manual_seed(E * 17 + H)
    n = torch.nn.functional.normalize(torch.randn(E, 3, H, W, device="cuda", generator=g), dim=1)
    n[:, 2] += 0.5
    n = torch.nn.functional.normalize(n, dim=1)
    if E >= 2:
        for k in range(E // 2):
            n[2 * k + 1, :, 0:2] = -n[2 * k, :, 0:2]
        if E % 2:
            n[E - 1, :, 0:2] = 0.0
        n[1, 2, 1] = torch.nextafter(n[1, 2, 1], torch.full_like(n[1, 2, 1], 2.0))   # row 1: nearly cancels
        n[1, :, 2] = -n[0, :, 2]                                                      # row 2: antiparallel pair
        n[min(2, E - 1), :, 3] = n[0, :, 3]                                           # row 3: duplicates
    return n.contiguous()


@pytest.mark.parametrize("shape,E", NORMALS_CASES, ids=[_shape_id(c) for c in NORMALS_CASES])
def test_normals_sizes(shape, E):
    """Mean normals, argmax and gathered normals bit for bit against the kernel's arithmetic restated; the uncertainty
    within its float64 bound. The degenerate rows reach the 1e-6 clamp."""
    from marigold_b200.ensemble import ensemble_normals

    H, W = shape
    n = _normals_input(E, H, W)
    for closest in (True, False):
        out, unc, aux = ensemble_normals(n, True, "closest" if closest else "mean", return_aux=True)
        ro, ri, ru, ub, _ = R.normals(n, closest)
        if E >= 2 and not closest:
            assert bool((ro[:, 0] == 0).all())                                  # exact cancellation
            assert bool((ro[:, 1].norm(dim=0) < 0.999).any())                   # below the clamp: not unit
        assert torch.equal(aux["member_idx"][0, 0], ri)
        assert torch.equal(out[0], ro)
        r = record(f"ens_sizes/normals_unc/E{E}", _ratio((unc[0, 0].double() - ru).abs(), ub))
        assert r <= 1.0, r


# ---- limits and the shared staging area ------------------------------------------------------------------------------
def test_ensemble_size_limit_raises_before_any_launch():
    """65 members: depth and IID raise, naming the limit, before any kernel is launched."""
    from marigold_b200 import _lib
    from marigold_b200._lib import MgbError
    from marigold_b200.ensemble import ensemble_depth, ensemble_iid

    lib = _lib.load()
    d = torch.rand(65, 1, 16, 16, device="cuda")
    x = torch.rand(65, 3, 16, 16, device="cuda")
    for fn in (lambda: ensemble_depth(d), lambda: ensemble_iid(x)):
        torch.cuda.synchronize()
        l0 = lib.mgb_launch_count()
        with pytest.raises(MgbError, match="64"):
            fn()
        torch.cuda.synchronize()
        assert lib.mgb_launch_count() == l0


@pytest.mark.parametrize("E", [8, 64])
def test_reduce_then_cost_leaves_reduce_output_intact(E):
    """The reduce is asynchronous and reads its parameters from the pinned staging area that the next cost call
    rewrites: a cost call at other parameters, issued without a synchronisation, must not change the reduce's map."""
    d, p = _scene(E, 768, 768)
    pred, unc, aux = _call(d, p, True, True)
    aux["cost_fn"](p * 1.5)
    a = R.align(d.reshape(E, -1), p, True)
    med, idx = R.lower_median(a)
    pr, ur, _ = R.renorm(med, R.mad(a, med), True)
    assert torch.equal(pred.reshape(-1), pr) and torch.equal(unc.reshape(-1), ur)
    assert torch.equal(aux["member_idx"].reshape(-1), idx)
