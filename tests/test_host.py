"""CPU tests of the host-side logic: scheduler coefficient tables vs the oracle's op-by-op `step`,
the C-ABI library (loads, exports every symbol the header declares), pipeline argument handling."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from marigold_b200.schedulers import DDIMScheduler, LCMScheduler
from oracle.schedulers import DDIMSchedulerOracle, LCMSchedulerOracle, SchedulerConfig

ROOT = Path(__file__).resolve().parents[1]


@pytest.mark.parametrize("n", [1, 2, 4, 10, 50, 7])
@pytest.mark.parametrize("pred", ["v_prediction"])
def test_ddim_coefficients_match_oracle_step(n, pred):
    s = DDIMScheduler(prediction_type=pred)
    s.set_timesteps(n)
    o = DDIMSchedulerOracle(SchedulerConfig(prediction_type=pred))
    o.set_timesteps(n)
    assert list(map(int, s.timesteps)) == o.timesteps.tolist()
    kx, kv, kz = s.coefficients()
    g = torch.Generator().manual_seed(n)
    x = torch.randn(2, 4, 8, 8, generator=g)
    for i, t in enumerate(o.timesteps):
        v = torch.randn(2, 4, 8, 8, generator=g)
        ref = o.step(v, t, x)
        mine = kx[i] * x + kv[i] * v
        assert (ref - mine).abs().max() < 2e-5 * max(1.0, ref.abs().max().item())
        x = ref
    assert (kz == 0).all()


def test_ddim_epsilon_prediction_without_zero_snr():
    s = DDIMScheduler(prediction_type="epsilon", rescale_betas_zero_snr=False, timestep_spacing="leading")
    s.set_timesteps(10)
    o = DDIMSchedulerOracle(SchedulerConfig(prediction_type="epsilon", rescale_betas_zero_snr=False,
                                            timestep_spacing="leading"))
    o.set_timesteps(10)
    assert list(map(int, s.timesteps)) == o.timesteps.tolist()
    kx, kv, _ = s.coefficients()
    x, v = torch.randn(1, 4, 4, 4), torch.randn(1, 4, 4, 4)
    for i, t in enumerate(o.timesteps):
        assert torch.allclose(o.step(v, t, x), kx[i] * x + kv[i] * v, atol=3e-5)
    with pytest.raises(RuntimeError):
        z = DDIMScheduler(prediction_type="epsilon")   # zero-SNR + epsilon is undefined at t=999
        z.set_timesteps(4)
        z.coefficients()


@pytest.mark.parametrize("n", [1, 2, 4, 8])
def test_lcm_coefficients_match_oracle_step(n):
    s = LCMScheduler()
    s.set_timesteps(n)
    o = LCMSchedulerOracle()
    o.set_timesteps(n)
    assert list(map(int, s.timesteps)) == o.timesteps.tolist()
    kx, kv, kz = s.coefficients()
    g = torch.Generator().manual_seed(100 + n)
    x = torch.randn(2, 4, 8, 8, generator=g)
    for i, t in enumerate(o.timesteps):
        v = torch.randn(2, 4, 8, 8, generator=g)
        z = torch.randn(2, 4, 8, 8, generator=g)
        ref = o.step(v, t, x, noise=z)
        mine = kx[i] * x + kv[i] * v + kz[i] * z
        assert (ref - mine).abs().max() < 2e-5 * max(1.0, ref.abs().max().item())
        x = ref
    assert kz[-1] == 0 and (kz[:-1] > 0).all()


def test_library_exports_every_declared_symbol():
    from marigold_b200 import _lib

    header = (ROOT / "include" / "marigold_b200.h").read_text()
    declared = set(re.findall(r"\b(mgb_[a-z0-9_]+)\s*\(", header))
    declared -= {"mgb_status", "mgb_dtype", "mgb_decode_mode"}
    assert declared, "no declarations parsed"
    lib = ctypes.CDLL(str(_lib.lib_path())) if _lib.lib_path().exists() else None
    if lib is None:
        _lib.load()          # builds (nvcc cross-compiles without a GPU)
        lib = ctypes.CDLL(str(_lib.lib_path()))
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, f"header declares symbols the library does not export: {missing}"
    assert declared == set(_lib.SIGNATURES), "ctypes SIGNATURES out of sync with include/marigold_b200.h"
    loaded = _lib.load()
    assert b"sm_90a" in loaded.mgb_build_info()


def test_no_cpu_fallback_on_missing_gpu():
    """On a box without a GPU the product path must fail loudly, never silently compute on the CPU."""
    from marigold_b200 import _lib
    from marigold_b200.engine import Engine

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.MgbError):
        Engine()
    from marigold_b200.ensemble import ensemble_depth, ensemble_normals

    with pytest.raises(_lib.MgbError):
        ensemble_depth(torch.rand(2, 1, 8, 8))
    with pytest.raises(_lib.MgbError):
        ensemble_normals(torch.nn.functional.normalize(torch.randn(2, 3, 8, 8), dim=1))


def test_product_never_imports_oracle():
    for py in (ROOT / "marigold_b200").glob("*.py"):
        src = py.read_text()
        assert "import oracle" not in src and "from oracle" not in src, f"{py.name} imports the oracle"


def test_colorize_and_resize_helpers():
    from marigold_b200.pipeline import colorize_depth_maps, get_tv_resample_method, resize_max_res

    c = colorize_depth_maps(np.linspace(0, 1, 12).reshape(3, 4), 0, 1)
    assert c.shape == (1, 3, 3, 4) and c.min() >= 0 and c.max() <= 1      # [B, 3, H, W] like image_util.py:38-76
    c = c.squeeze()
    np.testing.assert_allclose(c[:, 0, 0], np.array([158, 1, 66]) / 255.0)
    np.testing.assert_allclose(c[:, 2, 3], np.array([94, 79, 162]) / 255.0)
    # matplotlib semantics: cm(x) indexes a 256-entry table with int(x * 256); LUT[i] = interpolation at i / 255
    from marigold_b200.pipeline import _SPECTRAL_LUT

    assert _SPECTRAL_LUT.shape == (256, 3)
    np.testing.assert_allclose(_SPECTRAL_LUT[51], np.array([244, 109, 67]) / 255.0, atol=1e-12)     # 51 / 255 = 0.2 = anchor 2
    w = 127 / 25.5 - 4                                                                            # 127 / 255 lies between anchors 4, 5
    np.testing.assert_allclose(_SPECTRAL_LUT[127], (np.array([254, 224, 139]) * (1 - w) + np.array([255, 255, 191]) * w) / 255.0,
                               atol=1e-12)
    x = np.array([[0.4999, 0.5, 0.50195, 0.50391]])                         # 127.97 -> 127, 128, 128.5 -> 128, 129.0 -> 129
    idx = [127, 128, 128, 129]
    np.testing.assert_array_equal(colorize_depth_maps(np.repeat(x, 2, 0), 0, 1).squeeze()[:, 0].T, _SPECTRAL_LUT[idx])
    m = colorize_depth_maps(np.ones((2, 2)), 0, 1, valid_mask=np.array([[True, False], [True, True]])).squeeze()
    assert (m[:, 0, 1] == 0).all() and (m[:, 0, 0] > 0).any()
    with pytest.raises(ValueError):
        get_tv_resample_method("lanczos")
    img = torch.randint(0, 256, (1, 3, 90, 130), dtype=torch.uint8)
    assert resize_max_res(img, 64).shape == (1, 3, 44, 64)     # int() truncation: 90 * 64/130 = 44.3


def test_iid_output_container_follows_the_reference():
    """marigold_b200/iid.py vs marigold_iid_pipeline.py:59-160,393-411: channel ownership, visualisation spaces,
    error behaviour (KeyError on unknown names, RuntimeError on refill)."""
    import numpy as np
    import torch

    from marigold_b200.iid import MarigoldIIDOutput, fill_outputs

    g = torch.Generator().manual_seed(5)
    pred = torch.rand(1, 6, 8, 12, generator=g)
    unc = torch.rand(1, 6, 8, 12, generator=g)
    props = {"target_names": ["albedo", "shading"], "albedo": {"prediction_space": "srgb"},
             "shading": {"prediction_space": "linear", "up_to_scale": True}}
    out = MarigoldIIDOutput(props["target_names"])
    assert not out.is_complete
    fill_outputs(out, pred, unc, props["target_names"], props)
    assert out.is_complete and [e.name for e in out] == ["albedo", "shading"]
    a, s = out["albedo"], out["shading"]
    assert a.array.shape == (3, 8, 12) and np.array_equal(a.array, pred[0, :3].numpy())
    assert np.array_equal(s.uncertainty, unc[0, 3:].numpy())
    assert np.array_equal(np.asarray(a.image), np.moveaxis((pred[0, :3].numpy() * 255).astype(np.uint8), 0, -1))
    lin = pred[0, 3:].numpy()
    lin = (lin / max(lin.max(), 1e-6)) ** (1 / 2.2)
    assert np.array_equal(np.asarray(s.image), np.moveaxis((lin * 255).astype(np.uint8), 0, -1))
    import pytest

    with pytest.raises(RuntimeError):
        out.fill_entry("albedo", pred[:, :3], None, props)
    with pytest.raises(KeyError):
        out.fill_entry("normals", pred[:, :3], None, props)


def test_bfgs_driver_one_callback_follows_scipy_default_finite_differences():
    """marigold_b200.ensemble._bfgs hands scipy one callback that returns f and a gradient built from one batch of
    forward-difference points (jac=True); the trajectory must be the one scipy's own default (jac=None, as the
    reference calls it: marigold/util/ensemble.py:165-171) produces, bit for bit."""
    import scipy.optimize

    from marigold_b200.ensemble import _bfgs, _fd_grad, _scipy_fd_points

    rng = np.random.default_rng(0)
    A = rng.standard_normal((6, 6))
    A = A @ A.T + np.eye(6)
    b = rng.standard_normal(6)

    def f(x):
        x = np.asarray(x, dtype=np.float64)
        return float(np.float32(0.5 * x @ A @ x - b @ x + 0.1 * np.abs(x).sum()))   # fp32-rounded like the device cost

    batches = []

    def fun(x):
        x = np.asarray(x, dtype=np.float64)
        pert = _scipy_fd_points(x)
        xs = np.repeat(x[None], x.size, 0)
        xs[np.arange(x.size), np.arange(x.size)] = pert
        batches.append(len(xs))
        f0 = f(x)
        return f0, _fd_grad(x, f0, np.array([f(r) for r in xs]), pert)

    for x0 in (rng.standard_normal(6), np.array([0.0, 1e9, -1e9, 1.0, -1.0, 3e17])):   # incl. x + eps == x coordinates
        ref = scipy.optimize.minimize(f, x0, method="BFGS", tol=1e-6, options={"maxiter": 50, "disp": False})
        x1, nit1 = _bfgs(fun, x0, 1e-6, 50)
        np.testing.assert_array_equal(x1, ref.x)
        assert nit1 == ref.nit and batches and all(c == 6 for c in batches)


def test_gelu_exponent_polynomial_matches_erf():
    """The GEGLU epilogue's erf (csrc/common.cuh gelu_erf: erfc(|x|/sqrt 2) = 2^-Q(|x|), degree-8 Q evaluated in
    n = -|x|/2) restated in fp32 numpy with the constants read from the source: |gelu error| <= 5e-7 against the exact
    erf form diffusers' GEGLU uses (F.gelu, approximate="none"), over [-12, 12] and at the extremes."""
    import math
    import re
    from pathlib import Path

    src = (Path(__file__).resolve().parents[1] / "marigold_b200" / "csrc" / "common.cuh").read_text()
    K = {int(k): np.float32(float(v)) for k, v in re.findall(r"constexpr float kGeluK(\d) = ([-+0-9.e]+)f;", src)}
    assert sorted(K) == list(range(1, 9))
    x = np.concatenate([np.linspace(-12, 12, 400001), [0.0, -0.0, 1e-30, -1e-30, 50.0, -50.0, 1e4, -1e4]]).astype(np.float32)
    h = np.float32(0.5) * x
    n = -np.abs(h)
    p = K[8] * n + K[7]
    for k in range(6, 0, -1):
        p = (p * n + K[k]).astype(np.float32)
    with np.errstate(over="ignore", under="ignore"):
        e = np.exp2((p * n).astype(np.float32).astype(np.float64)).astype(np.float32)
        g = (n * e + (h - n)).astype(np.float32)
    exact = np.array([0.5 * v * (1.0 + math.erf(v / math.sqrt(2.0))) for v in x.astype(np.float64)])
    assert np.isfinite(g).all()
    assert np.abs(g - exact).max() <= 5e-7
