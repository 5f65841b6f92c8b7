"""End-to-end drop-in pipelines (tiny config) against the oracle pipelines on identical weights,
image and explicit noise; plus the reference's error behaviour at the call surface."""
import numpy as np
import pytest
import torch

from tests.helpers import engine_from_oracle, oracle_models, record, synthetic_image

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup():
    unet, vae, text = oracle_models("tiny")
    eng = engine_from_oracle(unet, vae, text)
    yield unet, vae, text, eng
    eng.close()


def _noise(E, lh, lw, n, seed=2024):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(E, 4, lh, lw, generator=g), torch.randn(max(n - 1, 1), E, 4, lh, lw, generator=g)


def test_depth_pipeline_single_member_matches_oracle(setup):
    from marigold_b200.pipeline import MarigoldDepthPipeline
    from marigold_b200.schedulers import DDIMScheduler
    from oracle.pipeline import OracleDepthPipeline
    from oracle.schedulers import DDIMSchedulerOracle

    unet, vae, text, eng = setup
    img = synthetic_image(128)
    z0, _ = _noise(1, 16, 16, 4)
    pipe = MarigoldDepthPipeline(eng, DDIMScheduler(), text, default_denoising_steps=4,
                                 default_processing_resolution=128)
    out = pipe(img, ensemble_size=1, noise=z0, show_progress_bar=False)
    ora = OracleDepthPipeline(unet, vae, DDIMSchedulerOracle(), text, 4, 128)
    ref, _, _ = ora(img, ensemble_size=1, noise=z0)
    assert out.depth_np.shape == (128, 128) and out.uncertainty is None and out.depth_colored is not None
    # bf16 operand tolerance for a 4-step trajectory + decoder (the map lives in [0,1])
    assert record("tiny/pipe_depth_max", np.abs(out.depth_np - ref).max()) < 1.5e-2      # measured 8.2e-3 (H100)
    assert record("tiny/pipe_depth_mean", np.abs(out.depth_np - ref).mean()) < 2e-3   # measured 8.6e-4 (H100)
    # run-to-run reproducibility: every kernel sums in a fixed order (no data atomics anywhere on the path)
    out2 = pipe(img, ensemble_size=1, noise=z0, show_progress_bar=False)
    np.testing.assert_array_equal(out.depth_np, out2.depth_np)


def test_depth_pipeline_ensemble_and_resize(setup):
    from marigold_b200.pipeline import MarigoldDepthPipeline
    from marigold_b200.schedulers import DDIMScheduler
    from oracle.pipeline import OracleDepthPipeline
    from oracle.schedulers import DDIMSchedulerOracle

    unet, vae, text, eng = setup
    img = synthetic_image(256)[:, :, :128, :]                    # 128 x 256 input -> processed at 64 x 128
    z0, _ = _noise(3, 8, 16, 2)
    pipe = MarigoldDepthPipeline(eng, DDIMScheduler(), text, default_denoising_steps=2,
                                 default_processing_resolution=128)
    # processing_res=100 -> 50 x 100 pixels -> 6 x 12 latents -> 48 x 96 decoded, resized back to the input size:
    # sizes that are not multiples of 64 run like in the reference (image_util.py:90-120, VAE floor semantics)
    z1 = torch.randn(1, 4, 6, 12, generator=torch.Generator().manual_seed(5))
    odd = pipe(img, ensemble_size=1, noise=z1, processing_res=100, show_progress_bar=False)
    ora100 = OracleDepthPipeline(unet, vae, DDIMSchedulerOracle(), text, 2, 100)
    ref100, _, _ = ora100(img, ensemble_size=1, noise=z1)
    assert odd.depth_np.shape == ref100.shape == (128, 256)
    assert record("tiny/pipe_depth_50x100_max", np.abs(odd.depth_np - ref100).max()) < 1.5e-2   # measured 8.2e-3 (H100)
    out = pipe(img, ensemble_size=3, noise=z0, batch_size=2, show_progress_bar=False,
               ensemble_kwargs=dict(output_uncertainty=True))
    ora = OracleDepthPipeline(unet, vae, DDIMSchedulerOracle(), text, 2, 128)
    ref, unc, ref_members = ora(img, ensemble_size=3, noise=z0, batch_size=2,
                                ensemble_kwargs=dict(output_uncertainty=True))
    assert out.depth_np.shape == (128, 256)
    assert out.uncertainty.shape == (64, 128)      # like the reference, the uncertainty map is NOT resized back (:317-318)
    assert out.depth_np.min() >= 0 and out.depth_np.max() <= 1
    # per-member predictions (before the ensemble) agree with the oracle at bf16-operand tolerance ...
    rgb_norm, _ = pipe._preprocess(img, 128, "bilinear")
    members = pipe._infer_members(rgb_norm, 3, 2, 2, None, z0, None, 0)
    assert members.shape == ref_members.shape == (3, 1, 64, 128)
    assert record("tiny/pipe_members_max", (members.cpu() - ref_members).abs().max()) < 2e-2   # measured 1.3e-2 (H100)
    # ... and the ensemble of IDENTICAL members matches the oracle's ensemble when given the same alignment
    # (the BFGS trajectory itself is rounding-chaotic on such near-flat random-weight maps; test_ensemble_gpu)
    from marigold_b200.ensemble import ensemble_depth
    from oracle.ensemble import ensemble_depth as oracle_ensemble

    o_pred, _, o_param = oracle_ensemble(ref_members, return_param=True)
    m_pred, _ = ensemble_depth(ref_members.cuda(), param=o_param, engine=eng)
    assert (m_pred.cpu() - o_pred).abs().max() < 5e-6


def test_depth_pipeline_lcm(setup):
    from marigold_b200.pipeline import MarigoldDepthPipeline
    from marigold_b200.schedulers import LCMScheduler
    from oracle.pipeline import OracleDepthPipeline
    from oracle.schedulers import LCMSchedulerOracle

    unet, vae, text, eng = setup
    img = synthetic_image(128)
    z0, zs = _noise(2, 16, 16, 4)
    pipe = MarigoldDepthPipeline(eng, LCMScheduler(), text, default_denoising_steps=4,
                                 default_processing_resolution=128)
    out = pipe(img, ensemble_size=1, noise=z0[:1], step_noise=zs[:, :1], show_progress_bar=False)
    ora = OracleDepthPipeline(unet, vae, LCMSchedulerOracle(), text, 4, 128)
    ref, _, _ = ora(img, ensemble_size=1, noise=z0[:1], step_noise=zs[:, :1])
    assert record("tiny/pipe_lcm_max", np.abs(out.depth_np - ref).max()) < 2e-2   # measured 1.4e-2 (H100)


def test_normals_pipeline_and_errors(setup):
    from marigold_b200.pipeline import MarigoldNormalsPipeline
    from marigold_b200.schedulers import DDIMScheduler, LCMScheduler
    from oracle.pipeline import OracleNormalsPipeline
    from oracle.schedulers import DDIMSchedulerOracle

    unet, vae, text, eng = setup
    img = synthetic_image(128)
    z0, _ = _noise(4, 16, 16, 2)
    pipe = MarigoldNormalsPipeline(eng, DDIMScheduler(), text, default_denoising_steps=2,
                                   default_processing_resolution=128)
    out = pipe(img, ensemble_size=4, noise=z0, show_progress_bar=False)
    ora = OracleNormalsPipeline(unet, vae, DDIMSchedulerOracle(), text, 2, 128)
    ref, _, _ = ora(img, ensemble_size=4, noise=z0)
    assert out.normals_np.shape == (3, 128, 128)
    strong = np.linalg.norm(ref, axis=0) > 0.5
    cos = (out.normals_np * ref).sum(0)[strong]
    assert np.median(cos) > 0.99
    # (the ensembled map can legitimately differ at single pixels: "closest" picks ONE member per pixel and two
    # near-equidistant members swap under bf16 noise.) Channel order and sign are checked on every strong pixel of every
    # MEMBER, before the ensemble:
    rgb_norm, _ = pipe._preprocess(img, 128, "bilinear")
    members = pipe._infer_members(rgb_norm, 4, 2, 0, None, z0, None, 1).cpu().numpy()
    _, _, ref_members = ora(img, ensemble_size=4, noise=z0)
    ref_members = ref_members.numpy()
    # (unit vectors: where the raw decoder output is short the direction is ill-conditioned, so single pixels may differ;
    # a swapped channel or a flipped sign would move the whole distribution)
    cos_m = (members * ref_members).sum(1).reshape(-1)
    assert record("tiny/pipe_normals_members_frac_cos98", float(np.mean(cos_m > 0.98))) > 0.99
    assert np.median(cos_m) > 0.999
    with pytest.raises(RuntimeError):
        MarigoldNormalsPipeline(eng, LCMScheduler(), text, 2, 128)(img, noise=z0[:1])
    with pytest.raises(TypeError):
        pipe("not an image")
    with pytest.raises(AssertionError):
        pipe(torch.zeros(3, 64, 64))
