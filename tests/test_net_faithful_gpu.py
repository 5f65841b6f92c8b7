"""GPU network graphs (through the C ABI) against the float64 restatement that rounds where the kernels round
(tests/net_ref.py, bf16=True), on oracle models whose every norm affine and bias has been redrawn (net_ref.randomise).

The check is element-wise: |ours - ref| <= TAU[stage] * rms(ref), so errors in small-valued regions count. What is left
between the two is fp32 accumulation order, but through a deep network it does not stay small: where the two
accumulations differ, a bf16 rounding can go the other way, and the difference it makes is rounded again downstream, so
the two computations' rounding decisions decorrelate (DESIGN.md section 4). TAU is therefore close to the gap to the fp32
oracle; the randomised weights are what give the tests their power over the loader and the folds. Each case also checks
the fp32 oracle at the tolerances of tests/test_net_gpu.py, which shows that the randomised model stays in the regime
those tests describe."""
import pytest
import torch

from tests import net_ref as N
from tests.helpers import engine_from_oracle, oracle_models, record, rel_err

pytestmark = pytest.mark.gpu


def _check(fails, name, stage, out, ref, mask=None):
    """|ours - ref| <= TAU[stage] rms(ref) at every element (of `mask`); records max |ours - ref| / rms(ref) and appends
    a message to `fails` when the bound is exceeded (every value of a test is recorded before it fails)."""
    out, ref = out.detach().cpu().to(torch.float64), ref.detach().cpu().to(torch.float64)
    d = (out - ref).abs().nan_to_num(float("inf"))
    if mask is not None:
        d = d[mask]
    e = record(f"faithful/{name}", float(d.max().item()) / N.rms(ref))
    if not e <= N.TAU[stage]:
        fails.append(f"{name}: max |ours - ref| / rms(ref) = {e:.3g} > {N.TAU[stage]:.3g}")


def _oracle_gap(fails, name, out, oracle, tol):
    record(f"oracle_rms/{name}", N.rms_err(out, oracle))
    e = record(f"oracle/{name}", rel_err(out, oracle))
    if not e < tol:
        fails.append(f"{name}: rel err to the fp32 oracle {e:.3g} >= {tol}")


@pytest.fixture(scope="module")
def tiny():
    unet, vae, text = oracle_models("tiny")
    N.randomise(unet, vae, seed=1)
    eng = engine_from_oracle(unet, vae, text)
    yield unet, vae, text, eng
    eng.close()


def _ddim(n):
    from marigold_b200.schedulers import DDIMScheduler

    s = DDIMScheduler()
    s.set_timesteps(n)
    return s


def _steps(name, unet, text, eng, B, lh, lw, seed=11, steps=(0, 2)):
    fails = []
    s = _ddim(4)
    kx, kv, kz = s.coefficients()
    eng.set_schedule(s.timesteps, kx, kv, kz)
    g = torch.Generator().manual_seed(seed)
    ct = unet.cfg.out_channels
    rgb = torch.randn(B, 4, lh, lw, generator=g)
    x = torch.randn(B, ct, lh, lw, generator=g)
    for step in steps:
        t = int(s.timesteps[step])
        mo_ref, x_ref = N.unet_step(unet, text, rgb, x, t, kx[step], kv[step])
        tgt = x.cuda().clone()
        out = eng.unet_step(rgb.cuda(), tgt, step, want_model_out=True)
        torch.cuda.synchronize()
        _check(fails, f"{name}/step{step}/model_out", "unet", out, mo_ref)
        _check(fails, f"{name}/step{step}/latent", "latent", tgt, x_ref)
        with torch.no_grad():
            ora = unet(torch.cat([rgb, x], 1), t, text.repeat(B, 1, 1))
        _oracle_gap(fails, f"{name}/step{step}", out, ora, 1.6e-2)
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("B,lh,lw", [(1, 16, 16), (2, 8, 24), (1, 27, 12), (2, 7, 9)])
def test_unet_step_faithful(tiny, B, lh, lw):
    unet, vae, text, eng = tiny
    _steps(f"tiny/unet_B{B}_{lh}x{lw}", unet, text, eng, B, lh, lw)


@pytest.mark.parametrize("n_targets", [2, 3])
def test_unet_step_iid_faithful(n_targets):
    """The IID configurations: in 4 (n + 1), out 4 n channels (the scheduler epilogue's 8- and 12-column rows)."""
    from marigold_b200.engine import Engine, EngineConfig
    from oracle.unet import UNet2DConditionOracle, UNetConfig
    from oracle.vae import AutoencoderKLOracle, VAEConfig

    torch.manual_seed(0)
    ucfg = UNetConfig.tiny()
    ucfg.in_channels, ucfg.out_channels = 4 * (n_targets + 1), 4 * n_targets
    unet, vae = UNet2DConditionOracle(ucfg).eval(), AutoencoderKLOracle(VAEConfig.tiny()).eval()
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=torch.Generator().manual_seed(7))
    N.randomise(unet, vae, seed=2)
    eng = Engine(EngineConfig(unet_in_channels=ucfg.in_channels, unet_out_channels=ucfg.out_channels,
                              unet_block_channels=list(ucfg.block_out_channels), unet_cross_dim=ucfg.cross_attention_dim,
                              vae_block_channels=list(vae.cfg.block_out_channels)))
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    eng.set_text_embedding(text)
    try:
        _steps(f"tiny/iid{n_targets}", unet, text, eng, 1, 16, 12)
    finally:
        eng.close()


@pytest.mark.parametrize("B,H,W", [(2, 64, 128), (1, 100, 50), (1, 77, 131)])
def test_vae_encode_faithful(tiny, B, H, W):
    unet, vae, text, eng = tiny
    rgb = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(12)) * 2 - 1
    out = eng.encode(rgb.cuda())
    torch.cuda.synchronize()
    fails = []
    _check(fails, f"tiny/encode_{H}x{W}", "encode", out, N.encode(vae, rgb))
    with torch.no_grad():
        ora = vae.quant_conv(vae.encoder(rgb))[:, :4] * 0.18215
    _oracle_gap(fails, f"tiny/encode_{H}x{W}", out, ora, 2e-2)
    assert not fails, "\n".join(fails)


def _decode_case(fails, name, vae, eng, lat, mode):
    out = eng.decode(lat.cuda(), mode)
    torch.cuda.synchronize()
    raw = N.decode(vae, lat, N.DECODE_RAW)
    ref = N.decode_head(raw, mode)
    mask = None
    if mode == N.DECODE_NORMALS:
        # unit normalisation amplifies every error by 1 / |clip(raw)|: compare where the vector is not short, and
        # require unit length everywhere
        o = out.cpu().double()
        assert torch.allclose(torch.norm(o, dim=1), torch.ones_like(o[:, 0]), atol=1e-4)
        mask = (torch.norm(raw.clip(-1, 1), dim=1, keepdim=True) > 0.3).expand_as(ref)
    _check(fails, name, "decode", out, ref, mask)
    return out


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_vae_decode_faithful(tiny, mode):
    unet, vae, text, eng = tiny
    g = torch.Generator().manual_seed(13)
    lat = torch.randn(2, 4, 9, 13, generator=g) if mode in (0, 3) else torch.randn(2, 4, 8, 16, generator=g)
    fails = []
    out = _decode_case(fails, f"tiny/decode_mode{mode}", vae, eng, lat, mode)
    if mode != N.DECODE_NORMALS:
        with torch.no_grad():
            ora = N.decode_head(vae.decoder(vae.post_quant_conv(lat / 0.18215)).double(), mode)
        _oracle_gap(fails, f"tiny/decode_mode{mode}", out, ora, 2e-2)
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("kind", ["ddim", "lcm"])
def test_denoise_trajectory_faithful(tiny, kind):
    """Four steps through mgb_denoise, which captures one step as a CUDA graph and replays it with the step index read
    from the device counter: a wrong step selection changes the bias table and the scheduler coefficients."""
    from marigold_b200.schedulers import LCMScheduler
    from oracle.schedulers import DDIMSchedulerOracle, LCMSchedulerOracle

    unet, vae, text, eng = tiny
    g = torch.Generator().manual_seed(14)
    B, lh, lw, n = 2, 16, 16, 4
    rgb = torch.randn(B, 4, lh, lw, generator=g)
    x0 = torch.randn(B, 4, lh, lw, generator=g)
    zs = torch.randn(n - 1, B, 4, lh, lw, generator=g)
    if kind == "ddim":
        s, o = _ddim(n), DDIMSchedulerOracle()
    else:
        s, o = LCMScheduler(), LCMSchedulerOracle()
        s.set_timesteps(n)
    o.set_timesteps(n)
    kx, kv, kz = s.coefficients()
    eng.set_schedule(s.timesteps, kx, kv, kz)
    x, xo = x0.double(), x0.clone()
    for i, t in enumerate(s.timesteps):
        z = zs[i] if i < n - 1 else None
        _, x = N.unet_step(unet, text, rgb, x, int(t), kx[i], kv[i], kz[i], z)
        x = x.float().double()                      # the product keeps the latent in fp32 between steps
        with torch.no_grad():
            v = unet(torch.cat([rgb, xo], 1), int(t), text.repeat(B, 1, 1))
            xo = o.step(v, int(t), xo, noise=zs[i] if (kind == "lcm" and i < n - 1) else None)
    out = eng.denoise(rgb.cuda(), x0.cuda(), zs.cuda() if kind == "lcm" else None)
    torch.cuda.synchronize()
    fails = []
    _check(fails, f"tiny/trajectory_{kind}", "trajectory", out, x)
    _oracle_gap(fails, f"tiny/trajectory_{kind}", out, xo, 1e-2)
    assert not fails, "\n".join(fails)


# ---- SD-2 widths: the 20-head C = 1280 cross-attention kernel, split-K on the small levels, GEGLU at N = 5120 ----
@pytest.fixture(scope="module")
def sd2():
    unet, vae, text = oracle_models("full")
    N.randomise(unet, vae, seed=3)
    eng = engine_from_oracle(unet, vae, text)
    yield unet, vae, text, eng
    eng.close()


@pytest.mark.parametrize("lh,lw", [(16, 16), (27, 12)])
def test_sd2_unet_step_faithful(sd2, lh, lw):
    unet, vae, text, eng = sd2
    _steps(f"sd2/unet_{lh}x{lw}", unet, text, eng, 1, lh, lw, steps=(2,))


@pytest.mark.parametrize("H,W", [(64, 64), (72, 40)])
def test_sd2_vae_faithful(sd2, H, W):
    unet, vae, text, eng = sd2
    g = torch.Generator().manual_seed(15)
    rgb = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    out = eng.encode(rgb.cuda())
    torch.cuda.synchronize()
    fails = []
    _check(fails, f"sd2/encode_{H}x{W}", "encode", out, N.encode(vae, rgb))
    lat = torch.randn(1, 4, H // 8, W // 8, generator=g)
    _decode_case(fails, f"sd2/decode_{H}x{W}", vae, eng, lat, N.DECODE_RAW)
    assert not fails, "\n".join(fails)
