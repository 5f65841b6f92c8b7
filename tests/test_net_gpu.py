"""GPU parity of the network graphs (through the C ABI) against the fp32 CPU oracle on identical
seeded weights and inputs. Tolerances are bf16-operand tolerances, stated per test; the tight 1e-3
bar of north_star is checked (and its feasibility reported) in test_pipeline_gpu.py."""
import pytest
import torch

from tests.helpers import engine_from_oracle, oracle_models, record, rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny():
    unet, vae, text = oracle_models("tiny")
    eng = engine_from_oracle(unet, vae, text)
    yield unet, vae, text, eng
    eng.close()


def _ddim(n):
    from marigold_b200.schedulers import DDIMScheduler

    s = DDIMScheduler()
    s.set_timesteps(n)
    return s


# (27, 12), (7, 9): latent sizes that are not multiples of 8 exercise the ceil(s/2) stride-2 convs and the
# skip-sized ("upsample_size") nearest upsampling of diffusers, as a 16:9 photo at processing_res 768 does (54 x 96)
@pytest.mark.parametrize("B,lh,lw", [(1, 16, 16), (2, 8, 24), (1, 27, 12), (2, 7, 9)])
def test_unet_step_matches_oracle(tiny, B, lh, lw):
    unet, vae, text, eng = tiny
    s = _ddim(4)
    kx, kv, kz = s.coefficients()
    eng.set_schedule(s.timesteps, kx, kv, kz)
    g = torch.Generator().manual_seed(11)
    rgb = torch.randn(B, 4, lh, lw, generator=g)
    x = torch.randn(B, 4, lh, lw, generator=g)
    for step in (0, 2):
        with torch.no_grad():
            ref = unet(torch.cat([rgb, x], 1), int(s.timesteps[step]), text.repeat(B, 1, 1))
        tgt = x.cuda().clone()
        out = eng.unet_step(rgb.cuda(), tgt, step, want_model_out=True)
        torch.cuda.synchronize()
        e = record(f"tiny/unet_step{step}/B{B}", rel_err(out, ref))
        assert e < 1.6e-2, f"unet step {step}: rel err {e}"   # bf16 operands through ~60 GEMM layers; measured <= 1.07e-2 (H100)
        upd = kx[step] * x + kv[step] * out.cpu()
        assert rel_err(tgt, upd) < 1e-5                     # fused scheduler epilogue is fp32-exact


@pytest.mark.parametrize("B,H,W", [(2, 64, 128), (1, 100, 50), (1, 77, 131)])
def test_vae_encode_matches_oracle(tiny, B, H, W):
    """Any H x W >= 8 (the reference resizes to max-edge and encodes whatever results, image_util.py:90-120): the
    pad-(0,1,0,1) stride-2 convs give floor(s/2) at every level."""
    unet, vae, text, eng = tiny
    g = torch.Generator().manual_seed(12)
    rgb = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    with torch.no_grad():
        ref = vae.quant_conv(vae.encoder(rgb))[:, :4] * 0.18215
    out = eng.encode(rgb.cuda())
    torch.cuda.synchronize()
    assert out.shape == ref.shape == (B, 4, H // 8, W // 8)
    assert record(f"tiny/encode_{H}x{W}", rel_err(out, ref)) < 2e-2    # measured <= 1.5e-2 (H100)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_vae_decode_matches_oracle(tiny, mode):
    unet, vae, text, eng = tiny
    g = torch.Generator().manual_seed(13)
    lat = torch.randn(2, 4, 8, 16, generator=g) if mode != 0 else torch.randn(2, 4, 9, 13, generator=g)
    with torch.no_grad():
        raw = vae.decoder(vae.post_quant_conv(lat / 0.18215))
    if mode == 0:
        ref = (raw.mean(1, keepdim=True).clip(-1, 1) + 1) / 2
    elif mode == 1:
        c = raw.clip(-1, 1)
        ref = c / torch.norm(c, dim=1, keepdim=True).clamp(min=1e-6)
    else:
        ref = raw
    out = eng.decode(lat.cuda(), mode)
    torch.cuda.synchronize()
    if mode == 1:
        # unit-normalisation is ill-conditioned where the raw vector is short: compare directions where
        # |clip(raw)| > 0.3 (cosine), and only boundedness elsewhere
        o = out.cpu()
        assert torch.allclose(torch.norm(o, dim=1), torch.ones_like(o[:, 0]), atol=1e-4)
        strong = torch.norm(raw.clip(-1, 1), dim=1) > 0.3
        cos = (o * ref).sum(1)[strong]
        assert record("tiny/decode_normals_min_cos", cos.min()) > 0.995, f"min cosine {cos.min()}"
        # channel order and sign everywhere the vector is not tiny: max component error
        strong3 = strong[:, None].expand_as(o)
        assert record("tiny/decode_normals_max_abs", (o - ref).abs()[strong3].max()) < 8e-2   # ~ decode error 1.5e-2 / |raw| 0.3; measured 5.6e-2 (H100)
    else:
        assert record(f"tiny/decode_mode{mode}", rel_err(out, ref)) < 2e-2    # measured <= 1.5e-2 (H100)


def test_denoise_trajectory_ddim_and_lcm(tiny):
    from marigold_b200.schedulers import LCMScheduler
    from oracle.schedulers import DDIMSchedulerOracle, LCMSchedulerOracle

    unet, vae, text, eng = tiny
    g = torch.Generator().manual_seed(14)
    B, lh, lw, n = 2, 16, 16, 4
    rgb = torch.randn(B, 4, lh, lw, generator=g)
    x0 = torch.randn(B, 4, lh, lw, generator=g)
    zs = torch.randn(n - 1, B, 4, lh, lw, generator=g)
    for kind in ("ddim", "lcm"):
        if kind == "ddim":
            s, o = _ddim(n), DDIMSchedulerOracle()
        else:
            s, o = LCMScheduler(), LCMSchedulerOracle()
            s.set_timesteps(n)
        o.set_timesteps(n)
        assert list(map(int, s.timesteps)) == o.timesteps.tolist()
        kx, kv, kz = s.coefficients()
        eng.set_schedule(s.timesteps, kx, kv, kz)
        x = x0.clone()
        with torch.no_grad():
            for i, t in enumerate(o.timesteps):
                v = unet(torch.cat([rgb, x], 1), t, text.repeat(B, 1, 1))
                x = o.step(v, t, x, noise=zs[i] if (kind == "lcm" and i < n - 1) else None)
        out = eng.denoise(rgb.cuda(), x0.cuda(), zs.cuda() if kind == "lcm" else None)
        torch.cuda.synchronize()
        assert record(f"tiny/trajectory_{kind}", rel_err(out, x)) < 1e-2, kind   # measured 4.9e-3 (H100)
