"""SD-2-size parity at the benchmarked resolutions (`-m gpu`): every stage of the hot path — VAE encode, one
UNet + DDIM step (first and mid-schedule), VAE decode with the depth and the normals head — at 768 x 768,
1024 x 1024 and a non-square 768 x 576, on seeded random weights of the real architecture, through the C ABI.

Two references on the same weights and inputs (reference call sites marigold_depth_pipeline.py:461-463,491-495,510-515):
  * the fp32 oracle graph (oracle/unet.py, oracle/vae.py) run by torch on the GPU with TF32 disabled (checked
    against the CPU oracle on the tiny model below) — the parity target;
  * the SAME graph run under torch bf16 (cuDNN / cuBLAS / SDPA), i.e. what the reference pipeline computes with
    torch_dtype=bfloat16 — the yardstick: bf16 operands cannot reach fp32's 1e-3, so the assertion that ties the
    product to the reference is   err(ours vs fp32) <= err(torch-bf16 vs fp32) * 1.05 + 1e-3   per stage.
Both errors are recorded in $MGB_PARITY_DIR/fullsize_parity.json when that variable names a directory."""
import json
import os
from pathlib import Path

import pytest
import torch

from tests.helpers import engine_from_oracle, oracle_models, rel_err, synthetic_image

pytestmark = pytest.mark.gpu
RECORD = {}


def _record(key, ours, yard):
    RECORD[key] = {"ours_vs_fp32": ours, "torch_bf16_vs_fp32": yard}
    if os.environ.get("MGB_PARITY_DIR"):
        out = Path(os.environ["MGB_PARITY_DIR"])
        out.mkdir(parents=True, exist_ok=True)
        (out / "fullsize_parity.json").write_text(json.dumps(RECORD, indent=1))


def _check(key, ours, ref, yard):
    e_ours, e_yard = rel_err(ours, ref), rel_err(yard, ref)
    _record(key, e_ours, e_yard)
    assert torch.isfinite(ours).all()
    assert e_ours <= e_yard * 1.05 + 1e-3, f"{key}: ours {e_ours:.3e} vs torch-bf16 {e_yard:.3e}"
    return e_ours, e_yard


@pytest.fixture(scope="module")
def full():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    unet, vae, text = oracle_models("full")
    eng = engine_from_oracle(unet, vae, text)
    dev = torch.device("cuda")
    ref = {"unet": unet.to(dev), "vae": vae.to(dev), "text": text.to(dev)}
    import copy

    yard = {"unet": copy.deepcopy(ref["unet"]).to(torch.bfloat16), "vae": copy.deepcopy(ref["vae"]).to(torch.bfloat16),
            "text": ref["text"].to(torch.bfloat16)}
    yield eng, ref, yard
    eng.close()


def _image(h, w, seed=1234):
    s = max(h, w)
    return (synthetic_image(s, seed=seed)[..., :h, :w].float() / 255.0 * 2.0 - 1.0).cuda()


def _encode_refs(ref, yard, img):
    with torch.no_grad():
        r = ref["vae"].quant_conv(ref["vae"].encoder(img))[:, :4] * 0.18215
        y = (yard["vae"].quant_conv(yard["vae"].encoder(img.to(torch.bfloat16)))[:, :4] * 0.18215).float()
    return r, y


# 768 x 432: a 16:9 photo at processing_res 768 (54 x 96 latents: odd level sizes 27 x 48, 14 x 24, 7 x 12)
@pytest.mark.parametrize("h,w", [(768, 768), (1024, 1024), (768, 576), (432, 768)])
def test_stages_match_oracle_within_the_bf16_yardstick(full, h, w):
    from marigold_b200.schedulers import DDIMScheduler

    eng, ref, yard = full
    tag = f"{h}x{w}"
    img = _image(h, w)
    # ---- encode (two different images back to back: a stale-operand race in the VAE attention GEMMs would show)
    eng.encode(_image(h, w, seed=99))
    lat = eng.encode(img)
    r_lat, y_lat = _encode_refs(ref, yard, img)
    _check(f"{tag}/encode", lat, r_lat, y_lat)

    # ---- UNet + DDIM step, first and mid-schedule
    s = DDIMScheduler()
    s.set_timesteps(10)
    kx, kv, kz = s.coefficients()
    eng.set_schedule(s.timesteps, kx, kv, kz)
    g = torch.Generator().manual_seed(2024)
    x0 = torch.randn(1, 4, h // 8, w // 8, generator=g).cuda()
    for step in (0, 5):
        t = int(s.timesteps[step])
        x = x0.clone()
        mo = eng.unet_step(r_lat, x, step, want_model_out=True)
        with torch.no_grad():
            inp = torch.cat([r_lat, x0], 1)
            r_v = ref["unet"](inp, t, ref["text"])
            y_v = yard["unet"](inp.to(torch.bfloat16), t, yard["text"]).float()
        _check(f"{tag}/unet_step{step}", mo, r_v, y_v)
        # the fused scheduler epilogue is fp32-exact on the product's own model output
        upd = float(kx[step]) * x0 + float(kv[step]) * mo
        assert rel_err(x, upd) < 1e-5

    # ---- decode, depth and normals heads, from the image's own latent
    with torch.no_grad():
        r_dec = ref["vae"].decoder(ref["vae"].post_quant_conv(r_lat / 0.18215))
        y_dec = yard["vae"].decoder(yard["vae"].post_quant_conv((r_lat / 0.18215).to(torch.bfloat16))).float()
    dep = eng.decode(r_lat, 0)
    _check(f"{tag}/decode_depth", dep, (r_dec.mean(1, keepdim=True).clip(-1, 1) + 1) / 2,
           (y_dec.mean(1, keepdim=True).clip(-1, 1) + 1) / 2)
    if (h, w) == (768, 768):
        nrm = eng.decode(r_lat, 1)

        def head(v):
            c = v.clip(-1, 1)
            return c / torch.norm(c, dim=1, keepdim=True).clamp(min=1e-6)

        r_n, y_n = head(r_dec), head(y_dec)
        # unit vectors: compare where the raw prediction is not near zero (normalisation amplifies there)
        strong = (torch.norm(r_dec.clip(-1, 1), dim=1, keepdim=True) > 0.1).expand_as(r_n)
        e_ours = float((nrm - r_n).abs()[strong].max())
        e_yard = float((y_n - r_n).abs()[strong].max())
        _record(f"{tag}/decode_normals", e_ours, e_yard)
        assert e_ours <= e_yard * 1.05 + 1e-3
        assert torch.allclose(torch.norm(nrm, dim=1), torch.ones_like(nrm[:, 0]), atol=1e-5)


def test_full_size_denoising_is_bit_reproducible(full):
    """Two runs of the same 3-step 768 x 768 denoising loop (eager first step, then CUDA-graph replays) give identical
    bits: GroupNorm statistics, split-K and split-KV merges all sum in a fixed order."""
    from marigold_b200.schedulers import DDIMScheduler

    eng, ref, yard = full
    s = DDIMScheduler()
    s.set_timesteps(3)
    eng.set_schedule(s.timesteps, *s.coefficients())
    g = torch.Generator().manual_seed(7)
    rgb = torch.randn(1, 4, 96, 96, generator=g).cuda()
    x0 = torch.randn(1, 4, 96, 96, generator=g).cuda()
    a = eng.denoise(rgb, x0)
    b = eng.denoise(rgb, x0)
    torch.cuda.synchronize()
    assert torch.isfinite(a).all() and torch.equal(a, b)
    d1, d2 = eng.decode(a, 0), eng.decode(a, 0)
    assert torch.equal(d1, d2)


def test_gpu_fp32_oracle_equals_cpu_oracle_on_the_tiny_model():
    """The full-size target above is the oracle graph evaluated by torch on the GPU; pin that evaluation to the CPU
    oracle (the one the golden vectors freeze) where the CPU finishes in seconds."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    unet, vae, text = oracle_models("tiny")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 8, 16, 24, generator=g)
    img = torch.rand(1, 3, 64, 128, generator=g) * 2 - 1
    with torch.no_grad():
        a = unet(x, 499, text)
        b = vae.decoder(vae.post_quant_conv(vae.quant_conv(vae.encoder(img))[:, :4]))
        import copy

        ug, vg = copy.deepcopy(unet).cuda(), copy.deepcopy(vae).cuda()
        a2 = ug(x.cuda(), 499, text.cuda())
        b2 = vg.decoder(vg.post_quant_conv(vg.quant_conv(vg.encoder(img.cuda()))[:, :4]))
    assert rel_err(a2, a) < 1e-4 and rel_err(b2, b) < 1e-4   # fp32 accumulation order only
