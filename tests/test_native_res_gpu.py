"""Native-resolution inference (`-m gpu`): the VAE mid-block attention in row blocks, 12-megapixel photos end to end.

  * row-block invariance: encode and decode on the SD-size VAE (random weights) give the same bits whatever the number
    of query rows per block (mgb_debug_vae_attn_blocks forces it), at latents of 96 x 96, 77 x 131 (T not a multiple
    of 64) and 128 x 128, for one and two images; every size up to 1024 x 1024 runs as one block;
  * the pipelines at processing_res=0 on a 4032 x 3024 photo, and the refusal of an input one member cannot fit,
    before anything is allocated or launched. One phone photo's member needs 76.5 GB of workspace: these run before
    the torch graphs below, whose libraries keep device memory for the rest of the process;
  * parity at 4000 x 3000: encode, then decode the 500 x 375 latent with the depth, normals and one-IID-target heads,
    against the fp32 oracle run by torch on the GPU with TF32 off, with the bf16 yardstick of test_fullsize_gpu.py. Its
    mid-block attention is evaluated in row blocks (_blocked_attention): SDPA cannot hold the T x T scores here."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from tests.helpers import engine_from_oracle, oracle_models, rel_err, synthetic_image

pytestmark = pytest.mark.gpu


def _hook(name, res, args):
    from marigold_b200 import _lib

    f = getattr(_lib.load(), name)        # debug hooks outside the public header
    f.restype, f.argtypes = res, args
    return f


def attn_blocks(eng, NB, T, budget=0, force_rows=0):
    """(rows per block, blocks over the NB images) of an (NB, T) VAE attention; sets the handle's budget and forced rows
    (0: the library's)."""
    from marigold_b200._lib import check

    f = _hook("mgb_debug_vae_attn_blocks", C.c_int32,
              [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)])
    r, b = C.c_int32(), C.c_int32()
    check(f(eng._h, budget, force_rows, NB, T, C.byref(r), C.byref(b)), "mgb_debug_vae_attn_blocks")
    return r.value, b.value


@pytest.fixture(scope="module")
def models():
    return oracle_models("full")


@pytest.fixture
def engine(models):
    eng = engine_from_oracle(*models)
    yield eng
    eng.close()


def test_one_block_up_to_1024(engine):
    for lh, lw in ((96, 96), (128, 128), (96, 128), (128, 72)):
        for NB in (1, 2):
            assert attn_blocks(engine, NB, lh * lw) == (lh * lw, NB), (lh, lw, NB)
    # 1920 x 1080 (T = 32 400) is past the budget: blocks of a multiple of 128 rows
    R, n = attn_blocks(engine, 1, 240 * 135)
    assert R % 128 == 0 and n == -(-32400 // R) and n > 1


@pytest.mark.parametrize("NB", [1, 2])
@pytest.mark.parametrize("lh,lw", [(96, 96), (77, 131), (128, 128)])
def test_row_blocks_are_bit_identical(engine, lh, lw, NB):
    T = lh * lw
    g = torch.Generator().manual_seed(1000 * lh + lw + NB)
    img = (torch.rand(NB, 3, 8 * lh, 8 * lw, generator=g) * 2 - 1).cuda()
    lat = torch.randn(NB, 4, lh, lw, generator=g).cuda()
    assert attn_blocks(engine, NB, T) == (T, NB)
    enc, dec = engine.encode(img), engine.decode(lat, 2)
    # forced block heights (one ragged tail: T - 64 rows, then 64), and the budget path at a 1-byte budget, which leaves
    # only the one-wave floor of the P V GEMM
    for force, budget in ((128, 0), (640, 0), (T - 64, 0), (0, 1)):
        R, n = attn_blocks(engine, NB, T, budget=budget, force_rows=force)
        assert R == (force or R) and n == NB * -(-T // R) and (force or R % 128 == 0)
        assert torch.equal(engine.encode(img), enc), (force, budget)
        assert torch.equal(engine.decode(lat, 2), dec), (force, budget)
    attn_blocks(engine, NB, T)


# ---- pipelines at processing_res = 0 -----------------------------------------------------------------------------
def _photo(h, w, seed=3):
    return synthetic_image(max(h, w), seed=seed)[..., :h, :w].contiguous()


def test_depth_and_normals_at_native_resolution(models, engine):
    from marigold_b200.pipeline import MarigoldDepthPipeline, MarigoldNormalsPipeline, select_batch_size
    from marigold_b200.schedulers import DDIMScheduler

    text = models[2]
    H, W = 3024, 4032
    img = _photo(H, W)
    bs = select_batch_size(engine, 10, H, W)
    assert 1 <= bs <= 8
    assert engine.workspace_bytes(bs, H, W) <= torch.cuda.mem_get_info()[0] + engine.held_bytes()
    pipe = MarigoldDepthPipeline(engine, DDIMScheduler(), text, default_denoising_steps=1, default_processing_resolution=0)
    out = pipe(img, ensemble_size=10, generator=torch.Generator(device="cuda").manual_seed(0), color_map=None,
               show_progress_bar=False, ensemble_kwargs={"output_uncertainty": True})
    assert out.depth_np.shape == (H, W) and np.isfinite(out.depth_np).all()
    assert out.uncertainty is not None and out.uncertainty.shape == (H, W) and np.isfinite(out.uncertainty).all()
    npipe = MarigoldNormalsPipeline(engine, DDIMScheduler(), text, default_denoising_steps=1,
                                    default_processing_resolution=0)
    nout = npipe(img, ensemble_size=2, generator=torch.Generator(device="cuda").manual_seed(0), show_progress_bar=False,
                 ensemble_kwargs={"output_uncertainty": True})
    assert nout.normals_np.shape == (3, H, W) and np.isfinite(nout.normals_np).all()
    assert nout.uncertainty is not None


def test_iid_at_native_resolution():
    from marigold_b200.engine import Engine, EngineConfig
    from marigold_b200.pipeline import MarigoldIIDPipeline
    from marigold_b200.schedulers import DDIMScheduler
    from oracle.unet import UNet2DConditionOracle, UNetConfig
    from oracle.vae import AutoencoderKLOracle, VAEConfig

    torch.manual_seed(4)
    ucfg = UNetConfig()
    ucfg.in_channels, ucfg.out_channels = 12, 8
    unet, vae = UNet2DConditionOracle(ucfg).eval(), AutoencoderKLOracle(VAEConfig()).eval()
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=torch.Generator().manual_seed(7))
    eng = Engine(EngineConfig(unet_in_channels=12, unet_out_channels=8))
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    names = ["albedo", "shading"]
    props = {"target_names": names, "albedo": {"prediction_space": "srgb"},
             "shading": {"prediction_space": "linear", "up_to_scale": True}}
    H, W = 3024, 4032
    pipe = MarigoldIIDPipeline(eng, DDIMScheduler(), text, target_properties=props, default_denoising_steps=1,
                               default_processing_resolution=0)
    out = pipe(_photo(H, W), ensemble_size=2, generator=torch.Generator(device="cuda").manual_seed(0),
               show_progress_bar=False, ensemble_kwargs={"output_uncertainty": True})
    assert out.is_complete
    for name in names:
        assert out[name].array.shape == (3, H, W) and np.isfinite(out[name].array).all()
        assert out[name].uncertainty is not None
    eng.close()


def test_too_large_for_one_member_is_refused_before_any_work(models, engine):
    from marigold_b200.pipeline import MarigoldDepthPipeline
    from marigold_b200.schedulers import DDIMScheduler

    live = _hook("mgb_debug_live_device_bytes", C.c_int64, [])
    lib = engine.lib
    pipe = MarigoldDepthPipeline(engine, DDIMScheduler(), models[2], default_denoising_steps=1,
                                 default_processing_resolution=0)
    torch.cuda.synchronize()
    b0, l0, t0 = live(), lib.mgb_launch_count(), torch.cuda.memory_allocated()
    big = torch.zeros(1, 3, 8192, 8192, dtype=torch.uint8)          # the supported maximum; it cannot fit a card
    with pytest.raises(ValueError, match=r"needs \d+ bytes of device workspace, but \d+ bytes are available"):
        pipe(big, ensemble_size=1, show_progress_bar=False)
    with pytest.raises(ValueError, match="supported maximum"):
        pipe(torch.zeros(1, 3, 8192, 8200, dtype=torch.uint8), ensemble_size=1, show_progress_bar=False)
    assert (live(), lib.mgb_launch_count(), torch.cuda.memory_allocated()) == (b0, l0, t0)
    # the C ABI refuses a batch past the maximum before it reads an argument's memory or launches
    x = torch.zeros(16, device="cuda")
    assert lib.mgb_encode(engine._h, C.c_void_p(x.data_ptr()), 2, 8192, 8192, C.c_void_p(x.data_ptr()), None) == -5
    assert lib.mgb_decode(engine._h, C.c_void_p(x.data_ptr()), 2, 1024, 1024, 0, C.c_void_p(x.data_ptr()), None) == -5
    assert engine.workspace_bytes(2, 8192, 8192) == 0
    assert (live(), lib.mgb_launch_count()) == (b0, l0)


# ---- 12 MP parity ------------------------------------------------------------------------------------------------
def _blocked_attention(self, x, rows=4096):
    """oracle VAEAttention.forward with the queries in blocks of `rows`: fp32 scores and softmax on the block, then P V
    in the module's dtype (for bf16, SDPA's flash arithmetic: unrounded fp32 logits, bf16 probabilities)."""
    B, Cc, H, W = x.shape
    h = self.group_norm(x).reshape(B, Cc, H * W).transpose(1, 2)
    q, k, v = self.to_q(h), self.to_k(h), self.to_v(h)
    kt = k.float().transpose(1, 2)
    o = torch.empty_like(q)
    for r0 in range(0, H * W, rows):
        s = torch.matmul(q[:, r0:r0 + rows].float(), kt) * (Cc ** -0.5)
        o[:, r0:r0 + rows] = torch.matmul(torch.softmax(s, dim=-1).to(q.dtype), v)
        del s
    return x + self.to_out[0](o).transpose(1, 2).reshape(B, Cc, H, W)


def _blocked(vae):
    from oracle.vae import VAEAttention

    for m in vae.modules():
        if isinstance(m, VAEAttention):
            m.forward = types.MethodType(_blocked_attention, m)
    return vae


def _heads(raw):
    c = raw.clip(-1, 1)
    return {"depth": (raw.mean(1, keepdim=True).clip(-1, 1) + 1) / 2,
            "normals": c / torch.norm(c, dim=1, keepdim=True).clamp(min=1e-6), "iid": (c + 1) / 2}


def test_12mp_encode_decode_match_oracle(models):
    import copy

    unet, vae, text = models
    H, W = 3000, 4000
    img = (synthetic_image(W)[..., :H, :W].float() / 255.0 * 2.0 - 1.0)
    eng = engine_from_oracle(unet, vae, text)
    lat = eng.encode(img.cuda())
    ours = {"encode": lat.cpu()}
    for name, mode in (("depth", 0), ("normals", 1), ("iid", 3)):
        ours[name] = eng.decode(lat, mode).cpu()
    eng.close()                                  # the torch graphs below need the card to themselves
    torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    refs = {}
    for tag, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        v = _blocked(copy.deepcopy(vae)).cuda().to(dt)
        with torch.no_grad():
            refs[tag, "encode"] = (v.quant_conv(v.encoder(img.cuda().to(dt)))[:, :4] * 0.18215).float().cpu()
            raw = v.decoder(v.post_quant_conv((lat / 0.18215).to(dt))).float()
            for k, t in _heads(raw).items():
                refs[tag, k] = t.cpu()
            del raw, v
        torch.cuda.empty_cache()
    for key in ("encode", "depth", "iid"):
        e_ours, e_yard = rel_err(ours[key], refs["fp32", key]), rel_err(refs["bf16", key], refs["fp32", key])
        assert torch.isfinite(ours[key]).all()
        assert e_ours <= e_yard * 1.05 + 1e-3, f"{key}: ours {e_ours:.3e} vs torch-bf16 {e_yard:.3e}"
    # unit vectors: compared where the raw prediction is not near zero (test_fullsize_gpu.py)
    r = refs["fp32", "normals"]
    strong = (torch.norm(refs["fp32", "iid"] * 2 - 1, dim=1, keepdim=True) > 0.1).expand_as(r)
    e_ours = float((ours["normals"] - r).abs()[strong].max())
    e_yard = float((refs["bf16", "normals"] - r).abs()[strong].max())
    assert e_ours <= e_yard * 1.05 + 1e-3, (e_ours, e_yard)
