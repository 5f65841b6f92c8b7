"""Native-resolution inference (`-m gpu`): the VAE mid-block attention in row blocks, 12-megapixel photos end to end.

  * row-block invariance: encode and decode on the SD-size VAE (random weights) give the same bits whatever the number
    of query rows per block (mgb_debug_vae_attn_blocks forces it), at latents of 96 x 96, 77 x 131 (T not a multiple
    of 64) and 128 x 128, for one and two images; every size up to 1024 x 1024 runs as one block;
  * the pipelines at processing_res=0 on a 4032 x 3024 photo, and the refusal of an input one member cannot fit,
    before anything is allocated or launched. One phone photo's member needs 76.5 GB of workspace: these run before
    the torch graphs below, whose libraries keep device memory for the rest of the process;
  * parity at 4000 x 3000: encode, then decode the 500 x 375 latent with the depth, normals and one-IID-target heads,
    against the fp32 oracle run by torch on the GPU with TF32 off, with the bf16 yardstick of test_fullsize_gpu.py. Its
    mid-block attention is evaluated in row blocks (_blocked_attention): SDPA cannot hold the T x T scores here;
  * one UNet + DDIM step at the 504 x 378 and 500 x 375 latents of 4032 x 3024 and 4000 x 3000 photos (T = 190 512 and
    187 500 tokens at level 0; the 2H - 1 upsample crops fall on different levels), at steps 0 and 5 of 10, against
    the same fp32 oracle and bf16 yardstick; the fused DDIM update against kx x + kv model_out;
  * the VAE attention's core (score GEMM, row softmax, V^T, P V GEMM, in row blocks: mgb_debug_vae_attn_core) element
    by element against float64 at T = 187 500, 190 512, 2 x 32 400 and 10 087, on four kinds of input, and bit for bit
    across block heights at T = 190 512.

The VAE attention core's bound. The reference is o = softmax(s) v with s = q k^T / sqrt(C) in float64 on the same bf16
q, k, v; only rows are checked whose float64 probabilities fit (check_rows: both end blocks, both sides of every block
boundary, the last 64 rows, 2048 seeded rows). Per element of row i, with p the float64 probabilities, Tp the key count
rounded up to 64 and the constants of tests/ops_ref.py:
    |o~ - o| <= (2^-8 + 2 R_F32_OUT) |o|                      bf16 output, fp32 epilogue
              + C_P 2^-8 sum_j p_j |v_j|                      bf16 P
              + C_ACC Tp 2^-24 sum_j p_j |v_j|                P V fp32 accumulation
              + sum_j p_j |ds_j| (|v_j| + |o|)                the score error through the softmax (|v_j - o| bounded)
              + sum_j p_j softmax_rel(T, m - s_j) |v_j|       the softmax's fp32 exp and row sum (ops_ref.softmax_rel)
    |ds_j| <= C_ACC C 2^-24 |q||k_j| / sqrt(C) + R_F32_OUT |s_j|   the score GEMM's accumulation and epilogue.
softmax_rel's row-sum term grows with T: (ceil(T / 256) + 16) 2^-24, about 2^-14.4 at T = 190 512."""
import ctypes as C
import json
import os
import types
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import ops_ref
from tests.helpers import (VAE_C, _core_inputs, _core_ref, _photo, attn_blocks, attn_core, engine_from_oracle,
                           live_device_bytes, oracle_models, record, rel_err, synthetic_image)
from tests.ops_cases import check_rows

pytestmark = pytest.mark.gpu


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

    live = live_device_bytes
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


# ---- the UNet step at native resolution --------------------------------------------------------------------------
PARITY = {}


def _record_parity(key, ours, yard):
    PARITY[key] = {"ours_vs_fp32": ours, "torch_bf16_vs_fp32": yard}
    if os.environ.get("MGB_PARITY_DIR"):
        out = Path(os.environ["MGB_PARITY_DIR"])
        out.mkdir(parents=True, exist_ok=True)
        (out / "native_res_parity.json").write_text(json.dumps(PARITY, indent=1))


def test_unet_step_at_native_resolution_matches_oracle(models):
    """One UNet + DDIM step at steps 0 and 5 of a 10-step schedule on the latents of 4032 x 3024 and 4000 x 3000
    photos, within test_fullsize_gpu.py's bf16 yardstick of the fp32 oracle. The engine runs first and is closed before
    the torch graphs, which keep device memory for the rest of the process."""
    import copy

    from marigold_b200.schedulers import DDIMScheduler

    unet, vae, text = models
    s = DDIMScheduler()
    s.set_timesteps(10)
    kx, kv, kz = s.coefficients()
    eng = engine_from_oracle(unet, vae, text)
    eng.set_schedule(s.timesteps, kx, kv, kz)
    inputs, ours = {}, {}
    for lh, lw in ((378, 504), (375, 500)):
        g = torch.Generator().manual_seed(lh * lw)
        rgb, x0 = torch.randn(1, 4, lh, lw, generator=g), torch.randn(1, 4, lh, lw, generator=g)
        inputs[lh, lw] = rgb, x0
        for step in (0, 5):
            x = x0.cuda()
            mo = eng.unet_step(rgb.cuda(), x, step, want_model_out=True)
            # the fused scheduler epilogue is fp32-exact on the product's own model output
            assert rel_err(x, float(kx[step]) * x0.cuda() + float(kv[step]) * mo) < 1e-5, (lh, lw, step)
            assert torch.isfinite(mo).all()
            ours[lh, lw, step] = mo.cpu()
            del x, mo
    eng.close()
    torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    refs = {}
    for tag, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        u, tx = copy.deepcopy(unet).cuda().to(dt), text.cuda().to(dt)
        with torch.no_grad():
            for (lh, lw), (rgb, x0) in inputs.items():
                for step in (0, 5):
                    inp = torch.cat([rgb, x0], 1).cuda().to(dt)
                    refs[tag, lh, lw, step] = u(inp, int(s.timesteps[step]), tx).float().cpu()
        del u, tx
        torch.cuda.empty_cache()
    for (lh, lw, step), mo in ours.items():
        e_ours, e_yard = rel_err(mo, refs["fp32", lh, lw, step]), rel_err(refs["bf16", lh, lw, step],
                                                                        refs["fp32", lh, lw, step])
        _record_parity(f"{lw}x{lh}/unet_step{step}", e_ours, e_yard)
        assert e_ours <= e_yard * 1.05 + 1e-3, f"{lw}x{lh} step {step}: ours {e_ours:.3e} vs torch-bf16 {e_yard:.3e}"


# ---- the VAE attention core at native token counts ---------------------------------------------------------------
# 4000 x 3000 (T % 64 = 44), 4032 x 3024 (T % 64 = 48), two 1920 x 1080 images (blocks and per-image offsets) and
# 77 x 131 latents (one block)
CORE_SIZES = [(1, 187500), (1, 190512), (2, 32400), (1, 10087)]
# logits of std 1; of std 40 (up to about +-200); one key dominating every query (logit about 14 against a log-sum of
# the others of about 13) at T - 1, in the ragged last 64-key tile, and near T / 2
REGIMES = ("std1", "logits80", "key_last", "key_mid")


@pytest.fixture(scope="module")
def core_engine(models):
    eng = engine_from_oracle(*models)
    yield eng
    eng.close()


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("NB,T", CORE_SIZES, ids=lambda x: str(x))
def test_vae_attn_core_within_float64_bound(core_engine, NB, T, regime):
    R, blocks = attn_blocks(core_engine, NB, T)
    assert blocks == NB * -(-T // R)
    q, k, v = _core_inputs(NB, T, regime)
    o = attn_core(core_engine, q, k, v, NB, T)
    rows = check_rows(T, R, seed=T).cuda()
    ref, bound, pv_abs = _core_ref(q, k, v, NB, T, rows)
    out = o.view(NB, T, VAE_C)[:, rows]
    r = ops_ref.within(out, ref, bound)
    record(f"native_res/vae_attn_core/{NB}x{T}/{regime}/worst", r["worst"])
    # what the rows say about the bf16 P rounding: the error beyond every other term, over 2^-8 sum_j p_j |v_j|
    other = bound - ops_ref.C_P * ops_ref.U_BF16 * pv_abs
    c_p = ((out.double() - ref).abs() - other).clamp(min=0) / (ops_ref.U_BF16 * pv_abs + ops_ref.TINY)
    record(f"native_res/vae_attn_core/{NB}x{T}/{regime}/c_p", float(c_p.max()))
    assert not r["nan"] and r["worst"] <= 1.0, (R, len(rows), r)


def test_vae_attn_core_row_blocks_are_bit_identical_at_12mp(core_engine):
    """At T = 190 512 one block cannot run (S and P would take 218 GB): the default block height and forced heights
    of 128 and 1792 rows give the same bits."""
    T = 190512
    q, k, v = _core_inputs(1, T, "std1")
    R0, _ = attn_blocks(core_engine, 1, T)
    assert R0 not in (128, 1792, T)
    base = attn_core(core_engine, q, k, v, 1, T)
    for force in (128, 1792):
        assert attn_blocks(core_engine, 1, T, force_rows=force) == (force, -(-T // force))
        assert torch.equal(attn_core(core_engine, q, k, v, 1, T), base), force
    attn_blocks(core_engine, 1, T)
