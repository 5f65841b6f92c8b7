"""24-megapixel photos (`-m gpu`): the VAE forwards on their lifetime-planned arena.

  * address independence: encode and decode give the same bits with every arena buffer poisoned (0xFF bytes, NaN in
    fp32 and bf16, written before the forward uses it) and under the alternative placement (reverse allocation order),
    at latents of 96 x 96, 77 x 131 and 128 x 128, 768 x 768 photos two at a time, a 4032 x 3024 photo, and a poisoned
    decode at 6048 x 4032. A buffer read before it is written, or after its bytes were handed to another, shows here;
  * the plans at 6048 x 4032: no two buffers live at once share a byte; the decoder's peak is at most 4.3 U and the
    encoder's 2.6 U (U = one fp32 128-channel map at full resolution, 512 bytes per pixel; measured 4.000 U and
    2.500 U, 49.96 GB of workspace); the workspace of one member and the pipelines' reserve for normals with E = 10 fit
    the card beside the weights;
  * the UNet step's arena (bump-allocated, stack-shaped) is exactly what the planner makes of its lifetimes;
  * the operators past 2^32 elements, element by element against float64 with the bounds of tests/ops_ref.py, on rows
    that include the first and last ones and those holding elements 2^30, 2^31 and 2^32: GroupNorm (+ SiLU, raw copy)
    over [24.4M, 256] and [24.4M, 128] with a mean of 100; the full-resolution 256 -> 256 conv with fp32 output and
    conv2 with the shortcut K concatenation (128 + 256 -> 128); upsample2x to [24.4M, 256], bit for bit; the VAE
    attention core (row blocks, as the decoder runs it) at T = 381 024 with random logits and with a dominant last
    key, and softmax_rows at n = 381 024; the flash attention at T = 381 024, C = 320, with and without a dominant
    last key;
  * one UNet + DDIM step at the 756 x 504 latent against the fp32 oracle with TF32 off and the bf16 yardstick, as
    test_native_res_gpu.py does at 12 MP. The encoder and decoder oracles do not fit the card at 24 MP; their numerics
    are held by the 12 MP parity tests, which run on the same planned arena;
  * the pipelines at processing_res=0 on a 6048 x 4032 photo: depth with E = 2 and uncertainty, normals with E = 2, a
    2-target IID model with E = 1; 8192 x 8192 is still refused before any work."""
import copy
import gc

import numpy as np
import pytest
import torch

from tests import ops_ref as R
from tests.helpers import (U_PER_PIXEL, VAE_C, _block_rows, _core_inputs, _core_ref, _photo, arena_place, arena_plan,
                           attn_blocks, attn_core, conv_row_ref, engine_from_oracle, group_stats64, groupnorm_rows_ref,
                           live_device_bytes, no_overlap, oracle_models, record, rel_err, set_arena, weight_bytes)

pytestmark = pytest.mark.gpu

H24, W24 = 4032, 6048
P24 = H24 * W24
T24 = P24 // 64            # latent tokens: 756 x 504 = 381 024


@pytest.fixture(scope="module")
def models():
    return oracle_models("full")


@pytest.fixture(scope="module")
def engine(models):
    eng = engine_from_oracle(*models)
    yield eng
    eng.close()


@pytest.fixture(autouse=True)
def _give_back_memory():
    """Every test here needs most of the card: what one leaves in torch's cache is returned before the next."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def test_iid_at_24mp():
    """First in the file: its own engine needs the card before the module's engine holds a 24 MP workspace."""
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
    pipe = MarigoldIIDPipeline(eng, DDIMScheduler(), text, target_properties=props, default_denoising_steps=1,
                               default_processing_resolution=0)
    out = pipe(_photo(H24, W24), ensemble_size=1, generator=torch.Generator(device="cuda").manual_seed(0),
               show_progress_bar=False)
    assert out.is_complete
    for name in names:
        assert out[name].array.shape == (3, H24, W24) and np.isfinite(out[name].array).all()
    eng.close()


# ---- operators past 2^32 elements -------------------------------------------------------------------------------
def _rows(n_rows, widths, seed, n_random=64):
    """Rows of [n_rows, width] tensors to check: the first and the last 64, those holding elements 2^30, 2^31 and 2^32
    of a tensor of each width and their neighbours, and n_random seeded rows."""
    rows = set(range(64)) | set(range(n_rows - 64, n_rows))
    for w in widths:
        for e in (2 ** 30, 2 ** 31, 2 ** 32):
            rows |= {e // w - 1, e // w, e // w + 1}
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, n_rows, (n_random,), generator=g).tolist())
    return torch.tensor(sorted(r for r in rows if 0 <= r < n_rows), dtype=torch.long)


@pytest.mark.parametrize("C", [256, 128])
def test_groupnorm_past_2_32_elements(C):
    from marigold_b200 import ops

    G, eps = 32, 1e-6
    g = torch.Generator(device="cuda").manual_seed(C)
    x = torch.randn(1, P24, C, device="cuda", generator=g).mul_(2).add_(100.0)
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    y, raw = ops.groupnorm_ex(x, None, gamma, beta, 1, P24, G, eps, 1, raw_copy=True)
    torch.cuda.synchronize()
    assert y.numel() > 2 ** 31 and (C < 256 or y.numel() > 2 ** 32)
    mean, rstd = group_stats64(x[0], G, eps)
    rows = _rows(P24, [C], seed=C).cuda()
    ref, bound = groupnorm_rows_ref(x[0, rows], mean, rstd, gamma, beta, G)
    R.assert_within(y[0, rows], ref, bound, f"native_res_24mp/groupnorm_c{C}/worst")
    assert torch.equal(raw[0, rows], x[0, rows].to(torch.bfloat16))


@pytest.mark.parametrize("Cin,Cin2,Cout", [(256, 0, 256), (128, 256, 128)], ids=["up_256", "conv2_shortcut"])
def test_full_resolution_conv_past_2_32_elements(Cin, Cin2, Cout):
    from marigold_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(Cin + Cin2)
    K = 9 * Cin + Cin2
    x = torch.randn(1, H24, W24, Cin, device="cuda", generator=g, dtype=torch.bfloat16)
    x2 = torch.randn(1, H24, W24, Cin2, device="cuda", generator=g, dtype=torch.bfloat16) if Cin2 else None
    wb = (torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    wsc = (torch.randn(Cout, Cin2, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16) if Cin2 else None
    b = torch.randn(Cout, device="cuda", generator=g)
    wp = ops.pack_conv_weight(wb)
    if Cin2:
        wp = torch.cat([wp, wsc], dim=1).contiguous()
    out = torch.empty(1, H24, W24, Cout, device="cuda")
    ops.conv2d_ex(x, wp, b, 1, H24, W24, Cin, Cout, x2=x2, Cin2=Cin2, out=out)
    torch.cuda.synchronize()
    assert max(x.numel(), out.numel(), x2.numel() if Cin2 else 0) > 2 ** 32
    worst = 0.0
    for y in _rows(H24, [W24 * c for c in (Cin, Cin2, Cout) if c], seed=K, n_random=6).tolist():
        ref, bound = conv_row_ref(x, wb, y, b, x2, wsc)
        r = R.within(out[0, y], ref, bound)
        assert not r["nan"] and r["worst"] <= 1.0, (y, r)
        worst = max(worst, r["worst"])
    record(f"native_res_24mp/conv_{Cin}+{Cin2}_{Cout}/worst", worst)


@pytest.mark.parametrize("std", [3.0, 40.0])
def test_softmax_rows_at_24mp(std):
    from tests.ops_cases import case_softmax_rows

    res = case_softmax_rows(M=64, n=T24, ld=(T24 + 63) // 64 * 64, std=std)
    record(f"native_res_24mp/softmax_rows_std{std:g}/worst", res["worst"])
    assert res["ok"], res


@pytest.mark.parametrize("regime", ["std1", "key_last"])
def test_vae_attn_core_at_24mp(engine, regime):
    """The VAE attention core in the decoder's row blocks at T = 381 024, within test_native_res_gpu.py's float64
    bound (its module docstring)."""
    rows_per_block, blocks = attn_blocks(engine, 1, T24)
    assert rows_per_block < T24 and blocks == -(-T24 // rows_per_block)
    q, k, v = _core_inputs(1, T24, regime)
    o = attn_core(engine, q, k, v, 1, T24)
    rows = _block_rows(T24, rows_per_block, seed=T24, every=4).cuda()
    ref, bound, _ = _core_ref(q, k, v, 1, T24, rows)
    R.assert_within(o.view(1, T24, VAE_C)[:, rows], ref, bound, f"native_res_24mp/vae_attn_core/{regime}/worst")


@pytest.mark.parametrize("dominant_at", [None, T24 - 1], ids=["std1", "key_last"])
def test_flash_attention_at_24mp(dominant_at):
    """The head-dim-64 flash attention at the UNet's level 0 on a 24 MP photo (T = 381 024, C = 320), on rows of its
    128-row query tiles, within tests/ops_ref.attn_bound of float64."""
    from marigold_b200 import ops
    from tests.ops_cases import dominant_key

    T, Cc, heads = T24, 320, 5
    g = torch.Generator(device="cuda").manual_seed(3)
    q, k, v = (torch.randn(T, Cc, device="cuda", generator=g) for _ in range(3))
    if dominant_at is not None:
        dominant_key(q.view(1, T, Cc), k.view(1, T, Cc), dominant_at, 14.0, 0.125, 64, seed=T)
    qkv = torch.cat([q, k, v], 1).to(torch.bfloat16).contiguous()
    del q, k, v
    out = ops.flash_attn64(qkv, 1, T, Cc, 0.125)
    torch.cuda.synchronize()
    rows = _block_rows(T, 128, seed=T + 1, every=32).cuda()
    q64, k64, v64 = [R.f64(t).reshape(1, T, heads, 64).permute(0, 2, 1, 3) for t in qkv.split(Cc, dim=1)]
    ref = torch.empty(1, heads, len(rows), 64, dtype=torch.float64, device="cuda")
    pv_abs = torch.empty_like(ref)
    step = max(1, (1 << 26) // (heads * T))
    for i in range(0, len(rows), step):
        p = torch.softmax((q64[:, :, rows[i:i + step]] @ k64.transpose(-1, -2)) * 0.125, dim=-1)
        ref[:, :, i:i + step], pv_abs[:, :, i:i + step] = p @ v64, p @ v64.abs()
        del p
    ref, pv_abs = (t.permute(0, 2, 1, 3).reshape(len(rows), Cc) for t in (ref, pv_abs))
    R.assert_within(out[rows], ref, R.attn_bound(ref, pv_abs),
                    f"native_res_24mp/flash_attn_c320/{'key_last' if dominant_at else 'std1'}/worst")


def _forward_variants(eng, img, lat):
    out = {}
    for poison, placement in ((False, 0), (True, 0), (True, 1), (False, 1)):
        set_arena(eng, poison, placement)
        out[poison, placement] = (eng.encode(img), eng.decode(lat, 2))
    set_arena(eng)
    return out


@pytest.mark.parametrize("NB,lh,lw", [(1, 96, 96), (1, 77, 131), (1, 128, 128), (2, 96, 96), (1, 378, 504)])
def test_outputs_do_not_depend_on_addresses(engine, NB, lh, lw):
    g = torch.Generator().manual_seed(1000 * lh + lw + NB)
    img = (torch.rand(NB, 3, 8 * lh, 8 * lw, generator=g) * 2 - 1).cuda()
    lat = torch.randn(NB, 4, lh, lw, generator=g).cuda()
    # the alternative placement moves buffers (the switch takes effect)
    offs = []
    for placement in (0, 1):
        set_arena(engine, placement=placement)
        offs.append(arena_plan(engine, 2, NB, lh, lw)[3])
    set_arena(engine)
    assert (offs[0] != offs[1]).any()
    out = _forward_variants(engine, img, lat)
    enc, dec = out[False, 0]
    assert torch.isfinite(enc).all() and torch.isfinite(dec).all()
    for key, (e, d) in out.items():
        assert torch.equal(e, enc) and torch.equal(d, dec), key


def test_24mp_decode_does_not_depend_on_addresses(engine):
    lat = torch.randn(1, 4, H24 // 8, W24 // 8, generator=torch.Generator().manual_seed(24)).cuda()
    base = engine.decode(lat, 0)
    assert base.shape == (1, 1, H24, W24) and torch.isfinite(base).all()
    set_arena(engine, poison=True)
    try:
        assert torch.equal(engine.decode(lat, 0), base)
    finally:
        set_arena(engine)


def test_24mp_plans(engine):
    from marigold_b200.pipeline import call_reserve_bytes

    U = H24 * W24 * U_PER_PIXEL
    for op, d0, d1, limit in ((2, H24 // 8, W24 // 8, 4.3), (1, H24, W24, 2.6)):
        nbytes, t0, t1, off = arena_plan(engine, op, 1, d0, d1)
        assert (off % 1024 == 0).all()
        assert no_overlap(nbytes, t0, t1, off), op
        peak = int((off + nbytes).max())
        record(f"native_res_24mp/plan_peak_over_U/{'decode' if op == 2 else 'encode'}", peak / U)
        assert peak <= limit * U, (op, peak / U)
        # the plan is the placement of its own lifetimes, and the same on every call
        assert arena_place(nbytes, t0, t1)[1].tolist() == off.tolist()
        assert arena_plan(engine, op, 1, d0, d1)[3].tolist() == off.tolist()
    need = engine.workspace_bytes(1, H24, W24)
    weights = weight_bytes(engine)
    total = torch.cuda.get_device_properties(0).total_memory
    record("native_res_24mp/workspace_bytes", need)
    assert need + call_reserve_bytes(H24, W24, 10, 3) + weights < total, (need, weights, total)


@pytest.mark.parametrize("NB,lh,lw", [(1, 96, 96), (2, 77, 131)])
def test_unet_arena_is_the_planners_stack(engine, NB, lh, lw):
    nbytes, t0, t1, bump = arena_plan(engine, 0, NB, lh, lw)
    peak, off = arena_place(nbytes, t0, t1)
    assert off.tolist() == bump.tolist()
    assert peak == int((bump + nbytes).max())


def test_upsample2x_past_2_32_elements():
    from marigold_b200 import ops

    Hi, Wi, Cc = H24 // 2, W24 // 2, 256
    x = torch.randn(1, Hi, Wi, Cc, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    y = ops.upsample2x(x)
    assert y.numel() > 2 ** 32
    rows = torch.cat([torch.arange(0, 4), torch.randint(0, H24, (60,), generator=torch.Generator().manual_seed(5)),
                      torch.arange(H24 - 4, H24)])
    for r in rows.tolist():
        ref = x[0, r // 2].to(torch.bfloat16).repeat_interleave(2, dim=0)
        assert torch.equal(y[0, r], ref), r
    del x, y
    torch.cuda.empty_cache()


def test_depth_and_normals_at_24mp(models, engine):
    from marigold_b200.pipeline import MarigoldDepthPipeline, MarigoldNormalsPipeline
    from marigold_b200.schedulers import DDIMScheduler

    text = models[2]
    img = _photo(H24, W24)
    pipe = MarigoldDepthPipeline(engine, DDIMScheduler(), text, default_denoising_steps=1,
                                 default_processing_resolution=0)
    out = pipe(img, ensemble_size=2, generator=torch.Generator(device="cuda").manual_seed(0), color_map=None,
               show_progress_bar=False, ensemble_kwargs={"output_uncertainty": True})
    assert out.depth_np.shape == (H24, W24) and np.isfinite(out.depth_np).all()
    assert out.uncertainty is not None and out.uncertainty.shape == (H24, W24) and np.isfinite(out.uncertainty).all()
    del out
    npipe = MarigoldNormalsPipeline(engine, DDIMScheduler(), text, default_denoising_steps=1,
                                    default_processing_resolution=0)
    nout = npipe(img, ensemble_size=2, generator=torch.Generator(device="cuda").manual_seed(0), show_progress_bar=False)
    assert nout.normals_np.shape == (3, H24, W24) and np.isfinite(nout.normals_np).all()


def test_8192_is_still_refused_before_any_work(models, engine):
    from marigold_b200.pipeline import MarigoldDepthPipeline
    from marigold_b200.schedulers import DDIMScheduler

    live = live_device_bytes
    pipe = MarigoldDepthPipeline(engine, DDIMScheduler(), models[2], default_denoising_steps=1,
                                 default_processing_resolution=0)
    torch.cuda.synchronize()
    b0, l0, t0 = live(), engine.lib.mgb_launch_count(), torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match=r"needs \d+ bytes of device workspace, but -?\d+ bytes are available"):
        pipe(torch.zeros(1, 3, 8192, 8192, dtype=torch.uint8), ensemble_size=1, show_progress_bar=False)
    assert (live(), engine.lib.mgb_launch_count(), torch.cuda.memory_allocated()) == (b0, l0, t0)


# ---- the UNet step at the 24 MP latent ---------------------------------------------------------------------------
def test_unet_step_at_24mp_matches_oracle(models):
    """One UNet + DDIM step (step 0 of 10) on the 756 x 504 latent (T = 381 024 tokens at level 0), within the bf16
    yardstick of the fp32 oracle. The engine runs first and is closed before the torch graphs."""
    from marigold_b200.schedulers import DDIMScheduler

    unet, vae, text = models
    s = DDIMScheduler()
    s.set_timesteps(10)
    kx, kv, kz = s.coefficients()
    lh, lw = H24 // 8, W24 // 8
    g = torch.Generator().manual_seed(lh * lw)
    rgb, x0 = torch.randn(1, 4, lh, lw, generator=g), torch.randn(1, 4, lh, lw, generator=g)
    eng = engine_from_oracle(unet, vae, text)
    eng.set_schedule(s.timesteps, kx, kv, kz)
    x = x0.cuda()
    mo = eng.unet_step(rgb.cuda(), x, 0, want_model_out=True)
    assert rel_err(x, float(kx[0]) * x0.cuda() + float(kv[0]) * mo) < 1e-5
    assert torch.isfinite(mo).all()
    ours = mo.cpu()
    del x, mo
    eng.close()
    torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    refs = {}
    for tag, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        u, tx = copy.deepcopy(unet).cuda().to(dt), text.cuda().to(dt)
        with torch.no_grad():
            refs[tag] = u(torch.cat([rgb, x0], 1).cuda().to(dt), int(s.timesteps[0]), tx).float().cpu()
        del u, tx
        torch.cuda.empty_cache()
    e_ours, e_yard = rel_err(ours, refs["fp32"]), rel_err(refs["bf16"], refs["fp32"])
    record("native_res_24mp/unet_step0/ours_vs_fp32", e_ours)
    record("native_res_24mp/unet_step0/torch_bf16_vs_fp32", e_yard)
    assert e_ours <= e_yard * 1.05 + 1e-3, f"ours {e_ours:.3e} vs torch-bf16 {e_yard:.3e}"
