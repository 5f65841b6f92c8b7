"""60-megapixel photos (`-m gpu`): the decoder's full-resolution 256-channel stage in 2.5 U (net.cu, up_conv_low_memory
and resnet_shortcut_halves; U = one fp32 128-channel map at full resolution, 512 bytes per pixel; 30.8 GB at
9504 x 6336).

  * the plans: at 9504 x 6336 the decoder's peak is 2.5 U (plus the GroupNorm scratch), no two buffers live at once
    share a byte, and the library's rule gives the forced plan; forced at 8064 x 6048 and 6048 x 4032 the peak is
    2.5 U too;
  * the same bits: low-memory decodes equal the default path's for the depth, normals and raw-3 modes, one and two
    members, at 1920 x 1080 and 1000 x 744, with the library's bands, with forced band heights that leave a ragged
    last band, with one band, with a poisoned arena and under the reversed placement; at operator level the banded
    conv with the split output and with a row origin against one launch of the whole conv, and the two-source
    two-launch GroupNorm against the fused one;
  * float64 at the new scale: the two-source GroupNorm over two [60.2M, 128] halves in their own memory, and the
    banded up-conv writing both halves, on rows that include the first and last ones and those holding elements
    2^30 .. 2^33; the VAE attention core at T = 940 896 in its row blocks and the flash attention at T = 940 896;
  * the pipelines at processing_res=0 on a 9504 x 6336 photo: depth with E = 1 and with E = 2 and uncertainty;
    select_batch_size takes one depth member at 9504 x 6336 and 9528 x 6328; normals and a 2-target IID model
    (E = 1) either complete or are refused with ValueError before any work, and which is recorded."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from tests import ops_ref as R
from tests.helpers import (U_PER_PIXEL, VAE_C, _block_rows, _core_inputs, _core_ref, _photo, _rows, arena_place,
                           arena_plan, attn_blocks, attn_core, conv_row_ref, engine_from_oracle, group_stats64,
                           groupnorm_rows_ref, no_overlap, oracle_models, record, set_arena, set_bands, set_low_memory,
                           weight_bytes)

pytestmark = pytest.mark.gpu

H60, W60 = 6336, 9504
P60 = H60 * W60            # 60 217 344 pixels
T60 = P60 // 64            # latent tokens: 1188 x 792 = 940 896
SCRATCH = 1 << 20          # bytes of GroupNorm partials and statistics live beside the 2.5 U at the decoder's peak


def conv_band(x, src_y0, wp, bias, out, out_hi, split_col, ldo, out_y0, NB_tile, H, W, Cin, Cout, ty0, tiles):
    """One band of the decoder's banded conv (mgb_debug_conv2d_band); x None: only returns (tile_h, tiles_y)."""
    from marigold_b200 import _lib
    from marigold_b200.ops import ptr, stream_ptr

    f = _lib.load().mgb_debug_conv2d_band
    geom = (C.c_int32 * 2)()
    xp = None if x is None else ptr(x)
    src_rows = 0 if x is None else x.shape[-3]
    ob = None if out is None else C.c_void_p(out.data_ptr())
    oh = None if out_hi is None else C.c_void_p(out_hi.data_ptr())
    _lib.check(f(xp, src_y0, src_rows, None if wp is None else ptr(wp), None if bias is None else ptr(bias), ob, oh,
                 split_col, ldo, out_y0, NB_tile, H, W, Cin, Cout, ty0, tiles, geom, stream_ptr()),
               "mgb_debug_conv2d_band")
    return geom[0], geom[1]


def groupnorm_halves(a, b, gamma, beta, NB, HW, G, eps, silu):
    """The two-source two-launch GroupNorm (mgb_debug_groupnorm_halves): raw over a, the operand over b."""
    from marigold_b200 import _lib
    from marigold_b200.ops import ptr, stream_ptr

    lib = _lib.load()
    Ch = a.shape[-1]
    f = lib.mgb_debug_groupnorm_halves
    ws = torch.empty((int(lib.mgb_op_groupnorm_ws_bytes(NB, HW, 2 * Ch, G)) + 3) // 4, device="cuda")
    stats = torch.empty(NB * 2 * Ch * 2, device="cuda")
    _lib.check(f(ptr(a), ptr(b), Ch, ptr(gamma), ptr(beta), ptr(ws), ptr(stats), NB, HW, G, float(eps), int(silu),
                 stream_ptr()), "mgb_debug_groupnorm_halves")


def _conv_weights(Cin, Cout, seed):
    from marigold_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(seed)
    wb = (torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (9 * Cin) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, device="cuda", generator=g)
    return wb, ops.pack_conv_weight(wb), b


def _halo(ty0, tiles, th, H):
    """Image rows [lo, hi) a band of tile rows [ty0, ty0 + tiles) reads: the band and its halo inside the image."""
    return max(0, ty0 * th - 1), min(H, (ty0 + tiles) * th + 1)


@pytest.fixture(autouse=True)
def _give_back_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def test_iid_at_60mp():
    """First in the file: its own engine needs the card before the module's engine holds a 60 MP workspace. Its call
    reserve is 108 bytes per pixel; it completes with finite outputs or is refused before any work."""
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
    del unet, vae
    names = ["albedo", "shading"]
    props = {"target_names": names, "albedo": {"prediction_space": "srgb"},
             "shading": {"prediction_space": "linear", "up_to_scale": True}}
    pipe = MarigoldIIDPipeline(eng, DDIMScheduler(), text, target_properties=props, default_denoising_steps=1,
                               default_processing_resolution=0)
    lib = eng.lib
    launches = lib.mgb_launch_count()
    try:
        out = pipe(_photo(H60, W60), ensemble_size=1, generator=torch.Generator(device="cuda").manual_seed(0),
                   show_progress_bar=False)
    except ValueError as e:
        assert lib.mgb_launch_count() == launches, "refused after launching work"
        print(f"2-target IID at 9504 x 6336: refused ({e})")
        record("native_res_60mp/iid_completes", 0.0)
    else:
        assert out.is_complete
        for name in names:
            assert out[name].array.shape == (3, H60, W60) and np.isfinite(out[name].array).all()
        record("native_res_60mp/iid_completes", 1.0)
    finally:
        eng.close()


# ---- the pipelines at 60 MP (an engine of their own, before the float64 references load their libraries) ----------
@pytest.fixture(scope="module")
def models():
    return oracle_models("full")


def test_depth_and_normals_at_60mp(models):
    """select_batch_size takes one depth member at 9504 x 6336 and 9528 x 6328; depth with E = 1 and with E = 2 and
    uncertainty completes. Normals (E = 1) are borderline, a call reserve of 60 bytes per pixel: they complete with
    finite outputs or are refused before any work."""
    import time

    from marigold_b200.pipeline import (MarigoldDepthPipeline, MarigoldNormalsPipeline, call_reserve_bytes,
                                        select_batch_size)
    from marigold_b200.schedulers import DDIMScheduler

    eng = engine_from_oracle(*models)
    try:
        for h, w in ((H60, W60), (6328, 9528)):
            record(f"native_res_60mp/workspace_bytes_{w}x{h}", eng.workspace_bytes(1, h, w))
            assert select_batch_size(eng, 1, h, w, reserve_bytes=call_reserve_bytes(h, w, 1, 1)) == 1, (h, w)
        img = _photo(H60, W60)
        pipe = MarigoldDepthPipeline(eng, DDIMScheduler(), models[2], default_denoising_steps=1,
                                     default_processing_resolution=0)
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = pipe(img, ensemble_size=1, generator=torch.Generator(device="cuda").manual_seed(0), color_map=None,
                   show_progress_bar=False)
        torch.cuda.synchronize()
        record("native_res_60mp/depth_e1_seconds", time.perf_counter() - t)
        assert out.depth_np.shape == (H60, W60) and np.isfinite(out.depth_np).all()
        del out
        out = pipe(img, ensemble_size=2, generator=torch.Generator(device="cuda").manual_seed(0), color_map=None,
                   show_progress_bar=False, ensemble_kwargs={"output_uncertainty": True})
        assert out.depth_np.shape == (H60, W60) and np.isfinite(out.depth_np).all()
        assert out.uncertainty is not None and out.uncertainty.shape == (H60, W60)
        assert np.isfinite(out.uncertainty).all()
        del out
        gc.collect()
        torch.cuda.empty_cache()
        npipe = MarigoldNormalsPipeline(eng, DDIMScheduler(), models[2], default_denoising_steps=1,
                                        default_processing_resolution=0)
        launches = eng.lib.mgb_launch_count()
        try:
            nout = npipe(img, ensemble_size=1, generator=torch.Generator(device="cuda").manual_seed(0),
                         show_progress_bar=False)
        except ValueError as e:
            assert eng.lib.mgb_launch_count() == launches, "refused after launching work"
            print(f"normals at 9504 x 6336: refused ({e})")
            record("native_res_60mp/normals_completes", 0.0)
        else:
            assert nout.normals_np.shape == (3, H60, W60) and np.isfinite(nout.normals_np).all()
            record("native_res_60mp/normals_completes", 1.0)
    finally:
        eng.close()


# ---- float64 at 60 MP (before the module's engine: these need most of the card) ----------------------------------
def test_groupnorm_halves_past_2_33_elements():
    """[a | b] with a, b [60.2M, 128] each and a mean of 100: the statistics over both, the shortcut's copy written over
    a and the conv operand over b, as the decoder runs them."""
    G, eps = 32, 1e-6
    g = torch.Generator(device="cuda").manual_seed(60)
    a = torch.randn(P60, 128, device="cuda", generator=g).mul_(2).add_(100.0)
    b = torch.randn(P60, 128, device="cuda", generator=g).mul_(2).add_(100.0)
    gamma, beta = torch.randn(256, device="cuda", generator=g), torch.randn(256, device="cuda", generator=g)
    assert a.numel() > 2 ** 32
    ma, ra = group_stats64(a, G // 2, eps, chunk=1 << 18)
    mb, rb = group_stats64(b, G // 2, eps, chunk=1 << 18)
    mean, rstd = torch.cat([ma, mb], 1), torch.cat([ra, rb], 1)
    rows = torch.tensor(sorted(set(_rows(P60, 128, seed=60).tolist()) | set(_rows(P60, 256, seed=61).tolist())),
                        device="cuda")
    xr = torch.cat([a[rows], b[rows]], 1)
    groupnorm_halves(a, b, gamma, beta, 1, P60, G, eps, 1)
    torch.cuda.synchronize()
    ref, bound = groupnorm_rows_ref(xr, mean, rstd, gamma, beta, G)
    R.assert_within(b.view(torch.bfloat16).view(P60, 256)[rows], ref, bound, "native_res_60mp/groupnorm_halves/worst")
    assert torch.equal(a.view(torch.bfloat16).view(P60, 256)[rows], xr.to(torch.bfloat16))


def test_banded_up_conv_past_2_33_elements():
    """The up-conv's bands (256 -> 256, output split into two [60.2M, 128] maps) at 9504 x 6336: the bands holding image
    rows with elements 2^30 .. 2^33 of either half, and the first and last rows, each from its own seeded band operand
    (the band and its halo rows), against float64 with tests/ops_ref.py's conv bound."""
    Cin = Cout = 256
    wb, wp, bias = _conv_weights(Cin, Cout, seed=6336)
    th, tiles_y = conv_band(None, 0, None, None, None, None, 0, 0, 0, 1, H60, W60, Cin, Cout, 0, 0)
    half_a = torch.empty(P60, 128, device="cuda")
    half_b = torch.empty(P60, 128, device="cuda")
    assert half_a.numel() > 2 ** 32
    rows = {0, H60 - 1}
    for width in (W60 * 128, W60 * 256):
        for e in (2 ** 30, 2 ** 31, 2 ** 32, 2 ** 33):
            rows |= {e // width - 1, e // width, e // width + 1}
    rows = sorted(r for r in rows if 0 <= r < H60)
    bt = 2
    bands = sorted({r // th // bt * bt for r in rows})
    worst = 0.0
    for ty0 in bands:
        tiles = min(bt, tiles_y - ty0)
        lo, hi = _halo(ty0, tiles, th, H60)
        g = torch.Generator(device="cuda").manual_seed(ty0)
        x = torch.randn(1, hi - lo, W60, Cin, device="cuda", generator=g, dtype=torch.bfloat16)
        conv_band(x, lo, wp, bias, half_a, half_b, 128, 128, 0, 1, H60, W60, Cin, Cout, ty0, tiles)
        torch.cuda.synchronize()
        for y in rows:
            if not ty0 * th <= y < (ty0 + tiles) * th:
                continue
            ref, bound = conv_row_ref(x, wb, y - lo, bias)
            got = torch.cat([half_a.view(H60, W60, 128)[y], half_b.view(H60, W60, 128)[y]], 1)
            r = R.within(got, ref, bound)
            assert not r["nan"] and r["worst"] <= 1.0, (y, r)
            worst = max(worst, r["worst"])
    record("native_res_60mp/banded_up_conv/worst", worst)


@pytest.mark.parametrize("regime", ["std1", "key_last"])
def test_vae_attn_core_at_60mp(regime):
    """The VAE attention core in the decoder's row blocks at T = 940 896 (the 60 MP latent), within
    test_native_res_gpu.py's float64 bound. Its blocks are the one-wave minimum of the P V GEMM, 4 224 rows: their
    scores (23.8 GB) pass kVaeAttnBudget but stay far below the decoder's full-resolution peak."""
    eng = engine_from_oracle(*oracle_models("full"))
    try:
        rows_per_block, blocks = attn_blocks(eng, 1, T60)
        Tp = -(-T60 // 64) * 64
        assert rows_per_block < T60 and blocks == -(-T60 // rows_per_block)
        assert rows_per_block * Tp * 6 < 2 * P60 * U_PER_PIXEL, rows_per_block
        record("native_res_60mp/vae_attn_rows_per_block", rows_per_block)
        record("native_res_60mp/vae_attn_block_bytes", rows_per_block * Tp * 6)
        q, k, v = _core_inputs(1, T60, regime)
        o = attn_core(eng, q, k, v, 1, T60)
        rows = _block_rows(T60, rows_per_block, seed=T60, every=8).cuda()
        ref, bound, _ = _core_ref(q, k, v, 1, T60, rows)
        R.assert_within(o.view(1, T60, VAE_C)[:, rows], ref, bound, f"native_res_60mp/vae_attn_core/{regime}/worst")
    finally:
        eng.close()


@pytest.mark.parametrize("dominant_at", [None, T60 - 1], ids=["std1", "key_last"])
def test_flash_attention_at_60mp(dominant_at):
    """The head-dim-64 flash attention at the UNet's level 0 on a 60 MP photo (T = 940 896, C = 320), on rows of its
    128-row query tiles, within tests/ops_ref.attn_bound of float64."""
    from marigold_b200 import ops
    from tests.ops_cases import dominant_key

    T, Cc, heads = T60, 320, 5
    g = torch.Generator(device="cuda").manual_seed(5)
    q, k, v = (torch.randn(T, Cc, device="cuda", generator=g) for _ in range(3))
    if dominant_at is not None:
        dominant_key(q.view(1, T, Cc), k.view(1, T, Cc), dominant_at, 14.0, 0.125, 64, seed=T)
    qkv = torch.cat([q, k, v], 1).to(torch.bfloat16).contiguous()
    del q, k, v
    out = ops.flash_attn64(qkv, 1, T, Cc, 0.125)
    torch.cuda.synchronize()
    rows = _block_rows(T, 128, seed=T + 1, every=64).cuda()
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
                    f"native_res_60mp/flash_attn_c320/{'key_last' if dominant_at else 'std1'}/worst")


# ---- operator level, bit for bit ---------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(744, 1000), (1080, 1920), (259, 333)])
@pytest.mark.parametrize("bt", [1, 3, 1 << 20])
def test_conv_bands_equal_one_launch(H, W, bt):
    """The up-conv's bands (band operand from the 2x nearest upsampling, split output) and conv1's bands (row-origin
    output into a staging band) equal one launch of the whole conv bit for bit, with the whole conv's tile."""
    Cin, Cout = 256, 256
    _, wp, bias = _conv_weights(Cin, Cout, seed=H * W)
    th, tiles_y = conv_band(None, 0, None, None, None, None, 0, 0, 0, 1, H, W, Cin, Cout, 0, 0)
    g = torch.Generator(device="cuda").manual_seed(H + W)
    xh = torch.randn(1, (H + 1) // 2, (W + 1) // 2, Cin, device="cuda", generator=g).to(torch.bfloat16)
    x = xh.repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :H, :W].contiguous()
    whole = torch.empty(H * W, Cout, device="cuda")
    conv_band(x, 0, wp, bias, whole, None, 0, Cout, 0, 1, H, W, Cin, Cout, 0, tiles_y)
    # up-conv: band operands with their halo rows, output split at channel 128
    a = torch.full((H * W, 128), float("nan"), device="cuda")
    b = torch.full((H * W, 128), float("nan"), device="cuda")
    for ty0 in range(0, tiles_y, bt):
        tiles = min(bt, tiles_y - ty0)
        lo, hi = _halo(ty0, tiles, th, H)
        conv_band(x[:, lo:hi].contiguous(), lo, wp, bias, a, b, 128, 128, 0, 1, H, W, Cin, Cout, ty0, tiles)
    torch.cuda.synchronize()
    assert torch.equal(torch.cat([a, b], 1), whole)
    # conv1: the whole operand, each band's output to a staging band, then copied into place
    Cout1 = 128
    _, wp1, bias1 = _conv_weights(Cin, Cout1, seed=H * W + 1)
    whole1 = torch.empty(H * W, Cout1, device="cuda")
    conv_band(x, 0, wp1, bias1, whole1, None, 0, Cout1, 0, 1, H, W, Cin, Cout1, 0, tiles_y)
    out = torch.full((H * W, Cout1), float("nan"), device="cuda")
    stage = torch.empty(min(H, bt * th) * W, Cout1, device="cuda")
    for ty0 in range(0, tiles_y, bt):
        tiles = min(bt, tiles_y - ty0)
        r0, r1 = ty0 * th, min(H, (ty0 + tiles) * th)
        stage.fill_(float("nan"))
        conv_band(x, 0, wp1, bias1, stage, None, 0, Cout1, r0, 1, H, W, Cin, Cout1, ty0, tiles)
        out[r0 * W:r1 * W] = stage[:(r1 - r0) * W]
    torch.cuda.synchronize()
    assert torch.equal(out, whole1)


@pytest.mark.parametrize("NB,HW", [(1, 1920 * 1080), (2, 1000 * 744), (1, 4099)])
def test_groupnorm_halves_equal_fused(NB, HW):
    """The two-source GroupNorm in two launches, in the memory of its two sources, equals the fused GroupNorm's operand
    and raw copy of [a | b] bit for bit."""
    from marigold_b200 import ops

    G, eps = 32, 1e-6
    g = torch.Generator(device="cuda").manual_seed(NB * HW + 1)
    a = torch.randn(NB * HW, 128, device="cuda", generator=g).mul_(3).add_(1.0)
    b = torch.randn(NB * HW, 128, device="cuda", generator=g).mul_(2).sub_(0.5)
    gamma, beta = torch.randn(256, device="cuda", generator=g), torch.randn(256, device="cuda", generator=g)
    y_ref, raw_ref = ops.groupnorm_ex(a.view(NB, HW, 128), b.view(NB, HW, 128), gamma, beta, NB, HW, G, eps, 1,
                                      raw_copy=True)
    groupnorm_halves(a, b, gamma, beta, NB, HW, G, eps, 1)
    torch.cuda.synchronize()
    assert torch.equal(b.view(torch.bfloat16).view(NB * HW, 256), y_ref.view(NB * HW, 256))
    assert torch.equal(a.view(torch.bfloat16).view(NB * HW, 256), raw_ref.view(NB * HW, 256))


@pytest.fixture(scope="module")
def engine(models):
    eng = engine_from_oracle(*models)
    yield eng
    set_low_memory(eng, 0)
    set_bands(eng)
    eng.close()


# ---- plans -------------------------------------------------------------------------------------------------------
def test_60mp_plan(engine):
    set_low_memory(engine, 0)
    U = P60 * U_PER_PIXEL
    lh, lw = H60 // 8, W60 // 8
    nbytes, t0, t1, off = arena_plan(engine, 2, 1, lh, lw)
    assert (off % 1024 == 0).all()
    assert no_overlap(nbytes, t0, t1, off)
    peak = int((off + nbytes).max())
    record("native_res_60mp/plan_peak_over_U/decode", peak / U)
    assert peak <= 2.5 * U + SCRATCH, peak / U
    assert arena_place(nbytes, t0, t1)[1].tolist() == off.tolist()
    set_low_memory(engine, 1)
    try:
        assert [a.tolist() for a in arena_plan(engine, 2, 1, lh, lw)] == [a.tolist() for a in (nbytes, t0, t1, off)]
    finally:
        set_low_memory(engine, 0)
    enc = arena_plan(engine, 1, 1, H60, W60)
    record("native_res_60mp/plan_peak_over_U/encode", int((enc[3] + enc[0]).max()) / U)
    need = engine.workspace_bytes(1, H60, W60)
    record("native_res_60mp/workspace_bytes", need)
    print(f"9504 x 6336: decoder peak {peak / U:.3f} U, encoder {int((enc[3] + enc[0]).max()) / U:.3f} U, "
          f"workspace {need} B, weights {weight_bytes(engine)} B")


@pytest.mark.parametrize("h,w", [(6048, 8064), (4032, 6048)])
def test_low_memory_plan_when_forced(engine, h, w):
    set_low_memory(engine, 1)
    try:
        nbytes, t0, t1, off = arena_plan(engine, 2, 1, h // 8, w // 8)
    finally:
        set_low_memory(engine, 0)
    U = h * w * U_PER_PIXEL
    assert no_overlap(nbytes, t0, t1, off)
    assert int((off + nbytes).max()) <= 2.5 * U + SCRATCH, int((off + nbytes).max()) / U


# ---- the same bits -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NB", [1, 2])
@pytest.mark.parametrize("h,w", [(1080, 1920), (744, 1000)])
def test_low_memory_decode_is_bit_identical(engine, NB, h, w):
    lh, lw = h // 8, w // 8
    lat = torch.randn(NB, 4, lh, lw, generator=torch.Generator().manual_seed(NB * h + w + 60)).cuda()
    try:
        for mode in (0, 1, 2):            # depth, normals, raw 3-channel
            set_low_memory(engine, -1)
            ref = engine.decode(lat, mode)
            assert torch.isfinite(ref).all()
            set_low_memory(engine, 1)
            # the library's bands, ragged forced bands (3 and 5 tile rows), one band
            for bands in ((0, 0), (3, 5), (1 << 20, 1 << 20)):
                set_bands(engine, *bands)
                assert torch.equal(engine.decode(lat, mode), ref), (mode, bands)
            set_bands(engine)
            if mode == 2:
                for poison, placement in ((True, 0), (True, 1)):
                    set_arena(engine, poison, placement)
                    assert torch.equal(engine.decode(lat, mode), ref), (poison, placement)
                set_arena(engine)
    finally:
        set_arena(engine)
        set_bands(engine)
        set_low_memory(engine, 0)
    record(f"native_res_60mp/low_memory_vs_default/{w}x{h}_nb{NB}/max_abs_diff", 0.0)
