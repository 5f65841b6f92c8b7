"""45-48-megapixel photos (`-m gpu`): the decoder's first full-resolution resnet in place (net.cu,
resnet_shortcut_in_place), which takes the decoder's planned peak from 4 U to 3 U (U = one fp32 128-channel map at full
resolution, 512 bytes per pixel; 25.0 GB at 8064 x 6048).

  * the plans: at 8064 x 6048 the decoder's peak is 3 U (plus the GroupNorm scratch), no two buffers live at once share
    a byte, and the plan is its own lifetimes' placement on every call; at 6048 x 4032 and 768 x 768 the library's
    rule keeps the default path, so plans and workspace bytes are those of a handle that never runs in place;
  * the same bits: decodes forced in place equal the default path's for the depth, normals and raw-3 modes, one and two
    members, at 1920 x 1080 and 1000 x 744, also with a poisoned arena and the reversed placement; the two-launch
    GroupNorm over strided rows (in place for the shortcut's copy) equals the fused GroupNorm's operand and copy;
  * float64 at the new scale: that GroupNorm over [48.8M, 256] in place and over the [48.8M, 128] second halves of its
    rows, on rows that include the first and last ones and those holding elements 2^30 .. 2^33;
  * the pipelines at processing_res=0 on an 8064 x 6048 photo: depth with E = 1 and with E = 2 and uncertainty, normals
    with E = 1, a 2-target IID model with E = 1; select_batch_size takes one member at 7728 x 5152 (just past the
    default path's limit), 8192 x 5464 and 8256 x 5504;
  * the two convs of the in-place resnet in its layout at 8064 x 6048 (strided output over a [48.8M, 256] buffer, the
    shortcut's operand at a 1024-byte pixel stride) against float64 on rows holding elements 2^30 .. 2^33."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from tests import ops_ref as R
from tests.helpers import engine_from_oracle, oracle_models, record
from tests.test_native_res_24mp_gpu import (U_PER_PIXEL, _hook, _photo, _weight_bytes, arena_place, arena_plan,
                                            group_stats64, groupnorm_rows_ref, no_overlap, set_arena)

pytestmark = pytest.mark.gpu

H48, W48 = 6048, 8064
P48 = H48 * W48            # 48 771 072 pixels
SCRATCH = 1 << 20          # bytes of GroupNorm partials and statistics live beside the 3 U at the decoder's peak


def set_low_memory(eng, mode):
    """1: the decoder's first full-resolution resnet in place at every size; -1: never; 0: the library's rule."""
    from marigold_b200._lib import check

    f = _hook("mgb_debug_vae_low_memory", C.c_int32, [C.c_void_p, C.c_int32])
    check(f(eng._h, mode), "mgb_debug_vae_low_memory")


def groupnorm_rows(x, C_, ldx, raw, ldr, gamma, beta, NB, HW, G, eps, silu):
    """The two-launch GroupNorm (mgb_debug_groupnorm_rows) over rows of C_ channels at a stride of ldx floats of x."""
    from marigold_b200 import _lib
    from marigold_b200.ops import ptr, stream_ptr

    lib = _lib.load()
    x_p = C.c_void_p(x.data_ptr())                          # rows at a stride: x may be a column slice
    raw_p = None if raw is None else C.c_void_p(raw.data_ptr())
    f = _hook("mgb_debug_groupnorm_rows", C.c_int32,
              [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
               C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_void_p])
    y = torch.empty(NB * HW, C_, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty((int(lib.mgb_op_groupnorm_ws_bytes(NB, HW, C_, G)) + 3) // 4, device="cuda")
    stats = torch.empty(NB * C_ * 2, device="cuda")
    _lib.check(f(x_p, C_, ldx, ptr(y), raw_p, ldr, ptr(gamma), ptr(beta), ptr(ws), ptr(stats), NB, HW, G,
                 float(eps), int(silu), stream_ptr()), "mgb_debug_groupnorm_rows")
    return y


def _rows(n_rows, width, seed, n_random=64):
    """The first and last 64 rows of a [n_rows, width] tensor, those holding elements 2^30 .. 2^33 and their neighbours,
    and n_random seeded rows."""
    rows = set(range(64)) | set(range(n_rows - 64, n_rows))
    for e in (2 ** 30, 2 ** 31, 2 ** 32, 2 ** 33):
        rows |= {e // width - 1, e // width, e // width + 1}
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, n_rows, (n_random,), generator=g).tolist())
    return torch.tensor(sorted(r for r in rows if 0 <= r < n_rows), dtype=torch.long)


@pytest.fixture(autouse=True)
def _give_back_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def test_iid_at_48mp():
    """First in the file: its own engine needs the card before the module's engine holds a 48 MP workspace, and
    before the float64 conv references below load their libraries' kernels."""
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
    out = pipe(_photo(H48, W48), ensemble_size=1, generator=torch.Generator(device="cuda").manual_seed(0),
               show_progress_bar=False)
    assert out.is_complete
    for name in names:
        assert out[name].array.shape == (3, H48, W48) and np.isfinite(out[name].array).all()
    eng.close()


# ---- the two-launch GroupNorm ------------------------------------------------------------------------------------
# Before the module's engine: the largest runs here need the card before it holds a workspace.
def test_groupnorm_rows_past_2_33_elements():
    """[48.8M, 256] with a mean of 100: the strided [48.8M, 128] second halves first, then the whole rows with the
    shortcut's copy written over them, as the decoder runs them."""
    G, eps = 32, 1e-6
    g = torch.Generator(device="cuda").manual_seed(48)
    x = torch.randn(P48, 256, device="cuda", generator=g).mul_(2).add_(100.0)
    gamma, beta = torch.randn(256, device="cuda", generator=g), torch.randn(256, device="cuda", generator=g)
    assert x.numel() > 2 ** 33
    rows = _rows(P48, 256, seed=48).cuda()
    # second halves: [48.8M, 128] at a row stride of 256 floats
    mean, rstd = group_stats64(x[:, 128:], G, eps, chunk=1 << 18)
    y = groupnorm_rows(x[:, 128:], 128, 256, None, 0, gamma[128:], beta[128:], 1, P48, G, eps, 1)
    torch.cuda.synchronize()
    ref, bound = groupnorm_rows_ref(x[rows, 128:], mean, rstd, gamma[128:], beta[128:], G)
    R.assert_within(y[rows], ref, bound, "native_res_48mp/groupnorm_rows_c128_ld256/worst")
    del y
    # whole rows, in place
    mean, rstd = group_stats64(x, G, eps, chunk=1 << 18)
    xr = x[rows].clone()
    y = groupnorm_rows(x, 256, 256, x, 512, gamma, beta, 1, P48, G, eps, 1)
    torch.cuda.synchronize()
    ref, bound = groupnorm_rows_ref(xr, mean, rstd, gamma, beta, G)
    R.assert_within(y[rows], ref, bound, "native_res_48mp/groupnorm_rows_c256_in_place/worst")
    raw = x.view(torch.bfloat16).view(P48, 512)[:, :256]
    assert torch.equal(raw[rows], xr.to(torch.bfloat16))


def conv_strided(x, x2, ld2, wp, bias, out_ptr, ldo, H, W, Cin, Cin2, Cout):
    """The conv of the in-place resnet (mgb_debug_conv2d_strided): fp32 output at out_ptr with a row stride of ldo
    floats, shortcut operand x2 (or None) at a pixel stride of ld2 elements."""
    from marigold_b200 import _lib
    from marigold_b200.ops import ptr, stream_ptr

    f = _hook("mgb_debug_conv2d_strided", C.c_int32,
              [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int32] * 7 + [C.c_void_p])
    x2_p = None if x2 is None else C.c_void_p(x2.data_ptr())
    _lib.check(f(ptr(x), x2_p, ld2, ptr(wp), ptr(bias), C.c_void_p(out_ptr), ldo, 1, H, W, Cin, Cin2, Cout,
                 stream_ptr()), "mgb_debug_conv2d_strided")


@pytest.mark.parametrize("stage", ["conv1", "conv2_shortcut"])
def test_in_place_convs_past_2_33_elements(stage):
    """The two convs of the in-place resnet at 8064 x 6048 in its layout, over one [48.8M, 256] fp32 buffer: conv1
    (256 -> 128) into the second half of each row; conv2 (128 + 256 -> 128) reading the shortcut's bf16 operand from the
    first half of each row (1024-byte pixel stride) and writing the second half. Image rows holding elements 2^30 ..
    2^33 of the buffer, as fp32 and as bf16, and the first and last rows, against float64 with tests/ops_ref.py's conv
    bound."""
    from marigold_b200 import ops
    from tests.test_native_res_24mp_gpu import conv_row_ref

    Cin, Cin2, Cout = (256, 0, 128) if stage == "conv1" else (128, 256, 128)
    K = 9 * Cin + Cin2
    g = torch.Generator(device="cuda").manual_seed(K)
    buf = torch.empty(P48, 256, device="cuda")
    raw = None
    if Cin2:
        raw = buf.view(torch.bfloat16).view(1, H48, W48, 512)[..., :256]
        rv = raw.view(P48, 256)
        for a in range(0, P48, 1 << 22):
            rv[a:a + (1 << 22)] = torch.randn(min(1 << 22, P48 - a), 256, device="cuda", generator=g,
                                              dtype=torch.bfloat16)
    x = torch.randn(1, H48, W48, Cin, device="cuda", generator=g, dtype=torch.bfloat16)
    wb = (torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    wsc = (torch.randn(Cout, Cin2, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16) if Cin2 else None
    b = torch.randn(Cout, device="cuda", generator=g)
    wp = ops.pack_conv_weight(wb)
    if Cin2:
        wp = torch.cat([wp, wsc], dim=1).contiguous()
    conv_strided(x, raw, 512, wp, b, buf.data_ptr() + 128 * 4, 256, H48, W48, Cin, Cin2, Cout)
    torch.cuda.synchronize()
    out = buf.view(1, H48, W48, 256)[..., 128:]
    rows = set()
    for width in (W48 * 256, W48 * 512):
        rows |= set(_rows(H48, width, seed=K, n_random=0).tolist())
    rows |= set(torch.randint(0, H48, (4,), generator=torch.Generator().manual_seed(K)).tolist())
    worst = 0.0
    for y in sorted(rows):
        ref, bound = conv_row_ref(x, wb, y, b, raw, wsc)
        r = R.within(out[0, y], ref, bound)
        assert not r["nan"] and r["worst"] <= 1.0, (y, r)
        worst = max(worst, r["worst"])
    record(f"native_res_48mp/in_place_{stage}/worst", worst)


@pytest.mark.parametrize("NB,HW", [(1, 1920 * 1080), (2, 1000 * 744), (1, 4099)])
def test_groupnorm_rows_equal_fused(NB, HW):
    """Bit for bit the fused GroupNorm's operand and raw copy (mgb_op_groupnorm_ex): in place over 256 channels, and
    over 128 channels at a row stride of 256."""
    from marigold_b200 import ops

    G, eps = 32, 1e-6
    g = torch.Generator(device="cuda").manual_seed(NB * HW)
    x = torch.randn(NB * HW, 256, device="cuda", generator=g).mul_(3).add_(1.0)
    gamma, beta = torch.randn(256, device="cuda", generator=g), torch.randn(256, device="cuda", generator=g)
    half = x[:, 128:].contiguous()
    y_ref, _ = ops.groupnorm_ex(half.view(NB, HW, 128), None, gamma[128:], beta[128:], NB, HW, G, eps, 1)
    y = groupnorm_rows(x[:, 128:], 128, 256, None, 0, gamma[128:], beta[128:], NB, HW, G, eps, 1)
    assert torch.equal(y, y_ref.view(NB * HW, 128))
    y_ref, raw_ref = ops.groupnorm_ex(x.view(NB, HW, 256), None, gamma, beta, NB, HW, G, eps, 1, raw_copy=True)
    y = groupnorm_rows(x, 256, 256, x, 512, gamma, beta, NB, HW, G, eps, 1)
    torch.cuda.synchronize()
    assert torch.equal(y, y_ref.view(NB * HW, 256))
    assert torch.equal(x.view(torch.bfloat16).view(NB * HW, 512)[:, :256], raw_ref.view(NB * HW, 256))


@pytest.fixture(scope="module")
def models():
    return oracle_models("full")


@pytest.fixture(scope="module")
def engine(models):
    eng = engine_from_oracle(*models)
    yield eng
    set_low_memory(eng, 0)
    eng.close()


# ---- plans -------------------------------------------------------------------------------------------------------
def test_48mp_plan(engine):
    set_low_memory(engine, 0)
    U = P48 * U_PER_PIXEL
    lh, lw = H48 // 8, W48 // 8
    nbytes, t0, t1, off = arena_plan(engine, 2, 1, lh, lw)
    assert (off % 1024 == 0).all()
    assert no_overlap(nbytes, t0, t1, off)
    peak = int((off + nbytes).max())
    record("native_res_48mp/plan_peak_over_U/decode", peak / U)
    assert peak <= 3 * U + SCRATCH, peak / U
    assert arena_place(nbytes, t0, t1)[1].tolist() == off.tolist()
    assert arena_plan(engine, 2, 1, lh, lw)[3].tolist() == off.tolist()
    # the library's rule chose the in-place resnet: the plan is the forced one
    set_low_memory(engine, 1)
    try:
        assert [a.tolist() for a in arena_plan(engine, 2, 1, lh, lw)] == [a.tolist() for a in (nbytes, t0, t1, off)]
    finally:
        set_low_memory(engine, 0)
    enc = arena_plan(engine, 1, 1, H48, W48)
    record("native_res_48mp/plan_peak_over_U/encode", int((enc[3] + enc[0]).max()) / U)
    from marigold_b200.pipeline import call_reserve_bytes

    need = engine.workspace_bytes(1, H48, W48)
    record("native_res_48mp/workspace_bytes", need)
    total = torch.cuda.get_device_properties(0).total_memory
    assert need + call_reserve_bytes(H48, W48, 2, 1) + sum(_weight_bytes(engine)) < total, (need, total)


@pytest.mark.parametrize("NB,h,w", [(1, 4032, 6048), (1, 768, 768), (2, 768, 768)])
def test_plans_unchanged_where_the_default_fits(engine, NB, h, w):
    plans, need = {}, {}
    for mode in (0, -1):
        set_low_memory(engine, mode)
        plans[mode] = [a.tolist() for a in arena_plan(engine, 2, NB, h // 8, w // 8)]
        need[mode] = engine.workspace_bytes(NB, h, w)
    set_low_memory(engine, 0)
    assert plans[0] == plans[-1]
    assert need[0] == need[-1] > 0


# ---- the same bits -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NB", [1, 2])
@pytest.mark.parametrize("h,w", [(1080, 1920), (744, 1000)])
def test_in_place_decode_is_bit_identical(engine, NB, h, w):
    lh, lw = h // 8, w // 8
    lat = torch.randn(NB, 4, lh, lw, generator=torch.Generator().manual_seed(NB * h + w)).cuda()
    try:
        for mode in (0, 1, 2):            # depth, normals, raw 3-channel
            set_low_memory(engine, -1)
            ref = engine.decode(lat, mode)
            set_low_memory(engine, 1)
            out = engine.decode(lat, mode)
            assert torch.isfinite(ref).all()
            assert (out - ref).abs().max().item() == 0.0, mode
            if mode == 2:
                for poison, placement in ((True, 0), (True, 1)):
                    set_arena(engine, poison, placement)
                    assert torch.equal(engine.decode(lat, mode), ref), (poison, placement)
                set_arena(engine)
    finally:
        set_arena(engine)
        set_low_memory(engine, 0)
    record(f"native_res_48mp/in_place_vs_default/{w}x{h}_nb{NB}/max_abs_diff", 0.0)


def test_in_place_plan_at_24mp(engine):
    """Forced at 6048 x 4032 the in-place plan is 3 U too, and overlaps nothing."""
    set_low_memory(engine, 1)
    try:
        nbytes, t0, t1, off = arena_plan(engine, 2, 1, 504, 756)
    finally:
        set_low_memory(engine, 0)
    U = 4032 * 6048 * U_PER_PIXEL
    assert no_overlap(nbytes, t0, t1, off)
    assert int((off + nbytes).max()) <= 3 * U + SCRATCH


# ---- the pipelines at 48 MP --------------------------------------------------------------------------------------
def test_depth_and_normals_at_48mp(models, engine):
    from marigold_b200.pipeline import MarigoldDepthPipeline, MarigoldNormalsPipeline
    from marigold_b200.schedulers import DDIMScheduler

    text = models[2]
    img = _photo(H48, W48)
    pipe = MarigoldDepthPipeline(engine, DDIMScheduler(), text, default_denoising_steps=1,
                                 default_processing_resolution=0)
    out = pipe(img, ensemble_size=1, generator=torch.Generator(device="cuda").manual_seed(0), color_map=None,
               show_progress_bar=False)
    assert out.depth_np.shape == (H48, W48) and np.isfinite(out.depth_np).all()
    del out
    out = pipe(img, ensemble_size=2, generator=torch.Generator(device="cuda").manual_seed(0), color_map=None,
               show_progress_bar=False, ensemble_kwargs={"output_uncertainty": True})
    assert out.depth_np.shape == (H48, W48) and np.isfinite(out.depth_np).all()
    assert out.uncertainty is not None and out.uncertainty.shape == (H48, W48) and np.isfinite(out.uncertainty).all()
    del out
    npipe = MarigoldNormalsPipeline(engine, DDIMScheduler(), text, default_denoising_steps=1,
                                    default_processing_resolution=0)
    nout = npipe(img, ensemble_size=1, generator=torch.Generator(device="cuda").manual_seed(0), show_progress_bar=False)
    assert nout.normals_np.shape == (3, H48, W48) and np.isfinite(nout.normals_np).all()


def test_select_batch_size_at_45mp(engine):
    from marigold_b200.pipeline import call_reserve_bytes, select_batch_size

    gc.collect()
    torch.cuda.empty_cache()
    for h, w in ((5152, 7728), (5464, 8192), (5504, 8256)):     # 39.8, 44.8 and 45.4 MP
        assert select_batch_size(engine, 1, h, w, reserve_bytes=call_reserve_bytes(h, w, 1, 1)) == 1
    # reported, not asserted: 8160 x 6144 (50.1 MP)
    h, w = 6144, 8160
    need = engine.workspace_bytes(1, h, w)
    try:
        fits = select_batch_size(engine, 1, h, w, reserve_bytes=call_reserve_bytes(h, w, 1, 1)) == 1
    except ValueError:
        fits = False
    record("native_res_48mp/workspace_bytes_8160x6144", need)
    record("native_res_48mp/fits_8160x6144", float(fits))
    weights = sum(_weight_bytes(engine))
    print(f"8160 x 6144: workspace {need} B, weights {weights} B, fits: {fits}")
