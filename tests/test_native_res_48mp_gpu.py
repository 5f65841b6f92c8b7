"""45-48-megapixel photos (`-m gpu`): the library's rule runs the decoder's full-resolution stage in low memory
(net.cu, up_conv_low_memory and resnet_shortcut_halves) where one member's default decode does not fit (U = one fp32
128-channel map at full resolution, 512 bytes per pixel; 25.0 GB at 8064 x 6048).

  * the plans: at 8064 x 6048 the decoder's peak is 2.5 U (plus the GroupNorm scratch), no two buffers live at once
    share a byte, the plan is its own lifetimes' placement on every call, and the library's rule gives the forced plan;
    at 6048 x 4032 and 768 x 768 the rule keeps the default path, so plans and workspace bytes are those of a handle
    that never runs in low memory;
  * the pipelines at processing_res=0 on an 8064 x 6048 photo: depth with E = 1 and with E = 2 and uncertainty, normals
    with E = 1, a 2-target IID model with E = 1; select_batch_size takes one member at 7728 x 5152 (just past the
    default path's limit), 8192 x 5464 and 8256 x 5504;
  * the two convs of that stage's resnet at 8064 x 6048 on packed operands (conv1; conv2 with the shortcut's
    [48.8M, 256] bf16 operand) against float64 on rows holding elements 2^30 .. 2^33."""
import gc

import numpy as np
import pytest
import torch

from tests import ops_ref as R
from tests.helpers import (U_PER_PIXEL, _photo, _rows, arena_place, arena_plan, conv_row_ref, engine_from_oracle,
                           no_overlap, oracle_models, record, set_low_memory, weight_bytes)

pytestmark = pytest.mark.gpu

H48, W48 = 6048, 8064
P48 = H48 * W48            # 48 771 072 pixels
SCRATCH = 1 << 20          # bytes of GroupNorm partials and statistics live beside the 2.5 U at the decoder's peak


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


# Before the module's engine: conv2's operands and output take 62 GB of the card.
@pytest.mark.parametrize("stage", ["conv1", "conv2_shortcut"])
def test_resnet_convs_past_2_33_elements(stage):
    """The two convs of resnet_shortcut_halves at 8064 x 6048 on packed operands: conv1 (256 -> 128), and conv2
    (128 + 256 -> 128) reading the shortcut's [48.8M, 256] bf16 operand. Image rows holding elements 2^30 .. 2^33 of
    each operand and of the output, and the first and last rows, against float64 with tests/ops_ref.py's conv bound."""
    from marigold_b200 import ops
    Cin, Cin2, Cout = (256, 0, 128) if stage == "conv1" else (128, 256, 128)
    K = 9 * Cin + Cin2
    g = torch.Generator(device="cuda").manual_seed(K)
    x = torch.randn(1, H48, W48, Cin, device="cuda", generator=g, dtype=torch.bfloat16)
    x2 = torch.randn(1, H48, W48, Cin2, device="cuda", generator=g, dtype=torch.bfloat16) if Cin2 else None
    wb = (torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    wsc = (torch.randn(Cout, Cin2, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16) if Cin2 else None
    b = torch.randn(Cout, device="cuda", generator=g)
    wp = ops.pack_conv_weight(wb)
    if Cin2:
        wp = torch.cat([wp, wsc], dim=1).contiguous()
    out = torch.empty(1, H48, W48, Cout, device="cuda")
    ops.conv2d_ex(x, wp, b, 1, H48, W48, Cin, Cout, x2=x2, Cin2=Cin2, out=out)
    torch.cuda.synchronize()
    rows = set()
    for c in (Cin, Cin2, Cout):
        if c:
            rows |= set(_rows(H48, W48 * c, seed=K, n_random=0).tolist())
    rows |= set(torch.randint(0, H48, (4,), generator=torch.Generator().manual_seed(K)).tolist())
    worst = 0.0
    for y in sorted(rows):
        ref, bound = conv_row_ref(x, wb, y, b, x2, wsc)
        r = R.within(out[0, y], ref, bound)
        assert not r["nan"] and r["worst"] <= 1.0, (y, r)
        worst = max(worst, r["worst"])
    record(f"native_res_48mp/resnet_{stage}/worst", worst)


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
    assert peak <= 2.5 * U + SCRATCH, peak / U
    assert arena_place(nbytes, t0, t1)[1].tolist() == off.tolist()
    assert arena_plan(engine, 2, 1, lh, lw)[3].tolist() == off.tolist()
    # the library's rule chose the low-memory stage: the plan is the forced one
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
    assert need + call_reserve_bytes(H48, W48, 2, 1) + weight_bytes(engine) < total, (need, total)


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
    weights = weight_bytes(engine)
    print(f"8160 x 6144: workspace {need} B, weights {weights} B, fits: {fits}")
