"""Device LPIPS with the VGG16 and SqueezeNet 1.1 backbones (`-m gpu`): every step of evaluate_iid(..., lpips=...)
recomputed from the device's own input of that step (each conv, the squeeze's stride-2 conv1 included, held to the
float64 bound of tests/ops_ref.py; each pool bit for bit), the scalar against the float64 restatement that rounds where
the kernels round and against torchvision's float32 module (tests/lpips_nets_ref.py), exact properties, launch counts,
errors before any launch and the weight handle's memory."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import lpips_nets_ref, lpips_ref, ops_ref
from tests.helpers import CONFIGS, _inputs, _launches, live_device_bytes

pytestmark = pytest.mark.gpu
pytest.importorskip("torchvision")
NETS = ["vgg", "squeeze"]
MIN = {"vgg": 16, "squeeze": 17}
HEAD_TOL = 1e-6
# |lpips - restatement|, (against the float64 restatement that rounds where the kernels round, against torchvision's
# float32 module with TF32 off). Measured on an H100 80GB HBM3 (700 W power limit) over the test_scalar cases: VGG16 at
# most 1.4e-5 and 8.0e-5, SqueezeNet 1.1 at most 9.2e-5 and 2.3e-3. Unlike AlexNet's (4.1e-7), the float64 gap is not
# the head's: 8 of VGG16's 13 convolutions and 18 of SqueezeNet's 25 write only a bf16 operand, and where the device's
# fp32 accumulation error straddles a bf16 rounding boundary that element moves by one bf16 ulp, which no float64
# restatement can follow; every step is held to its own bound in test_steps_layer_local. The tolerances leave a margin
# of about 3x (float64) and 2x to 6x (float32).
SCALAR_TOL = {"vgg": (5e-5, 5e-4), "squeeze": (3e-4, 5e-3)}
# 81 x 146: SqueezeNet's three ceil-mode pools see even inputs (40 / 20 / 10 rows, 72 / 36 / 18 columns), so each has a
# partial last window in both dimensions; at the minimum size 17 they see 8 / 4 / 2. 77 x 131: odd extents, which VGG's
# floor-mode pools crop.
PARTIAL = (81, 146)
SIZES = {n: [(MIN[n], MIN[n]), (77, 131), PARTIAL, (480, 640), (1080, 1920)] for n in NETS}
OPS = {0: "conv", 1: "pool2", 2: "pool3", 3: "pool3_ceil"}


@pytest.fixture(scope="module", autouse=True)
def _give_back_memory():
    """The float64 restatements at 1080 x 1920 pass through tens of GB of torch's cache. Return it when the module ends, so
    that the tests after it, which size their batches by the free device memory, see the card as this module found it."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=NETS)
def net(request):
    from marigold_b200.evaluation import LPIPS

    net_type = request.param
    sd, lin = lpips_nets_ref.fabricated_weights(net_type, 0)
    h = LPIPS(sd, lin, device="cuda", net_type=net_type)
    ns = {"type": net_type, "sd": sd, "lin": lin, "lp": h,
          "r64": lpips_nets_ref.NetRound64(net_type, sd, lin, device="cuda"),
          "r32": lpips_nets_ref.Net32(net_type, sd, lin)}
    yield ns
    h.close()


def _eval(pred, gt, target, mask, transform, lp):
    from marigold_b200.evaluation import evaluate_iid

    return evaluate_iid(pred, gt, target, mask, transform, lpips=lp)


def _step(lp, H, W, s, copy=True):
    """(info dict, the bf16 output buffer of step s as float64 NHWC [2, h, w, ldo] or None)."""
    from marigold_b200 import _lib

    fn = _lib.load().mgb_debug_lpips_step
    info = (C.c_int32 * 11)()
    _lib.check(fn(lp._h, _lib.ptr(lp._ws), H, W, s, None, info), "mgb_debug_lpips_step")
    d = dict(zip(("op", "in", "buf", "col", "conv", "kind", "tap", "h", "w", "ldo", "nsteps"), list(info)))
    if not copy:
        return d, None
    planes = 4 if s < 0 and lp.net_type == "squeeze" else 1
    t = torch.empty(2 * planes, d["h"], d["w"], d["ldo"], device="cuda", dtype=torch.bfloat16)
    if fn(lp._h, _lib.ptr(lp._ws), H, W, s, _lib.ptr(t), info) != 0:
        return d, None
    return d, t.to(torch.float64)


def _features(lp, H, W, layer):
    from marigold_b200 import _lib

    fn = _lib.load().mgb_debug_lpips_net_features
    dims = (C.c_int32 * 3)()
    _lib.check(fn(lp._h, _lib.ptr(lp._ws), H, W, layer, None, dims), "mgb_debug_lpips_net_features")
    t = torch.empty(2, dims[0], dims[1], dims[2], device="cuda")
    _lib.check(fn(lp._h, _lib.ptr(lp._ws), H, W, layer, _lib.ptr(t), dims), "mgb_debug_lpips_net_features")
    return t.to(torch.float64)


def _prep_nchw(lp, x, H, W):
    """The prep operand's three colour channels as NCHW [2, 3, H, W]; the parity planes of SqueezeNet reassembled."""
    if lp.net_type != "squeeze":
        return x[..., :3].permute(0, 3, 1, 2)
    hs, ws = x.shape[1], x.shape[2]
    planes = x.reshape(2, 2, 2, hs, ws, 64)[..., :3]                     # [map, py, px, i, j, c]
    full = planes.permute(0, 5, 3, 1, 4, 2).reshape(2, 3, 2 * hs, 2 * ws)
    return full[:, :, :H, :W]


def _conv_modules(net_type, sd):
    """Conv index -> (bf16-rounded float64 weight, fp32 bias as float64, stride, padding), in the device's order."""
    from marigold_b200.evaluation import LPIPS_NETS

    out = []
    for key, shape in LPIPS_NETS[net_type][2]:
        w = lpips_ref.bf16(sd[f"{key}.weight"].to("cuda", torch.float64))
        b = sd[f"{key}.bias"].to("cuda", torch.float32).to(torch.float64)
        stride, pad = (2, 0) if net_type == "squeeze" and key == "features.0" else (1, (shape[2] - 1) // 2)
        out.append((w, b, stride, pad))
    return out


# ---- every step, from the device's own input ----------------------------------------------------------------------------
def _check_steps(ns, H, W):
    lp, net_type = ns["lp"], ns["type"]
    pred, gt, mask = _inputs(H, W, "albedo", "pixel", None, "noisy")
    got, _ = _eval(pred, gt, "albedo", mask, None, lp)
    p, g, _ = lpips_ref.metric_maps(pred, gt, "albedo", mask)
    ref_in = lpips_ref.bf16(lpips_ref.scaled_input(torch.cat([p, g])).to(torch.float64))
    _, pre = _step(lp, H, W, -1)
    x0 = _prep_nchw(lp, pre, H, W)
    ops_ref.assert_within(x0, ref_in, ops_ref.U_BF16 * ref_in.abs() + ops_ref.TINY, f"lpips_{net_type}_prep_{H}x{W}")
    assert (pre[..., 3:] == 0).all()
    convs, keys = _conv_modules(net_type, ns["sd"]), lpips_nets_ref.conv_keys(net_type)
    nsteps = _step(lp, H, W, 0, copy=False)[0]["nsteps"]
    last_read = {}                                                         # step -> the last step that reads its output
    for s in range(nsteps):
        last_read[_step(lp, H, W, s, copy=False)[0]["in"]] = s
    outs, ntaps = {}, 0
    for s in range(nsteps):
        for done in [t for t in outs if last_read.get(t, -1) < s]:        # hold only the outputs still to be read
            del outs[done]
        d, y = _step(lp, H, W, s)
        src = x0 if d["in"] < 0 else outs[d["in"]]
        name = f"lpips_{net_type}_step{s}_{OPS[d['op']]}_{H}x{W}"
        if d["op"] != 0:                                                   # pools: exact on the device's own input
            k = 2 if d["op"] == 1 else 3
            ref = F.max_pool2d(src, k, 2, ceil_mode=d["op"] == 3)
            assert y is not None and y.permute(0, 3, 1, 2).shape == ref.shape, (name, y.shape, ref.shape)
            assert torch.equal(y.permute(0, 3, 1, 2), ref), name
            outs[s] = ref
            continue
        w, b, stride, pad = convs[d["conv"]]
        xin = src[:, :w.shape[1]]
        pre, absprod = ops_ref.conv64(xin, w, stride=stride, padding=pad)
        pre = pre + b[None, :, None, None]
        ref = torch.relu(pre)
        # the GEMM's K, padded channels included: the accumulator is rounded at every MMA step, zero products or not
        K = w.shape[2] * w.shape[3] * ((w.shape[1] + 63) // 64 * 64)
        c0, c1 = d["col"], d["col"] + w.shape[0]
        if y is not None:
            got_b = y.permute(0, 3, 1, 2)
            assert got_b.shape[-2:] == ref.shape[-2:], (name, got_b.shape, ref.shape)
            ops_ref.assert_within(got_b[:, c0:c1], ref, ops_ref.gemm_bound(K, absprod, ref, True, pre=pre.abs()),
                                  name + "_bf16")
            if keys[d["conv"]].endswith("squeeze"):                    # its padded columns: ReLU(0 + 0)
                assert d["ldo"] == 64 and (got_b[:, w.shape[0]:] == 0).all(), name
            if d["buf"] == s:
                outs[s] = got_b
        if d["tap"] >= 0:
            f = _features(lp, H, W, d["tap"]).permute(0, 3, 1, 2)
            assert f.shape[-2:] == ref.shape[-2:], (name, f.shape, ref.shape)
            ops_ref.assert_within(f[:, c0:c1], ref, ops_ref.gemm_bound(K, absprod, ref, False, pre=pre.abs()),
                                  name + "_f32")
            ntaps += d["buf"] == s
    L = len(lpips_nets_ref.CHANNELS[net_type])
    assert ntaps == L
    feats = [_features(lp, H, W, l).permute(0, 3, 1, 2) for l in range(L)]
    assert [f.shape[1] for f in feats] == list(lpips_nets_ref.CHANNELS[net_type])
    head = ns["r64"].head([f[:1] for f in feats], [f[1:] for f in feats])
    assert abs(got["lpips"] - head) <= HEAD_TOL * abs(head) + 1e-12, (got["lpips"], head)


@pytest.mark.parametrize("size", range(5), ids=["min", "77x131", "81x146", "480x640", "1080x1920"])
def test_steps_layer_local(net, size):
    H, W = SIZES[net["type"]][size]
    _check_steps(net, H, W)


# ---- the scalar ---------------------------------------------------------------------------------------------------------
def _check_scalar(ns, pred, gt, target, mask, transform, tag):
    got, info = _eval(pred, gt, target, mask, transform, ns["lp"])
    p, g, _ = lpips_ref.metric_maps(pred, gt, target, mask, transform, scale=info["scale"])
    r64 = ns["r64"](p, g)
    with torch.backends.cudnn.flags(allow_tf32=False):
        r32 = float(ns["r32"](p, g))
    d64 = ops_ref.record(f"lpips_{ns['type']}_scalar_vs_f64_{tag}", abs(got["lpips"] - r64))
    d32 = ops_ref.record(f"lpips_{ns['type']}_scalar_vs_f32_{tag}", abs(got["lpips"] - r32))
    tol64, tol32 = SCALAR_TOL[ns["type"]]
    assert d64 <= tol64 and d32 <= tol32, (got["lpips"], r64, r32)
    return got


@pytest.mark.parametrize("size", range(4), ids=["min", "77x131", "81x146", "480x640"])
@pytest.mark.parametrize("target,mask,transform,kind", CONFIGS)
def test_scalar(net, size, target, mask, transform, kind):
    H, W = SIZES[net["type"]][size]
    pred, gt, m = _inputs(H, W, target, mask, transform, kind)
    got = _check_scalar(net, pred, gt, target, m, transform, f"{target}_{mask}_{transform}_{kind}_{H}x{W}")
    if kind == "dark":                                     # k = 0: both maps 0
        assert got["lpips"] == 0.0


def test_scalar_full_hd(net):
    pred, gt, m = _inputs(1080, 1920, "shading", "pixel", None, "noisy")
    _check_scalar(net, pred, gt, "shading", m, None, "shading_pixel_1080x1920")


# ---- exact properties, unchanged PSNR / SSIM, launch counts ------------------------------------------------------------
@pytest.mark.parametrize("mask", ["none", "pixel"])
def test_exact_properties(net, mask):
    lp = net["lp"]
    for H, W in [(MIN[net["type"]], MIN[net["type"]] + 3), PARTIAL]:
        pred, gt, m = _inputs(H, W, "albedo", mask, None, "noisy")
        a, _ = _eval(pred, gt, "albedo", m, None, lp)
        b, _ = _eval(pred, gt, "albedo", m, None, lp)
        c, _ = _eval(gt, pred, "albedo", m, None, lp)
        z, _ = _eval(gt, gt.clone(), "albedo", m, None, lp)
        assert a["lpips"] > 0
        assert np.float64(a["lpips"]).tobytes() == np.float64(b["lpips"]).tobytes() == np.float64(c["lpips"]).tobytes()
        assert z["lpips"] == 0.0


@pytest.mark.parametrize("size", range(5), ids=["min", "77x131", "81x146", "480x640", "1080x1920"])
@pytest.mark.parametrize("target", ["albedo", "shading"])
def test_psnr_ssim_unchanged_and_launches(net, size, target):
    from marigold_b200.evaluation import evaluate_iid

    H, W = SIZES[net["type"]][size]
    pred, gt, m = _inputs(H, W, target, "pixel", None, "noisy")
    (plain, pinfo), n_plain = _launches(lambda: evaluate_iid(pred, gt, target, m))
    (with_lp, info), n_lp = _launches(lambda: _eval(pred, gt, target, m, None, net["lp"]))
    (again, _), n_again = _launches(lambda: _eval(pred, gt, target, m, None, net["lp"]))
    assert set(plain) == {"psnr", "ssim"} and set(with_lp) == {"psnr", "ssim", "lpips"}
    for k in ("psnr", "ssim"):
        assert np.float64(plain[k]).tobytes() == np.float64(with_lp[k]).tobytes(), k
    assert repr(pinfo) == repr(info)
    assert np.float64(with_lp["lpips"]).tobytes() == np.float64(again["lpips"]).tobytes()
    # prep, every conv (+ a split-K reduce where split), every pool, head, final
    nconv, npool = {"vgg": (13, 4), "squeeze": (25, 3)}[net["type"]]
    delta = ops_ref.record(f"lpips_{net['type']}_launch_delta_{target}_{H}x{W}", n_lp - n_plain)
    assert n_again == n_lp
    assert 3 + nconv + npool <= delta <= 3 + 2 * nconv + npool, delta


# ---- errors before any launch, the handle -------------------------------------------------------------------------------
def test_errors_before_launch(net):
    from marigold_b200 import _lib
    from marigold_b200.evaluation import LPIPS

    lib = _lib.load()
    n = MIN[net["type"]]
    l0 = lib.mgb_launch_count()
    for H, W in [(n - 1, 40), (40, n - 1)]:
        pred, gt, m = _inputs(H, W, "albedo", "pixel", None, "noisy")
        torch.cuda.synchronize()
        l0 = lib.mgb_launch_count()
        with pytest.raises(ValueError, match=f">= {n}"):
            _eval(pred, gt, "albedo", m, None, net["lp"])
        assert lib.mgb_launch_count() == l0
    with pytest.raises(ValueError, match="net_type"):
        LPIPS(net["sd"], net["lin"], net_type="alexnet")
    missing = {k: v for k, v in net["sd"].items() if not k.endswith(".bias")}
    with pytest.raises(ValueError, match="bias"):
        LPIPS(missing, net["lin"], net_type=net["type"])
    assert lib.mgb_launch_count() == l0
    h = LPIPS(net["sd"], net["lin"], device="cuda", net_type=net["type"])
    h.close()
    pred, gt, m = _inputs(40, 40, "albedo", "pixel", None, "noisy")
    torch.cuda.synchronize()
    l0 = lib.mgb_launch_count()
    with pytest.raises(ValueError, match="closed"):
        _eval(pred, gt, "albedo", m, None, h)
    assert lib.mgb_launch_count() == l0


@pytest.mark.parametrize("net_type", NETS)
def test_handle_memory(net_type):
    from marigold_b200 import _lib
    from marigold_b200.evaluation import LPIPS, LPIPS_NETS

    fn = live_device_bytes
    sd, lin = lpips_nets_ref.fabricated_weights(net_type, 0)
    b0 = fn()
    h = LPIPS(sd, lin, device="cuda", net_type=net_type)
    want = 0
    for key, (co, ci, k, _) in LPIPS_NETS[net_type][2]:
        n = 64 if key.endswith("squeeze") else co              # a Fire squeeze: 64 GEMM columns
        want += 2 * n * k * k * ((ci + 63) // 64 * 64) + 4 * n
    want += 4 * sum(lpips_nets_ref.CHANNELS[net_type])
    assert fn() - b0 == want
    h.close()
    assert fn() == b0
    _lib.load()


def test_alex_default_unchanged():
    """net_type defaults to "alex": the same handle layout and workspace as before the other nets."""
    from marigold_b200 import _lib
    from marigold_b200.evaluation import LPIPS

    sd, lin = lpips_ref.fabricated_weights(0)
    a, b = LPIPS(sd, lin, device="cuda"), LPIPS(sd, lin, device="cuda", net_type="alex")
    try:
        lib = _lib.load()
        assert a.net_type == "alex" and a.min_size == 31
        for H, W in [(31, 31), (480, 640)]:
            assert lib.mgb_lpips_ws_bytes_h(a._h, H, W) == lib.mgb_lpips_ws_bytes(H, W) > 0
        pred, gt, m = _inputs(77, 131, "albedo", "pixel", None, "noisy")
        ra, _ = _eval(pred, gt, "albedo", m, None, a)
        rb, _ = _eval(pred, gt, "albedo", m, None, b)
        assert np.float64(ra["lpips"]).tobytes() == np.float64(rb["lpips"]).tobytes()
    finally:
        a.close()
        b.close()
