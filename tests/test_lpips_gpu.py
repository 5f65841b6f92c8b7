"""Device LPIPS (`-m gpu`): the new implicit-GEMM conv kinds and the ReLU epilogue against the float64 bounds of
tests/ops_ref.py; every AlexNet layer of evaluate_iid(..., lpips=...) through mgb_debug_lpips_features, each recomputed
in float64 from the device's previous-layer output; the scalar against the float64 restatement that rounds where the
kernels round and against the reference's float32 arithmetic (tests/lpips_ref.py); exact properties, errors, launch
counts and the weight handle's memory."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import iid_eval_ref, lpips_ref, ops_ref
from tests.helpers import CONFIGS, _inputs, _launches, live_device_bytes

pytestmark = pytest.mark.gpu
pytest.importorskip("torchvision")
SEED = 0
IID_LAUNCHES = {False: 2, True: 6}
# |lpips - restatement|. Measured on an H100 80GB HBM3 (700 W power limit) over these cases: at most 4.1e-7 against the
# float64 restatement that rounds where the kernels round, and 8.9e-5 against the reference's float32 arithmetic (TF32
# off). SCALAR_TOL_64 leaves a margin of 12x; SCALAR_TOL_32 is the design target, half the last of the three decimals
# LPIPS is usually reported to.
SCALAR_TOL_64, SCALAR_TOL_32 = 5e-6, 5e-4
HEAD_TOL = 1e-6              # relative: the device head (double) against the float64 head on the device's own features
FEATURE_SIZES = [(31, 31), (77, 131), (481, 642), (480, 640), (1080, 1920)]


@pytest.fixture(scope="module")
def weights():
    return lpips_ref.fabricated_weights(SEED)


@pytest.fixture(scope="module")
def lp(weights):
    from marigold_b200.evaluation import LPIPS

    h = LPIPS(*weights, device="cuda")
    yield h
    h.close()


@pytest.fixture(scope="module")
def ref64(weights):
    return lpips_ref.Lpips64(*weights, device="cuda")


@pytest.fixture(scope="module")
def ref32(weights):
    return lpips_ref.Lpips32(*weights)


def _eval(pred, gt, target, mask, transform, lp):
    from marigold_b200.evaluation import evaluate_iid

    return evaluate_iid(pred, gt, target, mask, transform, lpips=lp)


def _debug_features(lp, H, W):
    """The five fp32 feature maps of the last call, NCHW float64 [2, C, h, w] (pred, gt)."""
    from marigold_b200 import _lib

    fn = _lib.load().mgb_debug_lpips_features
    dims = (C.c_int32 * 3)()
    out = []
    for l in range(5):
        _lib.check(fn(_lib.ptr(lp._ws), H, W, l, None, dims), "mgb_debug_lpips_features")
        t = torch.empty(2, dims[0], dims[1], dims[2], device="cuda")
        _lib.check(fn(_lib.ptr(lp._ws), H, W, l, _lib.ptr(t), dims), "mgb_debug_lpips_features")
        out.append(t.permute(0, 3, 1, 2).to(torch.float64))
    return out


# ---- the new conv kinds and EPI_RELU ---------------------------------------------------------------------------------
CONV_CASES = [  # kind, NB, Hout, Wout, Cin, Cout, splits, block_n
    (4, 2, 7, 9, 64, 64, 0, 0),
    (4, 1, 33, 45, 64, 64, 3, 0),
    (4, 2, 5, 6, 64, 16, 1, 16),
    (5, 2, 11, 13, 64, 192, 0, 0),
    (5, 1, 29, 37, 128, 96, 4, 0),
    (5, 2, 3, 3, 64, 192, 1, 64),
    (0, 2, 9, 14, 192, 384, 2, 0),
]


@pytest.mark.parametrize("kind,NB,H,W,Cin,Cout,splits,block_n", CONV_CASES)
def test_conv_kind_relu(kind, NB, H, W, Cin, Cout, splits, block_n):
    from marigold_b200 import _lib, ops

    g = torch.Generator(device="cuda").manual_seed(kind * 100 + H)
    k = 5 if kind == 5 else 3
    Hs, Ws = (H + 3, W + 2) if kind == 4 else (H, W)        # kind 4: a source one row taller than it reads
    x = torch.randn(NB, Hs, Ws, Cin, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (k * Cin ** 0.5)).to(torch.bfloat16).float()
    b = 0.3 * torch.randn(Cout, device="cuda", generator=g)
    out = torch.empty(NB, H, W, Cout, device="cuda")
    outb = torch.empty(NB, H, W, Cout, device="cuda", dtype=torch.bfloat16)
    ws = torch.empty(16 * NB * H * W * Cout, device="cuda")          # choose_tile splits at most 16 ways
    ops.conv2d_ex(x, ops.pack_conv_weight(w), b, NB, H, W, Cin, Cout, kind=kind, Hsrc=Hs if kind == 4 else 0,
                  Wsrc=Ws if kind == 4 else 0, out=out, out_bf16=outb, flags=_lib.EPI_RELU, block_n=block_n, splits=splits,
                  ws=ws)
    torch.cuda.synchronize()
    pad = 0 if kind == 4 else (k - 1) // 2
    ref, absprod = ops_ref.conv64(x.permute(0, 3, 1, 2), w, padding=pad)
    pre = ref[:, :, :H, :W] + b.double()[None, :, None, None]
    ref, absprod = torch.relu(pre), absprod[:, :, :H, :W]
    K = k * k * Cin
    name = f"lpips_conv_kind{kind}_{NB}x{H}x{W}x{Cin}x{Cout}_s{splits}_bn{block_n}"
    ops_ref.assert_within(out.permute(0, 3, 1, 2), ref, ops_ref.gemm_bound(K, absprod, ref, False, pre=pre.abs()), name)
    ops_ref.assert_within(outb.permute(0, 3, 1, 2), ref, ops_ref.gemm_bound(K, absprod, ref, True, pre=pre.abs()),
                          name + "_bf16")
    assert (out >= 0).all()


def test_conv_kind4_needs_the_source_extent():
    """Kind 4 is a valid (unpadded) conv only over a source two rows and columns larger than the output."""
    from marigold_b200 import _lib, ops

    x = torch.zeros(1, 9, 11, 64, device="cuda", dtype=torch.bfloat16)
    w = ops.pack_conv_weight(torch.zeros(64, 64, 3, 3, device="cuda"))
    b = torch.zeros(64, device="cuda")
    out = torch.empty(1, 7, 9, 64, device="cuda")
    l0 = _lib.load().mgb_launch_count()
    with pytest.raises(_lib.MgbError, match="kind 4"):
        ops.conv2d(x, w, b, 1, 7, 9, 64, 64, kind=4)
    with pytest.raises(_lib.MgbError, match="kind 4"):
        ops.conv2d_ex(x, w, b, 1, 7, 9, 64, 64, kind=4, Hsrc=8, Wsrc=11, out=out)
    assert _lib.load().mgb_launch_count() == l0
    ops.conv2d_ex(x, w, b, 1, 7, 9, 64, 64, kind=4, Hsrc=9, Wsrc=11, out=out)
    torch.cuda.synchronize()


# ---- per layer --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", FEATURE_SIZES)
def test_features_layer_local(H, W, lp, ref64):
    pred, gt, mask = _inputs(H, W, "albedo", "pixel", None, "noisy")
    got, _ = _eval(pred, gt, "albedo", mask, None, lp)
    feats = _debug_features(lp, H, W)
    assert feats[0].shape[-2:] == ((H - 3) // 4, (W - 3) // 4)
    p, g, _ = lpips_ref.metric_maps(pred, gt, "albedo", mask)
    x = lpips_ref.bf16(lpips_ref.scaled_input(torch.cat([p, g])).to(torch.float64))
    for l in range(5):
        if l:
            x = ref64.layer_input(l, feats[l - 1])
        y, a, K = ref64.conv(l, x)
        assert feats[l].shape == y.shape, (l, feats[l].shape, y.shape)
        ops_ref.assert_within(feats[l], y, ops_ref.gemm_bound(K, a, y, False), f"lpips_layer{l + 1}_{H}x{W}")
    head = ref64.head([f[:1] for f in feats], [f[1:] for f in feats])
    assert abs(got["lpips"] - head) <= HEAD_TOL * abs(head) + 1e-12, (got["lpips"], head)


# ---- the scalar ---------------------------------------------------------------------------------------------------------
def _check_scalar(pred, gt, target, mask, transform, lp, ref64, ref32, tag):
    got, info = _eval(pred, gt, target, mask, transform, lp)
    p, g, _ = lpips_ref.metric_maps(pred, gt, target, mask, transform, scale=info["scale"])
    r64 = ref64(p, g)
    with torch.backends.cudnn.flags(allow_tf32=False):
        r32 = float(ref32(p, g))
    d64 = ops_ref.record(f"lpips_scalar_vs_f64_{tag}", abs(got["lpips"] - r64))
    d32 = ops_ref.record(f"lpips_scalar_vs_f32_{tag}", abs(got["lpips"] - r32))
    assert d64 <= SCALAR_TOL_64 and d32 <= SCALAR_TOL_32, (got["lpips"], r64, r32)
    return got


@pytest.mark.parametrize("H,W", [(31, 31), (77, 131), (480, 640)])
@pytest.mark.parametrize("target,mask,transform,kind", CONFIGS)
def test_scalar(H, W, target, mask, transform, kind, lp, ref64, ref32):
    pred, gt, m = _inputs(H, W, target, mask, transform, kind)
    got = _check_scalar(pred, gt, target, m, transform, lp, ref64, ref32, f"{target}_{mask}_{transform}_{kind}_{H}x{W}")
    if kind == "dark":                                     # k = 0: both maps 0
        assert got["lpips"] == 0.0


def test_scalar_full_hd(lp, ref64, ref32):
    pred, gt, m = _inputs(1080, 1920, "shading", "pixel", None, "noisy")
    _check_scalar(pred, gt, "shading", m, None, lp, ref64, ref32, "shading_pixel_1080x1920")


# ---- where eps sits in _normalize_tensor ---------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(77, 131), (480, 640)])
def test_norm_eps_on_small_features(H, W, weights):
    """conv5's weight and bias times 1e-4, so that its per-pixel feature norms come near sqrt(1e-8): there torchmetrics'
    x / sqrt(1e-8 + sum x^2), upstream lpips' x / (||x|| + 1e-10) and x / (||x|| + 1e-8) part by several times the
    scalar bound. With the trained-scale weights of the other tests they agree to 5e-9 relative."""
    from marigold_b200.evaluation import LPIPS

    alex, lin = weights
    small = lpips_ref.with_small_layer(alex, 4, 1e-4)
    h = LPIPS(small, lin, device="cuda")
    try:
        ref = lpips_ref.Lpips64(small, lin, device="cuda")
        pred, gt, m = _inputs(H, W, "albedo", "pixel", None, "noisy")
        got, _ = _eval(pred, gt, "albedo", m, None, h)
        feats = _debug_features(h, H, W)
        norms = feats[4].pow(2).sum(1).sqrt()
        assert 0 < norms.max() < 1e-3, float(norms.max())
        head = ref.head([f[:1] for f in feats], [f[1:] for f in feats])
        assert abs(got["lpips"] - head) <= HEAD_TOL * abs(head), (got["lpips"], head)
        p, g, _ = lpips_ref.metric_maps(pred, gt, "albedo", m)
        f0, f1 = ref.features(p), ref.features(g)
        r64 = float(lpips_ref.head(f0, f1, ref.lins).squeeze())
        d64 = ops_ref.record(f"lpips_scalar_vs_f64_small_conv5_{H}x{W}", abs(got["lpips"] - r64))
        assert d64 <= SCALAR_TOL_64, (got["lpips"], r64)
        # the case tells the placements apart
        for norm in (lpips_ref.normalize_upstream,
                     lambda f: f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + lpips_ref.EPS)):
            alt = float(lpips_ref.head(f0, f1, ref.lins, norm=norm).squeeze())
            assert abs(alt - r64) > 5 * SCALAR_TOL_64, (alt, r64)
    finally:
        h.close()


# ---- exact properties ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mask", ["none", "pixel"])
def test_exact_properties(mask, lp):
    pred, gt, m = _inputs(77, 131, "albedo", mask, None, "noisy")
    a, _ = _eval(pred, gt, "albedo", m, None, lp)
    b, _ = _eval(pred, gt, "albedo", m, None, lp)
    c, _ = _eval(gt, pred, "albedo", m, None, lp)
    z, _ = _eval(gt, gt.clone(), "albedo", m, None, lp)
    assert a["lpips"] > 0
    assert np.float64(a["lpips"]).tobytes() == np.float64(b["lpips"]).tobytes() == np.float64(c["lpips"]).tobytes()
    assert z["lpips"] == 0.0


# ---- errors -------------------------------------------------------------------------------------------------------------
def test_errors(lp):
    from marigold_b200 import _lib

    lib = _lib.load()
    pred, gt, m = _inputs(30, 40, "albedo", "pixel", None, "noisy")
    l0 = lib.mgb_launch_count()
    with pytest.raises(ValueError, match="31"):
        _eval(pred, gt, "albedo", m, None, lp)
    with pytest.raises(ValueError, match="31"):
        _eval(pred.transpose(1, 2).contiguous(), gt.transpose(1, 2).contiguous(), "albedo", m.transpose(1, 2).contiguous(),
              None, lp)
    assert lib.mgb_launch_count() == l0
    pred, gt, m = _inputs(48, 64, "albedo", "pixel", None, "noisy")
    big = pred.clone()
    idx = torch.nonzero(m[0])[0]
    big[1, idx[0], idx[1]] = 1.25
    with pytest.raises(ValueError, match=r"values are expected to be in the \[0, 1\] range"):
        _eval(big, gt, "albedo", m, None, lp)
    nan = gt.clone()
    nan[2, idx[0], idx[1]] = float("nan")
    with pytest.raises(ValueError, match="nan"):
        _eval(pred, nan, "albedo", m, None, lp)
    off = torch.nonzero(~m[0])[0]
    outside = gt.clone()
    outside[:, off[0], off[1]] = float("nan")
    got, _ = _eval(pred, outside, "albedo", m, None, lp)
    assert np.isfinite(got["lpips"])


# ---- unchanged behaviour, launch counts, the handle -----------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(31, 31), (77, 131), (480, 640), (1080, 1920)])
@pytest.mark.parametrize("target", ["albedo", "shading"])
def test_psnr_ssim_unchanged_and_launches(H, W, target, lp):
    from marigold_b200.evaluation import evaluate_iid

    pred, gt, m = _inputs(H, W, target, "pixel", None, "noisy")
    (plain, pinfo), n_plain = _launches(lambda: evaluate_iid(pred, gt, target, m))
    (with_lp, info), n_lp = _launches(lambda: _eval(pred, gt, target, m, None, lp))
    up = target in iid_eval_ref.UP_TO_SCALE
    assert n_plain == IID_LAUNCHES[up]
    assert set(plain) == {"psnr", "ssim"} and set(with_lp) == {"psnr", "ssim", "lpips"}
    for k in ("psnr", "ssim"):
        assert np.float64(plain[k]).tobytes() == np.float64(with_lp[k]).tobytes(), k
    assert repr(pinfo) == repr(info)
    # prep, five convs (+ a split-K reduce each where split), two pools, head, final
    ops_ref.record(f"lpips_launch_delta_{target}_{H}x{W}", n_lp - n_plain)
    assert n_lp - n_plain == LPIPS_LAUNCHES[(H, W)], (H, W, n_lp - n_plain)


# launches of mgb_eval_iid_lpips beyond mgb_eval_iid's, per image size: 10 + the convolutions that split K
LPIPS_LAUNCHES = {(31, 31): 14, (77, 131): 14, (480, 640): 12, (1080, 1920): 10}


def test_handle_memory(weights):
    from marigold_b200.evaluation import LPIPS

    fn = live_device_bytes
    b0 = fn()
    h = LPIPS(*weights, device="cuda")
    bf16_bytes = 2 * (64 * 9 * 64 + 192 * 25 * 64 + 384 * 9 * 192 + 256 * 9 * 384 + 256 * 9 * 256)
    fp32_bytes = 4 * 2 * (64 + 192 + 384 + 256 + 256)
    assert fn() - b0 == bf16_bytes + fp32_bytes
    h.close()
    assert fn() == b0


def test_bad_weights(weights):
    from marigold_b200.evaluation import LPIPS

    alex, lin = weights
    bad = dict(alex)
    bad["features.3.weight"] = bad["features.3.weight"][:, :32]
    with pytest.raises(ValueError, match="features.3.weight"):
        LPIPS(bad, lin)
    with pytest.raises(ValueError, match="lin4"):
        LPIPS(alex, {k: v for k, v in lin.items() if not k.startswith("lin4")})
