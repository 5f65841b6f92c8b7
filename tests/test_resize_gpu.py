"""The device resize (csrc/image.cu) against torch's two antialias kernels (`-m gpu`).

* arith "cuda" (predictions): bit-identical, sign of zero included, to torch CUDA
  `F.interpolate(..., antialias=True, align_corners=False)` and to the CUDA emulation in tests/resize_ref.py.
* arith "cpu" (images): tap windows, weights and every output bit-identical to torch CPU's (through the emulation)
  and to torchvision's CPU resize of a uint8 image followed by the reference's host normalisation.
* Every float output within the float64 bound of tests/resize_ref.py, which does not trust either emulation.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import resize_ref as R

pytestmark = pytest.mark.gpu
METHODS = ["bilinear", "bicubic"]


def _dev(x, size, method, arith, post=0):
    from marigold_b200 import imageops

    return imageops.resize(x.cuda(), size, method, post=post, arith=arith)


def _bits_equal(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a, b) and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _photo(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    base = (0.5 + 0.4 * torch.sin(9 * xx + 5 * yy * yy))[None] * torch.tensor([1.0, 0.8, 0.6])[:, None, None]
    img = base * 255 + torch.randn(3, H, W, generator=g) * 12
    img[:, H // 3: H // 3 + 7] = 255                                     # saturated edges: bicubic overshoot and clamp
    img[:, :, W // 2: W // 2 + 5] = 0
    return img.clamp(0, 255).round().to(torch.uint8)[None]


PAIRS = [(130, 64), (64, 130), (4032, 768), (768, 4032), (3024, 576), (576, 3024), (1, 7), (7, 1), (577, 1), (3, 7),
         (1000, 999), (999, 1000), (240, 768), (37, 19), (17, 17), (333, 100), (1024, 333)]


@pytest.mark.parametrize("arith", ["cpu", "cuda"])
@pytest.mark.parametrize("method", METHODS)
def test_device_weights_equal_emulation(method, arith):
    rng = np.random.default_rng(5)
    pairs = PAIRS + [tuple(int(v) for v in p) for p in rng.integers(1, 500, size=(30, 2))]
    for a, b in pairs:
        got = R.identity_weights(lambda x, s: _dev(x, s, method, arith), a, b)
        xm, xs, w = R.weights(a, b, method, arith)
        want = R.weight_matrix(xm, xs, w, a)
        assert np.array_equal(got, want), (a, b, int((got != want).sum()))


CUDA_CASES = [((1, 1, 576, 768), (3024, 4032)), ((1, 1, 576, 768), (4032, 3024)), ((1, 1, 768, 768), (480, 640)),
              ((1, 1, 768, 768), (1080, 1920)), ((1, 1, 1024, 768), (333, 100)), ((1, 3, 77, 131), (40, 41)),
              ((2, 3, 240, 320), (768, 576)), ((1, 9, 33, 17), (100, 333)), ((3, 2, 1, 50), (1, 7)),
              ((1, 1, 50, 1), (7, 1)), ((1, 1, 1, 1), (5, 9)), ((1, 1, 31, 47), (1, 1))]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("case", CUDA_CASES, ids=[f"{s}->{o}" for s, o in CUDA_CASES])
def test_prediction_resize_cuda_mode(method, case):
    shape, size = case
    x = (torch.rand(*shape, generator=torch.Generator().manual_seed(sum(shape))) * 4 - 2).cuda()
    x.view(-1)[::97] = 0.0
    x.view(-1)[1::101] = -0.0
    got = _dev(x, size, method, "cuda")
    torch_cuda = F.interpolate(x, size=size, mode=method, antialias=True, align_corners=False)
    assert _bits_equal(got, torch_cuda), int((got != torch_cuda).sum())
    assert _bits_equal(got, torch.from_numpy(R.emulate(x.cpu(), size, method, "cuda")))
    r64, b = R.resize64(x.cpu(), size, method), R.bound(x.cpu(), size, method)
    assert np.all(np.abs(got.cpu().numpy() - r64) <= b), float((np.abs(got.cpu().numpy() - r64) / b).max())


def test_pipeline_resize_routes_predictions_through_cuda_mode():
    from marigold_b200.pipeline import _resize

    x = torch.rand(1, 1, 96, 128, generator=torch.Generator().manual_seed(3)).cuda()
    want = F.interpolate(x, size=(333, 517), mode="bilinear", antialias=True, align_corners=False)
    assert _bits_equal(_resize(x, (333, 517), "bilinear"), want)


def _max_res_size(H, W, edge):
    f = min(edge / W, edge / H)
    return int(H * f), int(W * f)


IMAGE_CASES = [((4032, 3024), 768), ((3024, 4032), 768), ((3024, 4032), 1024), ((3024, 4032), 512), ((480, 640), 768),
               ((77, 131), 768), ((77, 131), 50), ((1, 500), 768), ((300, 2), 768)]


@pytest.mark.parametrize("method", METHODS + ["nearest-exact"])
@pytest.mark.parametrize("case", IMAGE_CASES, ids=[f"{s}->{e}" for s, e in IMAGE_CASES])
def test_image_resize_cpu_mode(method, case, record_property):
    import torchvision.transforms.functional as TF
    from torchvision.transforms import InterpolationMode

    (H, W), edge = case
    img = _photo(H, W, H + W)
    size = _max_res_size(H, W, edge)
    u8 = _dev(img, size, method, "cpu", post=1)
    nrm = _dev(img, size, method, "cpu", post=2)
    tv = TF.resize(img, list(size), interpolation=InterpolationMode(method), antialias=True)
    ref_norm = torch.from_numpy(R.normalise_cpu(tv.numpy()))
    if method == "nearest-exact":
        assert _bits_equal(u8, tv.float()) and _bits_equal(nrm, ref_norm)
        return
    emu = R.emulate(img.float(), size, method, "cpu")
    emu_u8 = R.to_u8(emu, method)
    assert np.array_equal(u8.cpu().numpy(), emu_u8.astype(np.float32))
    assert _bits_equal(nrm, torch.from_numpy(R.normalise_cpu(emu_u8)))
    d = u8.cpu().to(torch.int32) - tv.to(torch.int32)
    n_diff = int((d != 0).sum())
    record_property("uint8_px_differing_from_torchvision", n_diff)
    print(f"{method} {H}x{W} -> {size}: {n_diff} uint8 px differ from torchvision")
    assert n_diff == 0
    assert _bits_equal(nrm, ref_norm)
    # the float result before rounding: same bits as the emulation, and within the float64 bound
    f = _dev(img, size, method, "cpu").cpu().numpy()
    assert np.array_equal(f.view(np.int32), emu.view(np.int32))
    if img.numel() < 2e6:
        assert np.all(np.abs(f - R.resize64(img.float(), size, method)) <= R.bound(img.float(), size, method))


def test_uint8_rounding_is_half_to_even():
    """An alternating 0 / 1 row resized to half width is exactly 0.5 everywhere: rint gives 0, round would give 1."""
    img = torch.zeros(1, 3, 4, 64, dtype=torch.uint8)
    img[..., 1::2] = 1
    out = _dev(img, (4, 32), "bilinear", "cpu", post=1)
    assert torch.all(out[..., 1:-1] == 0)
    assert _bits_equal(_dev(img.float(), (4, 32), "bilinear", "cpu")[..., 1:-1], torch.full((1, 3, 4, 30), 0.5))


def test_float_normalisation_is_true_division():
    from marigold_b200 import imageops

    x = torch.arange(256, dtype=torch.float32).reshape(1, 1, 16, 16)
    got = imageops.resize(x.cuda(), (16, 16), "nearest-exact", post=3, arith="cpu")
    assert _bits_equal(got, x / 255.0 * 2.0 - 1.0)
    assert not torch.equal(got.cpu(), (x.cuda() / 255.0 * 2.0 - 1.0).cpu())   # the CUDA reciprocal differs


def _reference_preprocess(inp, processing_res, method):
    """The reference's preprocessing restated on the host: pil_to_tensor, resize_max_res (torchvision, CPU), then
    rgb / 255.0 * 2.0 - 1.0 on the CPU tensor."""
    import torchvision.transforms.functional as TF
    from torchvision.transforms import InterpolationMode

    if not isinstance(inp, torch.Tensor):
        inp = TF.pil_to_tensor(inp.convert("RGB")).unsqueeze(0)
    rgb = inp                                                            # used where it lives, as the reference does
    if processing_res > 0:
        rgb = TF.resize(rgb, list(_max_res_size(*rgb.shape[-2:], processing_res)), interpolation=InterpolationMode(method),
                        antialias=True)
    return (rgb / 255.0 * 2.0 - 1.0).float()


@pytest.mark.parametrize("kind", ["pil", "uint8", "float", "float64", "cuda_uint8", "cuda_float"])
@pytest.mark.parametrize("processing_res", [0, 100, 513, 768])
def test_preprocess_bit_identical_to_reference(kind, processing_res):
    from PIL import Image

    from marigold_b200.pipeline import _MarigoldBase

    img = _photo(120, 160, 9)
    # the float image stays below 255 so that neither side's resize overshoots 255 and trips the range assertion
    if kind == "float64" and processing_res > 0:
        pytest.skip("a float64 image is resized in float64 by the reference; only its native-resolution dtype is kept")
    inp = {"pil": Image.fromarray(img[0].permute(1, 2, 0).numpy()), "uint8": img, "float": img.float() * 0.99,
           "float64": img.double() * 0.99, "cuda_uint8": img.cuda(), "cuda_float": img.float().cuda() * 0.99}[kind]
    fake = SimpleNamespace(device=torch.device("cuda"), dtype=torch.float32)
    got, size = _MarigoldBase._preprocess(fake, inp, processing_res, "bilinear")
    assert tuple(size[-2:]) == (120, 160)
    assert _bits_equal(got, _reference_preprocess(inp, processing_res, "bilinear"))


@pytest.mark.parametrize("method", METHODS)
def test_match_input_res_tail(method):
    from marigold_b200 import imageops
    from marigold_b200.pipeline import _resize, colorize_depth_maps

    pred = torch.rand(1, 1, 48, 96, generator=torch.Generator().manual_seed(4)) * 1.2 - 0.1
    ours = _resize(pred.cuda(), (71, 203), method).squeeze().cpu().numpy().clip(0, 1)
    ours_c = imageops.colorize_u8(torch.from_numpy(np.ascontiguousarray(ours)).cuda(), 0, 1,
                                  imageops.spectral_lut_u8()).cpu().numpy()
    ref = F.interpolate(pred.cuda(), size=(71, 203), mode=method, antialias=True, align_corners=False)
    ref = ref.squeeze().cpu().numpy().clip(0, 1)
    ref_c = np.moveaxis((colorize_depth_maps(ref, 0, 1).squeeze() * 255).astype(np.uint8), 0, -1)
    assert np.array_equal(ours.view(np.int32), ref.view(np.int32)) and np.array_equal(ours_c, ref_c)


def test_two_launches_per_resize_in_both_modes():
    from marigold_b200 import _lib

    lib = _lib.load()
    x = torch.rand(1, 3, 64, 80).cuda()
    for arith in ("cpu", "cuda"):
        torch.cuda.synchronize()
        n0 = lib.mgb_launch_count()
        _dev(x, (33, 41), "bicubic", arith, post=0)
        torch.cuda.synchronize()
        assert lib.mgb_launch_count() - n0 == 2


def test_largest_case_fits():
    """The 12 MP cases stay within a few hundred MB of device memory."""
    torch.cuda.reset_peak_memory_stats()
    _dev(torch.zeros(1, 1, 576, 768), (4032, 3024), "bicubic", "cuda")
    _dev(_photo(4032, 3024, 1), (1024, 768), "bicubic", "cpu", post=2)
    assert torch.cuda.max_memory_allocated() < 1 << 30
