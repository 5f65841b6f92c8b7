"""The resize restatements (tests/resize_ref.py) against torch's CPU `F.interpolate(antialias=True)`, which is what
torchvision's `resize` runs on the reference's host-side image. Needs no GPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import resize_ref as R

CAP = torch.backends.cpu.get_cpu_capability()
METHODS = ["bilinear", "bicubic"]
needs_fma = pytest.mark.skipif(CAP not in ("AVX2", "AVX512"),
                               reason=f"CPU capability {CAP}: torch's kernel is built without FMA contraction there, and "
                                      "the emulation restates the AVX2 / AVX512 build")


def _tcpu(x, size, method):
    return F.interpolate(x, size=size, mode=method, antialias=True, align_corners=False)


def _window_sensitive(limit, method, count):
    """(in, out) pairs whose float32 tap windows differ from the float64 definition's."""
    out = []
    for a in range(1, limit):
        for b in range(1, limit):
            x1, s1, _ = R.weights(a, b, method, "cpu")
            x2, s2, _, _ = R.windows64(a, b, method)
            if not (np.array_equal(x1, x2) and np.array_equal(s1, s2)):
                out.append((a, b))
                if len(out) == count:
                    return out
    return out


PAIRS = [(130, 64), (64, 130), (4032, 768), (768, 4032), (3024, 576), (576, 3024), (1, 1), (1, 7), (1, 100), (7, 1),
         (100, 1), (577, 1), (3, 7), (7, 3), (1000, 999), (999, 1000), (240, 768), (768, 240), (37, 19), (17, 17)]


def test_cpu_capability_recorded(record_property):
    record_property("cpu_capability", CAP)
    print("torch CPU capability:", CAP)


@needs_fma
@pytest.mark.parametrize("method", METHODS)
def test_cpu_weights_bit_exact(method):
    rng = np.random.default_rng(11)
    pairs = PAIRS + [tuple(int(v) for v in p) for p in rng.integers(1, 700, size=(60, 2))]
    pairs += _window_sensitive(120, method, 80)
    for a, b in pairs:
        got = R.identity_weights(lambda x, s: _tcpu(x, s, method), a, b)
        xm, xs, w = R.weights(a, b, method, "cpu")
        want = R.weight_matrix(xm, xs, w, a)
        assert np.array_equal(got.view(np.int32) & 0x7FFFFFFF, want.view(np.int32) & 0x7FFFFFFF) and \
            np.array_equal(got, want), (method, a, b, int((got != want).sum()))


def test_window_sensitive_pairs_exist():
    """The float32 window arithmetic differs from float64 often enough that windows must be restated exactly."""
    assert len(_window_sensitive(120, "bilinear", 50)) == 50 and len(_window_sensitive(120, "bicubic", 50)) == 50


@needs_fma
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("shape", [(50, 60, 123, 99), (30, 20, 72, 48), (1, 40, 1, 80), (90, 130, 64, 92), (1, 1, 5, 3),
                                   (240, 320, 77, 131), (400, 300, 37, 97), (31, 17, 5, 64), (1000, 50, 77, 20),
                                   (40, 1, 13, 2)])
def test_cpu_output_bit_exact(method, shape):
    """Every output bit (sign of zero included) of torch CPU, over windows of 2 to 52 taps: t0 w0, then the products of
    the later taps rounded and added in order in groups of four, the last (n - 1) % 4 taps fused."""
    H, W, h, w = shape
    x = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(H * W)) * 4 - 2
    want = _tcpu(x, (h, w), method).numpy()
    got = R.emulate(x, (h, w), method, "cpu")
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


@needs_fma
@pytest.mark.parametrize("method", METHODS)
def test_cpu_photo_bit_exact(method):
    """A 12 MP photo to 768 x 576 (windows of 11 and 23 taps): every float bit of torch CPU."""
    g = torch.Generator().manual_seed(2)
    x = torch.randint(0, 256, (1, 3, 3024, 4032), generator=g).float()
    want = _tcpu(x, (576, 768), method).numpy()
    assert np.array_equal(R.emulate(x, (576, 768), method, "cpu").view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("shape", [(240, 320, 77, 131), (50, 60, 123, 99), (1, 40, 1, 13), (40, 1, 13, 1),
                                   (31, 17, 5, 64), (64, 64, 1, 1), (3, 5, 700, 1)])
def test_float64_within_bound_of_both_emulations_and_torch_cpu(method, shape):
    H, W, h, w = shape
    x = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(7)) * 4 - 2
    r64 = R.resize64(x, (h, w), method)
    b = R.bound(x, (h, w), method)
    outs = [R.emulate(x, (h, w), method, "cpu"), R.emulate(x, (h, w), method, "cuda")]
    if w > 1:                      # torch's CPU antialias kernel returns wrong values when the output is one column wide
        outs.append(_tcpu(x, (h, w), method).numpy())
    for out in outs:
        assert np.all(np.abs(out - r64) <= b), float((np.abs(out - r64) / b).max())


@pytest.mark.parametrize("method", METHODS)
def test_bound_catches_a_dropped_tap(method):
    """The bound is tight enough that losing a window's last tap shows on a smooth photo-sized row."""
    x = torch.linspace(0, 255, 4032).reshape(1, 1, 1, 4032).repeat(1, 1, 2, 1)
    xm, xs, w = R.weights(4032, 768, method, "cpu")
    M = R.weight_matrix(xm, np.maximum(xs - 1, 1), w, 4032).astype(np.float64)
    dropped = x.numpy().astype(np.float64) @ M.T
    r64 = R.resize64(x, (2, 768), method)
    assert np.any(np.abs(dropped - r64) > R.bound(x, (2, 768), method))


def test_to_u8_rule():
    v = np.array([-3.0, -0.5, 0.5, 1.5, 2.5, 254.5, 255.4, 300.0], dtype=np.float32)
    assert R.to_u8(v, "bicubic").tolist() == [0, 0, 0, 2, 2, 254, 255, 255]
    assert R.to_u8(v[2:7], "bilinear").tolist() == [0, 2, 2, 254, 255]


def test_normalise_is_true_division():
    u = np.arange(256, dtype=np.uint8)
    got = R.normalise_cpu(u)
    want = (((u.astype(np.float32) / np.float32(255)).astype(np.float32) * np.float32(2)).astype(np.float32)
            - np.float32(1)).astype(np.float32)
    assert np.array_equal(got, want)
    recip = ((u.astype(np.float32) * (np.float32(1) / np.float32(255))) * np.float32(2) - np.float32(1)).astype(np.float32)
    assert int((recip != got).sum()) > 0


def test_golden_resize_reproduced_exactly():
    """The reference's own resize_max_res outputs (bilinear) from the emulation, every byte."""
    from pathlib import Path

    from tests.golden.cases import RESIZE_CASES, resize_input

    gold = np.load(Path(__file__).resolve().parent / "golden" / "ensemble_golden.npz")
    for name, cfg in RESIZE_CASES.items():
        if cfg["method"] != "bilinear":
            continue
        img = resize_input(cfg)
        H, W = img.shape[-2:]
        f = min(cfg["max_edge"] / W, cfg["max_edge"] / H)
        got = R.to_u8(R.emulate(img.float(), (int(H * f), int(W * f)), "bilinear", "cpu"), "bilinear")
        assert np.array_equal(got, gold[f"resize/{name}"])
