"""LPIPS with the VGG16 and SqueezeNet 1.1 backbones, without a GPU: each net's minimum map size against the torchvision
module, the float64 restatements of tests/lpips_nets_ref.py against torchvision's float32 module, and the weight checks
that raise before anything reaches the device."""
import ctypes as C

import pytest
import torch

from tests import lpips_nets_ref

pytest.importorskip("torchvision")
NETS = ["vgg", "squeeze"]


@pytest.mark.parametrize("net_type", ["alex", "vgg", "squeeze"])
def test_min_size_is_torchvisions(net_type):
    from marigold_b200.evaluation import lpips_min_size

    if net_type == "alex":
        from tests import lpips_ref

        net = lpips_ref._features_module(lpips_ref.fabricated_weights(0)[0], torch.float32)
        want = next(n for n in range(1, 64) if _non_empty(net, lpips_ref.SLICES, n))
    else:
        want = lpips_nets_ref.min_size(net_type)
    assert lpips_min_size(net_type) == want
    assert want == {"alex": 31, "vgg": 16, "squeeze": 17}[net_type]


def _non_empty(net, slices, n):
    x = torch.zeros(1, 3, n, n)
    try:
        with torch.no_grad():
            for a, b in slices:
                x = net[a:b](x)
                if x.numel() == 0:
                    return False
    except RuntimeError:
        return False
    return True


@pytest.mark.parametrize("net_type", NETS)
def test_restatements_agree(net_type):
    """The definition restatement equals torchvision's module up to float32 rounding; the rounding restatement stays
    within the bf16 operands' effect of it; the taps have the documented channels."""
    sd, lin = lpips_nets_ref.fabricated_weights(net_type, 0)
    g = torch.Generator().manual_seed(3)
    a, b = torch.rand(1, 3, 37, 45, generator=g), torch.rand(1, 3, 37, 45, generator=g)
    d64 = lpips_nets_ref.NetDef64(net_type, sd, lin)
    f = d64.features(a)
    assert [t.shape[1] for t in f] == list(lpips_nets_ref.CHANNELS[net_type])
    assert all(t.numel() > 0 for t in f)
    r_def = d64(a, b)
    r_round = lpips_nets_ref.NetRound64(net_type, sd, lin)(a, b)
    r32 = float(lpips_nets_ref.Net32(net_type, sd, lin)(a, b))
    assert r_def > 0
    assert abs(r32 - r_def) <= 1e-5 * r_def, (r32, r_def)
    assert abs(r_round - r_def) <= 2e-2 * r_def, (r_round, r_def)
    assert lpips_nets_ref.NetRound64(net_type, sd, lin)(a, a.clone()) == 0.0


def test_bad_arguments_raise_before_the_device():
    from marigold_b200.evaluation import LPIPS

    sd, lin = lpips_nets_ref.fabricated_weights("squeeze", 0)
    with pytest.raises(ValueError, match="net_type"):
        LPIPS(sd, lin, net_type="resnet")
    with pytest.raises(ValueError, match="features.12.expand3x3.weight"):
        LPIPS({k: v for k, v in sd.items() if k != "features.12.expand3x3.weight"}, lin, net_type="squeeze")
    bad = dict(sd)
    bad["features.9.squeeze.weight"] = bad["features.9.squeeze.weight"][:40]
    with pytest.raises(ValueError, match="features.9.squeeze.weight"):
        LPIPS(bad, lin, net_type="squeeze")
    with pytest.raises(ValueError, match="lin6"):
        LPIPS(sd, {k: v for k, v in lin.items() if not k.startswith("lin6")}, net_type="squeeze")
    vsd, vlin = lpips_nets_ref.fabricated_weights("vgg", 0)
    with pytest.raises(ValueError, match="lin_state_dict"):
        LPIPS(vsd, dict(vlin, **{"lin3.model.1.weight": torch.rand(1, 256, 1, 1)}), net_type="vgg")
    with pytest.raises(ValueError, match="features.28.bias"):
        LPIPS({k: v for k, v in vsd.items() if k != "features.28.bias"}, vlin, net_type="vgg")
    with pytest.raises(ValueError, match="net_state_dict has no 'features.2.weight'"):
        LPIPS(sd, lin, net_type="vgg")                 # a SqueezeNet state dict handed as VGG16's


def test_c_abi_checks_net_and_counts():
    """mgb_lpips_create_net validates the net type, the counts and every shape before it allocates anything."""
    from marigold_b200 import _lib

    lib = _lib.load()
    h = C.c_void_p()
    vp = (C.c_void_p * 25)(*([1] * 25))
    shapes = (C.c_int32 * 100)()
    chans = (C.c_int32 * 7)(64, 128, 256, 384, 384, 512, 512)
    assert lib.mgb_lpips_create_net(3, 25, vp, shapes, vp, 7, vp, chans, C.byref(h)) == -1
    assert b"unknown net type" in lib.mgb_last_error()
    assert lib.mgb_lpips_create_net(2, 13, vp, shapes, vp, 7, vp, chans, C.byref(h)) == -1
    assert lib.mgb_lpips_create_net(2, 25, vp, shapes, vp, 7, vp, chans, C.byref(h)) == -1   # shapes all zero
    assert b"conv 0" in lib.mgb_last_error()
    assert lib.mgb_lpips_min_size(3) == 0
    assert lib.mgb_lpips_ws_bytes_h(None, 480, 640) == 0
