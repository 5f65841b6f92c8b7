"""LPIPS with the VGG16 and SqueezeNet 1.1 backbones restated for the tests: torchmetrics'
LearnedPerceptualImagePatchSimilarity(net_type="vgg" | "squeeze", normalize=True) of one image pair. The taps are those
of torchmetrics' vendored lpips pretrained_networks, slices of torchvision's features module:
  vgg16().features         [0:4] [4:9] [9:16] [16:23] [23:30]                  (relu1_2 .. relu5_3; 64, 128, 256, 512, 512)
  squeezenet1_1().features [0:2] [2:5] [5:8] [8:10] [10:11] [11:12] [12:13]    (64, 128, 256, 384, 384, 512, 512)
The input handling and the head are those of tests/lpips_ref.py (its `head`, `scaled_input`, `check_inputs`).

Three forms of the backbone:
- `NetDef64`: float64 from the definition, walking the torchvision module's layers with float64 weights;
- `NetRound64`: float64, rounding where csrc/lpips.cu rounds: the scaled input and the conv weights in bf16, every conv
  in float64 with the fp32 bias, a tapped layer's post-ReLU output rounded to fp32 (the features the head reads) and
  from there to bf16 (the next operand), every other post-ReLU output (a Fire squeeze included) to bf16, the pools on
  the bf16 values;
- `Net32`: the torchvision module itself in float32 (run it with TF32 off), with the float32 head.
Fabricated weights as tests/lpips_ref.py makes them: torchvision's default init from a seed, every bias redrawn,
non-negative lin weights."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from tests import lpips_ref

SLICES = {
    "vgg": ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30)),
    "squeeze": ((0, 2), (2, 5), (5, 8), (8, 10), (10, 11), (11, 12), (12, 13)),
}
CHANNELS = {"vgg": (64, 128, 256, 512, 512), "squeeze": (64, 128, 256, 384, 384, 512, 512)}


def features_module(net_type: str, sd=None, dtype=torch.float32):
    from torchvision.models import squeezenet1_1, vgg16

    net = vgg16(weights=None) if net_type == "vgg" else squeezenet1_1(weights=None)
    if sd is not None:
        net.features.load_state_dict({k[len("features."):]: v for k, v in sd.items() if k.startswith("features.")})
    return net.features.to(dtype).eval()


def conv_keys(net_type: str):
    """The state-dict key prefix of every convolution, in the order the device runs them (evaluation.LPIPS_NETS)."""
    from marigold_b200.evaluation import LPIPS_NETS

    return [k for k, _ in LPIPS_NETS[net_type][2]]


def fabricated_weights(net_type: str, seed: int = 0):
    """(net_state_dict, lin_state_dict) in the checkpoints' key layout."""
    torch.manual_seed(seed)
    feats = features_module(net_type)
    sd = {f"features.{k}": v.detach().clone() for k, v in feats.state_dict().items()}
    g = torch.Generator().manual_seed(seed + 1)
    for k in conv_keys(net_type):
        sd[f"{k}.bias"] = 0.1 * torch.randn(sd[f"{k}.bias"].shape, generator=g)
    lin = {f"lin{l}.model.1.weight": torch.rand(1, c, 1, 1, generator=g) for l, c in enumerate(CHANNELS[net_type])}
    return sd, lin


def min_size(net_type: str, limit: int = 64) -> int:
    """The smallest n for which every tapped layer of the torchvision module is non-empty on an n x n input."""
    net = features_module(net_type)
    for n in range(1, limit):
        x = torch.zeros(1, 3, n, n)
        try:
            with torch.no_grad():
                for a, b in SLICES[net_type]:
                    x = net[a:b](x)
                    if x.numel() == 0:
                        raise RuntimeError("empty")
        except RuntimeError:
            continue
        return n
    raise AssertionError("no size up to the limit works")


class _Walk:
    """Walks the torchvision features module layer by layer in float64. rounding: the kernels' roundings (NetRound64)."""

    def __init__(self, net_type, sd, device, rounding):
        self.net_type, self.rounding = net_type, rounding
        self.net = features_module(net_type, sd, torch.float64).to(device)
        r = lpips_ref.bf16 if rounding else (lambda t: t)
        self.w = {id(m): r(m.weight.detach()) for m in self.net.modules() if isinstance(m, torch.nn.Conv2d)}
        # the bias in fp32, as the epilogue adds it
        self.b = {id(m): (m.bias.detach().float().double() if rounding else m.bias.detach())
                  for m in self.net.modules() if isinstance(m, torch.nn.Conv2d)}

    def conv_relu(self, m, x, out_round):
        y = torch.relu(F.conv2d(x, self.w[id(m)], self.b[id(m)], m.stride, m.padding))
        return out_round(y) if self.rounding else y

    def layer(self, m, x, tap):
        """One module of the features Sequential. tap: its output is the slice's (a tapped layer's) output."""
        out_round = (lambda t: t.float().double()) if tap else lpips_ref.bf16
        if isinstance(m, torch.nn.Conv2d):
            return self.conv_relu(m, x, out_round)       # the ReLU that follows is folded in (idempotent below)
        if isinstance(m, torch.nn.ReLU):
            return x
        if isinstance(m, torch.nn.MaxPool2d):
            return F.max_pool2d(x, m.kernel_size, m.stride, m.padding, ceil_mode=m.ceil_mode)
        # torchvision Fire
        s = self.conv_relu(m.squeeze, x, lpips_ref.bf16)
        return torch.cat([self.conv_relu(m.expand1x1, s, out_round), self.conv_relu(m.expand3x3, s, out_round)], 1)

    @torch.no_grad()
    def features(self, img: torch.Tensor):
        x = lpips_ref.scaled_input(img.float()).double()
        if self.rounding:
            x = lpips_ref.bf16(x)
        out = []
        for a, b in SLICES[self.net_type]:
            for i in range(a, b):
                x = self.layer(self.net[i], x, i == b - 1 or (i == b - 2 and isinstance(self.net[b - 1], torch.nn.ReLU)))
            out.append(x)
            if self.rounding:
                x = lpips_ref.bf16(x)                    # the next operand: bf16 of the fp32 features
        return out


class _Lpips64:
    def __init__(self, net_type, net_sd, lin_sd, device, rounding):
        self.walk = _Walk(net_type, net_sd, device, rounding)
        self.lins = [lin_sd[f"lin{l}.model.1.weight"].to(device, torch.float32).to(torch.float64)
                     for l in range(len(SLICES[net_type]))]

    def features(self, img):
        return self.walk.features(img)

    @torch.no_grad()
    def __call__(self, img1: torch.Tensor, img2: torch.Tensor) -> float:
        lpips_ref.check_inputs(img1, img2)
        return float(lpips_ref.head(self.features(img1), self.features(img2), self.lins).squeeze())

    def head(self, feats0, feats1) -> float:
        return float(lpips_ref.head(feats0, feats1, self.lins).squeeze())


class NetDef64(_Lpips64):
    """float64 from the definition."""

    def __init__(self, net_type, net_sd, lin_sd, device="cpu"):
        super().__init__(net_type, net_sd, lin_sd, device, False)


class NetRound64(_Lpips64):
    """float64 rounding where the kernels round."""

    def __init__(self, net_type, net_sd, lin_sd, device="cpu"):
        super().__init__(net_type, net_sd, lin_sd, device, True)


class Net32:
    """The reference's arithmetic: the torchvision module in float32 and the float32 head; metric(pred, gt) for
    [1, 3, H, W] float32 maps, a 0-dim tensor on the inputs' device."""

    def __init__(self, net_type, net_sd, lin_sd):
        self.net_type, self.sd = net_type, net_sd
        self.lins = [lin_sd[f"lin{l}.model.1.weight"].float() for l in range(len(SLICES[net_type]))]
        self._net = {}

    def net(self, device):
        if device not in self._net:
            self._net[device] = features_module(self.net_type, self.sd, torch.float32).to(device)
        return self._net[device]

    def features(self, x):
        net, out = self.net(x.device), []
        for a, b in SLICES[self.net_type]:
            x = net[a:b](x)
            out.append(x)
        return out

    @torch.no_grad()
    def __call__(self, img1: torch.Tensor, img2: torch.Tensor) -> torch.Tensor:
        lpips_ref.check_inputs(img1, img2)
        f0, f1 = self.features(lpips_ref.scaled_input(img1)), self.features(lpips_ref.scaled_input(img2))
        return lpips_ref.head(f0, f1, [w.to(img1.device) for w in self.lins]).squeeze()
