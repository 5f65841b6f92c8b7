"""One launch of every kernel family at its production shape (768 x 768 member), for `ncu --set full`:

    ncu --set full --clock-control none --import-source on -k regex:mgb -o out/r02_zoo python tools/kernel_zoo.py
    python tools/ncu_kernel_table.py out/r02_zoo.ncu-rep > out/kernel_table.md

Every launch goes through the operator-level C ABI (marigold_b200.ops) or the ensemble entry points, i.e. the same
kernels with the same tile choices the network graph makes for these shapes."""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from marigold_b200 import _lib, ops  # noqa: E402
from marigold_b200.ensemble import ensemble_depth, ensemble_normals  # noqa: E402

g = torch.Generator(device="cuda").manual_seed(0)
bf = torch.bfloat16


def rn(*s):
    return torch.randn(*s, device="cuda", generator=g)


def conv(H, W, cin, cout, kind=0, flags=0, bias=True, block_n=0):
    stride = 2 if kind in (2, 3) else 1
    x = rn(1, H * stride, W * stride, cin)
    xin = ops.space_to_depth(x) if stride == 2 else x.to(bf)
    w = ops.pack_conv_weight((rn(cout, cin, 3, 3) / (9 * cin) ** 0.5).to(bf))
    ws = torch.empty(16 * H * W * cout, device="cuda")
    ops.conv2d(xin, w, rn(cout) if bias else None, 1, H, W, cin, cout, kind=kind, flags=flags, block_n=block_n, ws=ws)


def linear(M, N, K, flags=0, residual=False, bf16out=False):
    a = rn(M, K).to(bf)
    w = (rn(N, K) / K ** 0.5).to(bf)
    n_out = N // 2 if flags & _lib.EPI_GEGLU else N
    ws = torch.empty(16 * M * N, device="cuda")
    ops.linear(a, w, rn(N), rn(M, n_out) if residual else None, out_f32=not bf16out, out_bf16=bf16out, flags=flags, ws=ws)


# ---- UNet, 96 x 96 level (C = 320) ----
conv(96, 96, 320, 320)                                   # resnet conv: gemm_tc<160> 144 CTAs, K = 2880
conv(96, 96, 960, 320)                                   # up-block conv on the concat: K = 8640
linear(9216, 2560, 320, flags=_lib.EPI_GEGLU, bf16out=True)   # FF-in + GEGLU
linear(9216, 320, 1280, residual=True, bf16out=True)     # FF-out
linear(9216, 960, 320, bf16out=True)                     # fused QKV
linear(9216, 320, 320, residual=True)                    # attention out-projection / proj_in / proj_out
qkv = rn(9216, 960).to(bf)
ops.flash_attn64(qkv, 1, 9216, 320, 0.125)               # flash attention (split-KV) + attn_combine
ops.groupnorm(rn(1, 9216, 320), rn(320), rn(320), 1, 9216, 320, 32, 1e-5, 1)
ops.groupnorm(rn(1, 9216, 960), rn(960), rn(960), 1, 9216, 960, 32, 1e-5, 1)
ops.layernorm(rn(9216, 320), rn(320), rn(320))
# ---- 48 x 48 (C = 640), 24 x 24 and 12 x 12 (C = 1280) ----
conv(48, 48, 640, 640)
conv(48, 48, 320, 320, kind=2)                           # stride-2 downsample over parity planes
linear(2304, 5120, 640, flags=_lib.EPI_GEGLU, bf16out=True)
ops.flash_attn64(rn(2304, 1920).to(bf), 1, 2304, 640, 0.125)
conv(24, 24, 1280, 1280)                                 # split-K + deferred epilogue
linear(576, 1280, 1280, residual=True)
linear(576, 10240, 1280, flags=_lib.EPI_GEGLU, bf16out=True)
conv(12, 12, 1280, 1280)
ops.groupnorm(rn(1, 144, 2560), rn(2560), rn(2560), 1, 144, 2560, 32, 1e-5, 1)
ops.upsample2x(rn(1, 48, 48, 640))
# ---- VAE decoder, 768 x 768 (C = 128) and 384 x 384 (C = 256) ----
conv(768, 768, 128, 128)                                 # 4608 tiles, two CTAs per SM
conv(768, 768, 128, 3, flags=_lib.EPI_DEPTH, block_n=16)  # conv_out + channel mean / clip / shift head (16-column tile)
conv(384, 384, 256, 256)
ops.groupnorm(rn(1, 768 * 768, 128), rn(128), rn(128), 1, 768 * 768, 128, 32, 1e-6, 1)
# ---- test-time ensemble, E = 10 members at 768 x 768 ----
d = torch.rand(10, 1, 768, 768, device="cuda", generator=g)
p0 = np.concatenate([np.ones(10), np.zeros(10)])
_, _, aux = ensemble_depth(d, return_aux=True, param=p0, output_uncertainty=True)     # minmax + reduce + renorm
aux["cost_fd"](p0, p0 + 1.5e-8)                          # f and one BFGS gradient: base pass + perturbation rows
n = torch.nn.functional.normalize(rn(10, 3, 768, 768), dim=1)
ensemble_normals(n, output_uncertainty=True)
# ---- bookends and evaluation ----
from marigold_b200 import imageops  # noqa: E402
from marigold_b200.evaluation import evaluate_depth  # noqa: E402

img = torch.randint(0, 256, (1, 3, 1080, 1920), dtype=torch.uint8, device="cuda")
rgb = imageops.resize(img, (432, 768), "bilinear", post=2)                      # resize_max_res + normalise
pred = torch.rand(1, 1, 432, 768, device="cuda", generator=g)
full = imageops.resize(pred, (1080, 1920), "bilinear")                          # final resize
imageops.colorize_u8(full[0, 0], 0, 1, imageops.spectral_lut_u8())
gt = full[0, 0] * 5 + 1 + 0.05 * rn(1080, 1920)
evaluate_depth(full[0, 0], gt, torch.rand(1080, 1920, device="cuda", generator=g) > 0.2, min_depth=0.5, max_depth=10.0)
torch.cuda.synchronize()
print("kernel zoo done")
