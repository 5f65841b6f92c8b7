"""Reference-vs-reference precision gap: the SAME torch graph (the oracle restatement of the SD-2 UNet) evaluated in
fp32 and under torch's bf16 autocast / pure-bf16 weights on the CPU, on the tiny seeded configuration of the parity
tests. This is what `torch_dtype=torch.bfloat16` does to the reference itself and makes north_star's 1e-3 bar
interpretable: our GPU path (bf16 operands, fp32 accumulate / trunk / statistics) is compared with the same fp32
oracle in tests/test_net_gpu.py. CPU only; writes out/ref_bf16_gap.json.
"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import copy  # noqa: E402

import torch  # noqa: E402

from oracle.schedulers import DDIMSchedulerOracle  # noqa: E402
from tests.helpers import oracle_models, rel_err, usable_cores  # noqa: E402

torch.set_num_threads(usable_cores())
unet, vae, text = oracle_models("tiny")
unet_bf = copy.deepcopy(unet).to(torch.bfloat16)
res = {}
g = torch.Generator().manual_seed(11)
for (B, lh, lw) in [(1, 16, 16), (2, 8, 24)]:
    rgb = torch.randn(B, 4, lh, lw, generator=g)
    x = torch.randn(B, 4, lh, lw, generator=g)
    with torch.no_grad():
        ref = unet(torch.cat([rgb, x], 1), 999, text.repeat(B, 1, 1))
        with torch.autocast("cpu", dtype=torch.bfloat16):
            ac = unet(torch.cat([rgb, x], 1), 999, text.repeat(B, 1, 1)).float()
        pure = unet_bf(torch.cat([rgb, x], 1).to(torch.bfloat16), 999, text.repeat(B, 1, 1).to(torch.bfloat16)).float()
    res[f"unet_step_{B}x{lh}x{lw}"] = {"autocast_bf16_vs_fp32": rel_err(ac, ref), "pure_bf16_vs_fp32": rel_err(pure, ref)}

# 4-step DDIM trajectory + decode to depth
o = DDIMSchedulerOracle()
o.set_timesteps(4)
rgb = torch.randn(1, 4, 16, 16, generator=g)
x0 = torch.randn(1, 4, 16, 16, generator=g)


def traj(model, cast):
    x = x0.clone()
    with torch.no_grad():
        for t in o.timesteps:
            inp = torch.cat([rgb, x], 1)
            v = model(inp.to(cast), int(t), text.to(cast)).float()
            x = o.step(v, t, x)
        d = vae.decoder(vae.post_quant_conv(x / 0.18215)).mean(1, keepdim=True).clip(-1, 1)
    return x, (d + 1) / 2


xr, dr = traj(unet, torch.float32)
xb, db = traj(unet_bf, torch.bfloat16)
res["ddim4_latent_pure_bf16_vs_fp32"] = rel_err(xb, xr)
res["ddim4_depth_pure_bf16_vs_fp32"] = rel_err(db, dr)
res["note"] = ("rel_err = max|a-b| / max|b| (tests/helpers.py). The product's figures against the same fp32 oracle: UNet step "
               "~0.9e-2, final depth (smoke) ~0.9e-2 with bf16 operands and fp32 accumulation/trunk.")
print(json.dumps(res, indent=1))
(ROOT / "out").mkdir(exist_ok=True)
(ROOT / "out" / "ref_bf16_gap.json").write_text(json.dumps(res, indent=1))
