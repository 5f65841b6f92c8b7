"""Shared builders for the parity tests: seeded oracle networks (the checker) and an Engine (the
product) loaded with the same weights."""
from __future__ import annotations

import numpy as np
import torch

from oracle.unet import UNet2DConditionOracle, UNetConfig
from oracle.vae import AutoencoderKLOracle, VAEConfig


def usable_cores() -> int:
    """Cores this process may actually use (affinity mask and cgroup CPU quota), not os.cpu_count():
    on the GPU box the container sees 128 CPUs but is limited, and 128 torch threads thrash."""
    import os

    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:  # noqa: BLE001
        pass
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(p))))
    except Exception:  # noqa: BLE001
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            p_ = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                n = min(n, max(1, q // p_))
        except Exception:  # noqa: BLE001
            pass
    return max(1, n)


def oracle_models(kind: str = "tiny", seed: int = 0):
    torch.manual_seed(seed)
    if kind == "tiny":
        ucfg, vcfg = UNetConfig.tiny(), VAEConfig.tiny()
    else:
        ucfg, vcfg = UNetConfig(), VAEConfig()
    unet = UNet2DConditionOracle(ucfg).eval()
    vae = AutoencoderKLOracle(vcfg).eval()
    g = torch.Generator().manual_seed(7)
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=g)
    return unet, vae, text


def engine_from_oracle(unet, vae, text):
    from marigold_b200.engine import Engine, EngineConfig

    cfg = EngineConfig(unet_block_channels=list(unet.cfg.block_out_channels),
                       unet_cross_dim=unet.cfg.cross_attention_dim,
                       vae_block_channels=list(vae.cfg.block_out_channels))
    eng = Engine(cfg)
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    eng.set_text_embedding(text)
    return eng


def synthetic_image(S: int, seed: int = 1234) -> torch.Tensor:
    """uint8 [1,3,S,S]: smooth sinusoids + rectangles + pixel noise (SURVEY.md §8(d))."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, S), np.linspace(0, 1, S), indexing="ij")
    img = np.zeros((3, S, S))
    for _ in range(6):
        fx, fy, ph = rng.uniform(0.5, 4, 2).tolist() + [rng.uniform(0, 6.28)]
        amp = rng.uniform(20, 50, 3)
        img += amp[:, None, None] * np.sin(2 * np.pi * (fx * xx + fy * yy) + ph)[None]
    img += 128
    for _ in range(5):
        x0, y0 = rng.integers(0, S - 8, 2)
        w, h = rng.integers(8, max(9, S // 3), 2)
        img[:, y0:y0 + h, x0:x0 + w] = rng.uniform(0, 255, 3)[:, None, None]
    img += rng.normal(0, 4, img.shape)
    return torch.from_numpy(np.clip(img, 0, 255).astype(np.uint8))[None]


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def record(name: str, value: float) -> float:
    """Append a measured parity value to $MGB_PARITY_DIR/parity_values.jsonl when that variable names a directory (the
    tolerances asserted in the GPU tests are these measurements plus a margin). Without it nothing is written."""
    import json
    import os
    from pathlib import Path

    if not os.environ.get("MGB_PARITY_DIR"):
        return float(value)
    out = Path(os.environ["MGB_PARITY_DIR"])
    try:
        out.mkdir(parents=True, exist_ok=True)
        with open(out / "parity_values.jsonl", "a") as f:
            f.write(json.dumps({"name": name, "value": float(value)}) + "\n")
    except OSError:
        pass
    return float(value)
