"""Diagnostics on a GPU box: (1) per-graph parity numbers of the tiny config vs the CPU oracle,
(2) timing of the full SD-2-size graphs with random weights (CUDA events).

    python tools/net_check.py [--skip-full] [--res 768] [--steps 5]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from tests.helpers import engine_from_oracle, oracle_models, rel_err  # noqa: E402


def parity():
    from marigold_b200.schedulers import DDIMScheduler

    out = {}
    unet, vae, text = oracle_models("tiny")
    eng = engine_from_oracle(unet, vae, text)
    s = DDIMScheduler()
    s.set_timesteps(4)
    kx, kv, kz = s.coefficients()
    eng.set_schedule(s.timesteps, kx, kv, kz)
    g = torch.Generator().manual_seed(11)
    B, lh, lw = 2, 16, 16
    rgb = torch.randn(B, 4, lh, lw, generator=g)
    x = torch.randn(B, 4, lh, lw, generator=g)
    with torch.no_grad():
        ref = unet(torch.cat([rgb, x], 1), int(s.timesteps[0]), text.repeat(B, 1, 1))
    tgt = x.cuda().clone()
    mo = eng.unet_step(rgb.cuda(), tgt, 0, want_model_out=True)
    torch.cuda.synchronize()
    out["unet_step_rel"] = rel_err(mo, ref)
    out["unet_ref_absmax"] = ref.abs().max().item()
    out["sched_rel"] = rel_err(tgt, kx[0] * x + kv[0] * mo.cpu())
    img = torch.rand(2, 3, 64, 128, generator=g) * 2 - 1
    with torch.no_grad():
        ref = vae.quant_conv(vae.encoder(img))[:, :4] * 0.18215
    out["encode_rel"] = rel_err(eng.encode(img.cuda()), ref)
    lat = torch.randn(2, 4, 8, 16, generator=g)
    with torch.no_grad():
        raw = vae.decoder(vae.post_quant_conv(lat / 0.18215))
    out["decode_raw_rel"] = rel_err(eng.decode(lat.cuda(), 2), raw)
    out["decode_depth_rel"] = rel_err(eng.decode(lat.cuda(), 0), (raw.mean(1, keepdim=True).clip(-1, 1) + 1) / 2)
    eng.close()
    return out


def full(res, steps):
    from marigold_b200 import _lib
    from marigold_b200.schedulers import DDIMScheduler

    out = {}
    t0 = time.time()
    unet, vae, text = oracle_models("full")
    out["oracle_build_s"] = round(time.time() - t0, 1)
    t0 = time.time()
    eng = engine_from_oracle(unet, vae, text)
    out["engine_load_s"] = round(time.time() - t0, 1)
    del unet, vae
    s = DDIMScheduler()
    s.set_timesteps(steps)
    kx, kv, kz = s.coefficients()
    eng.set_schedule(s.timesteps, kx, kv, kz)
    lh = lw = res // 8
    rgb = torch.randn(1, 4, lh, lw, device="cuda")
    x = torch.randn(1, 4, lh, lw, device="cuda")
    lib = _lib.load()
    out["workspace_gb"] = eng.workspace_bytes(1, res, res) / 1e9

    def timed(fn, iters=3):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = lib.mgb_launch_count()
        t0 = time.time()
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        cpu_ms = (time.time() - t0) * 1e3 / iters
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters, cpu_ms, (lib.mgb_launch_count() - l0) // iters

    ms, cpu_ms, launches = timed(lambda: eng.denoise(rgb, x))
    out["denoise_ms_per_step"] = ms / steps
    out["denoise_cpu_enqueue_ms_per_step"] = cpu_ms / steps
    out["launches_per_step"] = launches / steps
    out["steps_per_s"] = 1e3 / (ms / steps)
    f_unet = {384: 0.418e12, 768: 2.138e12, 1024: 4.658e12}.get(res)
    if f_unet:
        out["unet_tflops"] = f_unet / (ms / steps) / 1e9
    img = torch.rand(1, 3, res, res, device="cuda") * 2 - 1
    ms, _, launches = timed(lambda: eng.encode(img), 2)
    out["encode_ms"] = ms
    out["encode_launches"] = launches
    ms, _, launches = timed(lambda: eng.decode(x, 0), 2)
    out["decode_ms"] = ms
    out["decode_launches"] = launches
    o = eng.decode(eng.denoise(rgb, x), 0)
    out["finite"] = bool(torch.isfinite(o).all().item())
    out["depth_minmax"] = [o.min().item(), o.max().item()]
    eng.close()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-full", action="store_true")
    ap.add_argument("--skip-parity", action="store_true")
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--out", default=str(ROOT / "out" / "net_check.json"))
    a = ap.parse_args()
    res = {}
    if not a.skip_parity:
        res["parity_tiny"] = parity()
        print(json.dumps(res["parity_tiny"]), flush=True)
    if not a.skip_full:
        res["full"] = full(a.res, a.steps)
        print(json.dumps(res["full"]), flush=True)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(res, indent=1))
