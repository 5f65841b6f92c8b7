"""Native-resolution inference (processing_res = 0) on synthetic 12-megapixel photos, SD-size random weights: per run the
stage times from CUDA events (encode, denoise, decode, ensemble: summed over the member batches), mgb_workspace_bytes,
the member batch select_batch_size chose, and the VAE attention's rows per block and block count; the card's name and
power limit, read in the same run. Then 24 MP (6048 x 4032): depth with E = 1 and 1 step and with E = 10 and 4 steps,
normals, and a 2-target IID model (each its numbers, or the error with the bytes it needed); the largest 4:3 and 3:2
photos select_batch_size accepts for one depth member on this card; mgb_workspace_bytes at the batch caps and the
native sizes. Then a 1920 x 1080 decode with the VAE attention in one block against its default row blocks, alternated.
48 MP (8064 x 6048) and 60 MP (9504 x 6336), where the decoder runs its full-resolution 256-channel stage in low
memory: depth with E = 1 and 1 step.

    python tools/native_res.py [--out DIR] [--only-48mp] [--only-60mp]
        (prints one JSON line; with --out also writes DIR/native_res.json; --only-48mp / --only-60mp: the card, that
        run and the largest photos accepted)
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402

from bench import gpu_identity  # noqa: E402
from marigold_b200.ensemble import ensemble_depth, ensemble_iid, ensemble_normals  # noqa: E402
from marigold_b200.pipeline import call_reserve_bytes, select_batch_size  # noqa: E402
from marigold_b200.schedulers import DDIMScheduler  # noqa: E402
from tests.helpers import attn_blocks, synthetic_image  # noqa: E402


def make_engine(n_targets=1, seed=0):
    from marigold_b200.engine import Engine, EngineConfig
    from oracle.unet import UNet2DConditionOracle, UNetConfig
    from oracle.vae import AutoencoderKLOracle, VAEConfig

    torch.manual_seed(seed)
    ucfg = UNetConfig()
    ucfg.in_channels, ucfg.out_channels = 4 * (n_targets + 1), 4 * n_targets
    unet, vae = UNet2DConditionOracle(ucfg).eval(), AutoencoderKLOracle(VAEConfig()).eval()
    eng = Engine(EngineConfig(unet_in_channels=ucfg.in_channels, unet_out_channels=ucfg.out_channels))
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    eng.set_text_embedding(torch.randn(1, 2, ucfg.cross_attention_dim, generator=torch.Generator().manual_seed(7)))
    return eng


class Stages:
    """Event pairs per stage, summed after one synchronise."""

    def __init__(self):
        self.pairs = {}

    def time(self, name, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        self.pairs.setdefault(name, []).append((a, b))
        return out

    def ms(self):
        torch.cuda.synchronize()
        return {k: round(sum(a.elapsed_time(b) for a, b in v), 1) for k, v in self.pairs.items()}


def run(eng, task, H, W, E, steps):
    """One prediction of E members at H x W: the pipeline's stages (pipeline.py _infer_members + the ensembling)."""
    s = DDIMScheduler()
    s.set_timesteps(steps)
    eng.set_schedule(s.timesteps, *s.coefficients())
    rgb = (synthetic_image(max(H, W), seed=3)[..., :H, :W].float() / 255.0 * 2.0 - 1.0).cuda()
    ct = eng.cfg.unet_out_channels
    ch = {"depth": 1, "normals": 3, "iid": 3 * (ct // 4)}[task]
    bs = select_batch_size(eng, E, H, W, reserve_bytes=call_reserve_bytes(H, W, E, ch))
    g = torch.Generator(device="cuda").manual_seed(0)
    st = Stages()
    lat = st.time("encode", lambda: eng.encode(rgb))
    preds = []
    for s0 in range(0, E, bs):
        nb = min(bs, E - s0)
        z = torch.randn(nb, ct, H // 8, W // 8, device="cuda", generator=g)
        tgt = st.time("denoise", lambda: eng.denoise(lat.expand(nb, -1, -1, -1).contiguous(), z))
        if task == "iid":
            preds.append(st.time("decode", lambda: torch.cat([eng.decode(tgt[:, 4 * i:4 * i + 4].contiguous(), 3)
                                                              for i in range(ct // 4)], 1)))
        else:
            preds.append(st.time("decode", lambda: eng.decode(tgt, 0 if task == "depth" else 1)))
    pred = torch.cat(preds)
    if E > 1:
        ens = {"depth": lambda: ensemble_depth(pred, engine=eng, output_uncertainty=True),
               "normals": lambda: ensemble_normals(pred, engine=eng, output_uncertainty=True),
               "iid": lambda: ensemble_iid(pred, engine=eng, output_uncertainty=True)}[task]
        out = st.time("ensemble", ens)[0]
    else:
        out = pred
    ms = st.ms()
    assert torch.isfinite(out).all()
    R, blocks = attn_blocks(eng, 1, (H // 8) * (W // 8))
    return {"task": task, "H": H, "W": W, "E": E, "steps": steps, "stage_ms": ms, "batch_size": bs,
            "workspace_bytes": eng.workspace_bytes(bs, H, W), "attn_rows": R, "attn_blocks_per_image": blocks,
            "held_bytes_after": eng.held_bytes()}


def try_run(eng, task, H, W, E, steps):
    try:
        return run(eng, task, H, W, E, steps)
    except (ValueError, RuntimeError) as e:           # the batch selection's refusal, or an arena that cannot grow
        return {"task": task, "H": H, "W": W, "E": E, "steps": steps, "error": str(e)}


def largest_accepted(eng, aspect):
    """The largest photo of aspect (w, h) with sides multiples of 8 that select_batch_size accepts for one depth member
    (E = 1) in the memory free now: its size and workspace."""
    def fits(k):
        H, W = 8 * aspect[1] * k, 8 * aspect[0] * k
        try:
            select_batch_size(eng, 1, H, W, batch_size=1, reserve_bytes=call_reserve_bytes(H, W, 1, 1))
            return True
        except ValueError:
            return False
    if not fits(1):
        return {"error": f"no {aspect[0]}:{aspect[1]} photo fits"}
    lo, hi = 1, 2
    while fits(hi):
        lo, hi = hi, 2 * hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid)
    H, W = 8 * aspect[1] * lo, 8 * aspect[0] * lo
    return {"H": H, "W": W, "megapixels": round(H * W / 1e6, 1), "workspace_bytes": eng.workspace_bytes(1, H, W)}


def attention_ab(eng, reps=5):
    """Decode of a 1920 x 1080 latent (135 x 240) with the VAE attention in one block and in its default blocks,
    alternated in this one process; the difference is the attention's."""
    lat = torch.randn(1, 4, 135, 240, generator=torch.Generator().manual_seed(1)).cuda()
    T = 135 * 240
    arms = {"one_block": 8 << 30, "default": 0}
    ref = {}
    times = {k: [] for k in arms}
    for i in range(reps + 1):
        for name, budget in arms.items():
            attn_blocks(eng, 1, T, budget)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = eng.decode(lat, 0)
            b.record()
            torch.cuda.synchronize()
            if i:                                            # the first round warms both arms up
                times[name].append(a.elapsed_time(b))
            ref.setdefault(name, out)
    attn_blocks(eng, 1, T)
    med = {k: round(sorted(v)[len(v) // 2], 2) for k, v in times.items()}
    return {"decode_ms_median": med, "decode_ms_all": {k: [round(x, 2) for x in v] for k, v in times.items()},
            "rows": {k: attn_blocks(eng, 1, T, b)[0] for k, b in arms.items()},
            "bit_equal": bool(torch.equal(ref["one_block"], ref["default"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--only-48mp", action="store_true")
    ap.add_argument("--only-60mp", action="store_true")
    a = ap.parse_args()
    res = {"card": gpu_identity(torch.cuda.current_device()), "runs": []}
    eng = make_engine()
    if a.only_48mp or a.only_60mp:
        if a.only_48mp:
            res["mp48"] = try_run(eng, "depth", 6048, 8064, 1, 1)
        if a.only_60mp:
            res["mp60"] = try_run(eng, "depth", 6336, 9504, 1, 1)
        res["largest_accepted"] = {"4:3": largest_accepted(eng, (4, 3)), "3:2": largest_accepted(eng, (3, 2))}
        eng.close()
        return _emit(res, a.out)
    for (H, W) in ((3000, 4000), (3024, 4032)):
        for E in (1, 10):
            for steps in (1, 4):
                res["runs"].append(run(eng, "depth", H, W, E, steps))
                print(json.dumps(res["runs"][-1]), file=sys.stderr, flush=True)
    res["runs"].append(run(eng, "normals", 3000, 4000, 1, 1))
    res["mp24"] = try_run(eng, "depth", 4032, 6048, 1, 1)
    res["mp24_runs"] = [try_run(eng, "depth", 4032, 6048, 10, 4), try_run(eng, "normals", 4032, 6048, 1, 1)]
    res["mp48"] = try_run(eng, "depth", 6048, 8064, 1, 1)
    res["mp60"] = try_run(eng, "depth", 6336, 9504, 1, 1)
    res["workspace_bytes"] = {f"{B}x{H}x{W}": eng.workspace_bytes(B, H, W) for B, H, W in
                              ((16, 768, 768), (8, 1024, 1024), (1, 3024, 4032), (2, 3024, 4032), (1, 4032, 6048))}
    res["largest_accepted"] = {"4:3": largest_accepted(eng, (4, 3)), "3:2": largest_accepted(eng, (3, 2))}
    res["attention_1080p"] = attention_ab(eng)
    eng.close()
    torch.cuda.empty_cache()
    eng = make_engine(n_targets=2)
    res["runs"].append(run(eng, "iid", 3000, 4000, 1, 1))
    res["mp24_runs"].append(try_run(eng, "iid", 4032, 6048, 1, 1))
    eng.close()
    _emit(res, a.out)


def _emit(res, out):
    line = json.dumps(res)
    print(line, flush=True)
    if out:
        Path(out).mkdir(parents=True, exist_ok=True)
        (Path(out) / "native_res.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
