"""One image on several GPUs: what one rank's share of a row-split call costs (SD-size random weights, E = 1).

On one GPU, per size: the unsplit encode, the captured (graph) UNet + DDIM step and the decode; then every exchange of
a row-split run at world 1 is recorded, and for G in 1, 2, 4, 8 rank 0 runs its share of each stage with an exchange
that copies the other ranks' rows from the recording (a local copy standing in for the all-gather). Beside each G, the
all-gather time a model gives: the bytes a rank receives over NVLink's 450 GB/s per direction (the H100 SXM data
sheet's 900 GB/s bidirectional), not measured. The card's name, power limit and maximum SM clock are read in the same
run.

Under torchrun on a box with several GPUs (--torchrun): the wall time of a whole E = 1 depth call, max over the ranks,
with the row split and with it disabled.

    python tools/row_split.py [--out DIR] [--sizes 768x768,1080x1920,3024x4032,4032x6048,6048x8064]
    torchrun --nproc-per-node G tools/row_split.py --torchrun [--sizes ...]
"""
import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import torch  # noqa: E402

from bench import gpu_identity  # noqa: E402
from marigold_b200 import parallel  # noqa: E402
from marigold_b200.schedulers import DDIMScheduler  # noqa: E402
from native_res import make_engine  # noqa: E402
from tests.helpers import synthetic_image  # noqa: E402

NVLINK_BYTES_PER_S = 450e9          # one direction of the H100 SXM's NVLink (data sheet): a model, not measured


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def attn_shapes(eng, lh, lw):
    """(T, C) of the UNet step's 16 attentions, and of the VAE mid-block attention."""
    ch, L = eng.cfg.unet_block_channels, eng.cfg.unet_layers_per_block
    hs, ws = [lh], [lw]
    for _ in range(3):
        hs.append((hs[-1] + 1) // 2)
        ws.append((ws[-1] + 1) // 2)
    unet = [(hs[i] * ws[i], ch[i]) for i in range(3) for _ in range(L)] + [(hs[3] * ws[3], ch[3])] + \
        [(hs[3 - i] * ws[3 - i], ch[3 - i]) for i in range(1, 4) for _ in range(L + 1)]
    return unet, (lh * lw, eng.cfg.vae_block_channels[3])


def gather_model_ms(shapes, G):
    """Modelled all-gather time of one rank: (G - 1) chunks of each attention's output received over NVLink."""
    return sum((G - 1) * parallel.row_split_chunk(T, G) * C * 2 for T, C in shapes) / NVLINK_BYTES_PER_S * 1e3


def one_gpu(eng, H, W):
    lh, lw = H // 8, W // 8
    s = DDIMScheduler()
    s.set_timesteps(4)
    eng.set_schedule(s.timesteps, *s.coefficients())
    rgb = (synthetic_image(max(H, W), seed=3)[..., :H, :W].float() / 255.0 * 2.0 - 1.0).cuda().contiguous()
    g = torch.Generator(device="cuda").manual_seed(0)
    z = torch.randn(1, 4, lh, lw, device="cuda", generator=g)
    lat = eng.encode(rgb)
    tgt = z.clone()
    eng.denoise_range_(lat, tgt, 0, 1)                 # eager step, then the capture
    eng.decode(tgt, 0)                                 # the first decode at this shape loads modules, grows the arena
    unsplit = {"encode_ms": timed(lambda: eng.encode(rgb)),
               "step_ms": timed(lambda: eng.denoise_range_(lat, tgt, 1, 1)),
               "decode_ms": timed(lambda: eng.decode(tgt, 0))}
    unet_shapes, vae_shape = attn_shapes(eng, lh, lw)
    rec = []
    eng.set_row_split(0, 1, lambda buf, r, w: rec.append(buf.clone()))
    stages = {"encode": (lambda: eng.encode(rgb), [vae_shape]),
              "step": (lambda: eng.denoise_range_(lat, tgt.clone(), 1, 1), unet_shapes),
              "decode": (lambda: eng.decode(tgt, 0), [vae_shape])}
    recorded = {}
    for name, (fn, shapes) in stages.items():
        rec.clear()
        fn()                                            # records, and warms the eager path
        assert len(rec) == len(shapes), (name, len(rec))
        recorded[name] = list(rec)
    rec.clear()
    per_g = {}
    for G in (1, 2, 4, 8):
        row = {}
        for name, (fn, shapes) in stages.items():
            k = [0]

            def exchange(buf, r, w, name=name, shapes=shapes):
                T, C = shapes[k[0]]
                src = recorded[name][k[0]]
                k[0] += 1
                rows = parallel.row_split_rows(T, r, w)
                buf[:rows.start * C * 2] = src[:rows.start * C * 2]
                buf[rows.stop * C * 2:T * C * 2] = src[rows.stop * C * 2:T * C * 2]

            eng.set_row_split(0, G, exchange)
            fn()                                        # warm this G's launch shapes
            k[0] = 0
            row[f"{name}_ms"] = timed(fn)
            row[f"{name}_gather_model_ms"] = gather_model_ms(shapes, G)
        per_g[G] = {k: round(v, 3) for k, v in row.items()}
    eng.set_row_split()
    recorded.clear()
    torch.cuda.empty_cache()
    step_g2 = per_g[2]["step_ms"] + per_g[2]["step_gather_model_ms"]
    return {"H": H, "W": W, "tokens": lh * lw, "unsplit": {k: round(v, 3) for k, v in unsplit.items()},
            "rank0": per_g, "g2_step_beats_graph_step": step_g2 < unsplit["step_ms"]}


def multi_gpu(sizes):
    import torch.distributed as dist

    from marigold_b200.pipeline import MarigoldDepthPipeline

    dist.init_process_group("nccl")
    rank, G = parallel.world()
    torch.cuda.set_device(rank)
    eng = make_engine()
    text = torch.randn(1, 2, 1024, generator=torch.Generator().manual_seed(7))
    pipe = MarigoldDepthPipeline(eng, DDIMScheduler(), text, default_denoising_steps=4, default_processing_resolution=0)
    res = []
    for H, W in sizes:
        img = synthetic_image(max(H, W), seed=3)[..., :H, :W].contiguous()
        row = {"H": H, "W": W, "G": G}
        for label, min_tokens in (("split", 0), ("unsplit", 1 << 62)):
            parallel.ROW_SPLIT_MIN_TOKENS = min_tokens
            pipe(img, ensemble_size=1, generator=torch.Generator().manual_seed(0))      # warm
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe(img, ensemble_size=1, generator=torch.Generator().manual_seed(0))
            torch.cuda.synchronize()
            row[f"{label}_wall_ms"] = round(parallel.barrier_max_ms((time.perf_counter() - t0) * 1e3,
                                                                    torch.device("cuda", rank)), 1)
        res.append(row)
    eng.close()
    dist.destroy_process_group()
    return res, rank


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="768x768,1080x1920,3024x4032,4032x6048,6048x8064")
    ap.add_argument("--torchrun", action="store_true")
    a = ap.parse_args()
    sizes = [tuple(int(v) for v in s.split("x")) for s in a.sizes.split(",")]
    if a.torchrun:
        runs, rank = multi_gpu(sizes)
        res = {"card": gpu_identity(torch.cuda.current_device()), "torchrun": runs}
        if rank != 0:
            return
    else:
        res = {"card": gpu_identity(torch.cuda.current_device()), "runs": []}
        eng = make_engine()
        for H, W in sizes:
            res["runs"].append(one_gpu(eng, H, W))
            print(json.dumps(res["runs"][-1]), file=sys.stderr, flush=True)
        eng.close()
        passing = [r["tokens"] for r in res["runs"] if r["g2_step_beats_graph_step"]]
        res["smallest_tokens_g2_beats_graph_step"] = min(passing) if passing else None
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / ("row_split_torchrun.json" if a.torchrun else "row_split.json")).write_text(line + "\n")


if __name__ == "__main__":
    main()
