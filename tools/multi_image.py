"""Lists of images in one pipeline call against a loop of single calls: 16 synthetic 480 x 640 images (NYU / ScanNet
shaped), SD-size seeded weights, one fresh CPU generator per image (as script/*/infer.py seeds one per sample). Four
workloads: depth at processing_res 0 with E = 10 and 1 step; normals at 640 with E = 10 and 4 steps; a 3-target IID
model at 640 with E = 1 and 4 steps; depth at 768 with E = 1 and 4 steps; and, as a control, the first with
batch_size=10 (one image per batch, so both calls compute the same member maps). For each, the loop and the list call
alternate 3 times in this process after one warm-up of each; reported: images/s of every run (host clock around a call
that ends in a device synchronise), the (NB, lh, lw) sequence of member batches each call denoised (run-length
encoded; every change of shape recaptures the step graph), the largest difference between the two calls' maps, and per
run where the time went: the device time of the denoise and decode calls (CUDA events) and the host time of finishing
the images (ensemble, resize, host copy; synchronised on entry). The card's name, power limit and maximum SM clock are
read in the same run.

    python tools/multi_image.py [--out DIR] [--reps 3]    (prints one JSON line; with --out also writes DIR/multi_image.json)
"""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import gpu_identity  # noqa: E402
from marigold_b200.pipeline import MarigoldDepthPipeline, MarigoldIIDPipeline, MarigoldNormalsPipeline  # noqa: E402
from marigold_b200.schedulers import DDIMScheduler  # noqa: E402
from tests.helpers import synthetic_image  # noqa: E402
from tools.native_res import make_engine  # noqa: E402

N_IMAGES, H, W = 16, 480, 640
IID_PROPS = {"target_names": ["albedo", "shading", "residual"], "albedo": {"prediction_space": "srgb"},
             "shading": {"prediction_space": "linear", "up_to_scale": True},
             "residual": {"prediction_space": "linear", "up_to_scale": True}}


def maps(out):
    if hasattr(out, "depth_np"):
        return [out.depth_np]
    if hasattr(out, "normals_np"):
        return [out.normals_np]
    return [e.array for e in out]


def run_lengths(shapes):
    rle = []
    for s in shapes:
        if rle and rle[-1][0] == s:
            rle[-1][1] += 1
        else:
            rle.append([s, 1])
    return [[list(s), n] for s, n in rle]


def workload(pipe, images, reps, **kw):
    eng = pipe.engine
    shapes, denoise, decode, finish = [], eng.denoise, eng.decode, pipe._finish
    events = {"denoise": [], "decode": []}
    finish_s = []

    def timed(name, fn, *a):
        b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        b.record()
        out = fn(*a)
        e.record()
        events[name].append((b, e))
        return out

    def recording(rl, z, sn=None):
        shapes.append(tuple(z.shape[:1]) + tuple(z.shape[-2:]))
        return timed("denoise", denoise, rl, z, sn)

    def finishing(*a, **k):
        # synchronised on entry, so that the time is the finishing alone (ensemble, resize, host copy)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = finish(*a, **k)
        finish_s.append(time.perf_counter() - t0)
        return out

    eng.denoise = recording
    eng.decode = lambda t, mode: timed("decode", decode, t, mode)
    pipe._finish = finishing
    gens = lambda: [torch.Generator().manual_seed(1000 + i) for i in range(len(images))]  # noqa: E731

    def loop():
        return [pipe(im, generator=g, **kw) for im, g in zip(images, gens())]

    def listed():
        return pipe(images, generator=gens(), **kw)

    res = {"loop": [], "list": []}
    seq, outs, stages = {}, {}, {"loop": [], "list": []}
    try:
        for name, fn in (("loop", loop), ("list", listed)):      # warm-up: graphs, arena growth, scipy
            fn()
        for _ in range(reps):
            for name, fn in (("loop", loop), ("list", listed)):
                shapes.clear()
                finish_s.clear()
                for v in events.values():
                    v.clear()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[name] = fn()
                torch.cuda.synchronize()
                res[name].append(round(len(images) / (time.perf_counter() - t0), 3))
                seq[name] = run_lengths(shapes)
                stages[name].append({k: round(sum(b.elapsed_time(e) for b, e in v), 1) for k, v in events.items()}
                                    | {"finish": round(1e3 * sum(finish_s), 1)})
    finally:
        eng.denoise, eng.decode, pipe._finish = denoise, decode, finish
    diff = max(float(np.abs(a - b).max()) for x, y in zip(outs["loop"], outs["list"]) for a, b in zip(maps(x), maps(y)))
    return {"loop_images_per_s": res["loop"], "list_images_per_s": res["list"],
            "loop_median": statistics.median(res["loop"]), "list_median": statistics.median(res["list"]),
            "loop_batches": seq["loop"], "list_batches": seq["list"], "max_abs_diff_loop_vs_list": diff,
            "loop_stage_ms": stages["loop"], "list_stage_ms": stages["list"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    images = [synthetic_image(W, seed=100 + i)[:, :, :H, :W].contiguous() for i in range(N_IMAGES)]
    text = torch.randn(1, 2, 1024, generator=torch.Generator().manual_seed(7))
    result = {"gpu": gpu_identity(0), "images": N_IMAGES, "size": [H, W], "workloads": {}}
    eng = make_engine(1)
    depth = MarigoldDepthPipeline(eng, DDIMScheduler(), text)
    normals = MarigoldNormalsPipeline(eng, DDIMScheduler(), text)
    w = result["workloads"]
    w["depth_res0_E10_1step"] = workload(depth, images, args.reps, denoising_steps=1, ensemble_size=10,
                                         processing_res=0)
    # control: batches of one image's 10 members give both calls the same member maps, so the ensembles' BFGS runs the
    # same iterations; what is left is the cost of the list path itself
    w["depth_res0_E10_1step_bs10"] = workload(depth, images, args.reps, denoising_steps=1, ensemble_size=10,
                                              processing_res=0, batch_size=10)
    w["normals_640_E10_4steps"] = workload(normals, images, args.reps, denoising_steps=4, ensemble_size=10,
                                           processing_res=640)
    w["depth_768_E1_4steps"] = workload(depth, images, args.reps, denoising_steps=4, ensemble_size=1,
                                        processing_res=768)
    eng.close()
    eng = make_engine(3)
    iid = MarigoldIIDPipeline(eng, DDIMScheduler(), text, target_properties=IID_PROPS)
    w["iid3_640_E1_4steps"] = workload(iid, images, args.reps, denoising_steps=4, ensemble_size=1, processing_res=640)
    eng.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "multi_image.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
