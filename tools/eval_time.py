"""Time one evaluation call per sample (host clock around the synchronising call, after a warm-up) against the
reference's path restated on the same GPU: normals = torch CUDA error map, .cpu().numpy(), numpy metrics
(script/normals/eval.py:145-157); depth = numpy lstsq on the host, torch CUDA metrics with one .item() each
(script/depth/eval.py:171-217); IID = the float32 restatement of compute_iid_metric on the GPU (tests/iid_eval_ref.py:
torch lstsq, torch.quantile read back with float(), one .item() per metric; the reference repeats the fit and the
quantile for each metric it computes). LPIPS: evaluate_iid(..., lpips=...) against compute_iid_metric's "lpips" call
restated on the GPU (the lstsq and quantile of the up-to-scale targets, the zeroing, torchvision's AlexNet and the
restated head of tests/lpips_ref.py in float32, one .item()) under torch's default cuDNN TF32 setting, which the output
records. Both on the fabricated weights of tests/lpips_ref.py. The VGG16 and SqueezeNet 1.1 LPIPS the same way
(keys iid_<target>_lpips_<net>_*), against torchvision's float32 module and the head of tests/lpips_nets_ref.py, on its
fabricated weights. Prints one JSON line with the card's name and power limit.

    python tools/eval_time.py [--reps 20]
"""
import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import gpu_identity  # noqa: E402
from marigold_b200.evaluation import evaluate_depth, evaluate_iid, evaluate_normals  # noqa: E402
from marigold_b200.evaluation import LPIPS  # noqa: E402
from tests import eval_ref, iid_eval_ref, lpips_nets_ref, lpips_ref  # noqa: E402


def _time(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return {"median_us": float(np.median(ts) * 1e6), "min_us": float(np.min(ts) * 1e6)}


def _ref_depth(pred_np, gt_np, valid_np, gt_ts, mask_ts):
    """script/depth/eval.py:171-217 with least_square_disparity: host fit, device metrics with .item() each."""
    disp = np.zeros_like(gt_np)
    disp[gt_np > 0] = 1.0 / gt_np[gt_np > 0]
    s, t = eval_ref.lstsq(pred_np, disp, valid_np & (gt_np > 0) & (pred_np > 0))
    d = np.clip(pred_np * s + t, 1e-3, None)
    d = np.clip(np.clip(1.0 / d, 0.5, 8.0), 1e-6, None)
    o = torch.from_numpy(d).cuda()
    m = mask_ts
    n = m.sum()
    z = lambda v: torch.where(m, v, torch.zeros_like(v))  # noqa: E731
    dl = torch.log(o) - torch.log(gt_ts)
    r = torch.max(o / gt_ts, gt_ts / o)
    vals = [(z((o - gt_ts).abs() / gt_ts).sum() / n), (z((o - gt_ts) ** 2 / gt_ts).sum() / n), torch.sqrt(z((o - gt_ts) ** 2).sum() / n),
            torch.sqrt(z(dl ** 2).sum() / n), (torch.log10(o[m]) - torch.log10(gt_ts[m])).abs().mean(),
            z((r < 1.25).float()).sum() / n, z((r < 1.25 ** 2).float()).sum() / n, z((r < 1.25 ** 3).float()).sum() / n,
            torch.sqrt(z((1.0 / o - 1.0 / gt_ts) ** 2).sum() / n), torch.sqrt(z(dl ** 2).sum() / n - z(dl).sum() ** 2 / n ** 2) * 100]
    return [v.item() for v in vals]


def _ref_lpips(metric, pred, gt, target, mask):
    """compute_iid_metric(pred, gt, target, "lpips", metric, mask) (src/util/metric.py:263-288) on the GPU."""
    if target in iid_eval_ref.UP_TO_SCALE:
        s = torch.linalg.lstsq(pred[mask].reshape(-1, 1), gt[mask].reshape(-1, 1))[0]
        pred = s * pred
        q = torch.quantile(iid_eval_ref.brightness(gt)[mask[0]], 0.9)
        k = 0 if q < 1e-4 else float(0.8 / q)
        gt, pred = torch.clamp(k * gt, 0, 1), torch.clamp(k * pred, 0, 1)
    p, g = pred[None].clone(), gt[None].clone()
    p[~mask[None]] = 0
    g[~mask[None]] = 0
    return metric(p, g).item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    res = {"gpu": gpu_identity(torch.cuda.current_device()), "reps": a.reps, "cases": {},
           "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32}
    weights = lpips_ref.fabricated_weights(0)
    lp, metric = LPIPS(*weights), lpips_ref.Lpips32(*weights)
    nets = {}
    for net_type in ("vgg", "squeeze"):
        w = lpips_nets_ref.fabricated_weights(net_type, 0)
        nets[net_type] = (LPIPS(*w, net_type=net_type), lpips_nets_ref.Net32(net_type, *w))
    g = torch.Generator(device="cuda").manual_seed(0)
    for H, W in [(480, 640), (1080, 1920)]:
        gt = torch.randn(3, H, W, device="cuda", generator=g)
        gt[2] = gt[2].abs() + 1
        gt = gt / gt.norm(dim=0, keepdim=True)
        pred = gt + 0.3 * torch.randn(3, H, W, device="cuda", generator=g)

        def ref_normals():
            err, _ = eval_ref.cosine_error(pred, gt)
            return eval_ref.normals_metrics(err, decimals=4)

        dgt = 1.0 + 5.0 * torch.rand(H, W, device="cuda", generator=g)
        dpred = 0.8 / dgt - 0.05 + 0.01 * torch.randn(H, W, device="cuda", generator=g)
        dmask = torch.rand(H, W, device="cuda", generator=g) > 0.2
        gt_np, pred_np, valid_np = dgt.cpu().numpy(), dpred.cpu().numpy(), dmask.cpu().numpy()
        igt = torch.rand(3, H, W, device="cuda", generator=g)
        ipred = (0.6 * igt + 0.05 * torch.randn(3, H, W, device="cuda", generator=g)).abs()
        imask = (torch.rand(H, W, device="cuda", generator=g) > 0.2).expand(3, H, W).contiguous()
        res["cases"][f"{H}x{W}"] = {
            "normals_device": _time(lambda: evaluate_normals(pred, gt), a.reps),
            "normals_reference_path": _time(ref_normals, a.reps),
            "depth_device_lsd": _time(lambda: evaluate_depth(dpred, dgt, dmask, alignment="least_square_disparity",
                                                             min_depth=0.5, max_depth=8.0), a.reps),
            "depth_reference_path_lsd": _time(lambda: _ref_depth(pred_np, gt_np, valid_np, dgt, dmask), a.reps),
        }
        for target in ("albedo", "shading"):
            res["cases"][f"{H}x{W}"].update({
                f"iid_{target}_device": _time(lambda: evaluate_iid(ipred, igt, target, imask), a.reps),
                f"iid_{target}_reference_path": _time(lambda: iid_eval_ref.evaluate(ipred, igt, target, imask), a.reps),
                f"iid_{target}_lpips_device": _time(lambda: evaluate_iid(ipred.clamp(0, 1), igt, target, imask, lpips=lp),
                                                    a.reps),
                f"iid_{target}_lpips_reference_path": _time(lambda: _ref_lpips(metric, ipred.clamp(0, 1), igt, target,
                                                                               imask), a.reps),
            })
            for net_type, (nlp, nmetric) in nets.items():
                res["cases"][f"{H}x{W}"].update({
                    f"iid_{target}_lpips_{net_type}_device": _time(
                        lambda: evaluate_iid(ipred.clamp(0, 1), igt, target, imask, lpips=nlp), a.reps),
                    f"iid_{target}_lpips_{net_type}_reference_path": _time(
                        lambda: _ref_lpips(nmetric, ipred.clamp(0, 1), igt, target, imask), a.reps),
                })
    print(json.dumps(res))


if __name__ == "__main__":
    main()
