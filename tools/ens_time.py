"""Time ensemble_depth (host BFGS + device cost kernels) at the quoted size, and its per-iteration call alone: f and
the forward-difference points of its gradient (`cost_fd`).

    python tools/ens_time.py [--res 768] [--members 4 8 10]
"""
import argparse
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402

from marigold_b200.ensemble import _scipy_fd_points, ensemble_depth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=768)
    ap.add_argument("--members", type=int, nargs="+", default=[4, 8, 10])
    a = ap.parse_args()
    g = torch.Generator(device="cuda").manual_seed(0)
    for E in a.members:
        base = torch.rand(1, 1, a.res, a.res, device="cuda", generator=g)
        d = (base * (0.5 + torch.rand(E, 1, 1, 1, device="cuda", generator=g)) + 0.2 * torch.rand(E, 1, 1, 1, device="cuda", generator=g)
             + 0.02 * torch.randn(E, 1, a.res, a.res, device="cuda", generator=g))
        for _ in range(2):
            ensemble_depth(d, scale_invariant=True, shift_invariant=True, output_uncertainty=False)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 5
        for _ in range(n):
            ensemble_depth(d, scale_invariant=True, shift_invariant=True, output_uncertainty=False)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) / n * 1e3
        _, _, aux = ensemble_depth(d, scale_invariant=True, shift_invariant=True, output_uncertainty=False, return_aux=True)
        x = aux["param"]
        pert = _scipy_fd_points(x)
        t0 = time.perf_counter()
        for _ in range(50):
            aux["cost_fd"](x, pert)
        torch.cuda.synchronize()
        trip = (time.perf_counter() - t0) / 50 * 1e6
        print(f"E={E} res={a.res}: {ms:.2f} ms per ensemble_depth, {aux['round_trips']} round trips, nit {aux['nit']}, "
              f"{trip:.0f} us per f+grad-points call", flush=True)


if __name__ == "__main__":
    main()
