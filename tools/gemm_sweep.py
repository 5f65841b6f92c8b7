"""Device-time sweep of the wgmma GEMM / implicit-conv kernel (CUDA-graph replay, no host gaps).
    python tools/gemm_sweep.py [--out out/gemm_sweep.jsonl]
Reports us/launch, TFLOP/s and operand bytes pulled per SM-cycle, to separate pipeline-depth, TMA-shape
and L2-bandwidth effects."""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from marigold_b200 import _lib, ops  # noqa: E402
from marigold_b200._lib import check, ptr, stream_ptr  # noqa: E402

lib = _lib.load()


def graph_time(fn, n=20, reps=5):
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(n):
                fn()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (n * reps)


def linear_case(M, N, K, bn, stages, splits=1):
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).to(torch.bfloat16)
    out = torch.empty(M, N, device="cuda")
    ws = torch.empty(max(splits, 1) * M * N, device="cuda") if splits > 1 else None

    def fn():
        check(lib.mgb_op_linear(ptr(a), ptr(w), None, None, ptr(out), None, M, N, K, 0, bn, splits, stages, ptr(ws),
                                stream_ptr()), "linear")
    return graph_time(fn), 2.0 * M * N * K


def conv_case(NB, H, W, Cin, Cout, bn, stages, splits=1):
    x = torch.randn(NB, H, W, Cin, device="cuda").to(torch.bfloat16)
    w = ops.pack_conv_weight((torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5).to(torch.bfloat16))
    out = torch.empty(NB, H, W, Cout, device="cuda")
    ws = torch.empty(max(splits, 1) * NB * H * W * Cout, device="cuda") if splits > 1 else None

    def fn():
        check(lib.mgb_op_conv2d(ptr(x), ptr(w), None, None, ptr(out), None, NB, H, W, Cin, Cout, 0, 0, bn, splits,
                                stages, ptr(ws), stream_ptr()), "conv")
    return graph_time(fn), 2.0 * NB * H * W * Cout * Cin * 9


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "out" / "gemm_sweep.jsonl"))
    a = ap.parse_args()
    rows = []

    def rec(name, us, flop, ctas, kb, bn):
        byt = ctas * kb * (16384 + bn * 128)
        r = {"case": name, "us": round(us, 2), "tflops": round(flop / us / 1e6, 1), "ctas": ctas,
             "operand_GBps": round(byt / us / 1e3, 0), "us_per_kblock": round(us / kb, 3)}
        rows.append(r)
        print(json.dumps(r), flush=True)

    # 1) stage depth, linear M=9216 N=320 K=2880 (same GEMM as the 96x96 320->320 conv)
    for bn in (160, 64, 128, 256):
        for st in (2, 3, 4, 5, 6):
            if 1024 + st * (16384 + bn * 128) + 256 > 227 * 1024:
                continue
            us, fl = linear_case(9216, 320, 2880, bn, st)
            rec(f"lin9216x320x2880_bn{bn}_st{st}", us, fl, 72 * ((320 + bn - 1) // bn), 45, bn)
    # 2) the conv itself
    for bn in (160, 64):
        for st in (3, 5):
            us, fl = conv_case(1, 96, 96, 320, 320, bn, st)
            rec(f"conv96_320_bn{bn}_st{st}", us, fl, 72 * ((320 + bn - 1) // bn), 45, bn)
    # 3) big square GEMM (cuBLAS-like shape) to see the kernel's ceiling
    for bn in (256, 128):
        us, fl = linear_case(8192, 8192, 4096, bn, 4)
        rec(f"lin8192x8192x4096_bn{bn}", us, fl, 64 * (8192 // bn), 64, bn)
    # 4) K-only scaling (fixed tile count = 144 CTAs): per-k-block cost without wave effects
    for K in (320, 1280, 5120):
        us, fl = linear_case(9216, 320, K, 160, 5)
        rec(f"lin9216x320xK{K}_bn160", us, fl, 144, K // 64, 160)
    # 5) mid / low levels
    us, fl = conv_case(1, 48, 48, 640, 640, 128, 5)
    rec("conv48_640_bn128", us, fl, 18 * 5, 90, 128)
    us, fl = conv_case(1, 48, 48, 640, 640, 160, 5, splits=2)
    rec("conv48_640_bn160_sp2", us, fl, 18 * 4 * 2, 45, 160)
    us, fl = conv_case(1, 24, 24, 1280, 1280, 160, 5, splits=3)
    rec("conv24_1280_bn160_sp3", us, fl, 6 * 8 * 3, 60, 160)
    us, fl = conv_case(1, 12, 12, 1280, 1280, 128, 5, splits=7)
    rec("conv12_1280_bn128_sp7", us, fl, 2 * 10 * 7, 26, 128)
    us, fl = linear_case(9216, 2560, 320, 256, 4)
    rec("lin_ff1_9216x2560x320_bn256", us, fl, 72 * 10, 5, 256)
    us, fl = linear_case(9216, 320, 1280, 160, 5)
    rec("lin_ff2_9216x320x1280_bn160", us, fl, 144, 20, 160)
    us, fl = linear_case(9216, 960, 320, 160, 5)
    rec("lin_qkv_9216x960x320_bn160", us, fl, 72 * 6, 5, 160)
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text("\n".join(json.dumps(r) for r in rows) + "\n")
