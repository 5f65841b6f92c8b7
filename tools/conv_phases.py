"""Phase breakdown (clock64 stamps) + event timing of the dominant 3x3 conv (96x96, 320->320).
Usage: python tools/conv_phases.py [stages ...]"""
import ctypes as C
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from marigold_b200 import _lib, ops  # noqa: E402

lib = _lib.load()
raw = C.CDLL(str(_lib.lib_path()))
raw.mgb_debug_gemm_timing.argtypes = [C.c_void_p]


def run(H, W, Cin, Cout, bn, stages, reps=20, flags=0):
    x = torch.randn(1, H, W, Cin, device="cuda").to(torch.bfloat16)
    w = ops.pack_conv_weight((torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5))
    dbg = torch.zeros(4096, 8, dtype=torch.int64, device="cuda")
    fn = lambda: ops.conv2d(x, w, None, 1, H, W, Cin, Cout, kind=0, block_n=bn, stages=stages, flags=flags)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    raw.mgb_debug_gemm_timing(C.c_void_p(dbg.data_ptr()))
    fn()
    torch.cuda.synchronize()
    raw.mgb_debug_gemm_timing(None)
    d = dbg.cpu().double()
    d = d[d[:, 0] > 0]
    ph = {"prologue": d[:, 1] - d[:, 0], "first": d[:, 2] - d[:, 1], "mainloop": d[:, 3] - d[:, 2],
          "epilogue": d[:, 4] - d[:, 3], "total": d[:, 5] - d[:, 0]}
    s = " ".join(f"{k}={v.median().item():.0f}/{v.max().item():.0f}" for k, v in ph.items())
    fl = 2.0 * H * W * Cout * Cin * 9
    print(f"{H}x{W} {Cin}->{Cout} bn{bn} st{stages} flags={flags:#x}: {us:.1f} us ({fl / us * 1e-6:.0f} TF/s) ctas={len(d)} cycles(med/max): {s}",
          flush=True)


if __name__ == "__main__":
    st = [int(a) for a in sys.argv[1:]] or [0]
    for s in st:
        run(96, 96, 320, 320, 160, s)
        
    run(96, 96, 320, 640, 256, 4)

