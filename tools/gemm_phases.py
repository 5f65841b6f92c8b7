"""Per-phase cycle breakdown of gemm_tc_kernel via the clock64 debug hook.
stamps: 0 entry, 1 after prologue+pdl_wait, 2 first operand stage landed, 3 accumulator complete, 4 epilogue done, 5 exit"""
import ctypes as C
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from marigold_b200 import _lib  # noqa: E402
from marigold_b200._lib import check, ptr, stream_ptr  # noqa: E402

lib = _lib.load()
raw = C.CDLL(str(_lib.lib_path()))
raw.mgb_debug_gemm_timing.argtypes = [C.c_void_p]


def run(M, N, K, bn, stages, out_dtype="f32", flags=0):
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).to(torch.bfloat16)
    n_out = N // 2 if flags & 1 else N
    of = torch.empty(M, n_out, device="cuda") if out_dtype == "f32" else None
    ob = torch.empty(M, n_out, device="cuda", dtype=torch.bfloat16) if out_dtype == "bf16" else None
    bias = torch.randn(N, device="cuda")
    ctas = ((M + 127) // 128) * ((N + bn - 1) // bn)
    dbg = torch.zeros(ctas, 8, dtype=torch.int64, device="cuda")

    def fn():
        check(lib.mgb_op_linear(ptr(a), ptr(w), ptr(bias), None, ptr(of), ptr(ob), M, N, K, flags, bn, 1, stages, None, stream_ptr()), "lin")
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    raw.mgb_debug_gemm_timing(C.c_void_p(dbg.data_ptr()))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    raw.mgb_debug_gemm_timing(None)
    d = dbg.cpu().double()
    ph = {"prologue": (d[:, 1] - d[:, 0]), "first_stage": (d[:, 2] - d[:, 1]), "mainloop": (d[:, 3] - d[:, 2]),
          "epilogue": (d[:, 4] - d[:, 3]), "teardown": (d[:, 5] - d[:, 4]), "total": (d[:, 5] - d[:, 0])}
    s = " ".join(f"{k}={v.median().item():.0f}/{v.max().item():.0f}" for k, v in ph.items())
    s += f" mainloop/kb={ph['mainloop'].median().item() / (K // 64):.0f}"
    print(f"M{M} N{N} K{K} bn{bn} st{stages} {out_dtype} flags={flags:#x}: event_us={e0.elapsed_time(e1)*1e3:.1f} ctas={ctas} cycles(median/max): {s}", flush=True)


if __name__ == "__main__":
    for bn in (64, 128, 160, 256):                       # K-loop cycles per 64-deep K block vs the tile width
        run(9216, 1280, 2880, bn, 4)
    run(128, 160, 64, 160, 2)
    run(9216, 320, 320, 160, 5)
    run(9216, 320, 320, 160, 5, "bf16")
    run(9216, 320, 2880, 160, 5)
    run(9216, 2560, 320, 256, 4, "bf16")
    run(9216, 2560, 320, 256, 2, "bf16", flags=1)        # FF-in + GEGLU as the network launches it
    run(9216, 960, 320, 256, 2, "bf16")                  # fused QKV
    run(2304, 5120, 640, 256, 2, "bf16", flags=1)
