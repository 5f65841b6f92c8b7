"""Operator-level GPU parity: every case calls one C-ABI operator and holds each output element to a float64
reference on the same bf16-rounded inputs, within the per-element bounds of tests/ops_ref.py (cases in
tests/ops_cases.py; the data-movement kernels are exact). Run with MGB_PARITY_DIR set, every case records its worst
|d| / bound, and the GEMM / attention cases the accumulation constants c_acc / c_p they imply."""
import pytest

from tests.ops_cases import _record, cases

pytestmark = pytest.mark.gpu
_CASES = cases()


@pytest.mark.parametrize("name,fn,kw", _CASES, ids=[c[0] for c in _CASES])
def test_operator(name, fn, kw):
    import torch

    res = fn(**kw)
    torch.cuda.synchronize()
    _record(name, res)
    assert res["ok"], {k: v for k, v in res.items() if k != "ms"}


def _conv_call(flags, Cout, block_n, **kw):
    import torch

    from marigold_b200 import ops

    NB, H, W, Cin = 1, 8, 8, 64
    x = torch.zeros(NB, H, W, Cin, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(Cout, 9 * Cin, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(NB, max(Cout, 1), H, W, device="cuda")
    return ops.conv2d_ex(x, w, None, NB, H, W, Cin, Cout, out=out, flags=flags, block_n=block_n, **kw)


@pytest.mark.parametrize("flags,Cout,block_n", [
    ("EPI_DEPTH", 3, 64),       # a wider tile would take the plain NHWC epilogue
    ("EPI_NORMALS", 3, 32),
    ("EPI_NCHW", 32, 0),        # more columns than the 16-wide row a lane holds
    ("EPI_NCHW", 32, 16),
    ("EPI_DEPTH", 4, 16),       # depth / normals are defined for 3 channels only
])
def test_special_epilogue_rejected_before_launch(flags, Cout, block_n):
    import torch

    from marigold_b200 import _lib

    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.mgb_launch_count()
    with pytest.raises(_lib.MgbError, match="special epilogue"):
        _conv_call(getattr(_lib, flags), Cout, block_n)
    assert lib.mgb_launch_count() == n0


def test_special_epilogue_rejects_split_k_and_missing_inputs():
    import torch

    from marigold_b200 import _lib

    ws = torch.empty(1 << 16, device="cuda")
    with pytest.raises(_lib.MgbError):
        _conv_call(_lib.EPI_NCHW, 4, 16, splits=3, ws=ws)
    with pytest.raises(_lib.MgbError, match="special epilogue"):
        _conv_call(_lib.EPI_SCHED, 4, 0)          # no sched_x / sched_k
