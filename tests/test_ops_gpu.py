"""Operator-level GPU parity at production shapes (every case: one C-ABI operator vs torch fp32 on the same
bf16-rounded inputs; tolerances inside tests/ops_cases.py: 2e-3 linear, 3e-3 conv, 2e-2 attention output in bf16,
6e-3 norms in bf16, exact for the data-movement kernels)."""
import pytest

from tests.ops_cases import cases

pytestmark = pytest.mark.gpu
_CASES = cases()


@pytest.mark.parametrize("name,fn,kw", _CASES, ids=[c[0] for c in _CASES])
def test_operator(name, fn, kw):
    import torch

    res = fn(**kw)
    torch.cuda.synchronize()
    assert res["ok"], {k: v for k, v in res.items() if k != "ms"}
