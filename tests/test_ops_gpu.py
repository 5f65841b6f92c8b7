"""Operator-level GPU parity at production shapes (every case: one C-ABI operator vs torch fp32 on the same
bf16-rounded inputs; tolerances inside tests/ops_cases.py: 2e-3 linear, 3e-3 conv, 2e-2 attention output in bf16,
6e-3 norms in bf16, exact for the data-movement kernels)."""
import os
import subprocess
import sys

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


@pytest.mark.parametrize("variant", ["1", "3"])
def test_conv_halo_variants(variant):
    """The opt-in 3x3-conv operand-reuse path (MGB_CONV_HALO: one shared-memory halo per channel block, the 9 taps as
    descriptors into it) on every conv case. The library reads the switch once per process, hence the child process."""
    env = {**os.environ, "MGB_CONV_HALO": variant}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", __file__, "-k", "test_operator and conv"],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout, r.stdout[-2000:]
