"""CPU checks of the operator-test machinery (tests/ops_ref.py, tests/ops_cases.py): the per-element bound check
fails on a single element off by twice its bound, and the case list is well formed."""
import pytest
import torch

from tests import ops_ref


def _data(n=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(n, generator=g, dtype=torch.float64) * torch.logspace(-6, 3, n, dtype=torch.float64)
    bound = ops_ref.U_BF16 * ref.abs() + ops_ref.TINY
    return ref, bound


def test_assert_within_passes_at_the_bound():
    ref, bound = _data()
    out = ref + 0.999 * bound * torch.sign(torch.randn(ref.shape, generator=torch.Generator().manual_seed(1)))
    r = ops_ref.assert_within(out, ref, bound, "cpu.at_bound")
    assert r["worst"] <= 1.0


@pytest.mark.parametrize("where", [0, 1234, 4095])
def test_assert_within_catches_one_element_off_by_twice_its_bound(where):
    ref, bound = _data()
    out = ref.clone()
    out[where] += 2 * bound[where]
    with pytest.raises(AssertionError, match=rf"\({where},\)"):
        ops_ref.assert_within(out, ref, bound, "cpu.perturbed")
    r = ops_ref.within(out, ref, bound)
    assert r["index"] == (where,) and r["worst"] == pytest.approx(2.0)


def test_assert_within_rejects_nan():
    ref, bound = _data(16)
    out = ref.clone()
    out[3] = float("nan")
    with pytest.raises(AssertionError):
        ops_ref.assert_within(out, ref, bound, "cpu.nan")


def test_bf16_rounding_stays_inside_the_half_ulp_term():
    # the bf16 rounding of the exact value is exactly what U_BF16 * |ref| allows: never more
    ref = torch.randn(1 << 16, dtype=torch.float64) * 10
    out = ref.to(torch.bfloat16).to(torch.float64)
    assert ops_ref.within(out, ref, ops_ref.bf16_bound(ref, torch.zeros_like(ref)))["worst"] <= 1.0


def test_gemm_bound_is_far_below_a_dropped_k_block():
    # one 64-deep K block out of 10 missing moves an output by ~sqrt(64) |a||b|: the bound must not absorb it
    g = torch.Generator().manual_seed(2)
    a = torch.randn(64, 640, generator=g).to(torch.bfloat16)
    w = (torch.randn(32, 640, generator=g) / 640 ** 0.5).to(torch.bfloat16)
    ref, absprod = ops_ref.matmul64(a, w)
    dropped, _ = ops_ref.matmul64(a[:, 64:], w[:, 64:])
    bound = ops_ref.gemm_bound(640, absprod, ref, True)
    assert ops_ref.within(dropped, ref, bound)["worst"] > 10


def test_case_names_are_unique():
    from tests.ops_cases import cases

    names = [c[0] for c in cases()]
    assert len(names) == len(set(names))
