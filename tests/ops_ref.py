"""Float64 references and per-element error bounds for the operator cases (tests/ops_cases.py).

Every reference is computed in float64 from the SAME bf16-rounded operands the kernel receives, so the only
differences left are the kernel's own roundings. Each bound below is a sum of terms, one per rounding the kernel
performs, and `within()` reports the worst element as max(|out - ref| / bound): a value <= 1 passes.

Constants measured on an H100 80GB HBM3 (400 W power limit) with MGB_PARITY_DIR set (tests/helpers.record):
  C_ACC  wgmma's fp32 accumulation: an fp32 output's error beyond the epilogue's roundings, over K 2^-24 (|A| |B|^T).
         At most 0.0093 over the 56 GEMM / conv cases with a plain fp32 output. Set to 0.02 (about 2x margin).
  C_P    the bf16 rounding of the softmax probabilities fed to the P V MMA, relative to 2^-8 sum_j p_ij |v_j|:
         0.60 at T = 8, where a few keys do not average out, and <= 0.50 elsewhere. Set to 1, the worst case of
         rounding every p_ij by 2^-8.
The other terms are analytic (one or a few fp32 / bf16 roundings) and are not fitted.
"""
from __future__ import annotations

import math

import torch

U_F32 = 2.0 ** -24    # unit roundoff of fp32
U_BF16 = 2.0 ** -8    # unit roundoff of bf16 (8-bit significand): |bf16(x) - x| <= 2^-8 |x|
C_ACC = 0.02
C_P = 1.0
R_F32_OUT = 4 * U_F32   # a few fp32 roundings in the epilogue (scale / bias / residual / store)
R_ACT = 2.0 ** -20      # fast-math exp in SiLU / the GELU polynomial (|gelu error| <= 2.6e-7)
R_NORM = 2.0 ** -14     # fp32 statistics and affine of the norms, relative to the magnitudes they combine
TINY = 2.0 ** -100


def record(name: str, value: float) -> float:
    from tests import helpers

    return helpers.record(name, value)


def within(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> dict:
    """Worst element of |out - ref| / bound (all float64), its index and the usual summary figures."""
    out = out.detach().to(torch.float64)
    ref = ref.detach().to(torch.float64)
    bound = torch.broadcast_to(bound.detach().to(torch.float64), ref.shape)
    d = (out - ref).abs()
    ratio = d / bound
    nan = bool(torch.isnan(out).any().item())
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, math.inf), ratio)
    flat = int(torch.argmax(ratio).item())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), ratio.shape))
    worst = float(ratio.reshape(-1)[flat].item())
    return {"worst": worst, "index": idx, "out": float(out[idx].item()), "ref": float(ref[idx].item()),
            "bound": float(bound[idx].item()), "max_abs": float(d.nan_to_num(math.inf).max().item()),
            "rel_to_max": float(d.nan_to_num(math.inf).max().item() / (ref.abs().max().item() + 1e-30)), "nan": nan}


def assert_within(out, ref, bound, name: str) -> dict:
    """Fail unless |out - ref| <= bound element-wise; the message names the worst element. Records max(|d| / bound)."""
    r = within(out, ref, bound)
    record(name, r["worst"])
    assert not r["nan"] and r["worst"] <= 1.0, (
        f"{name}: |out - ref| / bound = {r['worst']:.3g} at {r['index']} (out {r['out']!r}, ref {r['ref']!r}, "
        f"bound {r['bound']:.3g})")
    return r


# ---- bounds -------------------------------------------------------------------------------------------------------
def acc_bound(K: int, absprod: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """fp32 accumulation of a K-long bf16 dot product: c_acc * K * 2^-24 * sum_k |a_k| |b_k|."""
    return C_ACC * K * U_F32 * abs(scale) * absprod


def gemm_bound(K, absprod, ref, bf16_out, pre=None, scale=1.0, act_gain=None, act_err=None):
    """|out - ref| for a GEMM with the fused epilogue.
    pre: the float64 value before the residual (None: ref); act_gain: |f'| applied to the accumulator error (None: 1);
    act_err: the activation's own absolute error."""
    pre = ref if pre is None else pre
    e = acc_bound(K, absprod, scale)
    if act_gain is not None:
        e = e * act_gain
    e = e + R_F32_OUT * (pre.abs() + ref.abs())
    if act_err is not None:
        e = e + act_err
    if bf16_out:
        e = e + U_BF16 * ref.abs()
    return e + TINY


def bf16_bound(ref, mag):
    """A bf16 result of a well-conditioned fp32 computation: half an ulp (2^-8 |ref|, which is at most one ulp of
    bf16(ref)) plus R_NORM times the magnitudes the fp32 arithmetic combined (the slack that matters near zero)."""
    return U_BF16 * ref.abs() + R_NORM * mag + TINY


def attn_bound(ref, pv_abs):
    """bf16 output rounding + the bf16 P operand: c_p * 2^-8 * sum_j p_ij |v_j|."""
    return U_BF16 * ref.abs() + C_P * U_BF16 * pv_abs + TINY


def softmax_rel(n, dist, p):
    """Relative error of softmax_rows_kernel's fp32 probability p_j = exp(s_j - m) / sum before its bf16 rounding, on
    rows of n logits; dist = m - s_j >= 0 (float64, [rows, n]), p the float64 softmax.
      * exp(s_j - m): the fp32 subtraction rounds the argument by 2^-24 dist_j and __expf is within 2 + 1.173 dist_j
        ulps (CUDA Programming Guide), an ulp being at most 2^-23 relative: 2^-22 (1 + dist_j) together.
      * the row sum carries its terms' relative errors, at most 2^-22 (1 + sum_j p_j dist_j) weighted by the terms,
        plus its own fp32 additions: 256 threads each add ceil(n / 256) terms in order, then 5 shuffle levels and 8
        warp partials: (ceil(n / 256) + 16) 2^-24. At n = 4096 that is 2^-19, at n = 190 512 about 2^-14.4.
      * 1 / sum and the product: 2^-23."""
    dbar = (p * dist).sum(dim=-1, keepdim=True)
    return 2.0 ** -22 * (2 + dist + dbar) + (math.ceil(n / 256) + 16) * U_F32 + 2.0 ** -23


# ---- references ---------------------------------------------------------------------------------------------------
def f64(t):
    return t.detach().to(torch.float64)


def matmul64(a, w):
    """A [M, K] x W [N, K]^T in float64 and the matching |A| |W|^T."""
    a, w = f64(a), f64(w)
    return a @ w.t(), a.abs() @ w.abs().t()


def conv64(x_nchw, w, stride=1, padding=1):
    """Convolution in float64 and the same convolution of the absolute values (x, w already bf16-rounded)."""
    import torch.nn.functional as F

    x, w = f64(x_nchw), f64(w)
    return (F.conv2d(x, w, stride=stride, padding=padding),
            F.conv2d(x.abs(), w.abs(), stride=stride, padding=padding))


def silu64(t):
    return t * torch.sigmoid(t)


def gelu64(t):
    return 0.5 * t * (1.0 + torch.erf(t / math.sqrt(2.0)))


# |silu'| <= 1.0999 and |gelu'| <= 1.1289 everywhere
SILU_GAIN = 1.1
GELU_GAIN = 1.13
