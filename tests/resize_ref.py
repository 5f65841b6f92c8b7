"""Plain restatements of the antialiased resize (torch `F.interpolate(..., antialias=True, align_corners=False)`, which
torchvision's `resize(antialias=True)` calls) that csrc/image.cu is held to.

Three forms, all separable with the horizontal pass (W -> w) first and the vertical pass (H -> h) over its float32 rows:

* `resize64` — float64 from the definition. scale = in / out, centre c = scale (o + 1/2), support S = (n / 2) max(scale, 1)
  (n = 2 for the triangle, 4 for Keys a = -0.5), taps k in [max(floor(c - S + 1/2), 0), min(floor(c + S + 1/2), in)),
  weight f((k - c + 1/2) / max(scale, 1)) normalised by the window's sum.
* `emulate(..., arith="cpu")` — torch's CPU kernel (aten/src/ATen/native/cpu/UpSampleKernel.cpp) step by step in
  float32, with the float64 intermediates C++ promotion gives it: the window bounds `int64(double(c - S) + 0.5)`, the tap
  offset `float((double(float(j + xmin) - c) + 0.5) * invscale)`, the bilinear `float(1.0 - double(x))`, a Keys
  polynomial whose multiply-adds the compiler contracts to FMAs (the AVX2 / AVX512 builds), `w / total`, the window
  length clamped to ceil(S) * 2 + 1, and the accumulation `out = t0 w0`, then taps 1 .. n - 1 in order: the compiler
  vectorises their products four at a time and adds them one by one (a rounded product, then a rounded add), and the
  last (n - 1) % 4 taps run in the scalar epilogue as `fma(tj, wj, out)`.
* `emulate(..., arith="cuda")` — torch's CUDA kernel (ATen/native/cuda/UpSample.cuh, `upsample_antialias`) step by
  step in float32 as nvcc compiles it: the centre scale (o + 0.5f) is never rounded on its own but contracted into
  each use, giving window bounds `int(fma(t, scale, -S) + 0.5f)` / `int(fma(t, scale, S) + 0.5f)` and the offset
  `(j + fma(-t, scale, xmin) + 0.5f) * invscale` (t = o + 0.5f); the filter functors with nvcc's default FMA
  contraction, `w / total`, and the same accumulation.

`bound` gives a per-element bound on |out - resize64| for either emulation (and so for the kernel), derived below with
u = 2^-24 and gamma_n = n u / (1 - n u). For one output of one pass, with m the number of taps, f_k the exact filter
values, T = sum f_k, F = sum |f_k|, and x the pass's input:

1. Centre: scale and c are rounded once each, so |c^ - c| <= dc = 2.01 u c.
2. Tap offset: (k - c) and (+ 1/2) are rounded at magnitude <= S + 2, the product with invscale (itself within u of
   1 / scale) once more, so |d^ - d| <= dd = invscale (dc + 2u (S + 2)) + 2.01 u A with A = n / 2 + 1 >= |d|.
3. Filter: f is L-Lipschitz (L = 1 for the triangle, 25/18 for Keys a = -0.5) and its few float32 operations on |x| <= 2
   add at most ef = 16 u, so |f^_k - f_k| <= df = L dd + ef.
4. Window ends: the start c - S + 1/2 (and the end) is computed within dv = dc + 2u (c + S + 1) of its value, so a tap
   present in one window and not the other sits within invscale dv of the filter's edge, where f = 0: its |f| is at most
   L invscale dv + df. With both ends, sum |f^_k - f_k| over the union of the windows is at most D = m df + 2 (L invscale
   dv + df).
5. Normalisation: the float32 sum of m values gives |T^ - T| <= dT = D + gamma_m (F + D); one division each, so
   sum |w^_k - w_k| <= W1 = D / T^ + F dT / (T T^) + u (F + D) / T^, with T^ >= T - dT.
6. Accumulation: the product-then-FMA chain over m taps adds at most gamma_m sum |w^_k x_k| <= gamma_m (1 + u) (F + D) /
   T^ * M, M = max |x| over the union window; the weight error adds W1 M.
7. The vertical pass applies 5 and 6 to the first pass's float32 rows (M grown by their bound), and carries the first
   pass's error e1 through its weights: + sum |w^_k| max e1 <= (F + D) / T^ (1 + u) max e1.

m is taken as the definition's window length plus two, so the bound does not trust any emulation's window.

`to_u8` is torchvision's uint8 rule: clamp to [0, 255] first for bicubic, round half to even, cast.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
INTERP = {"bilinear": 2, "bicubic": 4}
LIP = {"bilinear": 1.0, "bicubic": 25.0 / 18.0}
F32, F64 = np.float32, np.float64


# ---- float32 fused multiply-add, exactly -----------------------------------------------------------------------------
def fma32(a, b, c):
    """float32 fma(a, b, c) rounded once: the product is exact in float64, the sum's rounding error is recovered with
    TwoSum, and a float64 sum that lands on a float32 midpoint is moved off it in the direction of that error."""
    a, b, c = (np.asarray(v, dtype=F32) for v in (a, b, c))
    p = a.astype(F64) * b.astype(F64)
    cc = c.astype(F64)
    s = p + cc
    bb = s - p
    err = (p - (s - bb)) + (cc - bb)
    r = s.astype(F32)
    rd = r.astype(F64)
    other = np.nextafter(r, np.where(s > rd, F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (rd != s) & (np.abs(other.astype(F64) - s) == np.abs(s - rd)) & (err != 0)
    toward_other = np.sign(err) == np.sign(other.astype(F64) - rd)
    return np.where(mid & toward_other, other, r).astype(F32)


# ---- filters ----------------------------------------------------------------------------------------------------------
def _filter64(x, method):
    x = np.abs(np.asarray(x, dtype=F64))
    if method == "bilinear":
        return np.where(x < 1, 1 - x, 0.0)
    a = -0.5
    p1 = ((a + 2) * x - (a + 3)) * x * x + 1
    p2 = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1, p1, np.where(x < 2, p2, 0.0))


def _filter_cpu(x, method):
    x = np.abs(np.asarray(x, dtype=F32))
    if method == "bilinear":
        return np.where(x < 1, (1.0 - x.astype(F64)).astype(F32), F32(0))
    # cubic_convolution1 / 2 (ATen/native/UpSample.h) with A = -0.5, multiply-adds contracted
    p1 = fma32(fma32(F32(1.5), x, F32(-2.5)) * x, x, F32(1))
    p2 = fma32(fma32(fma32(F32(-0.5), x, F32(2.5)), x, F32(-4)), x, F32(2))
    return np.where(x < 1, p1, np.where(x < 2, p2, F32(0))).astype(F32)


def _filter_cuda(x, method):
    x = np.abs(np.asarray(x, dtype=F32))
    if method == "bilinear":
        return np.where(x < 1, F32(1) - x, F32(0)).astype(F32)
    # BicubicFilterFunctor: ((a + 2) x - (a + 3)) x x + 1 and (((x - 5) x + 8) x - 4) a, contracted by nvcc
    p1 = fma32(fma32(F32(1.5), x, F32(-2.5)) * x, x, F32(1))
    p2 = fma32(fma32(x - F32(5), x, F32(8)), x, F32(-4)) * F32(-0.5)
    return np.where(x < 1, p1, np.where(x < 2, p2, F32(0))).astype(F32)


# ---- tap windows and weights of one axis ------------------------------------------------------------------------------
def weights(in_len: int, out_len: int, method: str, arith: str):
    """(xmin [out], xsize [out], w float32 [out, K]) exactly as the `arith` ("cpu" / "cuda") kernel computes them;
    w[o, j] is the weight of input xmin[o] + j (zero past xsize)."""
    n = INTERP[method]
    scale = F32(in_len) / F32(out_len)
    support = F32(F64(n * 0.5) * F64(scale)) if scale >= 1 else F32(n * 0.5)
    invscale = F32(1.0 / F64(scale)) if scale >= 1 else F32(1)
    o = np.arange(out_len)
    if arith == "cpu":
        center = (F64(scale) * (o + 0.5)).astype(F32)
        xmin = np.maximum(np.trunc((center - support).astype(F64) + 0.5).astype(np.int64), 0)
        xmax = np.trunc((center + support).astype(F64) + 0.5).astype(np.int64)
        xsize = np.clip(np.minimum(xmax, in_len) - xmin, 0, int(math.ceil(support)) * 2 + 1)
    elif arith == "cuda":
        # nvcc contracts the centre into each use: fma(t, scale, -support), fma(t, scale, support) and
        # fma(-t, scale, xmin) with t = o + 0.5f, so the centre itself is never rounded
        t = (o.astype(F32) + F32(0.5)).astype(F32)
        xmin = np.maximum(np.trunc((fma32(t, scale, -support) + F32(0.5)).astype(F32)).astype(np.int64), 0)
        xmax = np.trunc((fma32(t, scale, support) + F32(0.5)).astype(F32)).astype(np.int64)
        xsize = np.minimum(xmax, in_len) - xmin
    else:
        raise ValueError(arith)
    K = max(int(xsize.max()), 1)
    j = np.arange(K)[None, :]
    live = j < xsize[:, None]
    if arith == "cpu":
        d = ((j + xmin[:, None]).astype(F32) - center[:, None]).astype(F32)
        arg = ((d.astype(F64) + 0.5) * F64(invscale)).astype(F32)
        f = _filter_cpu(arg, method)
    else:
        xmc = fma32(-t, scale, xmin.astype(F32))
        arg = ((((j.astype(F32) + xmc[:, None]).astype(F32) + F32(0.5)).astype(F32)) * invscale).astype(F32)
        f = _filter_cuda(arg, method)
    f = np.where(live, f, F32(0)).astype(F32)
    total = np.zeros(out_len, dtype=F32)
    for k in range(K):                                        # sequential float32 sum in tap order
        total = (total + f[:, k]).astype(F32)
    safe = np.where(total != 0, total, F32(1))
    w = np.where(total[:, None] != 0, (f / safe[:, None]).astype(F32), f).astype(F32)
    return xmin, xsize, np.where(live, w, F32(0)).astype(F32)


def windows64(in_len: int, out_len: int, method: str):
    """The definition's windows, centres and raw filter values in float64: (xmin, xsize, f [out, K], center)."""
    n = INTERP[method]
    scale = in_len / out_len
    support = n * 0.5 * max(scale, 1.0)
    invscale = 1.0 / max(scale, 1.0)
    o = np.arange(out_len)
    center = scale * (o + 0.5)
    xmin = np.maximum(np.floor(center - support + 0.5).astype(np.int64), 0)
    xsize = np.minimum(np.floor(center + support + 0.5).astype(np.int64), in_len) - xmin
    K = max(int(xsize.max()), 1)
    j = np.arange(K)[None, :]
    f = np.where(j < xsize[:, None], _filter64((j + xmin[:, None] - center[:, None] + 0.5) * invscale, method), 0.0)
    return xmin, xsize, f, center


def weight_matrix(xmin, xsize, w, in_len):
    """Dense [out, in] matrix of a tap table."""
    out_len, K = w.shape
    M = np.zeros((out_len, in_len), dtype=w.dtype)
    for j in range(K):
        live = j < xsize
        M[np.arange(out_len)[live], (xmin + j)[live]] = w[live, j]
    return M


# ---- the resize ------------------------------------------------------------------------------------------------------
def _pass_emul(x, in_len, out_len, method, arith, axis):
    """One float32 pass along `axis` of x (the other axes ride along), in tap order from out = t0 w0.

    CUDA: every later tap is an FMA. CPU: the compiler vectorises the products of taps 1 .. n - 1 in groups of four and
    adds them in order, so those taps are a rounded product then a rounded add; the (n - 1) % 4 taps left over run
    in the scalar epilogue as FMAs. Both passes follow this rule."""
    xmin, xsize, w = weights(in_len, out_len, method, arith)
    x = np.moveaxis(x, axis, -1)
    first_fma = np.ones_like(xsize) if arith == "cuda" else xsize - (xsize - 1) % 4     # taps j >= this are FMAs
    out = None
    for j in range(w.shape[1]):
        live = j < xsize
        idx = np.minimum(xmin + j, in_len - 1)
        t = x[..., idx]
        if j == 0:
            out = (t * w[:, 0]).astype(F32)
        else:
            fused = fma32(t, w[:, j], out)
            split = (out + (t * w[:, j]).astype(F32)).astype(F32)
            out = np.where(live, np.where(j >= first_fma, fused, split), out).astype(F32)
    return np.moveaxis(out, -1, axis)


def _to_np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def emulate(x, size, method: str, arith: str) -> np.ndarray:
    """float32 [..., H, W] -> [..., h, w] as torch's `arith` kernel computes it."""
    x = _to_np(x).astype(F32)
    H, W = x.shape[-2:]
    h, w = int(size[0]), int(size[1])
    t = _pass_emul(x, W, w, method, arith, -1)
    return _pass_emul(t, H, h, method, arith, -2)


def _pass64(x, in_len, out_len, method, axis):
    xmin, xsize, f, _ = windows64(in_len, out_len, method)
    T = f.sum(1)
    w = f / np.where(T != 0, T, 1.0)[:, None]
    M = weight_matrix(xmin, xsize, w, in_len)
    return np.moveaxis(np.moveaxis(x, axis, -1) @ M.T, -1, axis)


def resize64(x, size, method: str) -> np.ndarray:
    x = _to_np(x).astype(F64)
    H, W = x.shape[-2:]
    t = _pass64(x, W, int(size[1]), method, -1)
    return _pass64(t, H, int(size[0]), method, -2)


def _gamma(m):
    return m * U / (1 - m * U)


def _pass_bound(absx, e_in, in_len, out_len, method, axis):
    """Per-output bound of one pass (steps 1-7 of the module docstring). absx: |input| (its own rounding already
    included through e_in), e_in: the input's error bound (0 for the first pass)."""
    n = INTERP[method]
    L = LIP[method]
    scale = in_len / out_len
    S = n * 0.5 * max(scale, 1.0)
    inv = 1.0 / max(scale, 1.0)
    xmin, xsize, f, c = windows64(in_len, out_len, method)
    m = xsize + 2
    T = f.sum(1)
    F = np.abs(f).sum(1)
    dc = 2.01 * U * c
    dd = inv * (dc + 2 * U * (S + 2)) + 2.01 * U * (n / 2 + 1)
    df = L * dd + 16 * U
    dv = dc + 2 * U * (c + S + 1)
    D = m * df + 2 * (L * inv * dv + df)
    g = _gamma(m)
    dT = D + g * (F + D)
    Th = T - dT
    assert np.all(Th > 0), "bound undefined: window sum not bounded away from zero"
    W1 = D / Th + F * dT / (T * Th) + U * (F + D) / Th
    Wabs = (F + D) / Th * (1 + U)
    # M and max e_in over the union window [xmin - 1, xmin + xsize + 1)
    a = np.moveaxis(absx + e_in, axis, -1)
    e = np.moveaxis(np.broadcast_to(e_in, absx.shape), axis, -1)
    lo = np.maximum(xmin - 1, 0)
    hi = np.minimum(xmin + xsize + 1, in_len)
    Mx = np.stack([a[..., lo[o]:hi[o]].max(-1) for o in range(out_len)], -1)
    Me = np.stack([e[..., lo[o]:hi[o]].max(-1) for o in range(out_len)], -1)
    b = W1 * Mx + g * Wabs * Mx + Wabs * Me
    return np.moveaxis(b, -1, axis)


def bound(x, size, method: str) -> np.ndarray:
    """Per-element bound on |emulate(x, size, method, arith) - resize64(x, size, method)| for either arith."""
    x = np.abs(_to_np(x).astype(F64))
    H, W = x.shape[-2:]
    h, w = int(size[0]), int(size[1])
    zero = np.zeros_like(x)
    e1 = _pass_bound(x, zero, W, w, method, -1)
    t = np.abs(_pass64(x, W, w, method, -1))                     # |first pass| <= this + e1 (|w| sums bounded by Wabs)
    tx = np.abs(_pass64_abs(x, W, w, method, -1))
    return _pass_bound(np.maximum(t, tx), e1, H, h, method, -2)


def _pass64_abs(x, in_len, out_len, method, axis):
    """sum |w_k| |x_k|: a bound on the first pass's magnitude that does not depend on cancellation."""
    xmin, xsize, f, _ = windows64(in_len, out_len, method)
    T = f.sum(1)
    M = weight_matrix(xmin, xsize, np.abs(f) / np.abs(T)[:, None], in_len)
    return np.moveaxis(np.moveaxis(np.abs(x), axis, -1) @ M.T, -1, axis)


def to_u8(v, method: str) -> np.ndarray:
    """torchvision's cast back to uint8 (`_cast_squeeze_out`): bicubic clamps first, then round half to even."""
    v = _to_np(v).astype(F32)
    if method == "bicubic":
        v = np.clip(v, 0, 255)
    return np.rint(v).astype(np.uint8)


def normalise_cpu(u8) -> np.ndarray:
    """The reference's `rgb / 255.0 * 2.0 - 1.0` on a CPU tensor: float32 true division, then two roundings."""
    t = torch.from_numpy(np.ascontiguousarray(_to_np(u8)))
    return (t / 255.0 * 2.0 - 1.0).numpy()


def identity_weights(resize_fn, in_len: int, out_len: int) -> np.ndarray:
    """The [out, in] weight matrix of a resize, read off exactly: an [in, 1, 1, in] one-hot stack resized to (1, out)
    gives each input's weight in every output (one tap times 1.0; the 1 -> 1 vertical pass is the identity)."""
    eye = torch.eye(in_len, dtype=torch.float32).reshape(in_len, 1, 1, in_len)
    out = _to_np(resize_fn(eye, (1, out_len))).reshape(in_len, out_len)
    return out.T.copy()
