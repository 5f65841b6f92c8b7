"""Operator-level Python wrappers over the C ABI's mgb_op_* entry points (used by layer parity tests
and by tools/bringup.py). Tensors are torch CUDA tensors; layouts are the library's internal ones
(NHWC / token-major, bf16 operands, fp32 trunk)."""
from __future__ import annotations

import torch

from . import _lib
from ._lib import check, ptr, stream_ptr


def pack_conv_weight(w: torch.Tensor, cin_pad: int | None = None) -> torch.Tensor:
    """[Cout, Cin, kh, kw] (PyTorch) -> bf16 [Cout, kh*kw*Cin_pad] tap-major (tap = kh*3 + kw)."""
    cout, cin, kh, kw = w.shape
    cp = cin_pad or cin
    out = torch.zeros(cout, kh * kw, cp, dtype=torch.float32, device=w.device)
    out[:, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, kh * kw, cin).float()
    return out.reshape(cout, kh * kw * cp).to(torch.bfloat16).contiguous()


def linear(a, w, bias=None, residual=None, out_f32=True, out_bf16=False, flags=0, block_n=0, splits=0, stages=0,
           ws=None):
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if flags & _lib.EPI_GEGLU else N
    of = torch.empty(M, n_out, dtype=torch.float32, device=a.device) if out_f32 else None
    ob = torch.empty(M, n_out, dtype=torch.bfloat16, device=a.device) if out_bf16 else None
    check(lib.mgb_op_linear(ptr(a), ptr(w), ptr(bias), ptr(residual), ptr(of), ptr(ob), M, N, K, flags, block_n,
                            splits, stages, ptr(ws), stream_ptr()), "mgb_op_linear")
    return of, ob


def conv2d(x, w_packed, bias, NB, Hout, Wout, Cin, Cout, kind=0, residual=None, out_f32=True, out_bf16=False, flags=0,
           block_n=0, splits=0, stages=0, ws=None):
    lib = _lib.load()
    of = torch.empty(NB, Hout, Wout, Cout, dtype=torch.float32, device=x.device) if out_f32 else None
    ob = torch.empty(NB, Hout, Wout, Cout, dtype=torch.bfloat16, device=x.device) if out_bf16 else None
    check(lib.mgb_op_conv2d(ptr(x), ptr(w_packed), ptr(bias), ptr(residual), ptr(of), ptr(ob), NB, Hout, Wout, Cin,
                            Cout, kind, flags, block_n, splits, stages, ptr(ws), stream_ptr()), "mgb_op_conv2d")
    return of, ob


def linear_ex(a, w, bias=None, residual=None, a2=None, out=None, out_bf16=None, ldo=0, flags=0, scale=1.0,
              sched_x=None, sched_z=None, sched_k=None, aux_out=None, block_n=0, splits=0, stages=0, ws=None):
    """mgb_op_linear_ex: every input the network's GEMMs use; outputs are caller-allocated ([M, ldo] rows)."""
    lib = _lib.load()
    M, K = a.shape
    N = w.shape[0]
    K2 = a2.shape[1] if a2 is not None else 0
    check(lib.mgb_op_linear_ex(ptr(a), ptr(a2), ptr(w), ptr(bias), ptr(residual), ptr(out), ptr(out_bf16), M, N, K, K2,
                               ldo, flags, float(scale), ptr(sched_x), ptr(sched_z), ptr(sched_k), ptr(aux_out), block_n,
                               splits, stages, ptr(ws), stream_ptr()), "mgb_op_linear_ex")
    return out, out_bf16


def conv2d_ex(x, w_packed, bias, NB, Hout, Wout, Cin, Cout, kind=0, x2=None, Cin2=0, Hsrc=0, Wsrc=0, residual=None,
              out=None, out_bf16=None, flags=0, scale=1.0, sched_x=None, sched_z=None, sched_k=None, aux_out=None,
              block_n=0, splits=0, stages=0, ws=None):
    """mgb_op_conv2d_ex: second (1x1) operand, source extent, scale and scheduler inputs; outputs caller-allocated."""
    lib = _lib.load()
    check(lib.mgb_op_conv2d_ex(ptr(x), ptr(x2), ptr(w_packed), ptr(bias), ptr(residual), ptr(out), ptr(out_bf16), NB, Hout,
                               Wout, Cin, Cin2, Cout, kind, Hsrc, Wsrc, flags, float(scale), ptr(sched_x), ptr(sched_z),
                               ptr(sched_k), ptr(aux_out), block_n, splits, stages, ptr(ws), stream_ptr()),
          "mgb_op_conv2d_ex")
    return out, out_bf16


def flash_attn64(qkv, NB, T, C, scale):
    lib = _lib.load()
    out = torch.empty(NB * T, C, dtype=torch.bfloat16, device=qkv.device)
    check(lib.mgb_op_flash_attn64(ptr(qkv), ptr(out), NB, T, C, float(scale), stream_ptr()), "mgb_op_flash_attn64")
    return out


def groupnorm(x, gamma, beta, NB, HW, C, G, eps, silu):
    lib = _lib.load()
    y = torch.empty(NB, HW, C, dtype=torch.bfloat16, device=x.device)
    nbytes = int(lib.mgb_op_groupnorm_ws_bytes(NB, HW, C, G))
    if nbytes == 0:
        raise _lib.MgbError(f"groupnorm: unsupported shape NB={NB} HW={HW} C={C} G={G}")
    ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=x.device)
    check(lib.mgb_op_groupnorm(ptr(x), ptr(y), ptr(gamma), ptr(beta), ptr(ws), NB, HW, C, G, float(eps), int(silu),
                               stream_ptr()), "mgb_op_groupnorm")
    return y


def groupnorm_ex(xa, xb, gamma, beta, NB, HW, G, eps, silu, raw_copy=False):
    """GroupNorm over the channel concat [xa | xb] (xb may be None); returns (y, raw bf16 copy of the concat or None)."""
    lib = _lib.load()
    Ca = xa.shape[-1]
    Cb = xb.shape[-1] if xb is not None else 0
    y = torch.empty(NB, HW, Ca + Cb, dtype=torch.bfloat16, device=xa.device)
    raw = torch.empty_like(y) if raw_copy else None
    nbytes = int(lib.mgb_op_groupnorm_ws_bytes(NB, HW, Ca + Cb, G))
    if nbytes == 0:
        raise _lib.MgbError(f"groupnorm: unsupported shape NB={NB} HW={HW} C={Ca}+{Cb} G={G}")
    ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=xa.device)
    check(lib.mgb_op_groupnorm_ex(ptr(xa), Ca, ptr(xb), Cb, ptr(y), ptr(raw), ptr(gamma), ptr(beta), ptr(ws), NB, HW, G,
                                  float(eps), int(silu), stream_ptr()), "mgb_op_groupnorm_ex")
    return y, raw


def xattn2(x, ln2_g, ln2_b, ln3_g, ln3_b, GU, c1, H, scale, eps=1e-5):
    """Collapsed cross-attention against the fixed 2-token context, fused with norm2 / norm3 (see include/marigold_b200.h)."""
    lib = _lib.load()
    M, Cc = x.shape
    y = torch.empty(M, Cc, dtype=torch.bfloat16, device=x.device)
    a = torch.empty(M, Cc, dtype=torch.bfloat16, device=x.device)
    check(lib.mgb_op_xattn2(ptr(x), ptr(y), ptr(a), ptr(ln2_g), ptr(ln2_b), ptr(ln3_g), ptr(ln3_b), ptr(GU), ptr(c1), M, Cc,
                            H, float(scale), float(eps), stream_ptr()), "mgb_op_xattn2")
    return y, a


def layernorm(x, gamma, beta, eps=1e-5):
    lib = _lib.load()
    M, Cc = x.shape
    y = torch.empty(M, Cc, dtype=torch.bfloat16, device=x.device)
    check(lib.mgb_op_layernorm(ptr(x), ptr(y), ptr(gamma), ptr(beta), M, Cc, float(eps), stream_ptr()),
          "mgb_op_layernorm")
    return y


def space_to_depth(x):
    lib = _lib.load()
    NB, H, W, Cc = x.shape
    y = torch.empty(NB, 4, (H + 1) // 2, (W + 1) // 2, Cc, dtype=torch.bfloat16, device=x.device)
    check(lib.mgb_op_space_to_depth(ptr(x), ptr(y), NB, H, W, Cc, stream_ptr()), "mgb_op_space_to_depth")
    return y


def upsample2x(x, Ho=None, Wo=None):
    """Nearest x2 upsampling, optionally cropped to Ho = 2H - 1 / Wo = 2W - 1."""
    lib = _lib.load()
    NB, H, W, Cc = x.shape
    Ho, Wo = Ho or 2 * H, Wo or 2 * W
    y = torch.empty(NB, Ho, Wo, Cc, dtype=torch.bfloat16, device=x.device)
    check(lib.mgb_op_upsample2x_ex(ptr(x), ptr(y), NB, H, W, Cc, Ho, Wo, stream_ptr()), "mgb_op_upsample2x_ex")
    return y


def softmax_rows(s, n):
    """fp32 scores [M, ld] (first n columns valid) -> bf16 probabilities [M, ld], pad columns zero."""
    lib = _lib.load()
    M, ld = s.shape
    p = torch.empty(M, ld, dtype=torch.bfloat16, device=s.device)
    check(lib.mgb_op_softmax_rows(ptr(s), ptr(p), M, n, ld, stream_ptr()), "mgb_op_softmax_rows")
    return p


def pack_decoder_latent(latent, w, b, inv_scale):
    """fp32 latent NCHW [NB, 4, h, w] -> bf16 [NB * h * w, 64]: post_quant_conv(latent * inv_scale) (w fp32 [4, 4],
    b fp32 [4]) in channels 0..3, zeros in 4..63."""
    lib = _lib.load()
    NB, _, h, w_ = latent.shape
    z = torch.empty(NB * h * w_, 64, dtype=torch.bfloat16, device=latent.device)
    check(lib.mgb_op_pack_decoder_latent(ptr(latent), ptr(w), ptr(b), float(inv_scale), ptr(z), NB, h * w_, stream_ptr()),
          "mgb_op_pack_decoder_latent")
    return z


def transpose_bf16(x, ld):
    """bf16 [M, N] -> bf16 [N, ld], columns [M, ld) zero."""
    lib = _lib.load()
    M, N = x.shape
    y = torch.empty(N, ld, dtype=torch.bfloat16, device=x.device)
    check(lib.mgb_op_transpose_bf16(ptr(x), ptr(y), M, N, ld, stream_ptr()), "mgb_op_transpose_bf16")
    return y
