"""Device-side pre / post-processing bookends (csrc/image.cu) with the reference's semantics:

    resize          torchvision.transforms.functional.resize(img, size, interpolation, antialias=True)
                    (marigold/util/image_util.py:90-120; marigold_depth_pipeline.py:306-312)
    colorize_u8     colorize_depth_maps + chw2hwc + (x * 255).astype(uint8)   (image_util.py:38-76; depth_pipeline.py:326-331)

CUDA tensors only (the product path has no CPU fallback)."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr

_MODES = {"bilinear": 0, "bicubic": 1, "nearest-exact": 2}
_ARITH = {"cpu": 0, "cuda": 1}
_lut_cache = {}


def resize(img: torch.Tensor, size, mode: str, post: int = 0, arith: str = "cuda") -> torch.Tensor:
    """img [N,C,H,W] uint8 or float (CUDA) -> float32 [N,C,h,w]. post: 0 none; 1 clamp to [0,255] and round half to even
    (what a uint8 image becomes); 2 that, then x / 255 * 2 - 1; 3 x / 255 * 2 - 1 alone. arith: whose arithmetic the
    antialiased modes reproduce bit for bit in their tap windows and weights, torch's "cpu" kernel (an image the
    reference resizes on the host) or its "cuda" kernel (a prediction the reference resizes on the device)."""
    if not img.is_cuda:
        raise _lib.MgbError("marigold_b200.imageops.resize needs a CUDA tensor (no CPU fallback)")
    if mode not in _MODES:
        raise ValueError(f"Unknown resampling method: {mode}")
    if arith not in _ARITH:
        raise ValueError(f"Unknown resize arithmetic: {arith}")
    lib = _lib.load()
    N, Cc, H, W = img.shape
    h, w = int(size[0]), int(size[1])
    is_u8 = img.dtype == torch.uint8
    src = img.contiguous() if is_u8 else img.to(torch.float32).contiguous()
    with torch.cuda.device(img.device):
        dst = torch.empty(N, Cc, h, w, dtype=torch.float32, device=img.device)
        tmp = torch.empty(N * Cc * H * w, dtype=torch.float32, device=img.device)
        check(lib.mgb_resize_ex(ptr(src), int(is_u8), N * Cc, H, W, ptr(dst), h, w, _MODES[mode], _ARITH[arith],
                                int(post), ptr(tmp), stream_ptr()), "mgb_resize_ex")
    return dst


def spectral_lut_u8() -> np.ndarray:
    from .pipeline import _SPECTRAL_LUT

    return (_SPECTRAL_LUT * 255).astype(np.uint8)            # the cast the reference applies to the coloured map


def colorize_u8(depth: torch.Tensor, dmin: float, dmax: float, lut_u8: np.ndarray) -> torch.Tensor:
    """depth [H,W] float32 CUDA -> uint8 [H,W,3] CUDA through a 256-entry colour table (matplotlib's int(x * 256) lookup)."""
    if not depth.is_cuda:
        raise _lib.MgbError("marigold_b200.imageops.colorize_u8 needs a CUDA tensor (no CPU fallback)")
    lib = _lib.load()
    d = depth.to(torch.float32).contiguous()
    key = (d.device, lut_u8.tobytes())
    lut = _lut_cache.get(key)
    if lut is None:
        lut = torch.from_numpy(np.ascontiguousarray(lut_u8, dtype=np.uint8)).to(d.device)
        _lut_cache[key] = lut
    with torch.cuda.device(d.device):
        out = torch.empty(d.shape + (3,), dtype=torch.uint8, device=d.device)
        check(lib.mgb_colorize(ptr(d), d.numel(), float(dmin), float(dmax), ptr(lut), ptr(out), stream_ptr()), "mgb_colorize")
    return out
