"""Python face of one libmarigold_b200 handle: weights in, (encode / denoise / decode) on torch CUDA
tensors. torch is plumbing only here (device memory + current stream); all compute is the library's.

The engine is the object the drop-in pipelines (pipeline.py) hold where the reference pipeline holds
`unet`, `vae` and `scheduler` (marigold/marigold_depth_pipeline.py:133-139).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr


@dataclass
class EngineConfig:
    unet_in_channels: int = 8
    unet_out_channels: int = 4
    unet_block_channels: List[int] = field(default_factory=lambda: [320, 640, 1280, 1280])
    unet_layers_per_block: int = 2
    unet_cross_dim: int = 1024
    vae_block_channels: List[int] = field(default_factory=lambda: [128, 256, 512, 512])
    vae_layers_per_block: int = 2
    vae_latent_channels: int = 4
    norm_groups: int = 32
    latent_scale: float = 0.18215

    @staticmethod
    def tiny() -> "EngineConfig":
        return EngineConfig(unet_block_channels=[64, 128, 256, 256], unet_cross_dim=128,
                            vae_block_channels=[64, 64, 128, 128])

    def to_c(self) -> _lib.mgb_config:
        c = _lib.mgb_config()
        c.unet_in_channels, c.unet_out_channels = self.unet_in_channels, self.unet_out_channels
        c.unet_block_channels = (C.c_int32 * 4)(*self.unet_block_channels)
        c.unet_layers_per_block, c.unet_cross_dim = self.unet_layers_per_block, self.unet_cross_dim
        c.vae_block_channels = (C.c_int32 * 4)(*self.vae_block_channels)
        c.vae_layers_per_block, c.vae_latent_channels = self.vae_layers_per_block, self.vae_latent_channels
        c.norm_groups, c.latent_scale = self.norm_groups, self.latent_scale
        return c


_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


class _DeviceBytes:
    """n bytes of device memory at `addr`, for torch.as_tensor to view without a copy."""

    def __init__(self, addr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "|u1", "data": (int(addr), False),
                                         "strides": None, "version": 2}


class Engine:
    def __init__(self, cfg: EngineConfig = EngineConfig(), device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise _lib.MgbError("marigold_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = _lib.load()
        self.cfg = cfg
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            ccfg = cfg.to_c()
            check(self.lib.mgb_create(C.byref(ccfg), C.byref(self._h)), "mgb_create")
        self._finalized = False
        self.n_steps = 0
        self._exchange_cb = None         # the installed row-split callback, referenced while the library may call it
        self._exchange_error = None

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            with torch.cuda.device(self.device):
                self.lib.mgb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    # ---- weights --------------------------------------------------------------------------------
    def load_state_dict(self, prefix: str, sd: Dict[str, torch.Tensor]) -> None:
        """`prefix` is "unet" or "vae"; keys are diffusers state-dict names."""
        for k, v in sd.items():
            t = v.detach().to("cpu").contiguous()
            if t.dtype not in _DT:
                t = t.float()
            shape = (C.c_int64 * t.dim())(*t.shape)
            check(self.lib.mgb_load_tensor(self._h, f"{prefix}.{k}".encode(), C.c_void_p(t.data_ptr()), shape, t.dim(),
                                           _DT[t.dtype]), f"mgb_load_tensor({prefix}.{k})")

    def finalize(self) -> None:
        with torch.cuda.device(self.device):
            check(self.lib.mgb_finalize_weights(self._h), "mgb_finalize_weights")
        self._finalized = True

    # ---- conditioning / schedule ----------------------------------------------------------------
    def set_text_embedding(self, embed: torch.Tensor) -> None:
        e = embed.detach().to("cpu", torch.float32).reshape(-1, embed.shape[-1]).contiguous()
        with torch.cuda.device(self.device):
            check(self.lib.mgb_set_text_embedding(self._h, C.c_void_p(e.data_ptr()), e.shape[0]),
                  "mgb_set_text_embedding")

    def set_schedule(self, timesteps, kx, kv, kz) -> None:
        ts = np.ascontiguousarray(np.asarray(timesteps, dtype=np.int32))
        kx, kv, kz = (np.ascontiguousarray(np.asarray(a, dtype=np.float32)) for a in (kx, kv, kz))
        n = len(ts)
        assert len(kx) == len(kv) == len(kz) == n
        with torch.cuda.device(self.device):
            check(self.lib.mgb_set_schedule(self._h, n, ts.ctypes.data_as(C.c_void_p), kx.ctypes.data_as(C.c_void_p),
                                            kv.ctypes.data_as(C.c_void_p), kz.ctypes.data_as(C.c_void_p)),
                  "mgb_set_schedule")
        self.n_steps = n

    # ---- one image on several GPUs ------------------------------------------------------------------
    def set_row_split(self, rank: int = 0, world: int = 1, exchange=None) -> None:
        """Split every attention's query rows over `world` ranks (mgb_set_row_split); exchange=None clears it.
        exchange(buf, rank, world) receives one attention's output as a uint8 CUDA tensor of `world` equal chunks, chunk
        `rank` holding this rank's rows, and must fill the other chunks in place (an all-gather, parallel.exchange_rows).
        It runs with the library call's stream as torch's current stream. While the split is installed the hot-path
        calls take one image at a time."""
        if exchange is None:
            check(self.lib.mgb_set_row_split(self._h, 0, 1, None, None), "mgb_set_row_split")
            self._exchange_cb = None
            return

        def call(ctx, buf, chunk_bytes, r, g, stream):
            try:
                view = torch.as_tensor(_DeviceBytes(buf, chunk_bytes * g), device=self.device)
                s = torch.cuda.ExternalStream(stream, device=self.device) if stream else \
                    torch.cuda.default_stream(self.device)
                with torch.cuda.stream(s):
                    exchange(view, r, g)
                return 0
            except Exception as e:  # noqa: BLE001 -- a Python error must not unwind through the library
                self._exchange_error = e
                return -1

        cb = _lib.EXCHANGE_FN(call)
        check(self.lib.mgb_set_row_split(self._h, rank, world, C.cast(cb, C.c_void_p), None), "mgb_set_row_split")
        self._exchange_cb = cb

    def _check(self, status: int, what: str) -> None:
        """check(), with the exchange function's own exception as the cause of a failure it caused."""
        err, self._exchange_error = self._exchange_error, None
        if status != 0 and err is not None:
            try:
                check(status, what)
            except _lib.MgbError as e:
                raise _lib.MgbError(f"{e}: {err!r}") from err
        check(status, what)

    # ---- hot path -------------------------------------------------------------------------------
    def _f32(self, t: torch.Tensor) -> torch.Tensor:
        return t.to(self.device, torch.float32).contiguous()

    def encode(self, rgb: torch.Tensor) -> torch.Tensor:
        rgb = self._f32(rgb)
        B, _, H, W = rgb.shape
        out = torch.empty(B, 4, H // 8, W // 8, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            self._check(self.lib.mgb_encode(self._h, ptr(rgb), B, H, W, ptr(out), stream_ptr()), "mgb_encode")
        return out

    def unet_step(self, rgb_latent, target, step_index: int, noise=None, want_model_out=False):
        """In-place update of `target` (fp32 CUDA). Returns the raw model output if requested."""
        rgb_latent = self._f32(rgb_latent)
        assert target.is_cuda and target.dtype == torch.float32 and target.is_contiguous()
        B, _, lh, lw = target.shape
        mo = torch.empty_like(target) if want_model_out else None
        nz = self._f32(noise) if noise is not None else None
        with torch.cuda.device(self.device):
            self._check(self.lib.mgb_unet_step(self._h, ptr(rgb_latent), ptr(target), ptr(nz), ptr(mo), step_index, B, lh,
                                               lw, stream_ptr()), "mgb_unet_step")
        return mo

    def denoise(self, rgb_latent, target, step_noise=None) -> torch.Tensor:
        rgb_latent = self._f32(rgb_latent)
        target = self._f32(target).clone()
        B, _, lh, lw = target.shape
        sn = self._f32(step_noise) if step_noise is not None else None
        with torch.cuda.device(self.device):
            self._check(self.lib.mgb_denoise(self._h, ptr(rgb_latent), ptr(target), ptr(sn), B, lh, lw, stream_ptr()),
                        "mgb_denoise")
        return target

    def denoise_range_(self, rgb_latent, target, first_step: int, num_steps: int, step_noise=None) -> None:
        """In place on `target` (fp32 CUDA, contiguous): steps [first_step, first_step + num_steps)."""
        assert target.is_cuda and target.dtype == torch.float32 and target.is_contiguous()
        assert rgb_latent.is_cuda and rgb_latent.dtype == torch.float32 and rgb_latent.is_contiguous()
        B, _, lh, lw = target.shape
        with torch.cuda.device(self.device):
            self._check(self.lib.mgb_denoise_range(self._h, ptr(rgb_latent), ptr(target), ptr(step_noise), first_step,
                                                   num_steps, B, lh, lw, stream_ptr()), "mgb_denoise_range")

    def decode(self, latent, mode: int) -> torch.Tensor:
        """mode: 0 depth head [B,1,H,W], 1 normals head, 2 raw RGB, 3 (clip + 1) / 2 (one IID target); latent [B,4,h,w]."""
        latent = self._f32(latent)
        B, c, lh, lw = latent.shape
        assert c == 4, f"the VAE decodes 4-channel latents, got {c}"
        ch = 1 if mode == 0 else 3
        out = torch.empty(B, ch, lh * 8, lw * 8, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            self._check(self.lib.mgb_decode(self._h, ptr(latent), B, lh, lw, mode, ptr(out), stream_ptr()), "mgb_decode")
        return out

    def workspace_bytes(self, B, H, W) -> int:
        """Device workspace a batch of B members at H x W pixels needs; 0 beyond the supported maximum."""
        return int(self.lib.mgb_workspace_bytes(self._h, B, H, W))

    def held_bytes(self) -> int:
        """Device workspace the engine holds now (given back before it grows)."""
        return int(self.lib.mgb_workspace_held_bytes(self._h))
