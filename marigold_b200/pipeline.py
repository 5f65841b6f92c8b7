"""Drop-in pipelines with the reference's call surface:

    MarigoldDepthPipeline.__call__     marigold/marigold_depth_pipeline.py:155-338
    MarigoldNormalsPipeline.__call__   marigold/marigold_normals_pipeline.py:140-308

Same arguments, defaults, checks, warnings, output dataclasses and numpy post-processing; the objects
the reference holds as `unet`, `vae`, `scheduler` are replaced by one `Engine` (libmarigold_b200) plus
a host-side scheduler mirror. Two keyword-only additions exist because the reference draws noise from
a generator shared across batches (depth_pipeline.py:430-435), which cannot be reproduced once members
are sharded across GPUs:  noise=[E,4,h,w]  and  step_noise=[n-1,E,4,h,w] (LCM).
"""
from __future__ import annotations

import logging
from dataclasses import dataclass
from typing import Dict, Optional, Union

import numpy as np
import torch
import torch.nn.functional as F

from .engine import Engine
from .ensemble import ensemble_depth, ensemble_iid, ensemble_normals
from .schedulers import DDIMScheduler, LCMScheduler

try:  # PIL is optional at run time (tensor inputs work without it)
    from PIL import Image
except Exception:  # noqa: BLE001
    Image = None


@dataclass
class MarigoldDepthOutput:
    """reference marigold_depth_pipeline.py:60-75"""
    depth_np: np.ndarray
    depth_colored: Union[None, "Image.Image"]
    uncertainty: Union[None, np.ndarray]


@dataclass
class MarigoldNormalsOutput:
    """reference marigold_normals_pipeline.py:59-74"""
    normals_np: np.ndarray
    normals_img: "Image.Image"
    uncertainty: Union[None, np.ndarray]


_RESAMPLE = {"bilinear": "bilinear", "bicubic": "bicubic", "nearest": "nearest-exact", "nearest-exact": "nearest-exact"}


def get_tv_resample_method(method_str: str) -> str:
    """reference image_util.py:123-134 (returns an interpolate mode string instead of a torchvision enum)."""
    m = _RESAMPLE.get(method_str)
    if m is None:
        raise ValueError(f"Unknown resampling method: {method_str}")
    return m


def _resize(img: torch.Tensor, size, mode: str) -> torch.Tensor:
    """torchvision.transforms.functional.resize(img, size, interpolation, antialias=True) semantics. CUDA tensors (the
    pipelines' path) go through the library's own kernels (csrc/image.cu); CPU tensors (host-side helpers in the tests)
    through torch."""
    if img.is_cuda:
        from . import imageops

        out = imageops.resize(img, size, mode, post=1 if img.dtype == torch.uint8 else 0)
        return out.to(img.dtype)
    if mode == "nearest-exact":
        return F.interpolate(img.float(), size=size, mode=mode).to(img.dtype)
    out = F.interpolate(img.float(), size=size, mode=mode, antialias=True, align_corners=False)
    if img.dtype == torch.uint8:
        out = out.round().clamp(0, 255).to(torch.uint8)
    return out.to(img.dtype) if img.dtype.is_floating_point else out


def resize_max_res(img: torch.Tensor, max_edge_resolution: int, resample_method: str = "bilinear") -> torch.Tensor:
    """reference image_util.py:90-120 (int() truncation :116-117, antialias :119)."""
    assert 4 == img.dim(), f"Invalid input shape {img.shape}"
    h, w = img.shape[-2:]
    f = min(max_edge_resolution / w, max_edge_resolution / h)
    return _resize(img, (int(h * f), int(w * f)), resample_method)


# matplotlib's "Spectral" is the linear interpolation of ColorBrewer's 11-class Spectral palette.
_SPECTRAL11 = np.array([
    [158, 1, 66], [213, 62, 79], [244, 109, 67], [253, 174, 97], [254, 224, 139], [255, 255, 191],
    [230, 245, 152], [171, 221, 164], [102, 194, 165], [50, 136, 189], [94, 79, 162]], dtype=np.float64) / 255.0


def _spectral_lut() -> np.ndarray:
    """matplotlib's 256-entry lookup table of "Spectral" (LinearSegmentedColormap over the 11 evenly spaced ColorBrewer
    anchors, `_create_lookup_table(256, ...)`): LUT[i] = piecewise-linear interpolation at i / 255."""
    x = np.arange(256, dtype=np.float64) / 255.0 * 10.0
    i0 = np.clip(np.floor(x).astype(np.int64), 0, 9)
    w = (x - i0)[:, None]
    return np.clip(_SPECTRAL11[i0] * (1 - w) + _SPECTRAL11[i0 + 1] * w, 0.0, 1.0)


_SPECTRAL_LUT = _spectral_lut()


def colorize_depth_maps(depth, min_depth: float, max_depth: float, cmap: str = "Spectral", valid_mask=None) -> np.ndarray:
    """reference image_util.py:38-76. Returns [(B,) 3, H, W] float in [0,1]. "Spectral" (the pipeline default) is built
    in with matplotlib's exact semantics — `cm(x)` indexes a 256-entry table with int(x * 256) (x == 1 -> 255) — any other
    matplotlib colour map is looked up through matplotlib when it is installed."""
    depth = np.asarray(depth.detach().cpu().numpy() if isinstance(depth, torch.Tensor) else depth).squeeze()
    assert depth.ndim >= 2, "Invalid dimension"
    if depth.ndim < 3:
        depth = depth[np.newaxis]
    d = ((depth - min_depth) / (max_depth - min_depth)).clip(0, 1)
    if cmap == "Spectral":
        idx = np.minimum((d * 256).astype(np.int64), 255)
        rgb = _SPECTRAL_LUT[idx]                                          # [B, H, W, 3]
    else:
        try:
            import matplotlib
        except Exception:  # noqa: BLE001
            raise ValueError(f"colour map {cmap!r} needs matplotlib (only 'Spectral' is built in)") from None
        rgb = matplotlib.colormaps[cmap](d, bytes=False)[..., 0:3]
    out = np.moveaxis(rgb, -1, 1)                                         # [B, 3, H, W]
    if valid_mask is not None:
        vm = np.asarray(valid_mask.detach().cpu().numpy() if isinstance(valid_mask, torch.Tensor) else valid_mask).squeeze()
        vm = vm[np.newaxis, np.newaxis] if vm.ndim < 3 else vm[:, np.newaxis]
        out = out.copy()
        out[~np.repeat(vm, 3, axis=1)] = 0
    return out


def _check_ensemble_size(engine, ensemble_size: int) -> None:
    mx = int(engine.lib.mgb_ens_max_members())
    if ensemble_size > mx:
        raise ValueError(f"ensemble_size={ensemble_size} exceeds the {mx} members the ensembling kernels accept")


def find_batch_size(ensemble_size: int, input_res: int, dtype: torch.dtype) -> int:
    """reference batchsize.py:60-90 is a VRAM table for A100/3090/1080Ti; on an 80 GB H100 every supported
    configuration fits in batches of 16 members up to 768 px and 8 above, so that is the cap (it bounds the arena)."""
    return max(1, min(ensemble_size, 16 if input_res <= 768 else 8))


class _MarigoldBase:
    latent_scale_factor = 0.18215  # depth_pipeline.py:118

    def __init__(self, engine: Engine, scheduler, empty_text_embed: torch.Tensor,
                 default_denoising_steps: Optional[int] = None, default_processing_resolution: Optional[int] = None):
        self.engine = engine
        self.scheduler = scheduler
        self.empty_text_embed = empty_text_embed
        self.default_denoising_steps = default_denoising_steps
        self.default_processing_resolution = default_processing_resolution
        self.dtype = torch.float32           # ABI dtype; kernels compute in bf16 x bf16 -> fp32
        self.device = engine.device
        self._sched_key = None
        engine.set_text_embedding(empty_text_embed)

    def to(self, device=None, *a, **k):       # API compatibility with DiffusionPipeline.to
        return self

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, variant: Optional[str] = None, torch_dtype=None,
                        device=None, **kwargs):
        """Drop-in for `DiffusionPipeline.from_pretrained` as the reference calls it (script/depth/run.py:213-222):
        a LOCAL diffusers checkpoint directory (README.md:261-290). See marigold_b200/checkpoint.py."""
        from .checkpoint import load_pipeline

        return load_pipeline(cls, pretrained_model_name_or_path, variant=variant, torch_dtype=torch_dtype, device=device,
                             **kwargs)

    def _set_schedule(self, n: int):
        self.scheduler.set_timesteps(n, device=self.device)
        key = (type(self.scheduler).__name__, n)
        if key != self._sched_key:
            kx, kv, kz = self.scheduler.coefficients()
            self.engine.set_schedule(self.scheduler.timesteps, kx, kv, kz)
            self._sched_key = key

    def _preprocess(self, input_image, processing_res, resample_method):
        if Image is not None and isinstance(input_image, Image.Image):
            arr = np.asarray(input_image.convert("RGB"))
            rgb = torch.from_numpy(arr.copy()).permute(2, 0, 1).unsqueeze(0)
        elif isinstance(input_image, torch.Tensor):
            rgb = input_image
        else:
            raise TypeError(f"Unknown input type: {type(input_image) = }")
        input_size = rgb.shape
        assert 4 == rgb.dim() and 3 == input_size[-3], f"Wrong input shape {input_size}, expected [1, rgb, H, W]"
        rgb = rgb.to(self.device)
        if processing_res > 0 and rgb.dtype == torch.uint8:
            # resize_max_res (image_util.py:90-120) with the uint8 rounding and the [-1, 1] normalisation (:252-254) fused
            # into the second pass of the device resize
            from . import imageops

            h0, w0 = rgb.shape[-2:]
            f = min(processing_res / w0, processing_res / h0)
            rgb_norm = imageops.resize(rgb, (int(h0 * f), int(w0 * f)), resample_method, post=2).to(self.dtype)
        else:
            if processing_res > 0:
                rgb = resize_max_res(rgb, max_edge_resolution=processing_res, resample_method=resample_method)
            rgb_norm = (rgb / 255.0 * 2.0 - 1.0).to(self.dtype)
        assert rgb_norm.min() >= -1.0 and rgb_norm.max() <= 1.0
        return rgb_norm, input_size

    def _draw_noise(self, shape, generator, noise):
        if noise is not None:
            assert tuple(noise.shape) == tuple(shape), f"noise shape {tuple(noise.shape)} != {tuple(shape)}"
            return noise.to(self.device, torch.float32)
        dev = generator.device if generator is not None else self.device
        return torch.randn(shape, device=dev, dtype=self.dtype, generator=generator).to(self.device)

    @torch.no_grad()
    def encode_rgb(self, rgb_in: torch.Tensor) -> torch.Tensor:
        """depth_pipeline.py:479-496: the reference encodes the same image once per member (expand :258);
        the result is identical, so encode once and let the caller broadcast."""
        return self.engine.encode(rgb_in)

    def _infer_members(self, rgb_norm, ensemble_size, denoising_steps, batch_size, generator, noise, step_noise,
                       decode_mode):
        """The body of the reference's batch loop (depth_pipeline.py:281-290) + single_infer (:397-477).
        Under torch.distributed (one process per GPU) the members are sharded round-robin and joined by
        one all-gather of the decoded maps (parallel.py); the result is identical on every rank."""
        from . import parallel

        self._set_schedule(denoising_steps)
        rgb_latent1 = self.encode_rgb(rgb_norm)                      # [1,4,h,w]
        lh, lw = rgb_latent1.shape[-2:]
        is_lcm = isinstance(self.scheduler, LCMScheduler)
        need_sn = is_lcm and denoising_steps > 1
        rank, G = parallel.world()
        mine = parallel.member_indices(ensemble_size, rank, G)
        ct = self.engine.cfg.unet_out_channels               # 4, or 4 n for an n-target IID model
        if G > 1:
            # every rank draws (or receives) the FULL noise tensors and takes its rows, so member k's noise
            # does not depend on the partitioning (SURVEY.md F9)
            noise = self._draw_noise((ensemble_size, ct, lh, lw), generator, noise)
            if need_sn and step_noise is None:
                dev = generator.device if generator is not None else self.device
                step_noise = torch.randn((denoising_steps - 1, ensemble_size, ct, lh, lw), device=dev, dtype=self.dtype,
                                         generator=generator)
        _bs = batch_size if batch_size > 0 else find_batch_size(len(mine), max(rgb_norm.shape[1:]), self.dtype)
        preds = []
        for s in range(0, len(mine), _bs):
            ids = mine[s:s + _bs]
            nb = len(ids)
            if G > 1 or noise is not None:
                z0 = noise[ids].to(self.device, torch.float32).contiguous()
            else:
                z0 = self._draw_noise((nb, ct, lh, lw), generator, None)
            sn = None
            if need_sn:
                if step_noise is not None:
                    sn = step_noise[:, ids].to(self.device, torch.float32).contiguous()
                else:
                    # one randn per step, in step order after z0: the draw sequence of scheduler.step(generator=...)
                    # inside the reference loop (depth_pipeline.py:466-468), so a seeded generator gives the same stream
                    dev = generator.device if generator is not None else self.device
                    sn = torch.stack([torch.randn((nb, ct, lh, lw), device=dev, dtype=self.dtype, generator=generator)
                                      for _ in range(denoising_steps - 1)]).to(self.device)
            target = self.engine.denoise(rgb_latent1.expand(nb, -1, -1, -1).contiguous(), z0, sn)
            if decode_mode == _lib_decode_iid:
                # marigold_iid_pipeline.py:568-585: one VAE decode per 4-channel target slice, concatenated along channels
                preds.append(torch.cat([self.engine.decode(target[:, 4 * i:4 * i + 4].contiguous(), _lib_decode_iid)
                                        for i in range(ct // 4)], dim=1))
            else:
                preds.append(self.engine.decode(target, decode_mode))
        ch = 1 if decode_mode == 0 else (3 * (ct // 4) if decode_mode == _lib_decode_iid else 3)
        local = torch.concat(preds, dim=0) if preds else torch.empty((0, ch, lh * 8, lw * 8), device=self.device)
        return parallel.gather_members(local, ensemble_size)


class MarigoldDepthPipeline(_MarigoldBase):
    def __init__(self, engine, scheduler, empty_text_embed, scale_invariant: Optional[bool] = True,
                 shift_invariant: Optional[bool] = True, default_denoising_steps: Optional[int] = None,
                 default_processing_resolution: Optional[int] = None):
        super().__init__(engine, scheduler, empty_text_embed, default_denoising_steps, default_processing_resolution)
        self.scale_invariant = scale_invariant
        self.shift_invariant = shift_invariant

    def _check_inference_step(self, n_step: int) -> None:
        """depth_pipeline.py:340-379"""
        assert n_step >= 1
        if isinstance(self.scheduler, DDIMScheduler):
            if "trailing" != self.scheduler.config.timestep_spacing:
                logging.warning(
                    f'The loaded `DDIMScheduler` is configured with `timestep_spacing="'
                    f'{self.scheduler.config.timestep_spacing}"`; the recommended setting is `"trailing"`.')
            elif n_step > 10:
                logging.warning(f"Setting too many denoising steps ({n_step}) may degrade the prediction; consider "
                                f"relying on the default values.")
            if not self.scheduler.config.rescale_betas_zero_snr:
                logging.warning("The loaded `DDIMScheduler` is configured with `rescale_betas_zero_snr=False`; the "
                                "recommended setting is True.")
        elif isinstance(self.scheduler, LCMScheduler):
            logging.warning("DeprecationWarning: LCMScheduler will not be supported in the future.")
            if n_step > 10:
                logging.warning(f"Setting too many denoising steps ({n_step}) may degrade the prediction; consider "
                                f"relying on the default values.")
        else:
            raise RuntimeError(f"Unsupported scheduler type: {type(self.scheduler)}")

    @torch.no_grad()
    def __call__(self, input_image, denoising_steps: Optional[int] = None, ensemble_size: int = 1,
                 processing_res: Optional[int] = None, match_input_res: bool = True,
                 resample_method: str = "bilinear", batch_size: int = 0,
                 generator: Union[torch.Generator, None] = None, color_map: str = "Spectral",
                 show_progress_bar: bool = True, ensemble_kwargs: Dict = None, *,
                 noise: Optional[torch.Tensor] = None, step_noise: Optional[torch.Tensor] = None
                 ) -> MarigoldDepthOutput:
        if denoising_steps is None:
            denoising_steps = self.default_denoising_steps
        if processing_res is None:
            processing_res = self.default_processing_resolution
        assert processing_res >= 0
        assert ensemble_size >= 1
        _check_ensemble_size(self.engine, ensemble_size)          # fail before any inference work is spent
        self._check_inference_step(denoising_steps)
        resample = get_tv_resample_method(resample_method)
        rgb_norm, input_size = self._preprocess(input_image, processing_res, resample)

        target_preds = self._infer_members(rgb_norm, ensemble_size, denoising_steps, batch_size, generator, noise,
                                           step_noise, _lib_decode_depth)
        if ensemble_size > 1:
            final_pred, pred_uncert = ensemble_depth(target_preds, scale_invariant=self.scale_invariant,
                                                     shift_invariant=self.shift_invariant, engine=self.engine,
                                                     **(ensemble_kwargs or {}))
        else:
            final_pred, pred_uncert = target_preds, None
        if match_input_res:
            final_pred = _resize(final_pred, tuple(input_size[-2:]), resample)
        final_pred = final_pred.squeeze().cpu().numpy()
        if pred_uncert is not None:
            pred_uncert = pred_uncert.squeeze().cpu().numpy()
        final_pred = final_pred.clip(0, 1)
        depth_colored_img = None
        if color_map is not None:
            if color_map == "Spectral":
                from . import imageops

                hwc = imageops.colorize_u8(torch.from_numpy(np.ascontiguousarray(final_pred)).to(self.device), 0, 1,
                                           imageops.spectral_lut_u8()).cpu().numpy()            # :326-331 on the device
            else:
                col = (colorize_depth_maps(final_pred, 0, 1, cmap=color_map).squeeze() * 255).astype(np.uint8)
                hwc = np.moveaxis(col, 0, -1)
            depth_colored_img = Image.fromarray(hwc) if Image is not None else hwc
        return MarigoldDepthOutput(depth_np=final_pred, depth_colored=depth_colored_img, uncertainty=pred_uncert)


class MarigoldNormalsPipeline(_MarigoldBase):
    def _check_inference_step(self, n_step: int) -> None:
        """normals_pipeline.py:310-344: LCM is refused."""
        assert n_step >= 1
        if isinstance(self.scheduler, DDIMScheduler):
            if "trailing" != self.scheduler.config.timestep_spacing:
                logging.warning("The loaded `DDIMScheduler` is not configured with `timestep_spacing=\"trailing\"`.")
            elif n_step > 10:
                logging.warning(f"Setting too many denoising steps ({n_step}) may degrade the prediction.")
            if not self.scheduler.config.rescale_betas_zero_snr:
                logging.warning("The loaded `DDIMScheduler` is configured with `rescale_betas_zero_snr=False`.")
        elif isinstance(self.scheduler, LCMScheduler):
            raise RuntimeError("This pipeline implementation does not support the LCMScheduler. Please refer to the "
                               "project README.md for instructions about using LCM.")
        else:
            raise RuntimeError(f"Unsupported scheduler type: {type(self.scheduler)}")

    @torch.no_grad()
    def __call__(self, input_image, denoising_steps: Optional[int] = None, ensemble_size: int = 1,
                 processing_res: Optional[int] = None, match_input_res: bool = True,
                 resample_method: str = "bilinear", batch_size: int = 0,
                 generator: Union[torch.Generator, None] = None, show_progress_bar: bool = True,
                 ensemble_kwargs: Dict = None, *, noise: Optional[torch.Tensor] = None) -> MarigoldNormalsOutput:
        if denoising_steps is None:
            denoising_steps = self.default_denoising_steps
        if processing_res is None:
            processing_res = self.default_processing_resolution
        assert processing_res >= 0
        assert ensemble_size >= 1
        self._check_inference_step(denoising_steps)
        resample = get_tv_resample_method(resample_method)
        rgb_norm, input_size = self._preprocess(input_image, processing_res, resample)
        target_preds = self._infer_members(rgb_norm, ensemble_size, denoising_steps, batch_size, generator, noise,
                                           None, _lib_decode_normals)
        if ensemble_size > 1:
            final_pred, pred_uncert = ensemble_normals(target_preds, engine=self.engine, **(ensemble_kwargs or {}))
        else:
            final_pred, pred_uncert = target_preds, None
        if match_input_res:
            final_pred = _resize(final_pred, tuple(input_size[-2:]), resample)
        final_pred = final_pred.squeeze().cpu().numpy()
        if pred_uncert is not None:
            pred_uncert = pred_uncert.squeeze().cpu().numpy()
        final_pred = final_pred.clip(-1, 1)
        img = ((final_pred + 1) * 127.5).astype(np.uint8)
        hwc = np.moveaxis(img, 0, -1)
        normals_img = Image.fromarray(hwc) if Image is not None else hwc
        return MarigoldNormalsOutput(normals_np=final_pred, normals_img=normals_img, uncertainty=pred_uncert)


class MarigoldIIDPipeline(_MarigoldBase):
    """Intrinsic image decomposition with an arbitrary number of 3-channel targets (reference
    marigold/marigold_iid_pipeline.py:164-585): ONE UNet whose conv_in takes 4 (n + 1) latent channels and whose
    conv_out produces 4 n; every target's 4-channel latent is decoded separately; E > 1 goes through `ensemble_iid`."""

    def __init__(self, engine, scheduler, empty_text_embed, target_properties: Optional[Dict] = None,
                 default_denoising_steps: Optional[int] = None, default_processing_resolution: Optional[int] = None):
        super().__init__(engine, scheduler, empty_text_embed, default_denoising_steps, default_processing_resolution)
        self.target_properties = target_properties
        self.target_names = target_properties["target_names"]          # :228-229 (KeyError / TypeError like the reference)
        self.n_targets = len(self.target_names)
        if engine.cfg.unet_out_channels != 4 * self.n_targets:
            raise ValueError(f"the UNet predicts {engine.cfg.unet_out_channels} latent channels, but target_names "
                             f"{self.target_names} needs {4 * self.n_targets}")

    def _check_inference_step(self, n_step: int) -> None:
        """marigold_iid_pipeline.py:413-448: LCM is refused."""
        assert n_step >= 1
        if isinstance(self.scheduler, DDIMScheduler):
            if "trailing" != self.scheduler.config.timestep_spacing:
                logging.warning(f'The loaded `DDIMScheduler` is configured with `timestep_spacing="'
                                f'{self.scheduler.config.timestep_spacing}"`; the recommended setting is `"trailing"`.')
            elif n_step > 10:
                logging.warning(f"Setting too many denoising steps ({n_step}) may degrade the prediction; consider "
                                f"relying on the default values.")
            if not self.scheduler.config.rescale_betas_zero_snr:
                logging.warning("The loaded `DDIMScheduler` is configured with `rescale_betas_zero_snr=False`; the "
                                "recommended setting is True.")
        elif isinstance(self.scheduler, LCMScheduler):
            raise RuntimeError("This pipeline implementation does not support the LCMScheduler. Please refer to the "
                               "project README.md for instructions about using LCM.")
        else:
            raise RuntimeError(f"Unsupported scheduler type: {type(self.scheduler)}")

    @torch.no_grad()
    def __call__(self, input_image, denoising_steps: Optional[int] = None, ensemble_size: int = 1,
                 processing_res: Optional[int] = None, match_input_res: bool = True,
                 resample_method: str = "bilinear", batch_size: int = 0,
                 generator: Union[torch.Generator, None] = None, show_progress_bar: bool = True,
                 ensemble_kwargs: Dict = None, *, noise: Optional[torch.Tensor] = None):
        from .iid import MarigoldIIDOutput, fill_outputs

        if denoising_steps is None:
            denoising_steps = self.default_denoising_steps
        if processing_res is None:
            processing_res = self.default_processing_resolution
        assert processing_res >= 0
        assert ensemble_size >= 1
        self._check_inference_step(denoising_steps)
        resample = get_tv_resample_method(resample_method)
        rgb_norm, input_size = self._preprocess(input_image, processing_res, resample)
        target_preds = self._infer_members(rgb_norm, ensemble_size, denoising_steps, batch_size, generator, noise,
                                           None, _lib_decode_iid)
        assert target_preds.dim() == 4 and target_preds.shape[1] == 3 * self.n_targets      # :367-370
        if ensemble_size > 1:
            final_pred, pred_uncert = ensemble_iid(target_preds, engine=self.engine, **(ensemble_kwargs or {}))
        else:
            final_pred, pred_uncert = target_preds, None
        if match_input_res:
            final_pred = _resize(final_pred, tuple(input_size[-2:]), resample)      # (:386-392; uncertainty is NOT resized)
        output = MarigoldIIDOutput(target_names=self.target_names)
        fill_outputs(output, final_pred, pred_uncert, self.target_names, self.target_properties)
        assert output.is_complete
        return output


_lib_decode_depth, _lib_decode_normals, _lib_decode_iid = 0, 1, 3   # mgb_decode_mode
MarigoldPipeline = MarigoldDepthPipeline         # alias, reference marigold/__init__.py:41
