"""Drop-in pipelines with the reference's call surface:

    MarigoldDepthPipeline.__call__     marigold/marigold_depth_pipeline.py:155-338
    MarigoldNormalsPipeline.__call__   marigold/marigold_normals_pipeline.py:140-308
    MarigoldIIDPipeline.__call__       marigold/marigold_iid_pipeline.py:164-585

Same arguments, defaults, checks, warnings, output dataclasses and numpy post-processing; the objects
the reference holds as `unet`, `vae`, `scheduler` are replaced by one `Engine` (libmarigold_b200) plus
a host-side scheduler mirror. Two keyword-only additions exist because the reference draws noise from
a generator shared across batches (depth_pipeline.py:430-435), which cannot be reproduced once members
are sharded across GPUs:  noise=[E,4,h,w]  and  step_noise=[n-1,E,4,h,w] (LCM).

Each __call__ only carries its signature: one body (_MarigoldBase._call) checks everything before any work, then runs
one image through _infer_members or a list through _infer_list. Both loops take their member batch from one admission
rule (_admit_group), their noise from one drawer (_draw_image_noise), and finish an image with the pipeline's _finish.

Every pipeline also takes a list (or tuple) of images and returns a list of outputs in input order: the members of
several images share network batches, and each image is finished (ensembled, resized, copied to the host) by the single
call's code as soon as its last member is decoded. `generator` is then one generator, drawn from by the images in list
order, or a list with one generator (or None) per image; `noise` / `step_noise` are lists of per-image tensors (or
None). Image i's noise is what the single call with its generator draws (_MarigoldBase._infer_list).
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


def _resize(img: torch.Tensor, size, mode: str, arith: str = "cuda") -> torch.Tensor:
    """torchvision.transforms.functional.resize(img, size, interpolation, antialias=True) semantics. CUDA tensors (the
    pipelines' path) go through the library's own kernels (csrc/image.cu) in the rounding of torch's `arith` kernel:
    "cuda" for predictions, which the reference resizes on the device, "cpu" for images, which it resizes on the host.
    CPU tensors (host-side helpers in the tests) go through torch."""
    if img.is_cuda:
        from . import imageops

        out = imageops.resize(img, size, mode, post=1 if img.dtype == torch.uint8 else 0, arith=arith)
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
    return _resize(img, (int(h * f), int(w * f)), resample_method, arith="cpu")     # the reference's image is on the host


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


def find_batch_size(ensemble_size: int, input_res: int, dtype: torch.dtype) -> int:
    """reference batchsize.py:60-90 is a VRAM table for A100/3090/1080Ti; on an 80 GB H100 every supported
    configuration fits in batches of 16 members up to 768 px and 8 above, so that is the cap (it bounds the arena)."""
    return max(1, min(ensemble_size, 16 if input_res <= 768 else 8))


MAX_PIXELS = 1 << 26                 # kMaxPixels (csrc/net.h): members x height x width of one encode / decode call


def call_reserve_bytes(h: int, w: int, ensemble_size: int, channels: int) -> int:
    """Device memory a pipeline call holds beside the engine's workspace at h x w: the decoded members and their
    concatenation (ensemble_size fp32 maps of `channels` each), the ensembled prediction and its uncertainty, and the
    normalised fp32 input. At 24 MP it is 2.4 GB for depth and 6.7 GB for normals with 10 members. The engine's choice of
    the low-memory decoder stage counts the smallest of these, one depth member's 28 bytes per pixel
    (csrc/api_net.cu)."""
    return 4 * h * w * (channels * (2 * ensemble_size + 2) + 3)


def _on_free_memory(engine, free_bytes: Optional[int], select):
    """select(free_bytes), with the device's free memory measured when free_bytes is None. Memory that torch's caching
    allocator keeps for tensors already freed does not count as free there, and the engine's workspace cannot use it:
    the workspace comes from the driver. So where select refuses on that measure, the cache is handed back to the
    driver and select runs once more on a new measure. A call that fits without it leaves the cache alone."""
    if free_bytes is not None:
        return select(free_bytes)
    try:
        return select(torch.cuda.mem_get_info(engine.device)[0])
    except ValueError:
        torch.cuda.empty_cache()
        return select(torch.cuda.mem_get_info(engine.device)[0])


def select_batch_size(engine, n_members: int, h: int, w: int, batch_size: int = 0,
                      free_bytes: Optional[int] = None, reserve_bytes: int = 0) -> int:
    """Members per batch for n_members at h x w. batch_size > 0 is taken as given; 0 takes find_batch_size's value,
    lowered to the largest batch whose workspace (engine.workspace_bytes) fits the memory available to the engine: free
    device memory (`free_bytes`, or the device's, with torch's cache handed back where needed: _on_free_memory) plus
    the workspace the engine holds, which it gives back before it grows, less `reserve_bytes` that the call needs for
    its own tensors (call_reserve_bytes). A batch that cannot fit, explicit or of one member, raises ValueError before
    any inference work is spent."""
    return _on_free_memory(engine, free_bytes,
                           lambda free: _select_batch_size(engine, n_members, h, w, batch_size, free, reserve_bytes))


def _select_batch_size(engine, n_members, h, w, batch_size, free_bytes, reserve_bytes):
    avail = int(free_bytes) + engine.held_bytes() - int(reserve_bytes)
    explicit = batch_size > 0
    bs = min(batch_size, max(n_members, 1)) if explicit else find_batch_size(n_members, max(h, w), torch.float32)
    while True:
        need = engine.workspace_bytes(bs, h, w)
        if 0 < need <= avail:
            return bs
        if need == 0 and bs * h * w <= MAX_PIXELS:
            return bs                    # a shape the engine refuses for another reason, with its own error
        if explicit or bs == 1:
            break
        bs -= 1
    what = f"a batch of {bs} member{'s' if bs > 1 else ''} at {h} x {w}"
    if need == 0:
        raise ValueError(f"{what} exceeds the engine's supported maximum of {MAX_PIXELS} pixels per call")
    left = f" beside the call's own {int(reserve_bytes)}" if reserve_bytes else ""
    raise ValueError(f"{what} needs {need} bytes of device workspace, but {avail} bytes are available{left}")


def _processing_size(h0: int, w0: int, processing_res: int):
    """(h, w) of the image the pipelines process: resize_max_res's, or the input's own at processing_res = 0."""
    if processing_res > 0:
        f = min(processing_res / w0, processing_res / h0)
        return int(h0 * f), int(w0 * f)
    return int(h0), int(w0)


def _input_hw(image, i=None):
    """(H0, W0) of an input image, a PIL image or a 4-D tensor, from its shape alone, before any work. List element i
    that the single call would reject raises its error, prefixed with "image {i}: "; a single image (i None) that
    _preprocess rejects gives None, and _preprocess raises."""
    if Image is not None and isinstance(image, Image.Image):
        w0, h0 = image.size
        return int(h0), int(w0)
    if i is not None:
        if not isinstance(image, torch.Tensor):
            raise TypeError(f"image {i}: Unknown input type: {type(image) = }")
        assert 4 == image.dim() and 1 == image.shape[0] and 3 == image.shape[1], \
            f"image {i}: Wrong input shape {tuple(image.shape)}, expected [1, rgb, H, W]"
    elif not isinstance(image, torch.Tensor) or image.dim() != 4:
        return None
    return int(image.shape[-2]), int(image.shape[-1])


def size_groups(sizes):
    """[(size, [image indices])] in order of first appearance: the images of a list call that may share a batch."""
    groups = {}
    for i, s in enumerate(sizes):
        groups.setdefault(tuple(s), []).append(i)
    return list(groups.items())


def noise_draw_batches(ensemble_size: int, batch_size: int, h: int, w: int, world_size: int = 1):
    """Member counts of the successive noise draws for one image at h x w: what the single call draws, one batch at a
    time at world size 1 (batch_size members if given, else find_batch_size's), the whole ensemble under G > 1 ranks. A
    list call draws each image's noise in these pieces, whatever batches its members are later packed into."""
    if world_size > 1:
        return [ensemble_size]
    b = min(batch_size, ensemble_size) if batch_size > 0 else find_batch_size(ensemble_size, max(h, w), torch.float32)
    return [b] * (ensemble_size // b) + ([ensemble_size % b] if ensemble_size % b else [])


def select_list_batch_size(engine, n_jobs: int, h: int, w: int, ensemble_size: int, channels: int, n_images: int,
                           world_size: int = 1, batch_size: int = 0, free_bytes: Optional[int] = None) -> int:
    """Members per batch for a size group of a list call: select_batch_size over the group's n_jobs (image, member) jobs
    (one rank's share under world_size ranks), beside the call_reserve_bytes of every image one round of batches can
    hold open (parallel.open_images). The reserve grows with the batch, so the two are lowered together: the result is
    the largest batch that fits beside its own reserve. Raises ValueError like select_batch_size. The single call's
    selection is the one-image case."""
    if n_images == 1:                    # one image's reserve, whatever the batch
        return select_batch_size(engine, n_jobs, h, w, batch_size, free_bytes,
                                 call_reserve_bytes(h, w, ensemble_size, channels))
    return _on_free_memory(engine, free_bytes, lambda free: _select_list_batch_size(
        engine, n_jobs, h, w, ensemble_size, channels, n_images, world_size, batch_size, free))


def _select_list_batch_size(engine, n_jobs, h, w, ensemble_size, channels, n_images, world_size, batch_size,
                            free_bytes):
    from . import parallel

    per_image = call_reserve_bytes(h, w, ensemble_size, channels)
    explicit = batch_size > 0
    bs = min(batch_size, max(n_jobs, 1)) if explicit else find_batch_size(n_jobs, max(h, w), torch.float32)
    while True:
        reserve = parallel.open_images(bs, ensemble_size, world_size, n_images) * per_image
        if explicit or bs == 1:
            return select_batch_size(engine, n_jobs, h, w, bs, free_bytes, reserve)
        try:
            if select_batch_size(engine, bs, h, w, 0, free_bytes, reserve) == bs:
                return bs
        except ValueError:
            pass                         # not even one member fits beside this batch's reserve; a smaller one reserves less
        bs -= 1


def _image_runs(jobs, idx, ensemble_size):
    """[(image, [members])] of a job list, one entry per run of consecutive jobs of one image (idx: the group's images)."""
    runs = []
    for k in jobs:
        i, m = idx[k // ensemble_size], k % ensemble_size
        if runs and runs[-1][0] == i:
            runs[-1][1].append(m)
        else:
            runs.append((i, [m]))
    return runs


_lib_decode_depth, _lib_decode_normals, _lib_decode_iid = 0, 1, 3   # mgb_decode_mode


class _MarigoldBase:
    latent_scale_factor = 0.18215  # depth_pipeline.py:118
    member_channels = 1            # channels of one decoded member: 1 (depth), 3 (normals), 3 per target (IID)
    decode_mode = _lib_decode_depth
    # _check_inference_step: whether LCM runs (with a deprecation warning) or is refused, and the reference's DDIM
    # warnings (timestep spacing, too many steps, zero SNR) in the depth and IID pipelines' words
    lcm_supported = False
    step_warnings = ('The loaded `DDIMScheduler` is configured with `timestep_spacing="{spacing}"`; the recommended '
                     'setting is `"trailing"`.',
                     "Setting too many denoising steps ({n_step}) may degrade the prediction; consider relying on the "
                     "default values.",
                     "The loaded `DDIMScheduler` is configured with `rescale_betas_zero_snr=False`; the recommended "
                     "setting is True.")

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

    @torch.no_grad()
    def _call(self, input_image, denoising_steps, ensemble_size, processing_res, match_input_res, resample_method,
              batch_size, generator, ensemble_kwargs, noise, step_noise, **finish_kw):
        """The body of every pipeline's __call__ (depth_pipeline.py:155-338): one image, or a list of images with one
        output per image in input order (_infer_list). Every check runs before any inference work is spent."""
        if denoising_steps is None:
            denoising_steps = self.default_denoising_steps
        if processing_res is None:
            processing_res = self.default_processing_resolution
        assert processing_res >= 0
        assert ensemble_size >= 1
        mx = int(self.engine.lib.mgb_ens_max_members())
        if ensemble_size > mx:
            raise ValueError(f"ensemble_size={ensemble_size} exceeds the {mx} members the ensembling kernels accept")
        self._check_inference_step(denoising_steps)
        resample = get_tv_resample_method(resample_method)

        def finish(member_maps, out_hw):
            return self._finish(member_maps, out_hw, ensemble_size, resample, match_input_res, ensemble_kwargs,
                                **finish_kw)

        if isinstance(input_image, (list, tuple)):
            outputs = [None] * len(input_image)

            def finish_image(i, member_maps, out_hw):
                outputs[i] = finish(member_maps, out_hw)

            self._infer_list(input_image, ensemble_size, denoising_steps, processing_res, resample, batch_size,
                             generator, noise, step_noise, self.decode_mode, finish_image)
            return outputs
        batch_size, row_split = self._member_batch(input_image, processing_res, ensemble_size, batch_size)
        rgb_norm, input_size = self._preprocess(input_image, processing_res, resample)
        target_preds = self._infer_members(rgb_norm, ensemble_size, denoising_steps, batch_size, generator, noise,
                                           step_noise, self.decode_mode, row_split)
        return finish(target_preds, tuple(input_size[-2:]))

    def _check_inference_step(self, n_step: int) -> None:
        """depth_pipeline.py:340-379, normals_pipeline.py:310-344, marigold_iid_pipeline.py:413-448: the same checks in
        each pipeline's words (step_warnings); LCM is refused unless lcm_supported."""
        assert n_step >= 1
        spacing, too_many, zero_snr = self.step_warnings
        if isinstance(self.scheduler, DDIMScheduler):
            if "trailing" != self.scheduler.config.timestep_spacing:
                logging.warning(spacing.format(spacing=self.scheduler.config.timestep_spacing))
            elif n_step > 10:
                logging.warning(too_many.format(n_step=n_step))
            if not self.scheduler.config.rescale_betas_zero_snr:
                logging.warning(zero_snr)
        elif isinstance(self.scheduler, LCMScheduler):
            if not self.lcm_supported:
                raise RuntimeError("This pipeline implementation does not support the LCMScheduler. Please refer to "
                                   "the project README.md for instructions about using LCM.")
            logging.warning("DeprecationWarning: LCMScheduler will not be supported in the future.")
            if n_step > 10:
                logging.warning(too_many.format(n_step=n_step))
        else:
            raise RuntimeError(f"Unsupported scheduler type: {type(self.scheduler)}")

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
        # The reference resizes (image_util.py:90-120) and normalises (:252-254) the tensor where it lives: a host image
        # (PIL, or a CPU tensor) with torch CPU's resize and a true division, a CUDA tensor with torch CUDA's resize and
        # its division by a scalar, which multiplies by the reciprocal (1 ulp off for 111 of the 256 byte values).
        on_device = rgb.is_cuda
        rgb = rgb.to(self.device)
        from . import imageops

        size = _processing_size(*rgb.shape[-2:], processing_res)
        mode = resample_method if processing_res > 0 else "nearest-exact"
        if not on_device and rgb.dtype in (torch.uint8, torch.float32):
            # both fused into the resize's second pass; at native resolution the resize is the identity (nearest-exact
            # at the same size copies every value). uint8 is rounded back to uint8 first, float32 is used as it is.
            post = 2 if rgb.dtype == torch.uint8 else 3
            rgb_norm = imageops.resize(rgb, size, get_tv_resample_method(mode), post=post, arith="cpu").to(self.dtype)
        else:
            # a CUDA tensor, or a float dtype other than float32, which the reference normalises in its own dtype
            if processing_res > 0:
                rgb = _resize(rgb, size, get_tv_resample_method(mode), arith="cuda" if on_device else "cpu")
            if not on_device:
                rgb = rgb.cpu()
            rgb_norm = (rgb / 255.0 * 2.0 - 1.0).to(self.device, self.dtype)
        assert rgb_norm.min() >= -1.0 and rgb_norm.max() <= 1.0
        return rgb_norm, input_size

    def _admit_group(self, h, w, ensemble_size, n_images, n_mine, batch_size):
        """(member batch, row split, refusal) of a size group of n_images images at h x w, n_mine of whose jobs are this
        rank's: whether it runs row-split (parallel.row_split_rule), and select_list_batch_size's batch. A refused group
        raises ValueError, except a row-split one, which gives batch 0 and the error: the ranks must agree on its
        admission (each rank's depends on its own free memory) before any of them enters an exchange."""
        from . import parallel

        G = parallel.world()[1]
        split = parallel.row_split_rule(n_images * ensemble_size, h, w, G)
        try:
            with parallel.row_split(self.engine, split):
                bs = select_list_batch_size(self.engine, 1 if split else n_mine, h, w, ensemble_size,
                                            self.member_channels, n_images, G, batch_size)
        except ValueError as e:
            if not split:
                raise
            return 0, True, e
        return bs, split, None

    def _member_batch(self, input_image, processing_res, ensemble_size, batch_size):
        """(member batch, row split) of the single call, from the input's shape alone (_admit_group over this rank's
        members), so that an input that cannot run is refused before any work. Only a row-split call agrees with the
        other ranks, in one all-reduce. The caller passes the decision on to _infer_members."""
        from . import parallel

        hw0 = _input_hw(input_image)
        if hw0 is None:
            return batch_size, False                         # _preprocess rejects it
        h, w = _processing_size(*hw0, processing_res)
        rank, G = parallel.world()
        bs, split, err = self._admit_group(h, w, ensemble_size, 1, len(parallel.member_indices(ensemble_size, rank, G)),
                                           batch_size)
        if not split:
            return bs, False
        split, admitted = parallel.agree_batch_sizes([1, min(bs, 1)], self.device)
        if not admitted:
            raise err if err is not None else ValueError(f"another rank cannot admit one member at {h} x {w}")
        return 1, split == 1

    @torch.no_grad()
    def encode_rgb(self, rgb_in: torch.Tensor) -> torch.Tensor:
        """depth_pipeline.py:479-496: the reference encodes the same image once per member (expand :258);
        the result is identical, so encode once and let the caller broadcast."""
        return self.engine.encode(rgb_in)

    def _infer_members(self, rgb_norm, ensemble_size, denoising_steps, batch_size, generator, noise, step_noise,
                       decode_mode, row_split=False):
        """The body of the reference's batch loop (depth_pipeline.py:281-290) + single_infer (:397-477).
        Under torch.distributed (one process per GPU) the members are sharded round-robin and joined by
        one all-gather of the decoded maps (parallel.py); the result is identical on every rank. With row_split
        (the ranks' agreed decision, _member_batch) the one member runs on every rank, on rank 0's noise."""
        from . import parallel

        rank, G = parallel.world()
        split = row_split
        assert not split or ensemble_size == 1, "a row-split call runs one member"
        mine = [0] if split else parallel.member_indices(ensemble_size, rank, G)
        _bs = batch_size if batch_size > 0 else select_batch_size(self.engine, len(mine), *rgb_norm.shape[-2:])
        self._set_schedule(denoising_steps)
        with parallel.row_split(self.engine, split):
            rgb_latent1 = self.encode_rgb(rgb_norm)                      # [1,4,h,w]
            lh, lw = rgb_latent1.shape[-2:]
            ct = self.engine.cfg.unet_out_channels               # 4, or 4 n for an n-target IID model
            # one rank draws in the batches it runs; G ranks each draw (or receive) the FULL noise tensors and take
            # their rows, so member k's noise does not depend on the partitioning (SURVEY.md F9)
            pieces = None if G > 1 else noise_draw_batches(ensemble_size, _bs, *rgb_norm.shape[-2:])
            z, sn = self._draw_image_noise(generator, noise, step_noise, (ct, lh, lw), ensemble_size, denoising_steps,
                                           pieces)
            if split:
                z, sn = parallel.broadcast_from_first([z, sn], self.device)
            preds = []
            for s in range(0, len(mine), _bs):
                ids = mine[s:s + _bs]
                target = self.engine.denoise(rgb_latent1.expand(len(ids), -1, -1, -1).contiguous(), z[ids].contiguous(),
                                             sn[:, ids].contiguous() if sn is not None else None)
                preds.append(self._decode(target, decode_mode))
        ch = 1 if decode_mode == 0 else (3 * (ct // 4) if decode_mode == _lib_decode_iid else 3)
        local = torch.concat(preds, dim=0) if preds else torch.empty((0, ch, lh * 8, lw * 8), device=self.device)
        return local if split else parallel.gather_members(local, ensemble_size)

    def _draw_image_noise(self, generator, noise, step_noise, shape, ensemble_size, denoising_steps, pieces):
        """One image's z0 [E, *shape] and LCM step noise [n - 1, E, *shape] (None where no step draws noise), on the
        device, drawn from generator in the single call's order: at world size 1 per piece of b members (pieces), z0
        [b] then one [b] draw per step in step order, the draw sequence of scheduler.step(generator=...) inside the
        reference loop (depth_pipeline.py:466-468); under G > 1 ranks (pieces None) z0 [E] then the step noise
        [n - 1, E]. noise / step_noise, where given, replace their draws."""
        need_sn = isinstance(self.scheduler, LCMScheduler) and denoising_steps > 1
        dev = generator.device if generator is not None else self.device

        def randn(*size):
            return torch.randn(size + shape, device=dev, dtype=self.dtype, generator=generator)

        if pieces is None:
            if noise is not None:
                want = (ensemble_size,) + shape
                assert tuple(noise.shape) == want, f"noise shape {tuple(noise.shape)} != {want}"
            else:
                noise = randn(ensemble_size)
            if need_sn and step_noise is None:
                step_noise = randn(denoising_steps - 1, ensemble_size)
        else:
            zs, ss = [], []
            for b in pieces:
                if noise is None:
                    zs.append(randn(b))
                if need_sn and step_noise is None:
                    ss.append(torch.stack([randn(b) for _ in range(denoising_steps - 1)]))
            noise = torch.cat(zs) if zs else noise
            step_noise = torch.cat(ss, dim=1) if ss else step_noise
        return noise.to(self.device, torch.float32), (step_noise.to(self.device, torch.float32) if need_sn else None)

    def _decode(self, target, decode_mode):
        """The decode of one denoised member batch [NB, ct, lh, lw] -> [NB, member_channels, 8 lh, 8 lw]."""
        if decode_mode == _lib_decode_iid:
            # marigold_iid_pipeline.py:568-585: one VAE decode per 4-channel target slice, concatenated along channels
            return torch.cat([self.engine.decode(target[:, 4 * i:4 * i + 4].contiguous(), _lib_decode_iid)
                              for i in range(target.shape[1] // 4)], dim=1)
        return self.engine.decode(target, decode_mode)

    def _ensembled(self, target_preds, out_hw, ensemble_size, resample, match_input_res, ensemble_kwargs):
        """The head of every _finish: (prediction, uncertainty or None) of one image's member maps, ensembled by the
        pipeline's _ensemble when E > 1, and the prediction resized to out_hw when match_input_res."""
        if ensemble_size > 1:
            final_pred, pred_uncert = self._ensemble(target_preds, **(ensemble_kwargs or {}))
        else:
            final_pred, pred_uncert = target_preds, None
        if match_input_res:
            final_pred = _resize(final_pred, out_hw, resample)
        return final_pred, pred_uncert

    # ---- lists of images -------------------------------------------------------------------------------------------
    def _infer_list(self, images, ensemble_size, denoising_steps, processing_res, resample, batch_size, generator,
                    noise, step_noise, decode_mode, finish):
        """Every member of every image through shared member batches; finish(i, [E, C, H, W] member maps, (H0, W0)) is
        called for each image as soon as its last member is decoded, after which the call drops its device tensors.

        Images are grouped by processing size (in order of first appearance); a group's jobs are (image, member) in
        image-major order, job k on rank k mod G, and each batch takes the next bs of a rank's jobs (select_list_batch_size,
        agreed by MIN over ranks). An image is preprocessed and encoded alone, as in the single call, when its first
        member enters a batch. Under G ranks, round r runs every rank's r-th batch and one all-gather joins them.

        Noise: image i draws from generator[i] (a list), or from the one shared generator in list order, what the single
        call with that generator draws where free memory does not lower its batch (_draw_image_noise in
        noise_draw_batches pieces); noise[i] / step_noise[i] replace image i's draws. A member's maps depend only on its
        own inputs and on its batch's size, so a member packed beside other images' members has the single call's bits
        wherever the single call runs the same batch size."""
        from . import parallel

        N = len(images)
        rank, G = parallel.world()
        E = ensemble_size
        ct = self.engine.cfg.unet_out_channels
        need_sn = isinstance(self.scheduler, LCMScheduler) and denoising_steps > 1
        # ---- every check before any work
        hw0 = [_input_hw(im, i) for i, im in enumerate(images)]
        shared_gen = not isinstance(generator, (list, tuple))
        for name, per_image in (("generator", None if shared_gen else generator), ("noise", noise),
                                ("step_noise", step_noise)):
            if per_image is not None and (not isinstance(per_image, (list, tuple)) or len(per_image) != N):
                got = f"{len(per_image)} entries" if isinstance(per_image, (list, tuple)) else type(per_image).__name__
                raise ValueError(f"{name} must be None or a list of one entry per image ({N}); got {got}")
        groups = size_groups([_processing_size(h0, w0, processing_res) for h0, w0 in hw0])
        sizes, splits, refused = [], [], {}
        for (h, w), idx in groups:
            # a row-split group's admission is agreed with the batch sizes below, before any rank runs it
            try:
                bs, split, err = self._admit_group(h, w, E, len(idx), parallel.slots_per_rank(len(idx) * E, G),
                                                   batch_size)
            except ValueError as e:
                raise ValueError(f"image {idx[0]}: {e}") from None
            if err is not None:
                refused[len(sizes)] = err
            sizes.append(bs)
            splits.append(int(split))
            lh, lw = h // 8, w // 8
            for i in idx:
                if noise is not None and noise[i] is not None:
                    assert tuple(noise[i].shape) == (E, ct, lh, lw), \
                        f"image {i}: noise shape {tuple(noise[i].shape)} != {(E, ct, lh, lw)}"
                if need_sn and step_noise is not None and step_noise[i] is not None:
                    assert tuple(step_noise[i].shape) == (denoising_steps - 1, E, ct, lh, lw), \
                        f"image {i}: step_noise shape {tuple(step_noise[i].shape)} != " \
                        f"{(denoising_steps - 1, E, ct, lh, lw)}"
        if N == 0:
            return
        agreed = parallel.agree_batch_sizes(sizes + splits, self.device)
        sizes, splits = agreed[:len(groups)], agreed[len(groups):]
        for k, bs in enumerate(sizes):
            if bs == 0:
                why = refused.get(k, f"another rank cannot admit one member at {groups[k][0][0]} x {groups[k][0][1]}")
                raise ValueError(f"image {groups[k][1][0]}: {why}")
        self._set_schedule(denoising_steps)

        def draw(i):
            """Image i's z0 and step noise, drawn as the single call draws them with its generator."""
            h, w = _processing_size(*hw0[i], processing_res)
            return self._draw_image_noise(generator if shared_gen else generator[i],
                                          noise[i] if noise is not None else None,
                                          step_noise[i] if step_noise is not None else None, (ct, h // 8, w // 8), E,
                                          denoising_steps, None if G > 1 else noise_draw_batches(E, batch_size, h, w))

        drawn, next_draw = {}, 0

        def noise_of(i):
            nonlocal next_draw
            if not shared_gen:
                return draw(i)
            while next_draw <= i:                    # one generator: every image draws in list order
                drawn[next_draw] = draw(next_draw)
                next_draw += 1
            return drawn.pop(i)

        for ((h, w), idx), bs, split in zip(groups, sizes, splits):
            lh, lw = h // 8, w // 8
            n_jobs = len(idx) * E
            lat, z, sn, maps, done = {}, {}, {}, {}, {}
            with parallel.row_split(self.engine, split == 1):
                for rnd in range(parallel.num_rounds(n_jobs, bs, G)):
                    jobs, mine = parallel.round_jobs(n_jobs, bs, rnd, rank, G)
                    if split:
                        mine = jobs                      # every rank runs the one job
                    for k in jobs:                       # open the images this round reaches
                        i = idx[k // E]
                        if i not in maps:
                            z[i], sn[i] = noise_of(i)
                            if split:
                                z[i], sn[i] = parallel.broadcast_from_first([z[i], sn[i]], self.device)
                            maps[i] = torch.empty((E, self.member_channels, 8 * lh, 8 * lw), device=self.device)
                            done[i] = 0
                    if mine:
                        runs = _image_runs(mine, idx, E)
                        for i, _ in runs:
                            if i not in lat:
                                rgb_norm, _ = self._preprocess(images[i], processing_res, resample)
                                lat[i] = self.encode_rgb(rgb_norm)
                                del rgb_norm
                        rgb_latent = torch.cat([lat[i].expand(len(ms), -1, -1, -1) for i, ms in runs]).contiguous()
                        z0 = torch.cat([z[i][ms] for i, ms in runs]).contiguous()
                        s = torch.cat([sn[i][:, ms] for i, ms in runs], dim=1).contiguous() if need_sn else None
                        local = self._decode(self.engine.denoise(rgb_latent, z0, s), decode_mode)
                        del rgb_latent, z0, s
                    else:
                        local = torch.empty((0, self.member_channels, 8 * lh, 8 * lw), device=self.device)
                    pred = local if split else parallel.gather_round(local, bs, len(jobs))
                    del local
                    r0 = 0
                    for i, ms in _image_runs(jobs, idx, E):
                        maps[i][ms[0]:ms[-1] + 1] = pred[r0:r0 + len(ms)]
                        r0 += len(ms)
                        done[i] += len(ms)
                        if done[i] == E:
                            member_maps = maps.pop(i)
                            for held in (lat, z, sn, done):
                                held.pop(i, None)
                            finish(i, member_maps, hw0[i])
                            del member_maps
                    del pred


class MarigoldDepthPipeline(_MarigoldBase):
    lcm_supported = True

    def __init__(self, engine, scheduler, empty_text_embed, scale_invariant: Optional[bool] = True,
                 shift_invariant: Optional[bool] = True, default_denoising_steps: Optional[int] = None,
                 default_processing_resolution: Optional[int] = None):
        super().__init__(engine, scheduler, empty_text_embed, default_denoising_steps, default_processing_resolution)
        self.scale_invariant = scale_invariant
        self.shift_invariant = shift_invariant

    def __call__(self, input_image, denoising_steps: Optional[int] = None, ensemble_size: int = 1,
                 processing_res: Optional[int] = None, match_input_res: bool = True,
                 resample_method: str = "bilinear", batch_size: int = 0,
                 generator: Union[torch.Generator, None] = None, color_map: str = "Spectral",
                 show_progress_bar: bool = True, ensemble_kwargs: Dict = None, *,
                 noise: Optional[torch.Tensor] = None, step_noise: Optional[torch.Tensor] = None
                 ) -> MarigoldDepthOutput:
        return self._call(input_image, denoising_steps, ensemble_size, processing_res, match_input_res, resample_method,
                          batch_size, generator, ensemble_kwargs, noise, step_noise, color_map=color_map)

    def _ensemble(self, target_preds, **kwargs):
        return ensemble_depth(target_preds, scale_invariant=self.scale_invariant, shift_invariant=self.shift_invariant,
                              engine=self.engine, **kwargs)

    def _finish(self, target_preds, out_hw, ensemble_size, resample, match_input_res, ensemble_kwargs, color_map):
        """One image's [E, 1, h, w] member maps -> MarigoldDepthOutput (depth_pipeline.py:292-338)."""
        final_pred, pred_uncert = self._ensembled(target_preds, out_hw, ensemble_size, resample, match_input_res,
                                                  ensemble_kwargs)
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
    member_channels = 3
    decode_mode = _lib_decode_normals
    step_warnings = ('The loaded `DDIMScheduler` is not configured with `timestep_spacing="trailing"`.',
                     "Setting too many denoising steps ({n_step}) may degrade the prediction.",
                     "The loaded `DDIMScheduler` is configured with `rescale_betas_zero_snr=False`.")

    def __call__(self, input_image, denoising_steps: Optional[int] = None, ensemble_size: int = 1,
                 processing_res: Optional[int] = None, match_input_res: bool = True,
                 resample_method: str = "bilinear", batch_size: int = 0,
                 generator: Union[torch.Generator, None] = None, show_progress_bar: bool = True,
                 ensemble_kwargs: Dict = None, *, noise: Optional[torch.Tensor] = None) -> MarigoldNormalsOutput:
        return self._call(input_image, denoising_steps, ensemble_size, processing_res, match_input_res, resample_method,
                          batch_size, generator, ensemble_kwargs, noise, None)

    def _ensemble(self, target_preds, **kwargs):
        return ensemble_normals(target_preds, engine=self.engine, **kwargs)

    def _finish(self, target_preds, out_hw, ensemble_size, resample, match_input_res, ensemble_kwargs):
        """One image's [E, 3, h, w] member maps -> MarigoldNormalsOutput (normals_pipeline.py:278-308)."""
        final_pred, pred_uncert = self._ensembled(target_preds, out_hw, ensemble_size, resample, match_input_res,
                                                  ensemble_kwargs)
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
    decode_mode = _lib_decode_iid

    def __init__(self, engine, scheduler, empty_text_embed, target_properties: Optional[Dict] = None,
                 default_denoising_steps: Optional[int] = None, default_processing_resolution: Optional[int] = None):
        super().__init__(engine, scheduler, empty_text_embed, default_denoising_steps, default_processing_resolution)
        self.target_properties = target_properties
        self.target_names = target_properties["target_names"]          # :228-229 (KeyError / TypeError like the reference)
        self.n_targets = len(self.target_names)
        self.member_channels = 3 * self.n_targets
        if engine.cfg.unet_out_channels != 4 * self.n_targets:
            raise ValueError(f"the UNet predicts {engine.cfg.unet_out_channels} latent channels, but target_names "
                             f"{self.target_names} needs {4 * self.n_targets}")

    def __call__(self, input_image, denoising_steps: Optional[int] = None, ensemble_size: int = 1,
                 processing_res: Optional[int] = None, match_input_res: bool = True,
                 resample_method: str = "bilinear", batch_size: int = 0,
                 generator: Union[torch.Generator, None] = None, show_progress_bar: bool = True,
                 ensemble_kwargs: Dict = None, *, noise: Optional[torch.Tensor] = None):
        return self._call(input_image, denoising_steps, ensemble_size, processing_res, match_input_res, resample_method,
                          batch_size, generator, ensemble_kwargs, noise, None)

    def _ensemble(self, target_preds, **kwargs):
        return ensemble_iid(target_preds, engine=self.engine, **kwargs)

    def _finish(self, target_preds, out_hw, ensemble_size, resample, match_input_res, ensemble_kwargs):
        """One image's [E, 3 n, h, w] member maps -> MarigoldIIDOutput (marigold_iid_pipeline.py:367-411; the
        uncertainty is not resized, :386-392)."""
        from .iid import MarigoldIIDOutput, fill_outputs

        assert target_preds.dim() == 4 and target_preds.shape[1] == 3 * self.n_targets      # :367-370
        final_pred, pred_uncert = self._ensembled(target_preds, out_hw, ensemble_size, resample, match_input_res,
                                                  ensemble_kwargs)
        output = MarigoldIIDOutput(target_names=self.target_names)
        fill_outputs(output, final_pred, pred_uncert, self.target_names, self.target_properties)
        assert output.is_complete
        return output


MarigoldPipeline = MarigoldDepthPipeline         # alias, reference marigold/__init__.py:41
