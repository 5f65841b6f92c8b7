"""The pipeline calls' host logic (CPU), on a fake engine whose member maps are a known function of their noise: the
scheduler checks' exact warnings and errors, the errors every call raises before any work, the single call's noise
draws and member batches at world size 1, its admission from the input's shape and free memory, and the ensemble-size
check, for the depth, normals and IID pipelines, single and list calls alike."""
import logging
from types import SimpleNamespace

import pytest
import torch

from marigold_b200.pipeline import (MAX_PIXELS, MarigoldDepthPipeline, MarigoldIIDPipeline, MarigoldNormalsPipeline,
                                    call_reserve_bytes, find_batch_size)
from marigold_b200.schedulers import DDIMScheduler, LCMScheduler

GB = 1 << 30
PER_PIXEL = 4096                     # the fake engine's workspace bytes per member pixel, beside a fixed GB
MAX_MEMBERS = 64                     # the fake engine's mgb_ens_max_members


class _Lib:
    @staticmethod
    def mgb_ens_max_members():
        return MAX_MEMBERS


class FakeEngine:
    """encode: a constant latent, the image's mean; denoise: z0 + the latent's first channel (+ the step noise's sum);
    decode: the first channel, 8x nearest, in the decode mode's channels (1 for depth, 3 otherwise). Logs every encode
    and denoise."""
    lib, device = _Lib(), torch.device("cpu")

    def __init__(self, out_channels=4):
        self.cfg = SimpleNamespace(unet_out_channels=out_channels)
        self.log = []

    def set_text_embedding(self, t):
        pass

    def set_schedule(self, *a):
        pass

    def workspace_bytes(self, B, H, W):
        return 0 if B * H * W > MAX_PIXELS else GB + B * H * W * PER_PIXEL

    def held_bytes(self):
        return 0

    def encode(self, rgb):
        self.log.append(("encode",))
        return rgb.mean().reshape(1, 1, 1, 1).expand(1, 4, rgb.shape[-2] // 8, rgb.shape[-1] // 8).contiguous()

    def denoise(self, rl, z, sn=None):
        self.log.append(("denoise", tuple(z.shape)))
        return z + rl[:, :1] + (sn.sum(0) if sn is not None else 0)

    def decode(self, t, mode):
        return t[:, :1].repeat_interleave(8, 2).repeat_interleave(8, 3).repeat(1, 1 if mode == 0 else 3, 1, 1)


KINDS = ("depth", "normals", "iid")


def _pipe(kind, scheduler=None, real_preprocess=False):
    """A pipeline on the fake engine whose _finish returns the member maps; _preprocess normalises on the host."""
    if kind == "iid":
        pipe = MarigoldIIDPipeline(FakeEngine(8), scheduler or DDIMScheduler(), None,
                                   target_properties={"target_names": ["albedo", "shading"]})
    else:
        cls = MarigoldDepthPipeline if kind == "depth" else MarigoldNormalsPipeline
        pipe = cls(FakeEngine(), scheduler or DDIMScheduler(), None)
    if not real_preprocess:
        pipe._preprocess = lambda im, pr, rs: (im.float() / 255 * 2 - 1, im.shape)
    pipe._finish = lambda preds, out_hw, *a, **k: preds
    return pipe


def _image(h=64, w=64, seed=3):
    return torch.randint(0, 256, (1, 3, h, w), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def _call(pipe, image, as_list, **kw):
    kw = {"denoising_steps": 2, "processing_res": 0, **kw}
    return pipe([image] if as_list else image, **kw)


def _encoded(pipe):
    return any(e[0] == "encode" for e in pipe.engine.log)


@pytest.fixture(autouse=True)
def _free_memory(monkeypatch):
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (70 * GB, 80 * GB))


# ---- scheduler checks ----------------------------------------------------------------------------------------------
# the reference's texts: depth and IID share theirs (depth_pipeline.py:340-379, marigold_iid_pipeline.py:413-448),
# normals has its own (normals_pipeline.py:310-344)

def _ddim_warnings(kind, spacing, zero_snr, n):
    if kind == "normals":
        texts = ('The loaded `DDIMScheduler` is not configured with `timestep_spacing="trailing"`.',
                 f"Setting too many denoising steps ({n}) may degrade the prediction.",
                 "The loaded `DDIMScheduler` is configured with `rescale_betas_zero_snr=False`.")
    else:
        texts = (f'The loaded `DDIMScheduler` is configured with `timestep_spacing="{spacing}"`; the recommended '
                 'setting is `"trailing"`.',
                 f"Setting too many denoising steps ({n}) may degrade the prediction; consider relying on the default "
                 "values.",
                 "The loaded `DDIMScheduler` is configured with `rescale_betas_zero_snr=False`; the recommended "
                 "setting is True.")
    want = [texts[0]] if spacing != "trailing" else ([texts[1]] if n > 10 else [])
    return want + ([] if zero_snr else [texts[2]])


def _warnings(caplog):
    return [r.getMessage() for r in caplog.records if r.levelno >= logging.WARNING]


@pytest.mark.parametrize("as_list", [False, True])
@pytest.mark.parametrize("n", [4, 11])
@pytest.mark.parametrize("zero_snr", [True, False])
@pytest.mark.parametrize("spacing", ["trailing", "leading"])
@pytest.mark.parametrize("kind", KINDS)
def test_ddim_warnings(kind, spacing, zero_snr, n, as_list, caplog):
    caplog.set_level(logging.WARNING)
    pipe = _pipe(kind, DDIMScheduler(timestep_spacing=spacing, rescale_betas_zero_snr=zero_snr))
    _call(pipe, _image(), as_list, denoising_steps=n)
    assert _warnings(caplog) == _ddim_warnings(kind, spacing, zero_snr, n)


@pytest.mark.parametrize("as_list", [False, True])
@pytest.mark.parametrize("n", [4, 11])
@pytest.mark.parametrize("kind", KINDS)
def test_lcm(kind, n, as_list, caplog):
    caplog.set_level(logging.WARNING)
    pipe = _pipe(kind, LCMScheduler())
    if kind == "depth":                                   # accepted, with the reference's deprecation warning
        _call(pipe, _image(), as_list, denoising_steps=n)
        many = f"Setting too many denoising steps ({n}) may degrade the prediction; consider relying on the default " \
               "values."
        assert _warnings(caplog) == ["DeprecationWarning: LCMScheduler will not be supported in the future."] + \
            ([many] if n > 10 else [])
        return
    with pytest.raises(RuntimeError) as e:
        _call(pipe, _image(), as_list, denoising_steps=n)
    assert str(e.value) == ("This pipeline implementation does not support the LCMScheduler. Please refer to the "
                            "project README.md for instructions about using LCM.")
    assert _warnings(caplog) == [] and not _encoded(pipe)


@pytest.mark.parametrize("as_list", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_unsupported_scheduler_and_steps(kind, as_list):
    pipe = _pipe(kind, SimpleNamespace())
    with pytest.raises(RuntimeError) as e:
        _call(pipe, _image(), as_list)
    assert str(e.value) == f"Unsupported scheduler type: {SimpleNamespace}"
    with pytest.raises(AssertionError):
        _call(_pipe(kind), _image(), as_list, denoising_steps=0)
    assert not _encoded(pipe)


# ---- errors before any work ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_prologue_errors(kind):
    img = _image()
    cases = [  # (single-call input, list input, call arguments, exception, single text, list text)
        (img, [img], {"processing_res": -1}, AssertionError, "", ""),
        (img, [img], {"ensemble_size": 0}, AssertionError, "", ""),
        (img, [img], {"resample_method": "lanczos"}, ValueError, "Unknown resampling method: lanczos",
         "Unknown resampling method: lanczos"),
        ("img.png", [img, "img.png"], {}, TypeError, "Unknown input type: type(input_image) = <class 'str'>",
         "image 1: Unknown input type: type(image) = <class 'str'>"),
        (img[0], [img, img[0]], {}, AssertionError,
         "Wrong input shape torch.Size([3, 64, 64]), expected [1, rgb, H, W]",
         "image 1: Wrong input shape (3, 64, 64), expected [1, rgb, H, W]"),
        (img[:, :2], [img, img.expand(2, -1, -1, -1)], {}, AssertionError,
         "Wrong input shape torch.Size([1, 2, 64, 64]), expected [1, rgb, H, W]",
         "image 1: Wrong input shape (2, 3, 64, 64), expected [1, rgb, H, W]"),
    ]
    for single, listed, kw, exc, single_text, list_text in cases:
        for image, text in ((single, single_text), (listed, list_text)):
            pipe = _pipe(kind, real_preprocess=True)
            with pytest.raises(exc) as e:
                pipe(image, **{"denoising_steps": 2, "processing_res": 0, **kw})
            assert str(e.value) == text, (kw, image if isinstance(image, str) else None)
            assert not _encoded(pipe)


@pytest.mark.parametrize("as_list", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_ensemble_size_refused_before_any_work(kind, as_list):
    """Every call, single or list, refuses more members than the ensembling kernels accept before its first encode. The
    normals and IID single calls check it in the prologue they share with the depth call and the list calls."""
    pipe = _pipe(kind)
    with pytest.raises(ValueError) as e:
        _call(pipe, _image(), as_list, ensemble_size=MAX_MEMBERS + 1)
    assert str(e.value) == \
        f"ensemble_size={MAX_MEMBERS + 1} exceeds the {MAX_MEMBERS} members the ensembling kernels accept"
    assert pipe.engine.log == []


# ---- the single call's noise and batches at world size 1 -----------------------------------------------------------

def _expected(img, z, sn):
    lat = (img.float() / 255 * 2 - 1).mean()
    t = z[:, :1] + lat + (sn.sum(0)[:, :1] if sn is not None else 0)
    return t.repeat_interleave(8, 2).repeat_interleave(8, 3)


@pytest.mark.parametrize("case", ["lowered", "lowered-lcm", "lowered-lcm-noise", "explicit", "explicit-lcm"])
def test_single_call_noise_and_batches(case, monkeypatch):
    """The single call draws z0 and then the n - 1 LCM step-noise draws per member batch, in the batches it selected:
    free memory that fits 3 members lowers find_batch_size's 10, and an explicit batch_size of 4 is taken as given."""
    E, steps, h, w = 10, 3, 64, 48
    lcm, explicit, given = "lcm" in case, "explicit" in case, "noise" in case
    shape = (4, h // 8, w // 8)
    free = 70 * GB if explicit else FakeEngine().workspace_bytes(3, h, w) + call_reserve_bytes(h, w, E, 1)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (free, 80 * GB))
    pipe = _pipe("depth", LCMScheduler() if lcm else DDIMScheduler())
    img = _image(h, w)
    z_given = torch.randn((E,) + shape, generator=torch.Generator().manual_seed(1)) if given else None
    got = pipe(img, denoising_steps=steps, ensemble_size=E, processing_res=0, batch_size=4 if explicit else 0,
               generator=torch.Generator().manual_seed(7), noise=z_given)
    batches = [4, 4, 2] if explicit else [3, 3, 3, 1]
    assert find_batch_size(E, max(h, w), torch.float32) == E
    assert [e[1] for e in pipe.engine.log if e[0] == "denoise"] == [(b,) + shape for b in batches]
    g = torch.Generator().manual_seed(7)
    zs, ss = [], []
    for b in batches:
        if not given:
            zs.append(torch.randn((b,) + shape, generator=g))
        if lcm:
            ss.append(torch.stack([torch.randn((b,) + shape, generator=g) for _ in range(steps - 1)]))
    z = z_given if given else torch.cat(zs)
    assert torch.equal(got, _expected(img, z, torch.cat(ss, dim=1) if lcm else None))


# ---- the single call's admission -----------------------------------------------------------------------------------

def _need(b, h, w):
    return GB + b * h * w * PER_PIXEL


def _stub_device(monkeypatch, free, after=None):
    """The device's free memory: `free`, and `after` once torch's cache has been handed back (counted)."""
    state = {"free": free, "handed_back": 0}

    def empty_cache():
        state["handed_back"] += 1
        state["free"] = free if after is None else after

    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (state["free"], 80 * GB))
    monkeypatch.setattr(torch.cuda, "empty_cache", empty_cache)
    return state


ADMISSION = [  # (kind, input (H, W) or an input, processing_res, E, batch_size, free, free after the hand-back, result)
    ("depth", (768, 768), 0, 10, 0, 70 * GB, None, (10, False)),
    ("depth", (768, 768), 0, 10, 0, 10 * GB, None, (3, False)),
    ("depth", (768, 768), 0, 10, 0, 7 * GB + 7 * GB // 8, None, (3, False)),
    ("normals", (768, 768), 0, 10, 0, 7 * GB + 7 * GB // 8, None, (2, False)),    # 3 channels reserve more
    ("depth", (3024, 4032), 768, 10, 0, 70 * GB, None, (10, False)),
    ("depth", (3024, 4032), 768, 20, 0, 70 * GB, None, (16, False)),
    ("depth", (3024, 4032), 768, 20, 0, 12 * GB, None, (6, False)),
    ("depth", (768, 768), 0, 10, 4, 70 * GB, None, (4, False)),
    ("depth", (768, 768), 0, 10, 16, 70 * GB, None, (10, False)),
    ("iid", (3024, 4032), 0, 1, 0, 70 * GB, None, (1, False)),
    ("depth", (3024, 4032), 0, 1, 0, 40 * GB, 70 * GB, (1, False)),          # fits once torch's cache is handed back
    ("depth", "pil", 0, 10, 0, 10 * GB, None, (7, False)),
    ("depth", "not an image", 0, 10, 0, 70 * GB, None, (0, False)),          # _preprocess rejects it
]


@pytest.mark.parametrize("kind,size,processing_res,E,batch_size,free,after,want", ADMISSION)
def test_single_call_admission(kind, size, processing_res, E, batch_size, free, after, want, monkeypatch):
    from PIL import Image

    state = _stub_device(monkeypatch, free, after)
    if size == "pil":
        image = Image.new("RGB", (640, 480))
    elif isinstance(size, str):
        image = size
    else:
        image = torch.zeros(1, 3, 1, 1, dtype=torch.uint8).expand(1, 3, *size)
    assert _pipe(kind)._member_batch(image, processing_res, E, batch_size) == want
    assert state["handed_back"] == (1 if after is not None else 0)


@pytest.mark.parametrize("kind,ch", [("depth", 1), ("normals", 3), ("iid", 6)])
def test_single_call_refusal(kind, ch, monkeypatch):
    h, w = 4032, 6048
    state = _stub_device(monkeypatch, 70 * GB)
    image = torch.zeros(1, 3, 1, 1, dtype=torch.uint8).expand(1, 3, h, w)
    pipe = _pipe(kind)
    reserve = call_reserve_bytes(h, w, 2, ch)
    with pytest.raises(ValueError) as e:
        pipe._member_batch(image, 0, 2, 0)
    assert str(e.value) == f"a batch of 1 member at {h} x {w} needs {_need(1, h, w)} bytes of device workspace, but " \
                           f"{70 * GB - reserve} bytes are available beside the call's own {reserve}"
    assert state["handed_back"] == 1
    # past the engine's supported maximum of pixels per call
    with pytest.raises(ValueError) as e:
        pipe._member_batch(torch.zeros(1, 3, 1, 1).expand(1, 3, 8192, 8193), 0, 1, 0)
    assert str(e.value) == \
        f"a batch of 1 member at 8192 x 8193 exceeds the engine's supported maximum of {MAX_PIXELS} pixels per call"
    # and the call itself refuses before any work
    with pytest.raises(ValueError):
        pipe(image, denoising_steps=2, ensemble_size=2, processing_res=0)
    assert pipe.engine.log == []

