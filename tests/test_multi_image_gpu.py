"""Lists of images in one pipeline call (`-m gpu`, tiny model): a one-element list is the single call bit for bit; images
with one generator each and unmixed batches keep the single call's bits; a member packed beside other images' members
has the bits of the same member in any batch of that size; mixed sizes, determinism, errors before any work, and device
memory that does not grow with the length of the list."""
import numpy as np
import pytest
import torch

import tests.net_ref as N
from tests.helpers import engine_from_oracle, oracle_models, synthetic_image

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup():
    unet, vae, text = oracle_models("tiny")
    eng = engine_from_oracle(unet, vae, text)
    yield eng, text
    eng.close()


@pytest.fixture(scope="module")
def iid2():
    from marigold_b200.engine import Engine, EngineConfig
    from oracle.unet import UNet2DConditionOracle, UNetConfig
    from oracle.vae import AutoencoderKLOracle, VAEConfig

    torch.manual_seed(0)
    ucfg = UNetConfig.tiny()
    ucfg.in_channels, ucfg.out_channels = 12, 8
    unet, vae = UNet2DConditionOracle(ucfg).eval(), AutoencoderKLOracle(VAEConfig.tiny()).eval()
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=torch.Generator().manual_seed(7))
    eng = Engine(EngineConfig(unet_in_channels=12, unet_out_channels=8, unet_block_channels=list(ucfg.block_out_channels),
                              unet_cross_dim=ucfg.cross_attention_dim, vae_block_channels=list(vae.cfg.block_out_channels)))
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    yield eng, text
    eng.close()


IID_PROPS = {"target_names": ["albedo", "shading"], "albedo": {"prediction_space": "srgb"},
             "shading": {"prediction_space": "linear", "up_to_scale": True}}


def _depth(eng, text, lcm=False, steps=2):
    from marigold_b200.pipeline import MarigoldDepthPipeline
    from marigold_b200.schedulers import DDIMScheduler, LCMScheduler

    return MarigoldDepthPipeline(eng, LCMScheduler() if lcm else DDIMScheduler(), text, default_denoising_steps=steps,
                                 default_processing_resolution=128)


def _normals(eng, text):
    from marigold_b200.pipeline import MarigoldNormalsPipeline
    from marigold_b200.schedulers import DDIMScheduler

    return MarigoldNormalsPipeline(eng, DDIMScheduler(), text, default_denoising_steps=2,
                                   default_processing_resolution=128)


def _iid(eng, text):
    from marigold_b200.pipeline import MarigoldIIDPipeline
    from marigold_b200.schedulers import DDIMScheduler

    return MarigoldIIDPipeline(eng, DDIMScheduler(), text, target_properties=IID_PROPS, default_denoising_steps=2,
                               default_processing_resolution=128)


def _img(seed, h=128, w=128):
    return synthetic_image(max(h, w), seed=seed)[:, :, :h, :w].contiguous()


def _randn(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _arrays(out):
    """Every array an output object carries (maps, uncertainties, 8-bit images), in a fixed order."""
    from marigold_b200.iid import MarigoldIIDOutput

    if isinstance(out, MarigoldIIDOutput):
        return [a for e in out for a in (e.array, np.asarray(e.image), e.uncertainty)]
    img = getattr(out, "depth_colored", None) if hasattr(out, "depth_np") else out.normals_img
    m = out.depth_np if hasattr(out, "depth_np") else out.normals_np
    return [m, None if img is None else np.asarray(img), out.uncertainty]


def _assert_same(a, b):
    xa, xb = _arrays(a), _arrays(b)
    assert len(xa) == len(xb)
    for u, v in zip(xa, xb):
        assert (u is None) == (v is None)
        if u is not None:
            np.testing.assert_array_equal(u, v)


def _cuda_gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def test_one_element_list_is_the_single_call(setup, iid2):
    eng, text = setup
    img = _img(11)
    depth = _depth(eng, text)
    for E, kw in ((1, {}), (3, dict(batch_size=2, ensemble_kwargs=dict(output_uncertainty=True)))):
        z = _randn(E, E, 4, 16, 16)
        single = depth(img, ensemble_size=E, noise=z, **kw)
        (listed,) = depth([img], ensemble_size=E, noise=[z], **kw)
        assert single.depth_colored is not None and (E == 1 or single.uncertainty is not None)
        _assert_same(single, listed)
        single = depth(img, ensemble_size=E, generator=_cuda_gen(5), **kw)
        (listed,) = depth([img], ensemble_size=E, generator=_cuda_gen(5), **kw)
        _assert_same(single, listed)
        (listed,) = depth([img], ensemble_size=E, generator=[_cuda_gen(5)], **kw)
        _assert_same(single, listed)
    lcm = _depth(eng, text, lcm=True, steps=4)
    z, zs = _randn(1, 2, 4, 16, 16), _randn(2, 3, 2, 4, 16, 16)
    _assert_same(lcm(img, ensemble_size=2, noise=z, step_noise=zs),
                 lcm([img], ensemble_size=2, noise=[z], step_noise=[zs])[0])
    _assert_same(lcm(img, ensemble_size=2, generator=_cuda_gen(3)), lcm([img], ensemble_size=2, generator=_cuda_gen(3))[0])
    normals = _normals(eng, text)
    kw = dict(ensemble_size=4, ensemble_kwargs=dict(output_uncertainty=True))
    _assert_same(normals(img, generator=torch.Generator().manual_seed(9), **kw),
                 normals([img], generator=torch.Generator().manual_seed(9), **kw)[0])
    ieng, itext = iid2
    iid = _iid(ieng, itext)
    kw = dict(ensemble_size=2, ensemble_kwargs=dict(output_uncertainty=True))
    _assert_same(iid(img, generator=torch.Generator().manual_seed(4), **kw),
                 iid([img], generator=torch.Generator().manual_seed(4), **kw)[0])


def test_unmixed_batches_keep_each_generator(setup):
    """E = batch_size = 4: every batch holds one image's members, and each image draws what the single call draws."""
    eng, text = setup
    depth = _depth(eng, text)
    imgs = [_img(21), _img(22)]
    kw = dict(ensemble_size=4, batch_size=4, ensemble_kwargs=dict(output_uncertainty=True))
    outs = depth(imgs, generator=[torch.Generator().manual_seed(100 + i) for i in range(2)], **kw)
    assert len(outs) == 2
    for i, img in enumerate(imgs):
        _assert_same(depth(img, generator=torch.Generator().manual_seed(100 + i), **kw), outs[i])
    # one shared generator: the images draw in list order, each what the single call draws
    g = torch.Generator().manual_seed(7)
    outs = depth(imgs, generator=torch.Generator().manual_seed(7), **kw)
    for i, img in enumerate(imgs):
        _assert_same(depth(img, generator=g, **kw), outs[i])


def _members(pipe, images, E, batch_size, noise, decode_mode, processing_res=128, steps=2):
    """Every image's [E, C, H, W] member maps through the list path."""
    got = {}
    pipe._infer_list(images, E, steps, processing_res, "bilinear", batch_size, None, noise, None, decode_mode,
                     lambda i, maps, hw: got.__setitem__(i, maps.clone()))
    return [got[i] for i in range(len(images))]


def test_cross_image_batches_are_exact(setup):
    """Three images, E = 3, batches of 4: batches [i0 m0-2, i1 m0], [i1 m1-2, i2 m0-1], [i2 m2]. Member (i, m) in slot p
    of a batch of NB equals, bit for bit, the same inputs in slot p of a batch of NB whose other slots hold members of an
    unrelated image."""
    eng, text = setup
    depth = _depth(eng, text)
    E, bs = 3, 4
    imgs = [_img(31), _img(32), _img(33)]
    noise = [_randn(40 + i, E, 4, 16, 16) for i in range(3)]
    maps = _members(depth, imgs, E, bs, noise, 0)
    lat = [depth.encode_rgb(depth._preprocess(im, 128, "bilinear")[0]) for im in imgs]
    other = depth.encode_rgb(depth._preprocess(_img(99), 128, "bilinear")[0])
    n_jobs = 3 * E
    for start in range(0, n_jobs, bs):
        jobs = list(range(start, min(start + bs, n_jobs)))
        NB = len(jobs)
        for p, k in enumerate(jobs):
            i, m = divmod(k, E)
            rl = other.expand(NB, -1, -1, -1).clone()
            z0 = _randn(500 + k, NB, 4, 16, 16).cuda()
            rl[p], z0[p] = lat[i][0], noise[i][m].cuda()
            ref = eng.decode(eng.denoise(rl.contiguous(), z0.contiguous()), 0)
            assert torch.equal(ref[p], maps[i][m]), f"image {i} member {m} (slot {p} of {NB})"


def test_mixed_sizes(setup):
    """128 x 128, 96 x 160, 128 x 128 at processing_res = 0: two size groups, outputs in input order, each within the
    decoder's TAU of the single call (the batch sizes differ from the single call's, so the bits may)."""
    from marigold_b200.pipeline import _lib_decode_depth

    eng, text = setup
    depth = _depth(eng, text)
    imgs = [_img(51), _img(52, 96, 160), _img(53)]
    for E in (1, 3):
        noise = [_randn(60 + i, E, 4, im.shape[-2] // 8, im.shape[-1] // 8) for i, im in enumerate(imgs)]
        outs = depth(imgs, ensemble_size=E, processing_res=0, noise=noise)
        assert [o.depth_np.shape for o in outs] == [(128, 128), (96, 160), (128, 128)]
        if E == 1:
            for im, z, o in zip(imgs, noise, outs):
                ref = depth(im, ensemble_size=1, processing_res=0, noise=z).depth_np
                assert np.abs(o.depth_np - ref).max() <= N.TAU["decode"] * N.rms(torch.from_numpy(ref))
        else:
            maps = _members(depth, imgs, E, 0, noise, _lib_decode_depth, processing_res=0)
            for im, z, got in zip(imgs, noise, maps):
                ref = depth._infer_members(depth._preprocess(im, 0, "bilinear")[0], E, 2, 0, None, z, None, 0)
                assert got.shape == ref.shape
                for m in range(E):
                    assert (got[m] - ref[m]).abs().max() <= N.TAU["decode"] * N.rms(ref[m])


def test_list_calls_are_deterministic(setup):
    eng, text = setup
    depth = _depth(eng, text)
    imgs = [_img(71), _img(72), _img(73)]
    kw = dict(ensemble_size=3, batch_size=4, ensemble_kwargs=dict(output_uncertainty=True))
    a = depth(imgs, generator=torch.Generator().manual_seed(1), **kw)
    b = depth(imgs, generator=torch.Generator().manual_seed(1), **kw)
    for x, y in zip(a, b):
        _assert_same(x, y)


def test_errors_before_any_work(setup):
    from marigold_b200 import _lib
    from marigold_b200.pipeline import MAX_PIXELS

    eng, text = setup
    lib = _lib.load(build_if_missing=False)
    depth = _depth(eng, text)
    good = [_img(81), _img(82)]
    huge = torch.zeros(1, 3, 1, 1, dtype=torch.uint8).expand(1, 3, 9000, 8000)
    assert 9000 * 8000 > MAX_PIXELS
    z = [_randn(1, 1, 4, 16, 16)] * 3
    cases = [(TypeError, dict(input_image=good + ["not an image"])),
             (AssertionError, dict(input_image=good + [torch.zeros(3, 64, 64)])),
             (ValueError, dict(input_image=good + [huge], processing_res=0)),
             (ValueError, dict(input_image=good + [_img(83)], noise=z[:2])),
             (ValueError, dict(input_image=good + [_img(83)], generator=[None, None])),
             (ValueError, dict(input_image=good + [_img(83)], ensemble_size=65))]
    for exc, kw in cases:
        torch.cuda.synchronize()
        n0 = lib.mgb_launch_count()
        out = None
        with pytest.raises(exc) as info:
            out = depth(**kw)
        assert out is None and lib.mgb_launch_count() == n0, kw
        if exc is not ValueError or "processing_res" in kw:
            assert "image 2" in str(info.value), str(info.value)
    n0 = lib.mgb_launch_count()
    assert depth([]) == [] and lib.mgb_launch_count() == n0
    # single inputs keep their own errors
    with pytest.raises(TypeError):
        depth("not an image")


def test_memory_does_not_grow_with_the_list(setup):
    from marigold_b200.pipeline import call_reserve_bytes

    eng, text = setup
    depth = _depth(eng, text)
    kw = dict(ensemble_size=3, batch_size=4, ensemble_kwargs=dict(output_uncertainty=True))
    depth([_img(90)] * 3, **kw)                                  # warm-up: step graph, arena, scipy
    peaks = []
    for n in (3, 24):
        imgs = [_img(900 + i) for i in range(n)]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        outs = depth(imgs, **kw)
        torch.cuda.synchronize()
        assert len(outs) == n
        peaks.append(torch.cuda.max_memory_allocated() - base)
    assert peaks[1] - peaks[0] <= call_reserve_bytes(128, 128, 3, 1), peaks
