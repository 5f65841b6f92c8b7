"""Kernel launches each entry point adds to mgb_launch_count(). Every kernel the library enqueues counts once; memsets
and copies are not kernels and do not count; a replay of the cached step graph counts the kernels the graph holds.
bench.py reports this counter as gpu_launches."""
import numpy as np
import pytest
import torch

from tests.helpers import oracle_models

pytestmark = pytest.mark.gpu

EXPECTED = {
    "finalize": 16,
    "set_text_embedding": 48,
    "set_schedule": 25,
    "encode": 71,
    "unet_step": 299,
    "unet_step_noise_model_out": 301,
    "denoise_first": 893,
    "denoise_second": 894,
    "decode_0": 94,
    "decode_1": 94,
    "decode_2": 94,
    "decode_3": 94,
    "ens_depth_cost_fd_E4_shift": 3,
    "ens_depth_cost_fd_E4_scale": 3,
    "ens_depth_cost_fd_E20_shift": 2,
    "ens_depth_cost_fd_E20_scale": 2,
    "ens_minmax": 1,
    "ens_depth_reduce": 2,
    "ens_iid": 1,
    "ens_normals": 1,
    "eval_depth_ex": 4,
    "eval_normals": 4,
    "resize_u8": 2,
    "resize_f32": 2,
    "colorize": 1,
    "op_flash_attn64_split": 2,
    "op_flash_attn64_unsplit": 1,
    "op_groupnorm_ex": 1,
    "op_linear_splitk": 2,
}


def _delta(fn, *args, **kw):
    from marigold_b200 import _lib

    lib = _lib.load()
    torch.cuda.synchronize()
    l0 = lib.mgb_launch_count()
    r = fn(*args, **kw)
    torch.cuda.synchronize()
    return int(lib.mgb_launch_count() - l0), r


def _network(n, eng, models):
    from marigold_b200.schedulers import DDIMScheduler

    unet, vae, text = models
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    n["finalize"], _ = _delta(eng.finalize)
    n["set_text_embedding"], _ = _delta(eng.set_text_embedding, text)
    s = DDIMScheduler()
    s.set_timesteps(3)
    n["set_schedule"], _ = _delta(eng.set_schedule, s.timesteps, *s.coefficients())
    g = torch.Generator().manual_seed(0)
    img = (torch.rand(1, 3, 64, 64, generator=g) * 2 - 1).cuda()
    x = torch.randn(1, 4, 8, 8, generator=g).cuda()
    n["encode"], lat = _delta(eng.encode, img)
    n["unet_step"], _ = _delta(eng.unet_step, lat, x.clone(), 0)
    n["unet_step_noise_model_out"], _ = _delta(eng.unet_step, lat, x.clone(), 1, noise=torch.randn_like(x),
                                               want_model_out=True)
    n["denoise_first"], _ = _delta(eng.denoise, lat, x)       # step 0 eager, then captured; later steps replay
    n["denoise_second"], y = _delta(eng.denoise, lat, x)      # every step replays the graph
    for mode in range(4):
        n[f"decode_{mode}"], _ = _delta(eng.decode, y, mode)


def _ensemble(n, eng):
    from marigold_b200._lib import check, ptr, stream_ptr
    from marigold_b200.ensemble import ensemble_iid, ensemble_normals

    lib, h = eng.lib, eng._h
    g = torch.Generator(device="cuda").manual_seed(1)
    HW = 64 * 64
    for E in (4, 20):
        d = torch.rand(E, HW, device="cuda", generator=g) + 0.5
        base = np.concatenate([np.linspace(0.9, 1.1, E), np.linspace(-0.1, 0.1, E)])
        pert = base + 1e-3
        for shift in (1, 0):
            out = np.empty(1 + (2 * E if shift else E))
            key = f"ens_depth_cost_fd_E{E}_{'shift' if shift else 'scale'}"
            n[key], rc = _delta(lib.mgb_ens_depth_cost_fd, h, ptr(d), base.ctypes.data, pert.ctypes.data, E, HW, 1, shift,
                                1, 0.02, out.ctypes.data, stream_ptr())
            check(rc, "mgb_ens_depth_cost_fd")
    E = 4
    d = torch.rand(E, HW, device="cuda", generator=g) + 0.5
    mn, mx = np.zeros(E, np.float32), np.zeros(E, np.float32)
    n["ens_minmax"], rc = _delta(lib.mgb_ens_minmax, h, ptr(d), E, HW, mn.ctypes.data, mx.ctypes.data, stream_ptr())
    check(rc, "mgb_ens_minmax")
    param = np.concatenate([np.ones(E), np.zeros(E)])
    pred, unc = torch.empty(HW, device="cuda"), torch.empty(HW, device="cuda")
    idx = torch.empty(HW, dtype=torch.int32, device="cuda")
    n["ens_depth_reduce"], rc = _delta(lib.mgb_ens_depth_reduce, h, ptr(d), param.ctypes.data, E, HW, 1, 1, 1, ptr(pred),
                                       ptr(unc), ptr(idx), stream_ptr())
    check(rc, "mgb_ens_depth_reduce")
    n["ens_iid"], _ = _delta(ensemble_iid, torch.rand(E, 3, 32, 32, device="cuda", generator=g), True, engine=eng)
    nrm = torch.nn.functional.normalize(torch.randn(E, 3, 32, 32, device="cuda", generator=g), dim=1)
    n["ens_normals"], _ = _delta(ensemble_normals, nrm, True, engine=eng)


def _eval_and_image(n):
    from marigold_b200.evaluation import evaluate_depth, evaluate_normals
    from marigold_b200.imageops import colorize_u8, resize, spectral_lut_u8

    g = torch.Generator(device="cuda").manual_seed(2)
    pred = torch.rand(48, 64, device="cuda", generator=g) + 0.5
    gt = torch.rand(48, 64, device="cuda", generator=g) + 0.5
    n["eval_depth_ex"], _ = _delta(evaluate_depth, pred, gt, gt > 0.7, alignment="least_square_disparity",
                                   alignment_max_res=32)
    p3 = torch.nn.functional.normalize(torch.randn(3, 48, 64, device="cuda", generator=g), dim=0)
    g3 = torch.nn.functional.normalize(torch.randn(3, 48, 64, device="cuda", generator=g), dim=0)
    n["eval_normals"], _ = _delta(evaluate_normals, p3, g3)
    img = torch.randint(0, 256, (1, 3, 40, 56), dtype=torch.uint8, device="cuda", generator=g)
    n["resize_u8"], _ = _delta(resize, img, (24, 32), "bilinear", 2)
    n["resize_f32"], _ = _delta(resize, img.float(), (24, 32), "bicubic", 0)
    n["colorize"], _ = _delta(colorize_u8, pred, 0.5, 1.5, spectral_lut_u8())


def _ops(n):
    from marigold_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(3)
    for name, (NB, T, C) in (("split", (1, 4096, 64)), ("unsplit", (1, 128, 64))):
        qkv = torch.randn(NB * T, 3 * C, device="cuda", generator=g).to(torch.bfloat16)
        n[f"op_flash_attn64_{name}"], _ = _delta(ops.flash_attn64, qkv, NB, T, C, 0.125)
    xa = torch.randn(1, 64, 64, device="cuda", generator=g)
    xb = torch.randn(1, 64, 64, device="cuda", generator=g)
    gamma, beta = torch.ones(128, device="cuda"), torch.zeros(128, device="cuda")
    n["op_groupnorm_ex"], _ = _delta(ops.groupnorm_ex, xa, xb, gamma, beta, 1, 64, 32, 1e-5, 1)
    a = torch.randn(128, 512, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(128, 512, device="cuda", generator=g).to(torch.bfloat16)
    ws = torch.empty(2 * 128 * 128, device="cuda")
    n["op_linear_splitk"], _ = _delta(ops.linear, a, w, block_n=128, splits=2, stages=4, ws=ws)


def test_launch_count_of_every_entry_point():
    from marigold_b200.engine import Engine, EngineConfig

    models = oracle_models("tiny")
    unet, vae, _ = models
    eng = Engine(EngineConfig(unet_block_channels=list(unet.cfg.block_out_channels),
                              unet_cross_dim=unet.cfg.cross_attention_dim,
                              vae_block_channels=list(vae.cfg.block_out_channels)))
    n = {}
    _network(n, eng, models)
    _ensemble(n, eng)
    _eval_and_image(n)
    _ops(n)
    eng.close()
    assert n == EXPECTED, n
