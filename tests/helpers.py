"""Shared builders for the parity tests: seeded oracle networks (the checker) and an Engine (the
product) loaded with the same weights; the wrappers of the library's debug hooks; and the inputs, float64 references
and stub engines that more than one test module uses."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from oracle.unet import UNet2DConditionOracle, UNetConfig
from oracle.vae import AutoencoderKLOracle, VAEConfig


def usable_cores() -> int:
    """Cores this process may actually use (affinity mask and cgroup CPU quota), not os.cpu_count():
    on the GPU box the container sees 128 CPUs but is limited, and 128 torch threads thrash."""
    import os

    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:  # noqa: BLE001
        pass
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(p))))
    except Exception:  # noqa: BLE001
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            p_ = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                n = min(n, max(1, q // p_))
        except Exception:  # noqa: BLE001
            pass
    return max(1, n)


def oracle_models(kind: str = "tiny", seed: int = 0):
    torch.manual_seed(seed)
    if kind == "tiny":
        ucfg, vcfg = UNetConfig.tiny(), VAEConfig.tiny()
    else:
        ucfg, vcfg = UNetConfig(), VAEConfig()
    unet = UNet2DConditionOracle(ucfg).eval()
    vae = AutoencoderKLOracle(vcfg).eval()
    g = torch.Generator().manual_seed(7)
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=g)
    return unet, vae, text


def engine_from_oracle(unet, vae, text):
    from marigold_b200.engine import Engine, EngineConfig

    cfg = EngineConfig(unet_block_channels=list(unet.cfg.block_out_channels),
                       unet_cross_dim=unet.cfg.cross_attention_dim,
                       vae_block_channels=list(vae.cfg.block_out_channels))
    eng = Engine(cfg)
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    eng.set_text_embedding(text)
    return eng


def synthetic_image(S: int, seed: int = 1234) -> torch.Tensor:
    """uint8 [1,3,S,S]: smooth sinusoids + rectangles + pixel noise (SURVEY.md §8(d))."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, S), np.linspace(0, 1, S), indexing="ij")
    img = np.zeros((3, S, S))
    for _ in range(6):
        fx, fy, ph = rng.uniform(0.5, 4, 2).tolist() + [rng.uniform(0, 6.28)]
        amp = rng.uniform(20, 50, 3)
        img += amp[:, None, None] * np.sin(2 * np.pi * (fx * xx + fy * yy) + ph)[None]
    img += 128
    for _ in range(5):
        x0, y0 = rng.integers(0, S - 8, 2)
        w, h = rng.integers(8, max(9, S // 3), 2)
        img[:, y0:y0 + h, x0:x0 + w] = rng.uniform(0, 255, 3)[:, None, None]
    img += rng.normal(0, 4, img.shape)
    return torch.from_numpy(np.clip(img, 0, 255).astype(np.uint8))[None]


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def record(name: str, value: float) -> float:
    """Append a measured parity value to $MGB_PARITY_DIR/parity_values.jsonl when that variable names a directory (the
    tolerances asserted in the GPU tests are these measurements plus a margin). Without it nothing is written."""
    import json
    import os
    from pathlib import Path

    if not os.environ.get("MGB_PARITY_DIR"):
        return float(value)
    out = Path(os.environ["MGB_PARITY_DIR"])
    try:
        out.mkdir(parents=True, exist_ok=True)
        with open(out / "parity_values.jsonl", "a") as f:
            f.write(json.dumps({"name": name, "value": float(value)}) + "\n")
    except OSError:
        pass
    return float(value)


# ---- the library's debug hooks (marigold_b200/csrc/debug.h; typed by _lib.DEBUG_SIGNATURES) ---------------------------
def live_device_bytes() -> int:
    """Device and pinned host bytes the library's buffers hold now."""
    from marigold_b200 import _lib

    return _lib.load().mgb_debug_live_device_bytes()


def weight_bytes(eng) -> int:
    """Bytes of every device array the engine's weights own."""
    f = eng.lib.mgb_debug_weight_buffers
    n = f(eng._h, None, None, 0)
    size = (C.c_int64 * n)()
    assert f(eng._h, None, size, n) == n
    return sum(size)


def attn_blocks(eng, NB, T, budget=0, force_rows=0):
    """(rows per block, blocks over the NB images) of an (NB, T) VAE attention; sets the handle's budget and forced rows
    (0: the library's)."""
    from marigold_b200._lib import check

    r, b = C.c_int32(), C.c_int32()
    check(eng.lib.mgb_debug_vae_attn_blocks(eng._h, budget, force_rows, NB, T, C.byref(r), C.byref(b)),
          "mgb_debug_vae_attn_blocks")
    return r.value, b.value


def attn_core(eng, q, k, v, NB, T):
    """mgb_debug_vae_attn_core: bf16 q, k, v [NB T, 512] -> bf16 o, with the handle's row blocking."""
    from marigold_b200._lib import check

    o = torch.empty_like(q)
    check(eng.lib.mgb_debug_vae_attn_core(eng._h, q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), NB, T),
          "mgb_debug_vae_attn_core")
    torch.cuda.synchronize()
    return o


def set_arena(eng, poison=False, placement=0):
    from marigold_b200._lib import check

    check(eng.lib.mgb_debug_arena(eng._h, int(poison), placement), "mgb_debug_arena")


def set_low_memory(eng, mode):
    """1: the decoder's full-resolution stage in low memory at every size; -1: never; 0: the library's rule."""
    from marigold_b200._lib import check

    check(eng.lib.mgb_debug_vae_low_memory(eng._h, mode), "mgb_debug_vae_low_memory")


def set_bands(eng, up_tiles=0, conv1_tiles=0):
    """Tile rows per band of the low-memory decoder's banded up-conv and conv1 (0: the library's choice)."""
    from marigold_b200._lib import check

    check(eng.lib.mgb_debug_vae_bands(eng._h, up_tiles, conv1_tiles), "mgb_debug_vae_bands")


def _int64_ptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def arena_plan(eng, op, B, d0, d1):
    """(bytes, t_alloc, t_free, offset) per buffer of one forward's arena (op 0 UNet step, 1 encode, 2 decode)."""
    f = eng.lib.mgb_debug_arena_plan
    n = f(eng._h, op, B, d0, d1, None, None, None, None, 0)
    assert n > 0, n
    arrs = [np.zeros(n, dtype=np.int64) for _ in range(4)]
    assert f(eng._h, op, B, d0, d1, *map(_int64_ptr, arrs), n) == n
    return arrs


def arena_place(nbytes, t0, t1, placement=0):
    from marigold_b200 import _lib

    off = np.zeros(len(nbytes), dtype=np.int64)
    peak = _lib.load().mgb_debug_arena_place(len(off), _int64_ptr(nbytes), _int64_ptr(t0), _int64_ptr(t1), placement,
                                             _int64_ptr(off))
    assert peak >= 0
    return peak, off


# ---- native-resolution inputs and float64 references -------------------------------------------------------------
U_PER_PIXEL = 512          # bytes of one fp32 128-channel map per output pixel
VAE_C = 512


def _photo(h, w, seed=3):
    return synthetic_image(max(h, w), seed=seed)[..., :h, :w].contiguous()


def _rows(n_rows, width, seed, n_random=64):
    """The first and last 64 rows of a [n_rows, width] tensor, those holding elements 2^30 .. 2^33 and their neighbours,
    and n_random seeded rows."""
    rows = set(range(64)) | set(range(n_rows - 64, n_rows))
    for e in (2 ** 30, 2 ** 31, 2 ** 32, 2 ** 33):
        rows |= {e // width - 1, e // width, e // width + 1}
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, n_rows, (n_random,), generator=g).tolist())
    return torch.tensor(sorted(r for r in rows if 0 <= r < n_rows), dtype=torch.long)


def _block_rows(T, block, seed, every=1, n_random=128):
    """Query rows of a row-blocked (or row-tiled) kernel: the first 32 and last 64, both sides of every `every`-th block
    boundary, and n_random seeded rows."""
    rows = set(range(32)) | set(range(T - 64, T))
    for r0 in range(block, T, block * every):
        rows |= {r0 - 1, r0}
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, T, (n_random,), generator=g).tolist())
    return torch.tensor(sorted(rows), dtype=torch.long)


def no_overlap(nbytes, t0, t1, off):
    live = (t0[:, None] < t1[None, :]) & (t0[None, :] < t1[:, None])
    mem = (off[:, None] < (off + nbytes)[None, :]) & (off[None, :] < (off + nbytes)[:, None]) & (nbytes[:, None] > 0)
    both = live & mem & (nbytes[None, :] > 0)
    np.fill_diagonal(both, False)
    return not both.any()


def group_stats64(x, G, eps, chunk=1 << 20):
    """float64 mean and 1 / sqrt(var + eps) per group of x [HW, C] ([1, G, 1] each), two passes over row chunks."""
    from tests import ops_ref as R

    HW, C = x.shape
    n = HW * (C // G)
    s = torch.zeros(G, dtype=torch.float64, device=x.device)
    for a in range(0, HW, chunk):
        s += R.f64(x[a:a + chunk]).view(-1, G, C // G).sum(dim=(0, 2))
    mean = (s / n).view(1, G, 1)
    q = torch.zeros(G, dtype=torch.float64, device=x.device)
    for a in range(0, HW, chunk):
        q += ((R.f64(x[a:a + chunk]).view(-1, G, C // G) - mean) ** 2).sum(dim=(0, 2))
    return mean, (1.0 / torch.sqrt(q / n + eps)).view(1, G, 1)


def groupnorm_rows_ref(x_rows, mean, rstd, gamma, beta, G):
    """float64 SiLU(GroupNorm) of rows [n, C] given the statistics, and the bound of tests/ops_cases.py's GroupNorm case."""
    from tests import ops_ref as R
    from tests.ops_cases import _norm_mag

    n, C = x_rows.shape
    x64 = R.f64(x_rows).view(n, G, C // G)
    ga, be = R.f64(gamma).view(G, C // G), R.f64(beta).view(G, C // G)
    ref = R.silu64(((x64 - mean) * rstd * ga + be).reshape(n, C))
    mag = _norm_mag(x64, mean, rstd, ga, be).reshape(n, C)
    return ref, R.bf16_bound(ref, mag * R.SILU_GAIN)


def conv_row_ref(x, wb, y, b, x2=None, wsc=None):
    """float64 output row y [W, Cout] of the 3x3 pad-1 conv of NHWC x [1, H, W, Cin] (bf16) with bias b, plus the 1x1
    x2 [1, H, W, Cin2] @ wsc^T; and the bound of tests/ops_cases.py's conv case (K = 9 Cin + Cin2, fp32 output)."""
    from tests import ops_ref as R

    H, Cin = x.shape[1], x.shape[3]
    lo, hi = max(0, y - 1), min(H, y + 2)
    band = torch.zeros(1, Cin, 3, x.shape[2], dtype=torch.float64, device=x.device)
    band[0, :, lo - (y - 1):hi - (y - 1)] = R.f64(x[0, lo:hi]).permute(2, 0, 1)
    acc, absprod = R.conv64(band, wb, 1, (0, 1))
    acc, absprod = acc[0, :, 0].t(), absprod[0, :, 0].t()
    K = 9 * Cin
    if x2 is not None:
        a2, p2 = R.matmul64(x2[0, y], wsc)
        acc, absprod = acc + a2, absprod + p2
        K += x2.shape[3]
    ref = acc + R.f64(b)
    return ref, R.acc_bound(K, absprod) + 2 * R.R_F32_OUT * ref.abs() + R.TINY


def _core_inputs(NB, T, regime):
    from tests.ops_cases import dominant_key

    g = torch.Generator(device="cuda").manual_seed(7 * T + NB)
    std = 6.3 if regime == "logits80" else 1.0
    q = torch.randn(NB, T, VAE_C, device="cuda", generator=g) * std
    k = torch.randn(NB, T, VAE_C, device="cuda", generator=g) * std
    v = torch.randn(NB, T, VAE_C, device="cuda", generator=g)
    if regime in ("key_last", "key_mid"):
        dominant_key(q, k, T - 1 if regime == "key_last" else T // 2 + 7, 14.0, VAE_C ** -0.5, VAE_C, seed=T)
    return [t.reshape(NB * T, VAE_C).to(torch.bfloat16) for t in (q, k, v)]


def _core_ref(q, k, v, NB, T, rows):
    """float64 o, its bound (tests/test_native_res_gpu.py's docstring) and sum_j p_j |v_j| at `rows` of every image:
    [NB, len(rows), C]."""
    from tests import ops_ref as R

    Cc, Tp, scale = VAE_C, (T + 63) // 64 * 64, VAE_C ** -0.5
    ref = torch.empty(NB, len(rows), Cc, dtype=torch.float64, device="cuda")
    bound, pv_abs = torch.empty_like(ref), torch.empty_like(ref)
    step = max(1, (1 << 26) // T)
    for n in range(NB):
        k64, v64 = R.f64(k[n * T:(n + 1) * T]), R.f64(v[n * T:(n + 1) * T])
        ka, va = k64.abs(), v64.abs()
        for i in range(0, len(rows), step):
            qr = R.f64(q[n * T + rows[i:i + step]])
            s = qr @ k64.t() * scale
            ds = R.C_ACC * Cc * R.U_F32 * scale * (qr.abs() @ ka.t()) + R.R_F32_OUT * s.abs()
            dist = s.max(dim=1, keepdim=True).values - s
            del s
            p = torch.exp(-dist)
            p /= p.sum(dim=1, keepdim=True)
            o = p @ v64
            pds = p * ds
            del ds
            w = p * (R.softmax_rel(T, dist, p) + R.C_ACC * Tp * R.U_F32) + pds
            del dist
            pa = p @ va
            sl = slice(i, i + step)
            ref[n, sl], pv_abs[n, sl] = o, pa
            bound[n, sl] = ((R.U_BF16 + 2 * R.R_F32_OUT) * o.abs() + R.C_P * R.U_BF16 * pa + w @ va
                            + o.abs() * pds.sum(dim=1, keepdim=True) + R.TINY)
            del p, pds, w
    return ref, bound, pv_abs


# ---- stub engines of the host pipeline tests -----------------------------------------------------------------------
GB = 1 << 30


class StubEngine:
    """workspace_bytes: `per_member` bytes per member plus a fixed part; 0 past the supported maximum (like the
    library). held_bytes: what the engine holds now."""

    def __init__(self, per_member, fixed=GB, held=0):
        self.per_member, self.fixed, self.held = per_member, fixed, held
        self.asked = []

    def workspace_bytes(self, B, H, W):
        from marigold_b200.pipeline import MAX_PIXELS

        self.asked.append(B)
        return 0 if B * H * W > MAX_PIXELS else self.fixed + B * self.per_member

    def held_bytes(self):
        return self.held


class _Cfg:
    unet_out_channels = 4


class _Lib:
    @staticmethod
    def mgb_ens_max_members():
        return 64


class FakeEngine:
    """encode: a per-image constant latent; denoise: rgb_latent + z0 (+ the step noise's sum); decode: the first channel,
    8x nearest. Every member map is therefore a known function of its own image and noise. Records the batch shapes."""
    cfg, lib, device = _Cfg(), _Lib(), torch.device("cpu")

    def __init__(self):
        self.log = []

    def set_text_embedding(self, t):
        pass

    def set_schedule(self, *a):
        pass

    def workspace_bytes(self, B, H, W):
        return GB

    def held_bytes(self):
        return 0

    def encode(self, rgb):
        self.log.append(("encode",))
        return rgb.mean().reshape(1, 1, 1, 1).expand(1, 4, rgb.shape[-2] // 8, rgb.shape[-1] // 8).contiguous()

    def denoise(self, rl, z, sn=None):
        self.log.append(("denoise", tuple(z.shape)))
        return rl + z + (sn.sum(0) if sn is not None else 0)

    def decode(self, t, mode):
        return t[:, :1].repeat_interleave(8, 2).repeat_interleave(8, 3)


def _pipe(lcm=False, normals=False):
    from marigold_b200.pipeline import MarigoldDepthPipeline, MarigoldNormalsPipeline
    from marigold_b200.schedulers import DDIMScheduler, LCMScheduler

    cls = MarigoldNormalsPipeline if normals else MarigoldDepthPipeline
    pipe = cls(FakeEngine(), LCMScheduler() if lcm else DDIMScheduler(), None)
    pipe._preprocess = lambda im, pr, rs: (im.float() / 255 * 2 - 1, im.shape)
    return pipe


def _images(sizes):
    g = torch.Generator().manual_seed(3)
    return [torch.randint(0, 256, (1, 3, h, w), generator=g, dtype=torch.uint8) for h, w in sizes]


def _expected(img, z, sn):
    lat = (img.float() / 255 * 2 - 1).mean()
    t = lat + z + (sn.sum(0) if sn is not None else 0)
    return t[:, :1].repeat_interleave(8, 2).repeat_interleave(8, 3)


def _run(pipe, images, E, steps, bs, generator=None, noise=None, step_noise=None):
    done, log = {}, pipe.engine.log

    def finish(i, maps, hw):
        log.append(("finish", i))
        done[i] = maps.clone()

    pipe._infer_list(images, E, steps, 0, "bilinear", bs, generator, noise, step_noise, 0, finish)
    return done


# ---- ensembling and LPIPS ------------------------------------------------------------------------------------------
def _ref_cost(d, p, shift, reduction, reg):
    """reference cost_fn (ensemble.py:138-152) restated with torch CPU ops."""
    E = d.shape[0]
    if shift:
        s, t = np.split(p, 2)
        a = d * torch.from_numpy(s).float().view(E, 1, 1, 1) + torch.from_numpy(t).float().view(E, 1, 1, 1)
    else:
        a = d * torch.from_numpy(p).float().view(E, 1, 1, 1)
    c = 0.0
    for i in range(E):
        for j in range(i + 1, E):
            c += ((a[i] - a[j]) ** 2).mean().sqrt().item()
    if reg > 0:
        pr = a.median(0).values if reduction == "median" else a.mean(0)
        c += (abs(0.0 - pr.min().item()) + abs(1.0 - pr.max().item())) * reg
    return c


# (target, mask, transform, kind): see tests/golden/iid_eval_cases.py
CONFIGS = [
    ("albedo", "none", None, "noisy"),
    ("material", "pixel", "srgb2linear", "noisy"),
    ("shading", "split", "linear2srgb", "noisy"),
    ("residual", "pixel", None, "q255"),
    ("shading", "none", "srgb2linear", "q255"),
    ("residual", "split", None, "nan"),
    ("albedo", "split", "linear2srgb", "nan"),
    ("shading", "single", None, "noisy"),
    ("residual", "none", None, "dark"),
    ("albedo", "empty", None, "noisy"),
]


def _inputs(H, W, target, mask, transform, kind, seed=0):
    """CUDA (pred, gt, mask); the non-scale targets' predictions clipped to [0, 1], as LPIPS requires."""
    from tests import iid_eval_ref
    from tests.golden.iid_eval_cases import iid_eval_input

    cfg = dict(H=H, W=W, seed=1000 + seed + H + W, target=target, mask=mask, transform=transform, kind=kind)
    pred, gt, m = iid_eval_input(cfg)
    if target not in iid_eval_ref.UP_TO_SCALE:
        pred = np.clip(pred, 0.0, 1.0)
    return (torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(), torch.from_numpy(m).cuda() if m is not None else None)


def _launches(fn):
    from marigold_b200 import _lib

    lib = _lib.load()
    torch.cuda.synchronize()
    l0 = lib.mgb_launch_count()
    r = fn()
    return r, lib.mgb_launch_count() - l0
