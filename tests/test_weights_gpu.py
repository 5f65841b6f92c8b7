"""Every device table an engine builds, read back through the handle's debug hook and held to the float64 restatement
of the checkpoint in tests/weights_ref.py, one parameter at a time.

The network tests (tests/test_net_faithful_gpu.py) see a loader or fold error only when it moves a 60-layer output by
more than the bf16 rounding noise; most UNet body parameters do not. Here each table is compared on its own: the
repacked weights and fp32 copies bit for bit, the device-folded tables (fold_matmul, linear_small, xattn2_fold, the
time embedding and per-step bias table) element by element against a bound. A completeness check proves that every
device buffer the weights own was read, whole. The per-step state the captured UNet step selects on the device, the
in-place text folding, fp16 / bf16 checkpoints and the decoder's latent packing are checked the same way."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import net_ref as N
from tests import weights_ref as W
from tests.helpers import engine_from_oracle, oracle_models, record

pytestmark = pytest.mark.gpu


# ---- read-back ------------------------------------------------------------------------------------------------------
def _fn(name, res, args):
    from marigold_b200 import _lib

    f = getattr(_lib.load(), name)        # debug hooks outside the public header
    f.restype, f.argtypes = res, args
    return f


class Reader:
    """Reads device tables of one engine (mgb_debug_read) and remembers the address and size of each one read."""

    def __init__(self, eng):
        self.eng, self.seen, self._last = eng, {}, (None, None)
        self._rd = _fn("mgb_debug_read", C.c_int64, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64,
                                                      C.POINTER(C.c_uint64)])

    def addr(self, field):
        a = C.c_uint64()
        n = self._rd(self.eng._h, field.encode(), None, 0, C.byref(a))
        _raise(n, field)
        return a.value, n

    def read(self, field, dtype):
        if self._last[0] == field:
            return self._last[1]
        addr, n = self.addr(field)
        t = torch.empty(n // 4 if dtype == "f32" else n // 2, dtype=torch.float32 if dtype == "f32" else torch.bfloat16)
        _raise(self._rd(self.eng._h, field.encode(), C.c_void_p(t.data_ptr()), n, None), field)
        self.seen[addr] = n
        self._last = (field, t)
        return t


def _raise(status, field):
    from marigold_b200._lib import check

    if status < 0:
        check(int(status), f"mgb_debug_read({field})")


def weight_buffers(eng):
    f = _fn("mgb_debug_weight_buffers", C.c_int32, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.c_int32])
    n = f(eng._h, None, None, 0)
    assert n > 0
    addr, size = (C.c_uint64 * n)(), (C.c_int64 * n)()
    assert f(eng._h, addr, size, n) == n
    return dict(zip(addr, size))


# ---- comparison -----------------------------------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def compare(ratios, fails, name, kind, dev, ref, bound=None, dtype="f32"):
    """Bit-equal (bound None: ref holds fp32 values, the device their bf16 for a bf16 table) or |dev - ref| <= bound.
    Records the largest |dev - ref| / bound per kind in `ratios`; appends a message per failing table to `fails`."""
    if bound is None:
        want = ref.float().reshape(dev.shape)
        if dtype == "bf16":
            want = want.to(torch.bfloat16)
        bad = _bits(dev) != _bits(want.contiguous())
        if bad.any():
            i = int(bad.reshape(-1).nonzero()[0])
            fails.append(f"{name}: {int(bad.sum())} of {bad.numel()} elements differ, first at {i}: "
                         f"{dev.reshape(-1)[i].item()!r} != {want.reshape(-1)[i].item()!r}")
        return
    err = (dev.double() - ref.reshape(dev.shape)).abs()
    bound = bound.reshape(dev.shape)
    r = torch.where(err == 0, torch.zeros_like(err), err / bound).nan_to_num(float("inf"))
    worst = float(r.max())
    ratios[kind] = max(ratios.get(kind, 0.0), worst)
    if not worst <= 1.0:
        i = int(r.reshape(-1).argmax())
        fails.append(f"{name}: |dev - ref| / bound = {worst:.3g} at {i} (dev {dev.reshape(-1)[i].item()!r}, "
                     f"ref {ref.reshape(-1)[i].item()!r}, bound {bound.reshape(-1)[i].item():.3g})")


def check_table(reader, t, ratios, fails):
    dev = reader.read(t.field, t.dtype).reshape(t.shape)
    if t.cols is not None:
        dev = dev[:, t.cols]
    compare(ratios, fails, t.field, t.kind, dev, t.ref, t.bound, t.dtype)
    if t.given_kv is not None:
        # the fold alone, from the device's own kv
        kv = reader.read(t.field.rsplit(".", 1)[0] + ".kv", "f32").double().reshape(4, -1)
        dev = reader.read(t.field, t.dtype).reshape(t.shape)
        ref, bound = t.given_kv(kv)
        compare(ratios, fails, t.field + " (device kv)", t.kind + " (device kv)", dev, ref, bound)


def check_weights(eng, usd, vsd, text, label):
    """Every weight table against weights_ref, then the completeness check; returns the ratios per kind."""
    cfg = eng.cfg
    reader, ratios, fails = Reader(eng), {}, []
    ctx = text.reshape(-1, text.shape[-1])
    for t in W.unet_tables(usd, cfg.unet_block_channels, cfg.unet_layers_per_block, ctx):
        check_table(reader, t, ratios, fails)
    for t in W.vae_tables(vsd, cfg.vae_block_channels, cfg.vae_layers_per_block, N.LATENT_SCALE):
        check_table(reader, t, ratios, fails)
    # the encoder fold is summed on the host in fp32: besides its bound, it is those exact bits
    compare(ratios, fails, "vae.enc_out.w (host fp32 sum)", "", reader.read("vae.enc_out.w", "bf16"),
            W.enc_out_host(vsd, N.LATENT_SCALE), dtype="bf16")
    bufs = weight_buffers(eng)
    missing = {a: n for a, n in bufs.items() if a not in reader.seen}
    assert not missing, f"{label}: {len(missing)} weight buffers were not read ({sum(missing.values())} bytes)"
    assert set(reader.seen) == set(bufs), f"{label}: read arrays the weights do not own"
    wrong = {a: (reader.seen[a], n) for a, n in bufs.items() if reader.seen[a] != n}
    assert not wrong, f"{label}: bytes read != buffer size for {len(wrong)} buffers: {list(wrong.values())[:4]}"
    for k, v in sorted(ratios.items()):
        record(f"weights/{label}/{k}", v)
    assert not fails, f"{label}: {len(fails)} tables differ:\n" + "\n".join(fails[:40])
    return ratios


def _schedule(kind, n):
    from marigold_b200.schedulers import DDIMScheduler, LCMScheduler

    s = DDIMScheduler() if kind == "ddim" else LCMScheduler()
    s.set_timesteps(n)
    return s, s.coefficients()


def check_schedule(eng, usd, s, coeffs, label, ratios=None):
    """bias_table against its bound, row by row and resnet by resnet, and sched_k bit for bit."""
    cfg = eng.cfg
    reader = Reader(eng)
    n = len(s.timesteps)
    ref, bound, cols = W.bias_table(usd, cfg.unet_block_channels, cfg.unet_layers_per_block, s.timesteps)
    tab = reader.read("bias_table", "f32").reshape(n, -1)
    assert tab.shape == ref.shape
    ratios = {} if ratios is None else ratios
    fails = []
    for i in range(n):
        for key, off, w in cols:
            compare(ratios, fails, f"{label} row {i} (t = {int(s.timesteps[i])}) {key}", "bias table",
                    tab[i, off:off + w], ref[i, off:off + w], bound[i, off:off + w])
    k = torch.from_numpy(np.stack([np.asarray(c, dtype=np.float32) for c in coeffs], 1))
    compare(ratios, fails, f"{label} sched_k", "", reader.read("sched_k", "f32").reshape(n, 3), k)
    assert not fails, "\n".join(fails[:40])
    record(f"weights/{label}/bias table", ratios.get("bias table", 0.0))
    return tab, k


# ---- engines --------------------------------------------------------------------------------------------------------
def _iid_models(n_targets):
    from oracle.unet import UNet2DConditionOracle, UNetConfig
    from oracle.vae import AutoencoderKLOracle, VAEConfig

    torch.manual_seed(0)
    ucfg = UNetConfig.tiny()
    ucfg.in_channels, ucfg.out_channels = 4 * (n_targets + 1), 4 * n_targets
    unet, vae = UNet2DConditionOracle(ucfg).eval(), AutoencoderKLOracle(VAEConfig.tiny()).eval()
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=torch.Generator().manual_seed(7))
    return unet, vae, text


def _engine(unet, vae, text, usd=None, vsd=None):
    from marigold_b200.engine import Engine, EngineConfig

    eng = Engine(EngineConfig(unet_in_channels=unet.cfg.in_channels, unet_out_channels=unet.cfg.out_channels,
                              unet_block_channels=list(unet.cfg.block_out_channels),
                              unet_cross_dim=unet.cfg.cross_attention_dim,
                              vae_block_channels=list(vae.cfg.block_out_channels)))
    eng.load_state_dict("unet", unet.state_dict() if usd is None else usd)
    eng.load_state_dict("vae", vae.state_dict() if vsd is None else vsd)
    eng.finalize()
    eng.set_text_embedding(text)
    return eng


@pytest.fixture(scope="module")
def tiny():
    unet, vae, text = oracle_models("tiny")
    N.randomise(unet, vae, seed=1)
    eng = engine_from_oracle(unet, vae, text)
    yield unet, vae, text, eng
    eng.close()


# ---- every table ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("config", ["depth", "iid2", "iid3", "sd2"])
def test_every_table_matches_the_checkpoint(config):
    """Depth (conv_in 8 -> 64 padded input channels, conv_out N = 4), IID with 2 and 3 targets (12 / 16 input channels,
    N = 8 / 12) and the SD-2 widths (5 / 10 / 20 heads, C = 1280)."""
    if config == "depth":
        unet, vae, text = oracle_models("tiny")
    elif config == "sd2":
        unet, vae, text = oracle_models("full")
    else:
        unet, vae, text = _iid_models(int(config[-1]))
    N.randomise(unet, vae, seed=5)
    eng = _engine(unet, vae, text)
    try:
        usd, vsd = unet.state_dict(), vae.state_dict()
        ratios = check_weights(eng, usd, vsd, text, config)
        s, coeffs = _schedule("ddim", 4)
        eng.set_schedule(s.timesteps, *coeffs)
        check_schedule(eng, usd, s, coeffs, f"{config}/ddim4", ratios)
        print(f"\n{config}: max |dev - ref| / bound per table kind")
        for k, v in sorted(ratios.items()):
            print(f"  {k:28s} {v:.3g}")
    finally:
        eng.close()


def test_unknown_field_and_unfinalized_handle_are_refused():
    from marigold_b200._lib import MgbError, load
    from marigold_b200.engine import Engine, EngineConfig

    unet, vae, _ = oracle_models("tiny")
    eng = Engine(EngineConfig.tiny())
    rd = Reader(eng)
    with pytest.raises(MgbError, match="finalize"):
        rd.addr("unet.conv_in.w")
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    before = int(load().mgb_launch_count())
    for bad in ("unet.conv_in.x", "unet.resnets.99.c1.w", "unet.xfmrs.0.qkv.b", "vae.enc_res.0.temb_w", "unet",
                "unet.resnets.01x.c1.w", "nothing"):
        with pytest.raises(MgbError, match=bad.replace(".", r"\.")):
            rd.addr(bad)
    assert rd.addr("bias_table") == (0, 0)                           # no schedule yet
    rd.read("unet.conv_in.w", "bf16")
    assert int(load().mgb_launch_count()) == before                  # reading launches nothing
    eng.close()


# ---- per-step tables ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,n", [("ddim", 1), ("ddim", 4), ("ddim", 10), ("ddim", 50), ("lcm", 4)])
def test_bias_table_every_row_and_resnet(tiny, kind, n):
    unet, vae, text, eng = tiny
    s, coeffs = _schedule(kind, n)
    eng.set_schedule(s.timesteps, *coeffs)
    check_schedule(eng, unet.state_dict(), s, coeffs, f"depth/{kind}{n}")


def _state(reader):
    cur = reader.read("cur_bias", "f32").clone()
    k = reader.read("cur_sched_k", "f32").clone()
    reader._last = (None, None)
    c = torch.empty(1, dtype=torch.int32)
    assert reader.addr("step_counter")[1] == 4
    reader._rd(reader.eng._h, b"step_counter", C.c_void_p(c.data_ptr()), 4, None)
    return cur, k, int(c[0])


@pytest.mark.parametrize("B", [1, 2])
def test_steps_select_their_row(tiny, B):
    """mgb_unet_step(i) selects row i; mgb_denoise_range over [a, a + k) replays the captured step for every step after
    the first, with the counter armed to i before step i and advanced at its end: it ends at a + k, holding row a + k - 1."""
    unet, vae, text, eng = tiny
    s, coeffs = _schedule("ddim", 10)
    eng.set_schedule(s.timesteps, *coeffs)
    reader = Reader(eng)
    tab = reader.read("bias_table", "f32").reshape(10, -1).clone()
    sk = reader.read("sched_k", "f32").reshape(10, 3).clone()
    g = torch.Generator().manual_seed(40 + B)
    rgb, x = torch.randn(B, 4, 8, 8, generator=g).cuda(), torch.randn(B, 4, 8, 8, generator=g).cuda()
    for i in (0, 3, 9):
        eng.unet_step(rgb, x.clone(), i)
        torch.cuda.synchronize()
        cur, k, _ = _state(reader)
        assert torch.equal(_bits(cur), _bits(tab[i])), f"unet_step({i}): cur_bias is not row {i}"
        assert torch.equal(_bits(k), _bits(sk[i])), f"unet_step({i}): cur_sched_k is not row {i}"
    for a, n in ((0, 3), (4, 5), (2, 2)):
        eng.denoise_range_(rgb, x.clone(), a, n)
        torch.cuda.synchronize()
        cur, k, counter = _state(reader)
        assert counter == a + n, f"denoise_range({a}, {n}): step counter {counter}"
        assert torch.equal(_bits(cur), _bits(tab[a + n - 1])), f"denoise_range({a}, {n}): cur_bias is not row {a + n - 1}"
        assert torch.equal(_bits(k), _bits(sk[a + n - 1])), f"denoise_range({a}, {n}): cur_sched_k is not row {a + n - 1}"


def test_second_schedule_equals_a_fresh_engine(tiny):
    unet, vae, text, eng = tiny
    for kind, n in (("ddim", 10), ("lcm", 4)):
        s, coeffs = _schedule(kind, n)
        eng.set_schedule(s.timesteps, *coeffs)
    fresh = engine_from_oracle(unet, vae, text)
    try:
        fresh.set_schedule(s.timesteps, *coeffs)
        for field in ("bias_table", "sched_k"):
            a, b = Reader(eng).read(field, "f32"), Reader(fresh).read(field, "f32")
            assert torch.equal(_bits(a), _bits(b)), field
    finally:
        fresh.close()


def test_text_embedding_is_folded_in_place(tiny):
    """A second context rewrites kv, xGU and xc1 where the captured step graph reads them, and they then hold it."""
    unet, vae, text, eng = tiny
    reader = Reader(eng)
    fields = [f"unet.xfmrs.{i}.{f}" for i in range(len(W.unet_layout(eng.cfg.unet_block_channels, 2)[1]))
              for f in ("kv", "xGU", "xc1")]
    before = {f: reader.addr(f) for f in fields}
    other = torch.randn(text.shape, generator=torch.Generator().manual_seed(50)) * 2
    try:
        eng.set_text_embedding(other)
        assert {f: reader.addr(f) for f in fields} == before
        ratios, fails = {}, []
        for t in W.unet_tables(unet.state_dict(), eng.cfg.unet_block_channels, 2, other.reshape(2, -1)):
            if t.field in before:
                check_table(reader, t, ratios, fails)
        assert not fails, "\n".join(fails)
    finally:
        eng.set_text_embedding(text)


# ---- checkpoint dtypes ----------------------------------------------------------------------------------------------
def _crafted():
    """fp16 subnormals, +-0, fp16 max-normal, fp32 values on bf16 round-to-even ties in both directions, and values that
    round to bf16 inf (a tie above bf16's largest finite and fp32's largest finite)."""
    bits = [0x33800000, 0x34400000, 0x387FC000, 0xB5800000,      # 2^-24, 3 2^-24, 1023 2^-24, -2^-20 (fp16 subnormal)
            0x00000000, 0x80000000, 0x477FE000, 0xC77FE000,      # +0, -0, +-65504
            0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,      # 1 + 2^-8 (to even: down), 1 + 3 2^-8 (up), negated
            0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000]                  # round to +inf, +inf, -inf in bf16
    return torch.tensor(np.array(bits, dtype=np.uint32).view(np.float32))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=["f32", "f16", "bf16"])
def test_checkpoint_dtypes(dtype):
    """A checkpoint in fp16 or bf16: bf16 tables hold bf16(fp32(x)) and fp32 tables fp32(x), exactly, including a
    crafted norm affine and conv weight (fp16 subnormals, ties, overflow to inf)."""
    unet, vae, text = oracle_models("tiny")
    N.randomise(unet, vae, seed=6)
    usd, vsd = dict(unet.state_dict()), dict(vae.state_dict())
    v = _crafted()
    for key in ("down_blocks.1.resnets.0.norm2.weight", "conv_in.weight"):
        t = usd[key].clone().reshape(-1)
        t[:len(v)] = v
        usd[key] = t.reshape(usd[key].shape)
    usd = {k: x.to(dtype) for k, x in usd.items()}
    vsd = {k: x.to(dtype) for k, x in vsd.items()}
    eng = _engine(unet, vae, text, usd, vsd)
    try:
        check_weights(eng, {k: x.float() for k, x in usd.items()}, {k: x.float() for k, x in vsd.items()}, text,
                      f"load_{str(dtype).split('.')[-1]}")
    finally:
        eng.close()


# ---- the decoder's input --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NB,h,w", [(1, 8, 8), (2, 9, 13), (1, 96, 96), (2, 72, 54), (1, 1, 3)])
def test_pack_decoder_latent(tiny, NB, h, w):
    """post_quant_conv(latent * fp32(1 / scale)) as bf16 NHWC-64 at the latent shapes the decoder sees: channels 0..3
    within u_b |ref| + 5u (|b| + sum |w| |x s^-1|), channels 4..63 exactly +0."""
    from marigold_b200 import ops

    unet, vae, text, eng = tiny
    wq, bq = vae.post_quant_conv.weight.detach().float(), vae.post_quant_conv.bias.detach().float()
    lat = torch.randn(NB, 4, h, w, generator=torch.Generator().manual_seed(60 + h))
    lat[0, :, 0, 0] = torch.tensor([0.0, -0.0, 1e-30, -40.0])
    z = ops.pack_decoder_latent(lat.cuda(), wq.reshape(4, 4).contiguous().cuda(), bq.cuda(), N.INV_LATENT_SCALE)
    torch.cuda.synchronize()
    z = z.cpu()
    ref, bound = W.pack_decoder_latent(lat, wq, bq, N.INV_LATENT_SCALE)
    ratios, fails = {}, []
    compare(ratios, fails, f"pack_decoder_latent {NB}x{h}x{w}", "pack_decoder_latent", z[:, :4].contiguous(), ref, bound)
    assert not fails, fails[0]
    assert not _bits(z[:, 4:].contiguous()).any(), "pad channels 4..63 are not +0"
    record(f"weights/pack_decoder_latent/{NB}x{h}x{w}", ratios["pack_decoder_latent"])
