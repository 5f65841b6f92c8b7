"""The UNet step, the denoising loop and the VAE decode at the batch sizes the pipelines launch (`-m gpu`).

`_infer_members` hands `denoise` and `decode` batches of find_batch_size(E, res) members: up to 16 at <= 768 px and 8
above. The launch geometry depends on the batch: GroupNorm's chunks per image (gn_max_ctas() / NB), the GEMM tile and
split-K choices and the flash attention's KV split (all decided from M = NB HW), the CUDA step graph (keyed by
(NB, lh, lw)), and every per-image offset inside the graph. These tests run the SD-2-width graphs, on oracle weights
whose every norm affine and bias has been redrawn (net_ref.randomise), at those batch sizes with distinct inputs per
member, and hold them to:

  exact (torch.equal)  independence: replacing member j's inputs leaves every other member's outputs bit for bit;
                       permutation: reversing or rotating the members permutes the outputs bit for bit;
                       graph re-keying: denoise at NB = 8, 2, 8 (the 1024 px 8 + 2 split) gives the same bits as the
                       first call, and as the same steps driven one at a time through unet_step;
  bounded              every member against the same member run alone (NB = 1: other chunking and split choices),
                       |batched - alone| <= TAU[stage] rms(alone); members 0 and NB - 1 at 768 and 1024 px against the
                       fp32 oracle within test_fullsize_gpu's bf16 yardstick;
  memory               mgb_workspace_bytes at every batch cap, plus the weights, fits an 80 GB card; the NB = 16
                       768 x 768 decode runs.
Measured values go to $MGB_PARITY_DIR/parity_values.jsonl (tests/helpers.record) as batch/<case>/<output>."""
import copy

import pytest
import torch

from tests import net_ref as N
from tests.helpers import engine_from_oracle, oracle_models, record, rel_err, weight_bytes

pytestmark = pytest.mark.gpu

GIB = 1 << 30


# ---- models -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sd2():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    unet, vae, text = oracle_models("full")
    N.randomise(unet, vae, seed=5)
    eng = engine_from_oracle(unet, vae, text)
    dev = torch.device("cuda")
    ref = {"unet": unet.to(dev), "vae": vae.to(dev), "text": text.to(dev)}
    yard = {"unet": copy.deepcopy(ref["unet"]).to(torch.bfloat16), "vae": copy.deepcopy(ref["vae"]).to(torch.bfloat16),
            "text": ref["text"].to(torch.bfloat16)}
    yield eng, ref, yard
    eng.close()


def _iid_engine(n_targets=3, seed=6):
    """A full-width engine for the 3-target intrinsic-image models: in 16, out 12 channels. The tests that use it run
    first and close it: its workspace and the depth engine's largest one (55 GiB at NB = 16, 768 x 768) do not both fit
    an 80 GB card beside the torch references."""
    from marigold_b200.engine import Engine, EngineConfig
    from oracle.unet import UNet2DConditionOracle, UNetConfig
    from oracle.vae import AutoencoderKLOracle, VAEConfig

    torch.manual_seed(seed)
    ucfg = UNetConfig()
    ucfg.in_channels, ucfg.out_channels = 4 * (n_targets + 1), 4 * n_targets
    unet, vae = UNet2DConditionOracle(ucfg).eval(), AutoencoderKLOracle(VAEConfig()).eval()
    N.randomise(unet, vae, seed=seed)
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=torch.Generator().manual_seed(7))
    eng = Engine(EngineConfig(unet_in_channels=ucfg.in_channels, unet_out_channels=ucfg.out_channels))
    eng.load_state_dict("unet", unet.state_dict())
    eng.load_state_dict("vae", vae.state_dict())
    eng.finalize()
    eng.set_text_embedding(text)
    return eng


def _sched(eng, kind="ddim", n=4):
    from marigold_b200.schedulers import DDIMScheduler, LCMScheduler

    s = DDIMScheduler() if kind == "ddim" else LCMScheduler()
    s.set_timesteps(n)
    eng.set_schedule(s.timesteps, *s.coefficients())
    return s


def _randn(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).cuda()


# ---- runs: each takes its inputs (member dimension given per input) and returns a tuple of outputs, member first -------
def _step_run(eng, step):
    def run(rgb, x):
        tgt = x.clone()
        mo = eng.unet_step(rgb, tgt, step, want_model_out=True)
        return mo, tgt
    return run


def _denoise_run(eng):
    return lambda rgb, x0, zs=None: (eng.denoise(rgb, x0, zs),)


def _decode_run(eng, mode):
    return lambda lat: (eng.decode(lat, mode),)


def _call(run, inputs):
    out = run(*[t for t, _ in inputs])
    torch.cuda.synchronize()
    return out


def _member(t, dim, j):
    return t.narrow(dim, j, 1).contiguous()


# ---- exact properties -------------------------------------------------------------------------------------------------
def check_independence(run, inputs, base, seed=100):
    """Replace all of member j's inputs (j = 0, NB // 2, NB - 1): every other member's outputs keep their bits, and
    member j's change."""
    NB = base[0].shape[0]
    for j in sorted({0, NB // 2, NB - 1}):
        new = []
        for k, (t, dim) in enumerate(inputs):
            t = t.clone()
            sl = t.narrow(dim, j, 1)
            sl.copy_(_randn(seed + 17 * j + k, *sl.shape))
            new.append((t, dim))
        out = _call(run, new)
        keep = torch.arange(NB, device="cuda") != j
        for o, b in zip(out, base):
            assert torch.equal(o[keep], b[keep]), f"replacing member {j} of {NB} changed another member's output"
            assert not torch.equal(o[j], b[j]), f"member {j}'s new inputs left its output unchanged"


def check_permutation(run, inputs, base):
    """Reversed and rotated members give the same permutation of the outputs, bit for bit."""
    NB = base[0].shape[0]
    for name, perm in (("reversed", torch.arange(NB - 1, -1, -1)), ("rotated", torch.roll(torch.arange(NB), -1))):
        perm = perm.cuda()
        out = _call(run, [(t.index_select(dim, perm).contiguous(), dim) for t, dim in inputs])
        for o, b in zip(out, base):
            assert torch.equal(o, b.index_select(0, perm)), f"{name} members: outputs are not the permuted outputs"


# ---- bounded: batched member vs the same member alone -------------------------------------------------------------------
def check_against_alone(name, run, inputs, base, stages, masks=None):
    """|batched_j - alone_j| <= TAU[stage] rms(alone_j) for every member j and output; records the largest ratio per
    output (in units of TAU rms). masks[k](j, alone) -> (bool mask of the elements compared, weight of |batched - alone|
    or None), or masks[k] None: every element, unweighted."""
    NB = base[0].shape[0]
    worst = [0.0] * len(base)
    for j in range(NB):
        alone = _call(run, [(_member(t, dim, j), dim) for t, dim in inputs])
        for k, (b, a) in enumerate(zip(base, alone)):
            d = (b[j:j + 1].double() - a.double()).abs().nan_to_num(float("inf"))
            if masks and masks[k]:
                m, w = masks[k](j, a)
                record(f"batch/{name}/out{k}_{stages[k]}/masked_unweighted_over_tau",
                       float(d[m].max()) / N.rms(a) / N.TAU[stages[k]])
                d = d[m] if w is None else (d * w)[m]
            worst[k] = max(worst[k], float(d.max()) / N.rms(a))
    fails = []
    for k, stage in enumerate(stages):
        record(f"batch/{name}/out{k}_{stage}/alone_over_tau", worst[k] / N.TAU[stage])
        if not worst[k] <= N.TAU[stage]:
            fails.append(f"{name} output {k} ({stage}): max |batched - alone| / rms = {worst[k]:.3g} > {N.TAU[stage]}")
    assert not fails, "\n".join(fails)


def check_yardstick(name, ours, r, y):
    """test_fullsize_gpu's criterion: err(ours vs fp32 oracle) <= 1.05 err(torch bf16 vs fp32 oracle) + 1e-3."""
    e_ours, e_yard = rel_err(ours, r), rel_err(y, r)
    record(f"batch/{name}/ours_vs_fp32", e_ours)
    record(f"batch/{name}/torch_bf16_vs_fp32", e_yard)
    assert torch.isfinite(ours).all()
    assert e_ours <= e_yard * 1.05 + 1e-3, f"{name}: ours {e_ours:.3e} vs torch-bf16 {e_yard:.3e}"


def _depth(dec):
    return (dec.mean(1, keepdim=True).clip(-1, 1) + 1) / 2


@torch.no_grad()
def yardstick_decode(name, ref, yard, lat, dep):
    """Depth decode of one member (lat [1, 4, h, w]) by the fp32 oracle and by torch bf16."""
    r = _depth(ref["vae"].decoder(ref["vae"].post_quant_conv(lat / 0.18215)))
    y = _depth(yard["vae"].decoder(yard["vae"].post_quant_conv((lat / 0.18215).to(torch.bfloat16))).float())
    check_yardstick(name, dep, r, y)


def _normals_mask(eng, lats):
    """test_net_faithful_gpu's normals mask: compare where the clipped raw vector c is not short (|c| > 0.3). The unit
    normalisation c / |c| turns an error dc into at most |dc| / |c|, so the head's difference is weighted by |c| (of the
    member decoded alone): the weighted difference is in the units of the raw decode, which the bound is for. The raw
    decode itself is checked unweighted beside it."""
    def mask(j, alone):
        raw = eng.decode(_member(lats, 0, j), N.DECODE_RAW)
        c = torch.norm(raw.clip(-1, 1), dim=1, keepdim=True).double()
        return (c > 0.3).expand_as(alone), c.expand_as(alone)
    return mask


# ---- cases (the two that build the IID engine first) ----------------------------------------------------------------
def test_iid_3_targets_nb6():
    """NB = 6 at 54 x 96 on a full-width in 16 / out 12 UNet: one step, then the mode-3 decode of each target."""
    eng = _iid_engine()
    try:
        _sched(eng)
        NB = 6
        sin = [(_randn(18, NB, 4, 54, 96), 0), (_randn(19, NB, 12, 54, 96), 0)]
        srun = _step_run(eng, 1)
        sbase = _call(srun, sin)
        assert all(torch.isfinite(b).all() for b in sbase)
        check_permutation(srun, sin, sbase)
        check_independence(srun, sin, sbase)
        check_against_alone("iid3_54x96_nb6_step", srun, sin, sbase, ("unet", "latent"))
        drun = _decode_run(eng, N.DECODE_UNIT3)
        for k in range(3):
            din = [(sbase[1][:, 4 * k:4 * k + 4].contiguous(), 0)]
            dbase = _call(drun, din)
            check_independence(drun, din, dbase)
            check_against_alone(f"iid3_432x768_nb6_decode_target{k}", drun, din, dbase, ("decode",))
    finally:
        eng.close()


# ---- memory -------------------------------------------------------------------------------------------------------------


# 80 GB card; 6 GiB are left for the CUDA context, the caller's tensors (inputs, outputs, the ensemble) and fragmentation
CARD_BYTES, HEADROOM = 80 * 10 ** 9, 6 * GIB


def test_workspace_fits_at_the_batch_caps(sd2):
    """mgb_workspace_bytes (a host dry run: nothing is allocated) at the batch find_batch_size allows, for the depth /
    normals engine and the 3-target IID engine, at every processing shape the pipelines use."""
    from marigold_b200.pipeline import find_batch_size

    fails = []
    iid3 = _iid_engine()
    for name, e in (("depth", sd2[0]), ("iid3", iid3)):
        wb = weight_bytes(e)
        record(f"batch/workspace/{name}/weights_gib", wb / GIB)
        for H, W in ((768, 768), (432, 768), (768, 432), (1024, 1024), (576, 1024), (1024, 576)):
            B = find_batch_size(64, max(H, W), torch.float32)
            need = e.workspace_bytes(B, H, W)
            record(f"batch/workspace/{name}/{H}x{W}_nb{B}_gib", need / GIB)
            if need == 0 or need + wb + HEADROOM > CARD_BYTES:
                fails.append(f"{name} {H}x{W} NB={B}: workspace {need / GIB:.2f} GiB + weights {wb / GIB:.2f} GiB "
                             f"+ {HEADROOM / GIB:.0f} GiB headroom > {CARD_BYTES / GIB:.1f} GiB")
    iid3.close()
    assert not fails, "\n".join(fails)


# ---- cases on the depth / normals engine --------------------------------------------------------------------------------
def test_depth_768_nb16_step(sd2):
    """NB = 16 at 96 x 96: one DDIM step, independence, every member vs alone, members 0 and 15 vs the fp32 oracle."""
    eng, ref, yard = sd2
    s = _sched(eng)
    NB, step = 16, 1
    inputs = [(_randn(1, NB, 4, 96, 96), 0), (_randn(2, NB, 4, 96, 96), 0)]
    run = _step_run(eng, step)
    base = _call(run, inputs)
    assert all(torch.isfinite(b).all() for b in base)
    check_independence(run, inputs, base)
    check_against_alone("768_nb16_step", run, inputs, base, ("unet", "latent"))
    t = int(s.timesteps[step])
    for j in (0, NB - 1):
        with torch.no_grad():
            inp = torch.cat([inputs[0][0][j:j + 1], inputs[1][0][j:j + 1]], 1)
            r = ref["unet"](inp, t, ref["text"])
            y = yard["unet"](inp.to(torch.bfloat16), t, yard["text"]).float()
        check_yardstick(f"768_nb16_step/m{j}", base[0][j:j + 1], r, y)


def test_depth_768_nb16_denoise(sd2):
    """NB = 16 at 96 x 96: 4 DDIM steps through mgb_denoise (eager first step, then graph replays)."""
    eng, ref, yard = sd2
    _sched(eng)
    NB = 16
    inputs = [(_randn(3, NB, 4, 96, 96), 0), (_randn(4, NB, 4, 96, 96), 0)]
    run = _denoise_run(eng)
    base = _call(run, inputs)
    assert torch.isfinite(base[0]).all()
    check_independence(run, inputs, base)
    check_against_alone("768_nb16_denoise", run, inputs, base, ("trajectory",))


def test_depth_768_nb16_decode(sd2):
    """NB = 16 at 768 x 768, depth head: the largest decode the pipelines launch."""
    eng, ref, yard = sd2
    NB = 16
    need = eng.workspace_bytes(NB, 768, 768)
    out_bytes = NB * 768 * 768 * 4 * 2
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if need + out_bytes + 2 * GIB > free:
        pytest.skip(f"NB = 16 768 x 768 decode needs {need / GIB:.1f} GiB of workspace; {free / GIB:.1f} of "
                    f"{total / GIB:.1f} GiB free on this card")
    record("batch/768_nb16_decode/workspace_gib", need / GIB)
    lats = _randn(5, NB, 4, 96, 96)
    inputs = [(lats, 0)]
    run = _decode_run(eng, N.DECODE_DEPTH)
    base = _call(run, inputs)
    assert torch.isfinite(base[0]).all()
    check_independence(run, inputs, base)
    check_against_alone("768_nb16_decode_depth", run, inputs, base, ("decode",))
    for j in (0, NB - 1):
        yardstick_decode(f"768_nb16_decode/m{j}", ref, yard, lats[j:j + 1], base[0][j:j + 1])


def test_normals_nb10(sd2):
    """c4: NB = 10 at 96 x 96, normals head; permutation of the step and of the decode."""
    eng, ref, yard = sd2
    _sched(eng)
    NB = 10
    sin = [(_randn(6, NB, 4, 96, 96), 0), (_randn(7, NB, 4, 96, 96), 0)]
    srun = _step_run(eng, 2)
    sbase = _call(srun, sin)
    check_permutation(srun, sin, sbase)
    check_independence(srun, sin, sbase)
    check_against_alone("96_nb10_step", srun, sin, sbase, ("unet", "latent"))
    lats = _randn(8, NB, 4, 96, 96)
    din = [(lats, 0)]
    drun = _decode_run(eng, N.DECODE_NORMALS)
    dbase = _call(drun, din)
    assert torch.allclose(torch.norm(dbase[0], dim=1), torch.ones_like(dbase[0][:, 0]), atol=1e-4)
    check_permutation(drun, din, dbase)
    check_independence(drun, din, dbase)
    check_against_alone("768_nb10_decode_normals", drun, din, dbase, ("decode",), masks=[_normals_mask(eng, lats)])
    rrun = _decode_run(eng, N.DECODE_RAW)
    check_against_alone("768_nb10_decode_raw", rrun, din, _call(rrun, din), ("decode",))


def test_lcm_nb8_denoise(sd2):
    """c3: NB = 8 at 96 x 96, 4 LCM steps with step noise (the noise slice of member i is step_noise[s, i])."""
    eng, ref, yard = sd2
    _sched(eng, "lcm")
    NB, n = 8, 4
    inputs = [(_randn(9, NB, 4, 96, 96), 0), (_randn(10, NB, 4, 96, 96), 0), (_randn(11, n - 1, NB, 4, 96, 96), 1)]
    run = _denoise_run(eng)
    base = _call(run, inputs)
    assert torch.isfinite(base[0]).all()
    check_independence(run, inputs, base)
    check_permutation(run, inputs, base)
    check_against_alone("96_nb8_lcm_denoise", run, inputs, base, ("trajectory",))


def test_1024_graph_rekeying(sd2):
    """c5: denoise at NB = 8, then 2, then 8 (the step graph is captured again at each key); each call equals the same
    steps driven through unet_step at that NB, and the last equals the first."""
    eng, ref, yard = sd2
    s = _sched(eng)
    rgb, x0 = _randn(12, 10, 4, 128, 128), _randn(13, 10, 4, 128, 128)
    parts = [slice(0, 8), slice(8, 10), slice(0, 8)]
    outs = []
    for sl in parts:
        out = eng.denoise(rgb[sl], x0[sl])
        x = x0[sl].clone()
        for i in range(len(s.timesteps)):
            eng.unet_step(rgb[sl].contiguous(), x, i)
        torch.cuda.synchronize()
        assert torch.equal(out, x), f"denoise at NB = {sl.stop - sl.start} differs from its steps run one at a time"
        outs.append(out)
    assert torch.equal(outs[2], outs[0]), "denoise at NB = 8 changed after a call at NB = 2"
    inputs = [(rgb[:8].contiguous(), 0), (x0[:8].contiguous(), 0)]
    base = (outs[0],)
    check_independence(_denoise_run(eng), inputs, base)
    check_against_alone("128_nb8_denoise", _denoise_run(eng), inputs, base, ("trajectory",))
    # members 0 and 7 against the fp32 oracle's trajectory, within torch bf16's
    from oracle.schedulers import DDIMSchedulerOracle

    for j in (0, 7):
        xr, xy = x0[j:j + 1].clone(), x0[j:j + 1].clone()
        for m, xs in ((ref, xr), (yard, xy)):
            o = DDIMSchedulerOracle()
            o.set_timesteps(len(s.timesteps))
            dt = torch.float32 if m is ref else torch.bfloat16
            with torch.no_grad():
                for t in o.timesteps:
                    v = m["unet"](torch.cat([rgb[j:j + 1], xs], 1).to(dt), int(t), m["text"]).float()
                    xs.copy_(o.step(v, int(t), xs))
        check_yardstick(f"1024_nb8_denoise/m{j}", outs[0][j:j + 1], xr, xy)
    # depth decode of the 8 + 2 split
    lats = _randn(14, 10, 4, 128, 128)
    run = _decode_run(eng, N.DECODE_DEPTH)
    for sl in parts[:2]:
        inp = [(lats[sl].contiguous(), 0)]
        dbase = _call(run, inp)
        check_independence(run, inp, dbase)
        check_against_alone(f"1024_nb{sl.stop - sl.start}_decode_depth", run, inp, dbase, ("decode",))
        if sl.start == 0:
            for j in (0, 7):
                yardstick_decode(f"1024_nb8_decode/m{j}", ref, yard, lats[j:j + 1], dbase[0][j:j + 1])


def test_169_nb5(sd2):
    """NB = 5 at 54 x 96 (432 x 768): 5184 tokens = 40.5 tiles of 128, so token-GEMM tiles straddle members, and the
    levels are odd (27 x 48, 14 x 24, 7 x 12)."""
    eng, ref, yard = sd2
    _sched(eng)
    NB = 5
    sin = [(_randn(15, NB, 4, 54, 96), 0), (_randn(16, NB, 4, 54, 96), 0)]
    srun = _step_run(eng, 1)
    sbase = _call(srun, sin)
    check_permutation(srun, sin, sbase)
    check_independence(srun, sin, sbase)
    check_against_alone("54x96_nb5_step", srun, sin, sbase, ("unet", "latent"))
    din = [(_randn(17, NB, 4, 54, 96), 0)]
    drun = _decode_run(eng, N.DECODE_DEPTH)
    dbase = _call(drun, din)
    check_permutation(drun, din, dbase)
    check_independence(drun, din, dbase)
    check_against_alone("432x768_nb5_decode_depth", drun, din, dbase, ("decode",))
