"""CPU checks of the float64 network restatement (tests/net_ref.py) that the GPU graph tests compare against.

1. Without its bf16 roundings the restatement is the diffusers graph: it matches the fp32 oracle to fp32 precision on
   randomised weights, which shows that the folds (ffpo, the collapsed cross attention, the encoder's conv_out .
   quant_conv, the per-step bias table) are exact algebra.
2. Power: on the randomised tiny model, each parameter tensor is mutated: a norm affine reset, any other tensor zeroed,
   or swapped with a same-shaped sibling of its block. Its algebraic effect (restatement without rounding, on both
   sides) is scored in the GPU tests' metric, max |d| / rms(ref), in units of that stage's GPU tolerance tau. The test
   prints the weakest ten and how many clear 2 tau and 10 tau, and requires 2 tau of every encoder and decoder mutation
   outside a listed few, and of the UNet's stem and head. Most mutations inside the UNet body stay below 2 tau: the
   GPU tests do not show those.
"""
import re

import pytest
import torch

from tests import net_ref as N
from tests.helpers import oracle_models

# max |restatement - oracle| / rms(oracle) with bf16=False; measured <= 3.4e-6 (UNet), 2.8e-6 (encode),
# 4e-6 (decode): the fp32 rounding of the oracle itself
EXACT_TOL = 2e-5


@pytest.fixture(scope="module")
def tiny():
    unet, vae, text = oracle_models("tiny")
    N.randomise(unet, vae, seed=1)
    return unet, vae, text


def _ddim(n):
    from marigold_b200.schedulers import DDIMScheduler

    s = DDIMScheduler()
    s.set_timesteps(n)
    return s


def _unet_vs_oracle(unet, text, B, lh, lw):
    s = _ddim(4)
    kx, kv, _ = s.coefficients()
    g = torch.Generator().manual_seed(11)
    rgb = torch.randn(B, 4, lh, lw, generator=g)
    x = torch.randn(B, unet.cfg.out_channels, lh, lw, generator=g)
    for step in (0, 2):
        t = int(s.timesteps[step])
        with torch.no_grad():
            ora = unet(torch.cat([rgb, x], 1), t, text.repeat(B, 1, 1))
        mo, xn = N.unet_step(unet, text, rgb, x, t, kx[step], kv[step], bf16=False)
        e = N.rms_err(mo, ora)
        assert e < EXACT_TOL, f"step {step}: {e:.3g}"
        assert N.rms_err(xn, float(kx[step]) * x.double() + float(kv[step]) * ora.double()) < EXACT_TOL
        # the rounding switch is live: with bf16 the gap to fp32 is the bf16 operand noise
        mb, _ = N.unet_step(unet, text, rgb, x, t, kx[step], kv[step], bf16=True)
        assert 1e-3 < N.rms_err(mb, ora) < 1e-1


@pytest.mark.parametrize("B,lh,lw", [(1, 16, 16), (2, 8, 24), (1, 27, 12), (2, 7, 9)])
def test_unet_restatement_is_the_oracle_graph(tiny, B, lh, lw):
    unet, vae, text = tiny
    _unet_vs_oracle(unet, text, B, lh, lw)


@pytest.mark.parametrize("n_targets", [2, 3])
def test_unet_restatement_iid_is_the_oracle_graph(n_targets):
    from oracle.unet import UNet2DConditionOracle, UNetConfig
    from oracle.vae import AutoencoderKLOracle, VAEConfig

    torch.manual_seed(0)
    ucfg = UNetConfig.tiny()
    ucfg.in_channels, ucfg.out_channels = 4 * (n_targets + 1), 4 * n_targets
    unet, vae = UNet2DConditionOracle(ucfg).eval(), AutoencoderKLOracle(VAEConfig.tiny()).eval()
    text = torch.randn(1, 2, ucfg.cross_attention_dim, generator=torch.Generator().manual_seed(7))
    N.randomise(unet, vae, seed=2)
    _unet_vs_oracle(unet, text, 1, 16, 12)


@pytest.mark.parametrize("B,H,W", [(2, 64, 128), (1, 100, 50), (1, 77, 131)])
def test_encode_restatement_is_the_oracle_graph(tiny, B, H, W):
    unet, vae, text = tiny
    rgb = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(12)) * 2 - 1
    with torch.no_grad():
        ora = vae.quant_conv(vae.encoder(rgb))[:, :4] * 0.18215
    assert N.rms_err(N.encode(vae, rgb, bf16=False), ora) < EXACT_TOL
    assert 1e-3 < N.rms_err(N.encode(vae, rgb), ora) < 1e-1


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_decode_restatement_is_the_oracle_graph(tiny, mode):
    unet, vae, text = tiny
    lat = torch.randn(2, 4, 9, 13, generator=torch.Generator().manual_seed(13))
    with torch.no_grad():
        raw = vae.decoder(vae.post_quant_conv(lat / 0.18215)).double()
    ora = N.decode_head(raw, mode)
    out = N.decode(vae, lat, mode, bf16=False)
    if mode == N.DECODE_NORMALS:
        # unit vectors: compare where the clipped raw vector is not short (its direction is well conditioned)
        m = (torch.norm(raw.clip(-1, 1), dim=1, keepdim=True) > 0.3).expand_as(ora)
        out, ora = out[m], ora[m]
    assert N.rms_err(out, ora) < EXACT_TOL
    if mode == N.DECODE_RAW:
        assert 1e-3 < N.rms_err(N.decode(vae, lat, mode), ora) < 1e-1


# ---- power -------------------------------------------------------------------------------------------------------
_NORM = re.compile(r"(^|\.)(norm\d?|group_norm|conv_norm_out)\.(weight|bias)$")
# same-shaped siblings within a block: (pattern, replacement) on the key
_SIBLINGS = [(".norm1.", ".norm2."), (".norm3.", ".norm2."), (".conv1.", ".conv2."), (".to_q.", ".to_k."),
             (".to_k.", ".to_v."), (".attn1.to_out.", ".attn2.to_out."), (".attn1.to_q.", ".attn2.to_q."),
             (".proj_in.", ".proj_out.")]


# The VAE attention's key bias adds q . b_k to every logit of a row: softmax removes it, so no output can see it.
_INVISIBLE = re.compile(r"attentions\.0\.to_k\.bias$")


def _mutations(sd):
    """(label, mutated state dict) for every parameter tensor: norms reset to gamma = 1 / beta = 0, everything else
    zeroed; plus a swap with each same-shaped sibling of the block."""
    for k, v in sd.items():
        if _INVISIBLE.search(k):
            continue
        if _NORM.search(k):
            ident = torch.ones_like(v) if k.endswith(".weight") else torch.zeros_like(v)
            yield f"{k} = {'1' if k.endswith('.weight') else '0'}", {**sd, k: ident}
        else:
            yield f"{k} = 0", {**sd, k: torch.zeros_like(v)}
        for a, b in _SIBLINGS:
            if a in k:
                k2 = k.replace(a, b)
                if k2 in sd and sd[k2].shape == v.shape:
                    yield f"{k} <-> {k2}", {**sd, k: sd[k2], k2: v}


def _power(stage, unet, vae, text):
    """max |mutated - ref| / rms(ref) / tau for every mutation of the stage's parameters, weakest first. Both sides are
    the restatement without rounding: its algebraic effect. (With bf16 roundings any change of any value, however small,
    flips roundings that cascade through the network and would score at the rounding-noise level.)"""
    g = torch.Generator().manual_seed(21)
    if stage == "unet":
        s = _ddim(4)
        kx, kv, _ = s.coefficients()
        rgb, x = torch.randn(1, 4, 16, 16, generator=g), torch.randn(1, 4, 16, 16, generator=g)
        t = int(s.timesteps[2])

        def run(sd):
            return N.unet_step(unet, text, rgb, x, t, kx[2], kv[2], bf16=False, sd=sd)[0]
        sd = unet.state_dict()
    elif stage == "encode":
        rgb = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1

        def run(sd):
            return N.encode(vae, rgb, bf16=False, sd=sd)
        sd = {k: v for k, v in vae.state_dict().items() if k.startswith(("encoder.", "quant_conv."))}
    else:
        lat = torch.randn(1, 4, 8, 8, generator=g)

        def run(sd):
            return N.decode(vae, lat, N.DECODE_RAW, bf16=False, sd=sd)
        sd = {k: v for k, v in vae.state_dict().items() if k.startswith(("decoder.", "post_quant_conv."))}
    ref = run(sd)
    res = sorted((N.rms_err(run(m), ref) / N.TAU[stage], label) for label, m in _mutations(sd))
    return res, len(sd)


# A mutation is caught on the GPU only if its effect exceeds tau plus the GPU's own noise (about tau / 1.5), so the test
# asks for 2 tau. Mutations that stay below it on the input used here, with the reason:
_WEAK = {
    "encode": (r"^encoder\.mid_block\.attentions\.0\.to_[qk]\.",
               "the default-init q / k projections give logits of std ~0.3: the softmax is near uniform and q, k enter "
               "only at second order"),
    "decode": (r"^decoder\.mid_block\.attentions\.0\.(to_[qk]\.|group_norm\.)|^post_quant_conv\.bias",
               "as for the encoder (q, k and the GroupNorm before them), and post_quant_conv.bias moves this one 8 x 8 "
               "latent by 1.8 tau"),
}
# In the UNet only the stem and head reach 2 tau: every block between them is diluted by the default-init 1x1 shortcut
# convs of the up path (gain ~1 / sqrt(3) each) and most of its mutations stay below 2 tau (DESIGN.md section 4).
_UNET_ASSERTED = r"^(conv_in|conv_out|conv_norm_out|time_embedding)\."


@pytest.mark.parametrize("stage", ["unet", "encode", "decode"])
def test_every_parameter_moves_the_output(tiny, stage):
    unet, vae, text = tiny
    res, n = _power(stage, unet, vae, text)
    strong = sum(r >= 10.0 for r, _ in res)
    below = sum(r < 2.0 for r, _ in res)
    print(f"\n{stage}: {len(res)} mutations of {n} tensors; {strong} move the output by >= 10 tau, {below} by < 2 tau "
          f"(tau = {N.TAU[stage]:.3g}); weakest ten, in units of tau:")
    for r, label in res[:10]:
        print(f"  {r:10.4f}  {label}")
    if stage == "unet":
        checked = [(r, lb) for r, lb in res if re.search(_UNET_ASSERTED, lb)]
    else:
        checked = [(r, lb) for r, lb in res if not re.search(_WEAK[stage][0], lb)]
    assert checked and checked[0][0] >= 2.0, f"{stage}: {checked[0][1]} moves the output by only {checked[0][0]:.3g} tau"
