"""Float64 restatement of the product's network graphs (net.cu / api_net.cu) with the product's rounding points.

`unet_step`, `encode` and `decode` read the weights of the oracle models (oracle/unet.py, oracle/vae.py) from their
state dicts, apply the folds the library applies when it loads them, and round to bf16 exactly where the kernels do:

  weights   every GEMM / conv weight is bf16 (conv_in zero-padded to 64 input channels: zeros change nothing);
            ffpo = [bf16(W_po) | bf16(fp32 W_po W_ff2)], bias b_po + W_po b_ff2 (double);
            encoder conv_out . quant_conv: weight summed on the host in fp32 (w += q cw, j = 0..7), then bf16;
            bias float(double(qb + q cb) scale); the epilogue computes acc scale + bias;
            cross-attention tables G, U: bf16 of their fold; c1, the text K / V, the time MLP and the per-step bias
            table conv1.bias + time_emb_proj(silu(temb)): unrounded.
  resnet    t1 = bf16(silu(GN1([h | skip]))); the 1x1 shortcut reads bf16([h | skip]); h = conv1(t1) + bias (fp32);
            t2 = bf16(silu(GN2(h))); y = conv2(t2) + W_sc raw + (b2 + b_sc) + x, the residual x unrounded.
  xfmr      a = bf16(GN(x)) (eps 1e-6); hs0 = proj_in(a); qkv = bf16(bf16(LN1(hs0)) W_qkv);
            flash attention: P = bf16(exp(s - m_j)), m_j the running maximum over 64-key blocks within the KV split,
            o = bf16(.); hs1 = o W_o1 + b + hs0;
            cross attention (collapsed): z = LN2(hs1); acc = hs1 + c1 + sum_h sigmoid(0.125 z . G_h) U_h;
            hsb = bf16(acc); a = bf16(LN3(acc)); ffm = bf16(GEGLU(a)); y = [hsb | ffm] ffpo^T + bias + x.
  levels    space-to-depth and nearest x2 (2s or 2s - 1) read bf16 copies of the trunk; conv_in reads
            bf16([rgb | target]); conv_out fuses the scheduler: x' = kx x + kv (acc + b) + kz z.
  VAE       the encoder input is bf16(rgb); attention q, k, v = bf16(.), S unrounded, P = bf16(softmax(S)),
            o = bf16(P v); the decoder input is bf16(post_quant_conv(latent * fp32(1 / scale)));
            decode heads: depth (channel mean, clip, (d + 1) / 2), normals (clip, unit length), unit ((clip + 1) / 2), raw.

The folds themselves (ffpo, G / U / c1, the time MLP and the per-step bias, the encoder fold) are the functions of
tests/weights_ref.py, which holds the device's own tables to them.

Everything else is float64. With `bf16=False` no value is rounded and the folds are exact, so the result is the
diffusers graph algebra (tests/test_net_ref.py checks it against the fp32 oracle).

`randomise` redraws every norm affine and every conv / linear bias of the seeded oracle models, so that a wiring error
in any of them changes the output (the default init has gamma = 1, beta = 0 and biases of ~1 / sqrt(fan_in)).

Tolerances of the GPU comparison (tests/test_net_faithful_gpu.py), per stage: |ours - ref| <= TAU[stage] * rms(ref)
element-wise. See DESIGN.md section 4 for how they were measured.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests import weights_ref as WR

LATENT_SCALE = float(np.float32(0.18215))           # mgb_config.latent_scale (fp32)
INV_LATENT_SCALE = float(np.float32(1.0) / np.float32(0.18215))
GROUPS = 32
NUM_SMS = 132                                        # kNumSMs: the KV split of the flash attention depends on it

# Per-element bound of the GPU comparison, in units of rms(ref): about 1.5x the largest max |ours - ref| / rms(ref)
# measured per stage on an H100 80GB HBM3 at a 400 W power limit (UNet model output 1.9e-2, encode 1.3e-2, decode
# 5.1e-2 (normals, where the raw vector is not short), 4-step trajectories 9.5e-3). The updated latent carries
# kv times the model output's error and is dominated by kx x. DESIGN.md section 4.
TAU = {"unet": 3e-2, "latent": 1e-2, "encode": 2e-2, "decode": 7.5e-2, "trajectory": 1.5e-2}


# ---- test weights ---------------------------------------------------------------------------------------------------
def randomise(unet, vae, seed: int = 0, bias_std: float = 0.25):
    """Redraw, in place and distinct per tensor, every GroupNorm / LayerNorm gamma ~ U(0.5, 1.5) and beta ~ N(0, 0.3),
    and every conv / linear bias ~ N(0, bias_std). Weights keep their (seeded default) init. Returns (unet, vae)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for model in (unet, vae):
            for _, m in model.named_modules():
                if isinstance(m, (nn.GroupNorm, nn.LayerNorm)):
                    m.weight.uniform_(0.5, 1.5, generator=g)
                    m.bias.normal_(0.0, 0.3, generator=g)
                elif isinstance(m, (nn.Conv2d, nn.Linear)) and m.bias is not None:
                    m.bias.normal_(0.0, bias_std, generator=g)
    return unet, vae


# ---- rounding context -----------------------------------------------------------------------------------------------
class _Ctx:
    def __init__(self, sd, bf16: bool):
        self.sd, self.bf16 = sd, bf16

    def has(self, k):
        return k in self.sd

    def p(self, k):
        """fp32 parameter, unrounded (biases, norm affines, folded-table inputs)."""
        return self.sd[k].detach().to(torch.float64)

    def w(self, k):
        """GEMM / conv weight: bf16."""
        return self.r(self.sd[k].detach().float())

    def r(self, x):
        """bf16 rounding of an fp32 value (identity without bf16)."""
        if not self.bf16:
            return x.to(torch.float64)
        return x.float().to(torch.bfloat16).to(torch.float64)


def _gn(c, x, p, eps):
    return F.group_norm(x, GROUPS, c.p(p + ".weight"), c.p(p + ".bias"), eps)


def _ln(c, x, p, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), c.p(p + ".weight"), c.p(p + ".bias"), eps)


def _conv(c, x, p, stride=1, padding=1, bias=True):
    y = F.conv2d(x, c.w(p + ".weight"), stride=stride, padding=padding)
    return y + c.p(p + ".bias")[None, :, None, None] if bias else y


def _lin(c, x, p, bias=True):
    y = x @ c.w(p + ".weight").t()
    return y + c.p(p + ".bias") if bias else y


def _gelu(t):
    return 0.5 * t * (1.0 + torch.erf(t / math.sqrt(2.0)))


def _tokens(x):
    B, C, H, W = x.shape
    return x.permute(0, 2, 3, 1).reshape(B, H * W, C)


def _image(t, H, W):
    B, _, C = t.shape
    return t.reshape(B, H, W, C).permute(0, 3, 1, 2)


# ---- blocks -----------------------------------------------------------------------------------------------------------
def _resnet(c, p, x, skip, bias1, eps):
    inp = x if skip is None else torch.cat([x, skip], 1)
    t1 = c.r(F.silu(_gn(c, inp, p + ".norm1", eps)))
    h = _conv(c, t1, p + ".conv1", bias=False) + bias1[None, :, None, None]
    t2 = c.r(F.silu(_gn(c, h, p + ".norm2", eps)))
    y = _conv(c, t2, p + ".conv2")
    if c.has(p + ".conv_shortcut.weight"):
        return y + _conv(c, c.r(inp), p + ".conv_shortcut", padding=0)
    return y + x


def attn_splits(NB, T, C):
    """flash_attn64_splits (attn_tc.cu): the KV split of the flash attention."""
    units, nkv, slots = ((T + 127) // 128) * (C // 64) * NB, (T + 63) // 64, NUM_SMS * 2
    best, best_t = 1, 1e30
    for s in range(1, 9):
        if s > 1 and nkv // s < 6:
            break
        t = ((units * s + slots - 1) // slots) * (nkv / s + 15.0) + (8.0 if s > 1 else 0.0)
        if t < best_t - 1e-9:
            best_t, best = t, s
    return best


def _flash(c, q, k, v):
    """Self attention, head dim 64, scale 1/8. q, k, v [B, T, C] (bf16 values). With bf16 the probabilities fed to the
    P V MMA are bf16(exp(s - m_j)), m_j the running row maximum after KV block j within its split."""
    B, T, C = q.shape
    H = C // 64
    q, k, v = (t.reshape(B, T, H, 64).transpose(1, 2) for t in (q, k, v))
    s = (q @ k.transpose(-1, -2)) * 0.125
    if not c.bf16:
        o = torch.softmax(s, -1) @ v
    else:
        nkv = (T + 63) // 64
        sp = F.pad(s, (0, nkv * 64 - T), value=-math.inf).reshape(B, H, T, nkv, 64).amax(-1)
        splits = attn_splits(B, T, C)
        run = sp.clone()
        for si in range(splits):
            j0, j1 = si * nkv // splits, (si + 1) * nkv // splits
            run[..., j0:j1] = torch.cummax(sp[..., j0:j1], -1).values
        mk = run.repeat_interleave(64, -1)[..., :T]
        e = torch.exp(s - mk)
        w = torch.exp(mk - s.amax(-1, keepdim=True))
        o = ((c.r(e) * w) @ v) / (e * w).sum(-1, keepdim=True)
    return o.transpose(1, 2).reshape(B, T, C)


def _xfmr(c, p, x, ctx):
    B, C, H, W = x.shape
    a = c.r(_tokens(_gn(c, x, p + ".norm", 1e-6)))
    hs0 = _lin(c, a, p + ".proj_in")
    t = p + ".transformer_blocks.0"
    l1 = c.r(_ln(c, hs0, t + ".norm1"))
    q, k, v = (c.r(_lin(c, l1, f"{t}.attn1.to_{n}", bias=False)) for n in "qkv")
    o = c.r(_flash(c, q, k, v))
    hs1 = _lin(c, o, t + ".attn1.to_out.0") + hs0
    # cross attention against the two-token context, collapsed: G_h = Wq[h]^T (k0 - k1)_h, U_h = Wo[:, h] (v0 - v1)_h,
    # c1 = Wo v1 + bo
    kk, vv = ctx @ c.p(t + ".attn2.to_k.weight").t(), ctx @ c.p(t + ".attn2.to_v.weight").t()
    G, U, c1 = WR.xattn2_fold(c.p(t + ".attn2.to_q.weight"), c.p(t + ".attn2.to_out.0.weight"),
                             c.p(t + ".attn2.to_out.0.bias"), kk, vv)
    G, U = c.r(G), c.r(U)
    z = _ln(c, hs1, t + ".norm2")
    acc = hs1 + c1 + torch.sigmoid(0.125 * (z @ G.t())) @ U
    hsb = c.r(acc)
    a3 = c.r(_ln(c, acc, t + ".norm3"))
    pr = _lin(c, a3, t + ".ff.net.0.proj")
    ffm = c.r(pr[..., :4 * C] * _gelu(pr[..., 4 * C:]))
    # ff.net.2 folded into proj_out
    wpo = c.p(p + ".proj_out.weight")
    fold = c.r(WR.ffpo_fold(wpo, c.p(t + ".ff.net.2.weight")).float())
    bias = WR.ffpo_bias(c.p(p + ".proj_out.bias"), wpo, c.p(t + ".ff.net.2.bias"))
    y = hsb @ c.w(p + ".proj_out.weight").t() + ffm @ fold.t() + bias + _tokens(x)
    return _image(y, H, W)


def _vae_attn(c, p, x):
    B, C, H, W = x.shape
    a = c.r(_tokens(_gn(c, x, p + ".group_norm", 1e-6)))
    q, k, v = (c.r(_lin(c, a, f"{p}.to_{n}")) for n in "qkv")
    s = (q @ k.transpose(-1, -2)) * float(np.float32(1.0) / np.sqrt(np.float32(C), dtype=np.float32))
    o = c.r(c.r(torch.softmax(s, -1)) @ v)
    return x + _image(_lin(c, o, p + ".to_out.0"), H, W)


# ---- graphs -----------------------------------------------------------------------------------------------------------
@torch.no_grad()
def unet_step(unet, text, rgb, x, t, kx=1.0, kv=0.0, kz=0.0, noise=None, bf16=True, sd=None):
    """One UNet step with the fused scheduler update. rgb [B, 4, h, w], x [B, Ct, h, w], t the timestep, kx / kv / kz
    the step's coefficients (fp32 values). Returns (model_out, kx x + kv model_out + kz noise), float64 NCHW.
    sd: weights to use instead of unet.state_dict() (same keys)."""
    c = _Ctx(unet.state_dict() if sd is None else sd, bf16)
    cfg = unet.cfg
    ch, L, eps = cfg.block_out_channels, cfg.layers_per_block, cfg.norm_eps
    ctx = text.reshape(-1, text.shape[-1]).to(torch.float64)
    rgb, x = rgb.to(torch.float64), x.to(torch.float64)
    # the time MLP and the per-step bias table run on fp32 weights
    ste = F.silu(WR.time_mlp(c.p, WR.timestep_embedding([t], ch[0])))[0]

    def bias1(p):
        return WR.step_bias(c.p, p, ste)

    h = _conv(c, c.r(torch.cat([rgb, x], 1)), "conv_in")
    skips = [h]
    for i in range(4):
        b = f"down_blocks.{i}"
        for j in range(L):
            p = f"{b}.resnets.{j}"
            h = _resnet(c, p, h, None, bias1(p), eps)
            if i < 3:
                h = _xfmr(c, f"{b}.attentions.{j}", h, ctx)
            skips.append(h)
        if i < 3:
            h = _conv(c, c.r(h), f"{b}.downsamplers.0.conv", stride=2)
            skips.append(h)
    h = _resnet(c, "mid_block.resnets.0", h, None, bias1("mid_block.resnets.0"), eps)
    h = _xfmr(c, "mid_block.attentions.0", h, ctx)
    h = _resnet(c, "mid_block.resnets.1", h, None, bias1("mid_block.resnets.1"), eps)
    for i in range(4):
        b = f"up_blocks.{i}"
        for j in range(L + 1):
            p = f"{b}.resnets.{j}"
            h = _resnet(c, p, h, skips.pop(), bias1(p), eps)
            if i > 0:
                h = _xfmr(c, f"{b}.attentions.{j}", h, ctx)
        if i < 3:
            h = _conv(c, F.interpolate(c.r(h), size=tuple(skips[-1].shape[2:]), mode="nearest"),
                      f"{b}.upsamplers.0.conv")
    t_ = c.r(F.silu(_gn(c, h, "conv_norm_out", eps)))
    mo = _conv(c, t_, "conv_out")
    xn = float(kx) * x + float(kv) * mo
    if noise is not None and float(kz) != 0.0:
        xn = xn + float(kz) * noise.to(torch.float64)
    return mo, xn


@torch.no_grad()
def encode(vae, rgb, bf16=True, sd=None):
    """rgb [B, 3, H, W] -> the latent mean * latent_scale [B, 4, H // 8, W // 8], float64."""
    c = _Ctx(vae.state_dict() if sd is None else sd, bf16)
    n = len(vae.cfg.block_out_channels)
    h = _conv(c, c.r(rgb.float()), "encoder.conv_in")
    for i in range(n):
        b = f"encoder.down_blocks.{i}"
        for j in range(vae.cfg.layers_per_block):
            p = f"{b}.resnets.{j}"
            h = _resnet(c, p, h, None, c.p(p + ".conv1.bias"), 1e-6)
        if i < n - 1:
            h = _conv(c, F.pad(c.r(h), (0, 1, 0, 1)), f"{b}.downsamplers.0.conv", stride=2, padding=0)
    m = "encoder.mid_block"
    h = _resnet(c, m + ".resnets.0", h, None, c.p(m + ".resnets.0.conv1.bias"), 1e-6)
    h = _vae_attn(c, m + ".attentions.0", h)
    h = _resnet(c, m + ".resnets.1", h, None, c.p(m + ".resnets.1.conv1.bias"), 1e-6)
    t_ = c.r(F.silu(_gn(c, h, "encoder.conv_norm_out", 1e-6)))
    # conv_out (C -> 8) then quant_conv (1x1, 8 -> 8), mean half, folded
    sd = c.sd
    w, bias = WR.enc_out_fold(sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"], sd["quant_conv.weight"],
                             sd["quant_conv.bias"], LATENT_SCALE, host_fp32=bf16)
    if bf16:
        w, bias = c.r(w), bias.float().double()
    return F.conv2d(t_, w, padding=1) * LATENT_SCALE + bias[None, :, None, None]


DECODE_DEPTH, DECODE_NORMALS, DECODE_RAW, DECODE_UNIT3 = 0, 1, 2, 3


@torch.no_grad()
def decode(vae, latent, mode=DECODE_RAW, bf16=True, sd=None):
    """latent [B, 4, h, w] -> [B, 1 or 3, 8 h, 8 w] through the head `mode` (mgb_decode's modes), float64."""
    c = _Ctx(vae.state_dict() if sd is None else sd, bf16)
    n = len(vae.cfg.block_out_channels)
    xs = latent.float() * np.float32(INV_LATENT_SCALE) if bf16 else latent.double() * INV_LATENT_SCALE
    z = c.r(_conv(c, xs.double(), "post_quant_conv", padding=0))
    h = _conv(c, z, "decoder.conv_in")
    m = "decoder.mid_block"
    h = _resnet(c, m + ".resnets.0", h, None, c.p(m + ".resnets.0.conv1.bias"), 1e-6)
    h = _vae_attn(c, m + ".attentions.0", h)
    h = _resnet(c, m + ".resnets.1", h, None, c.p(m + ".resnets.1.conv1.bias"), 1e-6)
    for i in range(n):
        b = f"decoder.up_blocks.{i}"
        for j in range(vae.cfg.layers_per_block + 1):
            p = f"{b}.resnets.{j}"
            h = _resnet(c, p, h, None, c.p(p + ".conv1.bias"), 1e-6)
        if i < n - 1:
            h = _conv(c, F.interpolate(c.r(h), scale_factor=2.0, mode="nearest"), f"{b}.upsamplers.0.conv")
    t_ = c.r(F.silu(_gn(c, h, "decoder.conv_norm_out", 1e-6)))
    return decode_head(_conv(c, t_, "decoder.conv_out"), mode)


def decode_head(raw, mode):
    if mode == DECODE_DEPTH:
        return (raw.mean(1, keepdim=True).clip(-1, 1) + 1) / 2
    if mode == DECODE_NORMALS:
        cl = raw.clip(-1, 1)
        return cl / torch.norm(cl, dim=1, keepdim=True).clamp(min=1e-6)
    if mode == DECODE_UNIT3:
        return (raw.clip(-1, 1) + 1) / 2
    return raw


def rms(t) -> float:
    return float(t.to(torch.float64).pow(2).mean().sqrt().item())


def rms_err(out, ref) -> float:
    """max |out - ref| / rms(ref): the element-wise check |out - ref| <= tau rms(ref) passes iff this is <= tau."""
    out, ref = out.detach().cpu().to(torch.float64), ref.detach().cpu().to(torch.float64)
    d = (out - ref).abs()
    if torch.isnan(d).any():
        return math.inf
    return float(d.max().item()) / (rms(ref) + 1e-300)
