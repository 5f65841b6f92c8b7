"""Float64 restatement, from the diffusers state dict, of every device table the library builds: what
mgb_finalize_weights, mgb_set_text_embedding and mgb_set_schedule leave behind the handle (api_net.cu), in the layout
the kernels read, with a bound per element.

The folds are defined here once; tests/net_ref.py builds its network restatement from the same functions.

Bounds, per element, with u = 2^-24 and u_b = 2^-8 (the half-ulps of fp32 and bf16):
  bf16 weights (packed convs with their cin_pad zero columns, QKV, the GEGLU-interleaved ff1, linears, conv2 | 1x1
      shortcut, the left block of ffpo): the bits of torch's bf16 of the fp32 value;
  fp32 copies (norm affines, biases, temb_w, the cross-attention masters, te_*, pq_*): the same bits;
  host fp32 sums (conv2.b + conv_shortcut.b, time_emb_proj.b + conv1.b): the bits of the fp32 sum;
  enc_out.w: (1 + u_b) 8u sum_j |q||cw| + u_b |ref|; enc_out.b: 2u |ref|;
  ffpo right block (fold_matmul, K = C): (1 + u_b) K u (|W_po| |W_ff2|) + u_b |ref|; ffpo.b: u |ref| + 2 K 2^-53 (...);
  kv (linear_small, K = ctx): K u (|W| |ctx|);
  G, U (xattn2_fold, bf16): (1 + u_b) (66u sum_d |w| (|k0| + |k1|) + |w| e_kv) + u_b |ref|;
  c1: (C + 1) u (|Wo| |v1| + |bo|) + |Wo| e_v1, where e_kv is 0 when the fold is checked from the device's own kv;
  bias table: the embedding |d| <= 4u |angle| + 2u (the angle formed in fp32, the device's logf / expf may move it by
      an ulp or two), propagated to first order through linear_1 -> SiLU -> linear_2 -> SiLU -> time_emb_proj: a linear
      layer adds e_pre = |W| e_in + K u |W| |x| + u (|b| + |pre|), a SiLU gives e = 1.1 e_pre + 4u |silu|
      (|silu'| <= 1.1; fp32 expf, add and divide);
  pack_decoder_latent: (1 + u_b) 5u (|b| + sum |w| |x s^-1|) + u_b |ref|.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Iterator, Optional

import torch

U32 = 2.0 ** -24
UB = 2.0 ** -8
U64 = 2.0 ** -53


# ---- the folds (shared with tests/net_ref.py) ---------------------------------------------------------------------
def timestep_angle(ts, dim) -> torch.Tensor:
    """t f, f_i = exp(-ln(10000) i / half), formed in fp32 as the oracle forms it; float64 [n, dim / 2]."""
    half = dim // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    t = torch.tensor([float(x) for x in ts], dtype=torch.float32)
    return (t[:, None] * f[None, :]).to(torch.float64)


def timestep_embedding(ts, dim) -> torch.Tensor:
    """[cos | sin](t f), float64 [n, dim]."""
    ang = timestep_angle(ts, dim)
    return torch.cat([torch.cos(ang), torch.sin(ang)], -1)


def time_mlp(p, emb) -> torch.Tensor:
    """linear_2(silu(linear_1(emb))) on the fp32 weights; p maps a UNet key to its float64 value."""
    h = torch.nn.functional.silu(emb @ p("time_embedding.linear_1.weight").t() + p("time_embedding.linear_1.bias"))
    return h @ p("time_embedding.linear_2.weight").t() + p("time_embedding.linear_2.bias")


def step_bias(p, resnet, ste) -> torch.Tensor:
    """One resnet's conv1 bias at one step: conv1.bias + time_emb_proj(silu(temb)), ste = silu(temb)."""
    return p(resnet + ".conv1.bias") + ste @ p(resnet + ".time_emb_proj.weight").t() + p(resnet + ".time_emb_proj.bias")


def xattn2_fold(wq, wo, bo, kk, vv):
    """The cross attention against a two-token context, collapsed: G_h = Wq[h]^T (k0 - k1)_h, U_h = Wo[:, h] (v0 - v1)_h,
    c1 = Wo v1 + bo. kk, vv [2, C] (the two tokens' keys / values). Returns G [H, C], U [H, C], c1 [C]."""
    C = wq.shape[0]
    nh = C // 64
    G = torch.einsum("hdc,hd->hc", wq.reshape(nh, 64, C), (kk[0] - kk[1]).reshape(nh, 64))
    U = torch.einsum("chd,hd->hc", wo.reshape(C, nh, 64), (vv[0] - vv[1]).reshape(nh, 64))
    return G, U, wo @ vv[1] + bo


def ffpo_fold(wpo, w2):
    """ff.net.2 folded into proj_out: the right block W_po W_ff2 (float64 of the given values)."""
    return wpo.to(torch.float64) @ w2.to(torch.float64)


def ffpo_bias(bpo, wpo, b2):
    return bpo.to(torch.float64) + wpo.to(torch.float64) @ b2.to(torch.float64)


def enc_out_fold(cw, cb, qw, qb, scale, host_fp32):
    """conv_out (C -> 8) then quant_conv (1x1, 8 -> 8), the 4 mean channels: weight [4, C, 3, 3] and bias [4] (the
    bias times the latent scale, as the epilogue computes acc scale + bias). host_fp32: the weight summed in fp32 in the
    loader's order (w += q cw, j = 0..7); otherwise exact. Both float64."""
    q4 = qw.float()[:4, :, 0, 0]
    if host_fp32:
        w = torch.zeros_like(cw[:4], dtype=torch.float32)
        for j in range(8):
            w = w + q4[:, j, None, None, None] * cw[j].float()[None]
        w = w.to(torch.float64)
    else:
        w = torch.einsum("oj,jchw->ochw", q4.double(), cw.double())
    b = (qb.double()[:4] + q4.double() @ cb.double()) * scale
    return w, b


# ---- layouts --------------------------------------------------------------------------------------------------------
def pack_conv(w, cin_pad):
    """[cout, cin, 3, 3] -> tap-major [cout, 9 cin_pad] (tap = kh 3 + kw), columns cin..cin_pad - 1 of each tap zero."""
    cout, cin = w.shape[:2]
    o = torch.zeros(cout, 9, cin_pad, dtype=w.dtype)
    o[:, :, :cin] = w.reshape(cout, cin, 9).transpose(1, 2)
    return o.reshape(cout, 9 * cin_pad)


def geglu_rows(C):
    """Row order of the GEGLU-interleaved ff.net.0.proj: each 256-row tile holds 128 value rows, then their 128 gates."""
    i = torch.arange(8 * C)
    nt, r = i // 256, i % 256
    return torch.where(r < 128, nt * 128 + r, 4 * C + nt * 128 + r - 128)


def unet_layout(ch, nl):
    """Execution order of the UNet's resnets (prefix, cin, cout), transformers (prefix, C), down- and upsampler convs."""
    res, xf, downs, ups = [], [], [], []
    skip, prev = [ch[0]], ch[0]
    for i in range(4):
        b = f"down_blocks.{i}"
        for j in range(nl):
            res.append((f"{b}.resnets.{j}", prev if j == 0 else ch[i], ch[i]))
            if i < 3:
                xf.append((f"{b}.attentions.{j}", ch[i]))
            skip.append(ch[i])
        if i < 3:
            downs.append((f"{b}.downsamplers.0.conv", ch[i]))
            skip.append(ch[i])
        prev = ch[i]
    res.append(("mid_block.resnets.0", ch[3], ch[3]))
    xf.append(("mid_block.attentions.0", ch[3]))
    res.append(("mid_block.resnets.1", ch[3], ch[3]))
    for i in range(4):
        cout, b = ch[3 - i], f"up_blocks.{i}"
        for j in range(nl + 1):
            res.append((f"{b}.resnets.{j}", (prev if j == 0 else cout) + skip.pop(), cout))
            if i > 0:
                xf.append((f"{b}.attentions.{j}", cout))
        if i < 3:
            ups.append((f"{b}.upsamplers.0.conv", cout))
        prev = cout
    return res, xf, downs, ups


def vae_layout(vc, nl):
    """Encoder resnets, encoder downsamplers, decoder resnets and decoder upsamplers in execution order."""
    enc, down, dec, up = [], [], [], []
    prev = vc[0]
    for i in range(4):
        for j in range(nl):
            enc.append((f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else vc[i], vc[i]))
        if i < 3:
            down.append((f"encoder.down_blocks.{i}.downsamplers.0.conv", vc[i]))
        prev = vc[i]
    enc += [("encoder.mid_block.resnets.0", vc[3], vc[3]), ("encoder.mid_block.resnets.1", vc[3], vc[3])]
    dec += [("decoder.mid_block.resnets.0", vc[3], vc[3]), ("decoder.mid_block.resnets.1", vc[3], vc[3])]
    prev = vc[3]
    for i in range(4):
        cout = vc[3 - i]
        for j in range(nl + 1):
            dec.append((f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else cout, cout))
        if i < 3:
            up.append((f"decoder.up_blocks.{i}.upsamplers.0.conv", cout))
        prev = cout
    return enc, down, dec, up


# ---- tables ---------------------------------------------------------------------------------------------------------
@dataclass
class Table:
    """One device array, or a column block of one, and what it must hold.

    field: the mgb_debug_read path; dtype "bf16" or "f32", shape: the device array's; ref: without bound, fp32 values
    whose bits (of their bf16 for a bf16 table) the device must hold; with bound, float64 values and |dev - ref| <= bound
    at every element; kind: what the measured ratio is reported as; cols: the column block of a 2-D table this entry
    covers; given_kv: for xGU / xc1, (device kv float64 [4, C]) -> (ref, bound) of the fold alone."""
    field: str
    dtype: str
    shape: tuple
    ref: torch.Tensor
    bound: Optional[torch.Tensor] = None
    kind: str = ""
    cols: Optional[slice] = None
    given_kv: Optional[Callable] = None


def _cin_pad(cin):
    return (cin + 63) // 64 * 64


def _norm(field, sd, key):
    for s, k in (("g", "weight"), ("b", "bias")):
        v = sd[f"{key}.{k}"].float()
        yield Table(f"{field}.{s}", "f32", tuple(v.shape), v, kind="fp32 copies")


def _conv(field, sd, key):
    w = sd[key + ".weight"].float()
    pk = pack_conv(w, _cin_pad(w.shape[1]))
    yield Table(field + ".w", "bf16", tuple(pk.shape), pk, kind="bf16 weights")
    b = sd[key + ".bias"].float()
    yield Table(field + ".b", "f32", tuple(b.shape), b, kind="fp32 copies")


def _lin(field, sd, key, bias=True):
    w = sd[key + ".weight"].float()
    w = w.reshape(w.shape[0], -1)
    yield Table(field + ".w", "bf16", tuple(w.shape), w, kind="bf16 weights")
    if bias:
        b = sd[key + ".bias"].float()
        yield Table(field + ".b", "f32", tuple(b.shape), b, kind="fp32 copies")


def _f32(field, v, kind="fp32 copies"):
    v = v.float().reshape(-1) if v.dim() != 2 else v.float()
    return Table(field, "f32", tuple(v.shape), v, kind=kind)


def _resnet(field, sd, key, cin, cout, temb):
    yield from _norm(field + ".n1", sd, key + ".norm1")
    yield from _conv(field + ".c1", sd, key + ".conv1")
    yield from _norm(field + ".n2", sd, key + ".norm2")
    if cin == cout:
        yield from _conv(field + ".c2", sd, key + ".conv2")
    else:
        w = torch.cat([pack_conv(sd[key + ".conv2.weight"].float(), cout),
                       sd[key + ".conv_shortcut.weight"].float().reshape(cout, cin)], 1)
        yield Table(field + ".c2.w", "bf16", tuple(w.shape), w, kind="bf16 weights")
        yield _f32(field + ".c2.b", sd[key + ".conv2.bias"].float() + sd[key + ".conv_shortcut.bias"].float(),
                   "fp32 sums")
    if temb:
        yield _f32(field + ".temb_w", sd[key + ".time_emb_proj.weight"])
        yield _f32(field + ".temb_b", sd[key + ".time_emb_proj.bias"].float() + sd[key + ".conv1.bias"].float(),
                   "fp32 sums")


def xattn2_tables(wq, wo, bo, kv, e_kv=None):
    """G | U (bf16 [2 H, C]) and c1 ([C]) folded from kv float64 [4, C] (k0, k1, v0, v1), with their bounds; e_kv is
    kv's own error bound when kv is restated rather than the device's. Returns (GU, bound, c1, bound)."""
    wq, wo, bo = wq.double(), wo.double(), bo.double()
    C = wq.shape[0]
    nh = C // 64
    G, U, c1 = xattn2_fold(wq, wo, bo, kv[0:2], kv[2:4])
    aq, ao = wq.abs().reshape(nh, 64, C), wo.abs().reshape(C, nh, 64)
    eG = 66 * U32 * torch.einsum("hdc,hd->hc", aq, (kv[0].abs() + kv[1].abs()).reshape(nh, 64))
    eU = 66 * U32 * torch.einsum("chd,hd->hc", ao, (kv[2].abs() + kv[3].abs()).reshape(nh, 64))
    ec1 = (C + 1) * U32 * (wo.abs() @ kv[3].abs() + bo.abs())
    if e_kv is not None:
        eG = eG + torch.einsum("hdc,hd->hc", aq, (e_kv[0] + e_kv[1]).reshape(nh, 64))
        eU = eU + torch.einsum("chd,hd->hc", ao, (e_kv[2] + e_kv[3]).reshape(nh, 64))
        ec1 = ec1 + wo.abs() @ e_kv[3]
    GU = torch.cat([G, U])
    return GU, (1 + UB) * torch.cat([eG, eU]) + UB * GU.abs(), c1, ec1


def _xfmr(field, sd, key, C, ctx):
    t = key + ".transformer_blocks.0"
    yield from _norm(field + ".gn", sd, key + ".norm")
    yield from _lin(field + ".proj_in", sd, key + ".proj_in")
    for i in (1, 2, 3):
        yield from _norm(f"{field}.ln{i}", sd, f"{t}.norm{i}")
    qkv = torch.cat([sd[f"{t}.attn1.to_{n}.weight"].float() for n in "qkv"])
    yield Table(field + ".qkv.w", "bf16", tuple(qkv.shape), qkv, kind="bf16 weights")
    yield from _lin(field + ".o1", sd, t + ".attn1.to_out.0")
    wq, wo, bo = (sd[t + k].float() for k in (".attn2.to_q.weight", ".attn2.to_out.0.weight", ".attn2.to_out.0.bias"))
    wk, wv = sd[t + ".attn2.to_k.weight"].float(), sd[t + ".attn2.to_v.weight"].float()
    yield _f32(field + ".q2w", wq)
    yield _f32(field + ".o2w", wo)
    yield _f32(field + ".o2b", bo)
    yield _f32(field + ".k2w", wk)
    yield _f32(field + ".v2w", wv)
    # the text K / V: linear_small over K = ctx
    c = ctx.double()
    kv = torch.cat([c @ wk.double().t(), c @ wv.double().t()])
    K = c.shape[1]
    e_kv = K * U32 * torch.cat([c.abs() @ wk.double().abs().t(), c.abs() @ wv.double().abs().t()])
    yield Table(field + ".kv", "f32", (4, C), kv, e_kv, kind="kv")
    GU, bGU, c1, bc1 = xattn2_tables(wq, wo, bo, kv, e_kv)

    def own_gu(kv_dev, wq=wq, wo=wo, bo=bo):
        r = xattn2_tables(wq, wo, bo, kv_dev)
        return r[0], r[1]

    def own_c1(kv_dev, wq=wq, wo=wo, bo=bo):
        r = xattn2_tables(wq, wo, bo, kv_dev)
        return r[2], r[3]
    yield Table(field + ".xGU", "bf16", tuple(GU.shape), GU, bGU, kind="G, U", given_kv=own_gu)
    yield Table(field + ".xc1", "f32", (C,), c1, bc1, kind="c1", given_kv=own_c1)
    rows = geglu_rows(C)
    fw, fb = sd[t + ".ff.net.0.proj.weight"].float()[rows], sd[t + ".ff.net.0.proj.bias"].float()[rows]
    yield Table(field + ".ff1.w", "bf16", tuple(fw.shape), fw, kind="bf16 weights")
    yield Table(field + ".ff1.b", "f32", tuple(fb.shape), fb, kind="fp32 copies")
    # ffpo = [bf16(W_po) | bf16(W_po W_ff2)] (fold_matmul, K = C), bias b_po + W_po b_ff2 (double, then fp32)
    wpo, bpo = sd[key + ".proj_out.weight"].float(), sd[key + ".proj_out.bias"].float()
    w2, b2 = sd[t + ".ff.net.2.weight"].float(), sd[t + ".ff.net.2.bias"].float()
    shape = (C, 5 * C)
    yield Table(field + ".ffpo.w", "bf16", shape, wpo, kind="bf16 weights", cols=slice(0, C))
    right = ffpo_fold(wpo, w2)
    bound = (1 + UB) * C * U32 * (wpo.double().abs() @ w2.double().abs()) + UB * right.abs()
    yield Table(field + ".ffpo.w", "bf16", shape, right, bound, kind="ffpo right block", cols=slice(C, 5 * C))
    b = ffpo_bias(bpo, wpo, b2)
    bb = U32 * b.abs() + 2 * C * U64 * (bpo.double().abs() + wpo.double().abs() @ b2.double().abs())
    yield Table(field + ".ffpo.b", "f32", (C,), b, bb, kind="ffpo.b")


def unet_tables(sd, ch, nl, ctx) -> Iterator[Table]:
    """Every table of the UNet (fields unet.*), sd the UNet's state dict (fp32 values), ctx the text embedding [2, ctx]."""
    res, xf, downs, ups = unet_layout(ch, nl)
    yield from _conv("unet.conv_in", sd, "conv_in")
    for n, k in (("te_w1", "linear_1.weight"), ("te_b1", "linear_1.bias"), ("te_w2", "linear_2.weight"),
                 ("te_b2", "linear_2.bias")):
        yield _f32("unet." + n, sd["time_embedding." + k])
    for i, (key, cin, cout) in enumerate(res):
        yield from _resnet(f"unet.resnets.{i}", sd, key, cin, cout, True)
    for i, (key, C) in enumerate(xf):
        yield from _xfmr(f"unet.xfmrs.{i}", sd, key, C, ctx.reshape(-1, ctx.shape[-1]))
    for i, (key, _) in enumerate(downs):
        yield from _conv(f"unet.downs.{i}", sd, key)
    for i, (key, _) in enumerate(ups):
        yield from _conv(f"unet.ups.{i}", sd, key)
    yield from _norm("unet.norm_out", sd, "conv_norm_out")
    yield from _conv("unet.conv_out", sd, "conv_out")


def _vae_attn(field, sd, key):
    yield from _norm(field + ".gn", sd, key + ".group_norm")
    for n, k in (("q", "to_q"), ("k", "to_k"), ("v", "to_v"), ("o", "to_out.0")):
        yield from _lin(f"{field}.{n}", sd, f"{key}.{k}")


def vae_tables(sd, vc, nl, latent_scale) -> Iterator[Table]:
    """Every table of the VAE (fields vae.*), sd the VAE's state dict; latent_scale the fp32 mgb_config value."""
    enc, down, dec, up = vae_layout(vc, nl)
    yield from _conv("vae.enc_in", sd, "encoder.conv_in")
    for i, (key, cin, cout) in enumerate(enc):
        yield from _resnet(f"vae.enc_res.{i}", sd, key, cin, cout, False)
    for i, (key, _) in enumerate(down):
        yield from _conv(f"vae.enc_down.{i}", sd, key)
    yield from _vae_attn("vae.enc_attn", sd, "encoder.mid_block.attentions.0")
    yield from _norm("vae.enc_norm_out", sd, "encoder.conv_norm_out")
    cw, cb, qw, qb = (sd[k] for k in ("encoder.conv_out.weight", "encoder.conv_out.bias", "quant_conv.weight",
                                      "quant_conv.bias"))
    C = cw.shape[1]
    w, b = enc_out_fold(cw, cb, qw, qb, latent_scale, host_fp32=False)
    mag = torch.einsum("oj,jchw->ochw", qw.double()[:4, :, 0, 0].abs(), cw.double().abs())
    e = 8 * U32 * mag
    w, e = pack_conv(w, C), pack_conv(e, C)
    yield Table("vae.enc_out.w", "bf16", tuple(w.shape), w, (1 + UB) * e + UB * w.abs(), kind="enc_out.w")
    yield Table("vae.enc_out.b", "f32", (4,), b, 2 * U32 * b.abs(), kind="enc_out.b")
    yield _f32("vae.pq_w", sd["post_quant_conv.weight"])
    yield _f32("vae.pq_b", sd["post_quant_conv.bias"])
    yield from _conv("vae.dec_in", sd, "decoder.conv_in")
    for i, (key, cin, cout) in enumerate(dec):
        yield from _resnet(f"vae.dec_res.{i}", sd, key, cin, cout, False)
    yield from _vae_attn("vae.dec_attn", sd, "decoder.mid_block.attentions.0")
    for i, (key, _) in enumerate(up):
        yield from _conv(f"vae.dec_up.{i}", sd, key)
    yield from _norm("vae.dec_norm_out", sd, "decoder.conv_norm_out")
    yield from _conv("vae.dec_out", sd, "decoder.conv_out")


def enc_out_host(sd, latent_scale):
    """The encoder fold as the loader computes it (fp32 weight sum in its order): the bits the device must hold."""
    w, _ = enc_out_fold(sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"], sd["quant_conv.weight"],
                        sd["quant_conv.bias"], latent_scale, host_fp32=True)
    return pack_conv(w.float(), w.shape[1])


# ---- per-step tables ------------------------------------------------------------------------------------------------
def _silu(x):
    return torch.nn.functional.silu(x)


def _linear_err(W, b, x, e_x):
    """pre = x W^T + b and its bound: |W| e_x + K u |W| |x| + u (|b| + |pre|)."""
    pre = x @ W.t() + b
    aW = W.abs()
    return pre, e_x @ aW.t() + W.shape[1] * U32 * (x.abs() @ aW.t()) + U32 * (b.abs() + pre.abs())


def bias_table(sd, ch, nl, timesteps):
    """Rows of the per-step bias table: every resnet's conv1.bias + time_emb_proj(silu(temb_i)) in execution order,
    float64 [n, total], with its bound. Also returns each resnet's column offset and width."""
    def p(k):
        return sd[k].detach().double()
    ang = timestep_angle(timesteps, ch[0])
    emb = torch.cat([torch.cos(ang), torch.sin(ang)], -1)
    e = (4 * U32 * ang.abs() + 2 * U32).repeat(1, 2)
    pre, e = _linear_err(p("time_embedding.linear_1.weight"), p("time_embedding.linear_1.bias"), emb, e)
    h = _silu(pre)
    e = 1.1 * e + 4 * U32 * h.abs()
    temb, e = _linear_err(p("time_embedding.linear_2.weight"), p("time_embedding.linear_2.bias"), h, e)
    s = _silu(temb)
    e = 1.1 * e + 4 * U32 * s.abs()
    rows, bounds, cols = [], [], []
    off = 0
    for key, _, cout in unet_layout(ch, nl)[0]:
        y, ey = _linear_err(p(key + ".time_emb_proj.weight"), p(key + ".time_emb_proj.bias") + p(key + ".conv1.bias"),
                            s, e)
        rows.append(y)
        bounds.append(ey)
        cols.append((key, off, cout))
        off += cout
    return torch.cat(rows, 1), torch.cat(bounds, 1), cols


def pack_decoder_latent(lat, w, b, inv_scale):
    """z = post_quant_conv(latent * fp32(1 / scale)) float64 [NB h w, 4] with its bound; lat fp32 NCHW [NB, 4, h, w],
    w [4, 4, 1, 1], b [4], inv_scale the fp32 factor."""
    xs = (lat.float() * torch.tensor(inv_scale, dtype=torch.float32)).double()
    x = xs.permute(0, 2, 3, 1).reshape(-1, 4)
    W = w.double().reshape(4, 4)
    z = x @ W.t() + b.double()
    e = (1 + UB) * 5 * U32 * (b.double().abs() + x.abs() @ W.abs().t()) + UB * z.abs()
    return z, e
