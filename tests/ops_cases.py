"""Operator-level parity cases: every case calls ONE C-ABI operator (through marigold_b200.ops) and holds each output
element to a float64 reference on the same bf16-rounded inputs, within the per-element bound of tests/ops_ref.py.
Used by tests/test_ops_gpu.py (`-m gpu`) and by tools/bringup.py (crash-isolating battery with timings).

Covers the tile shapes the SD-2-size network launches (gemm_tc_kernel<160>/<128>/<256>, the two-CTA variants,
split-K + its deferred epilogue, split-KV flash attention + attn_combine, the space-to-depth stride-2 convs, the small-N
special epilogues) and the paths only the network used to reach: K concatenation in the linear and the conv
(conv2 + 1x1 shortcut), odd stride-2 inputs, the scheduler epilogue, GroupNorm over a concat with straddling groups and
its raw copy, the cropped upsample and the VAE attention helpers. The attention, softmax, transpose and VAE attention
GEMM cases also run at the token counts of a 4032 x 3024 photo at native resolution (T = 190 512 at the UNet's level 0
and in the VAE's mid block); there the attention's float64 reference is held to check_rows' rows only.

Each case returns {"ok": bool, "worst": max |d| / bound, ...}; "rel_to_max" is reported, never asserted."""
from __future__ import annotations

import math


def cases():
    cases = []

    def add(name, fn, **kw):
        cases.append((name, fn, kw))

    # ---- linear -----------------------------------------------------------------------------
    for bn in (128, 64, 256, 160, 32, 16):
        add(f"linear_bn{bn}_small", case_linear, M=256, N=320 if bn == 160 else 256, K=128, block_n=bn)
        add(f"linear_bn{bn}_ragged_n", case_linear, M=200, N=2 * bn - 12, K=192, block_n=bn, bias=True, bf16out=True)
        add(f"linear_bn{bn}_odd_n", case_linear, M=130, N=bn + 5, K=128, block_n=bn, bias=True, residual=True)
    for m in (1, 127, 129, 9217):
        add(f"linear_m{m}", case_linear, M=m, N=320, K=320, block_n=0, bias=True, bf16out=True)
    add("linear_qkv_96", case_linear, M=9216, N=960, K=320, block_n=160)
    add("linear_auto_96", case_linear, M=9216, N=320, K=1280, block_n=0)
    add("linear_bias_res_bf16", case_linear, M=2304, N=640, K=640, block_n=128, bias=True, residual=True, bf16out=True)
    add("linear_ragged_m144", case_linear, M=144, N=1280, K=1280, block_n=128, bias=True)
    add("linear_ragged_m576", case_linear, M=576, N=1280, K=1280, block_n=256, bias=True, residual=True)
    add("linear_geglu", case_linear, M=2304, N=5120, K=640, block_n=256, bias=True, geglu=True, bf16out=True)
    add("linear_geglu_bn128", case_linear, M=300, N=512, K=128, block_n=128, bias=True, geglu=True)
    for bn in (64, 128, 256):
        add(f"linear_geglu_bn{bn}_res", case_linear, M=300, N=512, K=128, block_n=bn, bias=True, geglu=True,
            residual=True)
    add("linear_splitk4", case_linear, M=144, N=1280, K=5120, block_n=128, splits=4, bias=True, residual=True)
    # 10 K blocks asked for 6 splits: 2 blocks per split, so 5 splits run
    add("linear_splitk_uneven", case_linear, M=144, N=640, K=640, block_n=128, splits=6, bias=True)
    add("linear_splitk_silu_scale_bf16_res", case_linear, M=200, N=512, K=1024, block_n=128, splits=4, bias=True,
        residual=True, bf16out=True, silu=True, scale=0.7)
    add("linear_stages2", case_linear, M=512, N=256, K=1024, block_n=128, stages=2)
    add("linear_silu_scale", case_linear, M=256, N=128, K=256, block_n=128, bias=True, silu=True)
    add("linear_silu_scale_bn16", case_linear, M=256, N=16, K=256, block_n=16, bias=True, silu=True, scale=-1.5)
    add("linear_n_ragged", case_linear, M=256, N=200, K=128, block_n=128, bias=True)
    add("linear_ldo", case_linear, M=300, N=256, K=256, block_n=128, bias=True, residual=True, bf16out=True, ldo=320)
    # the VAE score GEMM: EPI_SCALE, fp32 out with ldo = T rounded up to 64
    add("linear_vae_score", case_linear, M=84, N=84, K=512, block_n=0, scale=512 ** -0.5, ldo=128)
    # the VAE attention's GEMMs on a 4032 x 3024 photo (T = 190 512, Tp = 190 528): one block of score rows, and P V
    # over the whole key range
    add("linear_vae_score_t190512", case_linear, M=256, N=190512, K=512, block_n=0, scale=512 ** -0.5, ldo=190528)
    add("linear_vae_pv_k190528", case_linear, M=256, N=512, K=190528, block_n=0, bf16out=True, probs=True)
    # multi-wave grids take the two-CTAs-per-SM instantiation (MINB = 2)
    add("linear_2cta_bn64", case_linear, M=9216, N=256, K=640, block_n=64, bias=True, residual=True)
    add("linear_2cta_bn128", case_linear, M=9216, N=512, K=640, block_n=128, bias=True, bf16out=True)
    # K concatenation A = [A1 | A2]: K1 = one block, and K1 = 5 blocks (not a multiple of stages * 64)
    add("linear_kcat_k1_64", case_linear, M=300, N=256, K=64, K2=256, block_n=128, bias=True)
    add("linear_kcat_ffpo_320", case_linear, M=9216, N=320, K=320, K2=1280, block_n=0, bias=True, residual=True)
    # ---- conv -------------------------------------------------------------------------------
    add("conv3_16x16_c64", case_conv, NB=1, H=16, W=16, Cin=64, Cout=64, kind=0, block_n=64)
    add("conv3_96_c320", case_conv, NB=1, H=96, W=96, Cin=320, Cout=320, kind=0, block_n=160, bias=True)
    add("conv3_24_nb2", case_conv, NB=2, H=24, W=24, Cin=128, Cout=256, kind=0, block_n=128, bias=True, residual=True)
    add("conv3_nb3", case_conv, NB=3, H=20, W=12, Cin=128, Cout=128, kind=0, block_n=0, bias=True, residual=True)
    add("conv3_12_splitk", case_conv, NB=1, H=12, W=12, Cin=1280, Cout=1280, kind=0, block_n=128, splits=6, bias=True)
    add("conv3_rect_40x72", case_conv, NB=1, H=40, W=72, Cin=64, Cout=128, kind=0, block_n=128, bias=True)
    for wo in (8, 13, 33, 65, 129):
        add(f"conv3_wout{wo}", case_conv, NB=1, H=11, W=wo, Cin=64, Cout=96, kind=0, block_n=0, bias=True)
    add("conv1x1", case_conv, NB=2, H=24, W=24, Cin=640, Cout=320, kind=1, block_n=0, bias=True, residual=True)
    add("conv3_s2_pad1", case_conv, NB=2, H=24, W=24, Cin=128, Cout=128, kind=2, block_n=128, bias=True)
    add("conv3_s2_asym", case_conv, NB=1, H=48, W=48, Cin=128, Cout=128, kind=3, block_n=128, bias=True)
    # stride 2 on odd inputs: Hin x Win given; parity planes of ceil(Hin / 2) x ceil(Win / 2)
    for kind in (2, 3):
        add(f"conv3_s2_kind{kind}_77x131", case_conv, NB=1, Hin=77, Win=131, Cin=64, Cout=128, kind=kind, block_n=0,
            bias=True)
        add(f"conv3_s2_kind{kind}_27x13", case_conv, NB=2, Hin=27, Win=13, Cin=128, Cout=64, kind=kind, block_n=0,
            bias=True)
    # ResnetBlock conv2 + 1x1 shortcut as one implicit GEMM (second A operand, weights [W2 | Wsc])
    add("conv3_shortcut_24", case_conv, NB=1, H=24, W=24, Cin=640, Cout=1280, kind=0, block_n=0, bias=True, Cin2=640)
    add("conv3_shortcut_24_splitk", case_conv, NB=1, H=24, W=24, Cin=640, Cout=1280, kind=0, block_n=128, splits=4,
        bias=True, Cin2=640)
    add("conv3_shortcut_odd", case_conv, NB=2, H=13, W=7, Cin=128, Cout=64, kind=0, block_n=0, bias=True, Cin2=192)
    # small-N special epilogues, as the decoders / conv_out launch them (block_n = 0: the entry point picks 16)
    add("conv3_cout4_nchw", case_conv, NB=2, H=32, W=32, Cin=64, Cout=4, kind=0, block_n=16, bias=True, special="nchw")
    add("conv3_cout3_depth", case_conv, NB=2, H=32, W=32, Cin=128, Cout=3, kind=0, block_n=16, bias=True,
        special="depth")
    add("conv3_cout3_normals", case_conv, NB=1, H=32, W=32, Cin=128, Cout=3, kind=0, block_n=16, bias=True,
        special="normals")
    for cout in (4, 12):
        add(f"conv3_27x12_sched_c{cout}", case_conv, NB=2, H=27, W=12, Cin=320, Cout=cout, kind=0, block_n=0, bias=True,
            special="sched")
        add(f"conv3_27x12_nchw_c{cout}", case_conv, NB=2, H=27, W=12, Cin=128, Cout=cout, kind=0, block_n=0,
            bias=True, special="nchw")
        add(f"conv3_27x12_nchw_scale_c{cout}", case_conv, NB=2, H=27, W=12, Cin=128, Cout=cout, kind=0, block_n=0,
            bias=True, special="nchw", scale=0.18215)
        add(f"conv3_27x12_unit_c{cout}", case_conv, NB=2, H=27, W=12, Cin=128, Cout=cout, kind=0, block_n=0, bias=True,
            special="unit")
    add("conv3_27x12_depth", case_conv, NB=2, H=27, W=12, Cin=128, Cout=3, kind=0, block_n=0, bias=True,
        special="depth")
    add("conv3_27x12_normals", case_conv, NB=2, H=27, W=12, Cin=128, Cout=3, kind=0, block_n=0, bias=True,
        special="normals")
    add("conv3_auto_48", case_conv, NB=1, H=48, W=48, Cin=640, Cout=640, kind=0, block_n=0, bias=True)
    add("conv3_sched_exact", case_sched_exact, NB=2, H=27, W=12, Cin=320, Cout=4)
    # ---- attention --------------------------------------------------------------------------
    for T in (1, 8, 21, 63, 64, 65, 84, 127, 129, 324):
        for NB in (1, 3):
            for C in (64, 320, 1280):
                add(f"attn_t{T}_nb{NB}_c{C}", case_attn, NB=NB, T=T, C=C)
    add("attn_t128_h1", case_attn, NB=1, T=128, C=64)
    add("attn_t256_h2", case_attn, NB=1, T=256, C=128)
    add("attn_t144", case_attn, NB=1, T=144, C=1280)
    add("attn_t576_nb2", case_attn, NB=2, T=576, C=128)
    add("attn_t2304", case_attn, NB=1, T=2304, C=640)
    add("attn_t9216", case_attn, NB=1, T=9216, C=320)
    add("attn_t4096_c64", case_attn, NB=1, T=4096, C=64)
    add("attn_t1500_c64", case_attn, NB=1, T=1500, C=64)
    add("attn_t324_logits80", case_attn, NB=1, T=324, C=128, qk_std=6.3)
    add("attn_t1500_logits80", case_attn, NB=1, T=1500, C=64, qk_std=6.3)
    add("attn_t129_one_key", case_attn, NB=2, T=129, C=128, dominant=True)
    # the UNet's levels 0, 1 and 2 on a 4032 x 3024 photo (504 x 378 latents), checked on check_rows' rows; a key that
    # dominates every query late in the KV loop (past 256 key blocks: the running max grows there) and in the ragged
    # last key block
    add("attn_t190512_c320", case_attn, NB=1, T=190512, C=320)
    add("attn_t47628_c640", case_attn, NB=1, T=47628, C=640)
    add("attn_t11970_c1280", case_attn, NB=1, T=11970, C=1280)
    add("attn_t190512_late_key", case_attn, NB=1, T=190512, C=320, dominant_at=120001)
    add("attn_t190512_last_key", case_attn, NB=1, T=190512, C=320, dominant_at=190511)
    # ---- streaming kernels ------------------------------------------------------------------
    add("groupnorm_320", case_groupnorm, NB=2, HW=2304, C=320, G=32, eps=1e-5, silu=1)
    add("groupnorm_1920", case_groupnorm, NB=1, HW=576, C=1920, G=32, eps=1e-5, silu=1)
    add("groupnorm_2560", case_groupnorm, NB=1, HW=144, C=2560, G=32, eps=1e-6, silu=0)
    add("groupnorm_128_big", case_groupnorm, NB=1, HW=147456, C=128, G=32, eps=1e-6, silu=1)
    add("groupnorm_128_big_nb4", case_groupnorm, NB=4, HW=147456, C=128, G=32, eps=1e-6, silu=1)
    # concat [a | b] with groups that straddle the boundary (60 / 30 / 12 channels per group), and the raw copy
    add("groupnorm_cat_1280_640", case_groupnorm, NB=1, HW=576, C=1280, Cb=640, G=32, eps=1e-5, silu=1)
    add("groupnorm_cat_640_320", case_groupnorm, NB=2, HW=2304, C=640, Cb=320, G=32, eps=1e-5, silu=1)
    add("groupnorm_cat_256_128", case_groupnorm, NB=1, HW=4096, C=256, Cb=128, G=32, eps=1e-5, silu=0)
    # thread geometries Kq = 1 (C = 320), 2 (C = 640), 4 (C = 1280), with HW = 1 and 3
    for C in (320, 640, 1280):
        for HW in (1, 3):
            add(f"groupnorm_c{C}_hw{HW}", case_groupnorm, NB=2, HW=HW, C=C, G=32, eps=1e-5, silu=1)
    # one pixel past a whole number of 24-pixel rounds per chunk (C = 320: Tp = 3, R = 8)
    add("groupnorm_chunk_edge", case_groupnorm, NB=1, HW=24 * 264 + 1, C=320, G=32, eps=1e-5, silu=1)
    add("groupnorm_offset100", case_groupnorm, NB=1, HW=16384, C=128, G=32, eps=1e-6, silu=1, offset=100.0)
    add("groupnorm_offset100_cat", case_groupnorm, NB=1, HW=576, C=1280, Cb=640, G=32, eps=1e-5, silu=0,
        offset=100.0)
    # the batched geometry the pipelines launch (gn_max_ctas() / NB chunks per image): long per-thread fp32 runs (VAE
    # decoder at 768 x 768, NB = 16: 9216 values per thread and channel at C = 256), at a small and a large mean
    for off in (0.5, 100.0):
        o = "" if off == 0.5 else "_offset100"
        add(f"groupnorm_vae768_nb16_c256{o}", case_groupnorm, NB=16, HW=768 * 768, C=256, G=32, eps=1e-6, silu=1,
            offset=off)
        add(f"groupnorm_vae768_nb16_c128{o}", case_groupnorm, NB=16, HW=768 * 768, C=128, G=32, eps=1e-6, silu=1,
            offset=off)
        add(f"groupnorm_vae1024_nb8_c256{o}", case_groupnorm, NB=8, HW=1024 * 1024, C=256, G=32, eps=1e-6, silu=1,
            offset=off)
        add(f"groupnorm_unet96_nb16_cat_640_320{o}", case_groupnorm, NB=16, HW=9216, C=640, Cb=320, G=32, eps=1e-5,
            silu=1, offset=off)
        add(f"groupnorm_unet48_nb16_cat_1280_640{o}", case_groupnorm, NB=16, HW=2304, C=1280, Cb=640, G=32, eps=1e-5,
            silu=1, offset=off)
    # collapsed cross-attention (+ norm2 / norm3): one warp per token at three register sizes, four warps per token
    add("xattn2_c320", case_xattn2, M=9216, C=320)
    add("xattn2_c640", case_xattn2, M=2304, C=640)
    add("xattn2_c1280_wide", case_xattn2, M=576, C=1280)
    add("xattn2_c1280_wide_odd", case_xattn2, M=145, C=1280)
    add("xattn2_c1280_batched", case_xattn2, M=2 * 576, C=1280)
    add("xattn2_c320_offset", case_xattn2, M=2304, C=320, offset=100.0)
    add("layernorm_320", case_layernorm, M=9216, C=320)
    add("layernorm_1280", case_layernorm, M=576, C=1280)
    add("layernorm_320_offset", case_layernorm, M=9216, C=320, offset=100.0)
    add("layernorm_1280_offset", case_layernorm, M=576, C=1280, offset=100.0)
    add("s2d", case_s2d, NB=2, H=24, W=16, C=128)
    add("s2d_odd", case_s2d, NB=1, H=27, W=13, C=64)
    add("upsample", case_upsample, NB=2, H=12, W=8, C=64)
    add("upsample_crop", case_upsample, NB=2, H=14, W=7, C=64, crop=True)
    add("softmax_rows_84", case_softmax_rows, M=84, n=84, ld=128)
    add("softmax_rows_324_logits80", case_softmax_rows, M=324, n=324, ld=384, std=40.0)
    add("softmax_rows_4096", case_softmax_rows, M=64, n=4096, ld=4096)
    # VAE attention score rows at 4032 x 3024 and 4000 x 3000
    for n, ld in ((190512, 190528), (187500, 187520)):
        for std in (3.0, 40.0):
            add(f"softmax_rows_{n}_std{std:g}", case_softmax_rows, M=64, n=n, ld=ld, std=std)
    add("transpose_84x512", case_transpose, M=84, N=512, ld=128)
    add("transpose_4096x512", case_transpose, M=4096, N=512, ld=4096)
    add("transpose_190512x512", case_transpose, M=190512, N=512, ld=190528)
    return cases


# -------------------------------------------------------------------------------------------------
def _timeit(fn, iters=10):
    import torch

    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _check(res, key, out, ref, bound):
    """Per-element check of one output; the case passes when every output's worst |d| / bound is <= 1."""
    from tests import ops_ref

    r = ops_ref.within(out, ref, bound)
    res[key] = r
    res["worst"] = max(res.get("worst", 0.0), r["worst"])
    res["ok"] = res.get("ok", True) and (not r["nan"]) and r["worst"] <= 1.0
    return r


def _record(name, res):
    from tests import ops_ref

    ops_ref.record(f"ops.{name}.worst", res["worst"])
    for k in ("c_acc", "c_p"):
        if k in res:
            ops_ref.record(f"ops.{name}.{k}", res[k])


def _c_acc(res, out, ref, K, absprod, scale, pre):
    """What this case says about wgmma's accumulation: the error of an fp32 output beyond the epilogue's own roundings,
    over K 2^-24 |scale| |A||B|^T."""
    import torch

    from tests import ops_ref

    d = ((out.double() - ref).abs() - ops_ref.R_F32_OUT * (pre.abs() + ref.abs())).clamp(min=0)
    den = K * ops_ref.U_F32 * abs(scale) * absprod
    r = torch.where(den > 0, d / den, torch.zeros_like(d))
    res["c_acc"] = max(res.get("c_acc", 0.0), float(r.max().item()))


def _sched_k(kx, kv, kz):
    import torch

    return torch.tensor([kx, kv, kz], dtype=torch.float32, device="cuda")


def case_linear(M, N, K, block_n, bias=False, residual=False, bf16out=False, geglu=False, splits=0, stages=0,
                silu=False, scale=None, ldo=0, K2=0, probs=False):
    """probs: A holds rows of softmax probabilities (non-negative, summing to 1) and W unit-variance values, as in the
    VAE attention's P V GEMM."""
    import torch

    from marigold_b200 import _lib, ops
    from tests import ops_ref as R

    g = torch.Generator(device="cuda").manual_seed(1)
    Kt = K + K2
    a = torch.randn(M, K, device="cuda", generator=g)
    a = (torch.softmax(a, dim=1) if probs else a).to(torch.bfloat16)
    a2 = torch.randn(M, K2, device="cuda", generator=g).to(torch.bfloat16) if K2 else None
    w = (torch.randn(N, Kt, device="cuda", generator=g) / (1.0 if probs else Kt ** 0.5)).to(torch.bfloat16)
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    n_out = N // 2 if geglu else N
    ld = ldo or n_out
    r = torch.randn(M, ld, device="cuda", generator=g) if residual else None
    flags = (_lib.EPI_GEGLU if geglu else 0) | (_lib.EPI_SILU if silu else 0) | (_lib.EPI_SCALE if scale else 0)
    sc = scale if scale else 1.0
    ws = torch.empty(max(splits, 16) * M * N, device="cuda") if (splits > 1 or block_n == 0) else None
    # float64 reference on the bf16 operands
    acc, absprod = R.matmul64(torch.cat([a, a2], 1) if K2 else a, w)
    b64 = R.f64(b) if b is not None else torch.zeros(N, dtype=torch.float64, device="cuda")
    w_used, b_used = w, b
    act_gain = act_err = None
    if geglu:
        # the library expects [value | gate] halves per block_n tile (finalize_weights' packing)
        half, nt = block_n // 2, N // block_n
        val_rows = torch.arange(N // 2, device="cuda").reshape(nt, half)
        perm = torch.cat([val_rows, val_rows + N // 2], dim=1).reshape(-1)
        w_used = w[perm].contiguous()
        b_used = b[perm].contiguous() if b is not None else None
        t = acc + b64
        v, gt = t[:, : N // 2], t[:, N // 2:]
        pre = v * R.gelu64(gt)
        e_acc = R.acc_bound(Kt, absprod) + R.U_F32 * t.abs()
        act_gain = 1.0  # propagated explicitly below
        act_err = (R.gelu64(gt).abs() * e_acc[:, : N // 2] + v.abs() * R.GELU_GAIN * e_acc[:, N // 2:]
                   + R.R_ACT * (v.abs() + pre.abs()))
        absprod_b = torch.zeros_like(pre)
    else:
        t = acc * sc + b64
        pre = R.silu64(t) if silu else t
        if silu:
            act_gain = R.SILU_GAIN
            act_err = R.R_ACT * pre.abs() + R.SILU_GAIN * R.U_F32 * t.abs()
        absprod_b = absprod
    ref = pre + (R.f64(r)[:, :n_out] if r is not None else 0)
    sentinel = 12345.0
    of = torch.full((M, ld), sentinel, device="cuda")
    ob = torch.full((M, ld), sentinel, device="cuda", dtype=torch.bfloat16) if bf16out else None
    run = lambda: ops.linear_ex(a, w_used, b_used, r, a2=a2, out=of, out_bf16=ob, ldo=ldo, flags=flags, scale=sc,
                                block_n=block_n, splits=splits, stages=stages, ws=ws)
    run()
    torch.cuda.synchronize()
    res = {}
    kw = dict(pre=pre, scale=sc, act_gain=act_gain, act_err=act_err)
    _check(res, "f32", of[:, :n_out], ref, R.gemm_bound(Kt, absprod_b, ref, False, **kw))
    if ob is not None:
        _check(res, "bf16", ob[:, :n_out], ref, R.gemm_bound(Kt, absprod_b, ref, True, **kw))
    if not geglu and not silu:
        _c_acc(res, of[:, :n_out], ref, Kt, absprod, sc, pre)
    if ld > n_out:   # the row padding of an ldo > N output is never written
        res["pad_untouched"] = bool((of[:, n_out:] == sentinel).all().item()) and (
            ob is None or bool((ob[:, n_out:] == torch.tensor(sentinel, dtype=torch.bfloat16)).all().item()))
        res["ok"] = res["ok"] and res["pad_untouched"]
    res["ms"] = _timeit(run)
    res["tflops"] = 2.0 * M * N * Kt / res["ms"] / 1e9
    return res


def _conv_inputs(NB, Hin, Win, Cin, Cout, kind, Cin2, Hout, Wout, bias, residual, seed=2):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    taps = 1 if kind == 1 else 3
    x = torch.randn(NB, Hin, Win, Cin, device="cuda", generator=g)  # NHWC fp32
    wt = (torch.randn(Cout, Cin, taps, taps, device="cuda", generator=g) / (taps * taps * Cin + Cin2) ** 0.5)
    x2 = torch.randn(NB, Hout, Wout, Cin2, device="cuda", generator=g).to(torch.bfloat16) if Cin2 else None
    wsc = (torch.randn(Cout, Cin2, device="cuda", generator=g) / (9 * Cin + Cin2) ** 0.5).to(torch.bfloat16) if Cin2 else None
    b = torch.randn(Cout, device="cuda", generator=g) if bias else None
    r = torch.randn(NB, Hout, Wout, Cout, device="cuda", generator=g) if residual else None
    return x, wt.to(torch.bfloat16), x2, wsc, b, r


def _conv_ref(x, wb, x2, wsc, b, kind):
    """float64 conv (and |.| conv) NCHW of the bf16-rounded operands, with the 1x1 second operand added."""
    import torch.nn.functional as F

    from tests import ops_ref as R

    xn = x.to(torch_bf16()).permute(0, 3, 1, 2)
    if kind in (0, 1):
        acc, absprod = R.conv64(xn, wb, 1, 1 if kind == 0 else 0)
    elif kind == 2:
        acc, absprod = R.conv64(xn, wb, 2, 1)
    else:
        acc, absprod = R.conv64(F.pad(xn.double(), (0, 1, 0, 1)), wb, 2, 0)
    if x2 is not None:
        a2, p2 = R.conv64(x2.permute(0, 3, 1, 2), wsc[:, :, None, None], 1, 0)
        acc, absprod = acc + a2, absprod + p2
    if b is not None:
        acc = acc + R.f64(b)[None, :, None, None]
    return acc, absprod   # NCHW, bias included in acc


def torch_bf16():
    import torch

    return torch.bfloat16


def case_conv(NB, Cin, Cout, kind, block_n, H=None, W=None, Hin=None, Win=None, bias=False, residual=False, splits=0,
              special=None, Cin2=0, scale=None):
    import torch

    from marigold_b200 import _lib, ops
    from tests import ops_ref as R

    stride = 2 if kind in (2, 3) else 1
    Hin, Win = Hin or H * stride, Win or W * stride
    if kind == 2:
        H, W = (Hin + 1) // 2, (Win + 1) // 2
    elif kind == 3:
        H, W = Hin // 2, Win // 2
    else:
        H, W = Hin, Win
    x, wb, x2, wsc, b, r = _conv_inputs(NB, Hin, Win, Cin, Cout, kind, Cin2, H, W, bias, residual)
    K = (1 if kind == 1 else 9) * Cin + Cin2
    acc, absprod = _conv_ref(x, wb, x2, wsc, b, kind)
    sc = scale if scale else 1.0
    if scale:
        acc = (acc - (R.f64(b)[None, :, None, None] if b is not None else 0)) * sc + (
            R.f64(b)[None, :, None, None] if b is not None else 0)
    if kind in (2, 3):
        x_in = ops.space_to_depth(x)
        Hs, Ws = (Hin + 1) // 2, (Win + 1) // 2
    else:
        x_in = x.to(torch.bfloat16).contiguous()
        Hs = Ws = 0
    wp = ops.pack_conv_weight(wb)
    if Cin2:
        wp = torch.cat([wp, wsc], dim=1).contiguous()
    flags = _lib.EPI_SCALE if scale else 0
    hw = H * W
    sched = {}
    e_acc = R.acc_bound(K, absprod, sc) + R.R_F32_OUT * acc.abs()   # NCHW
    if special is None:
        ref = acc.permute(0, 2, 3, 1)
        pre = ref
        if r is not None:
            ref = ref + R.f64(r)
        of = torch.empty(NB, H, W, Cout, device="cuda")
        bound = e_acc.permute(0, 2, 3, 1) + R.R_F32_OUT * ref.abs() + R.TINY
    elif special in ("nchw", "unit"):
        flags |= _lib.EPI_NCHW | (_lib.EPI_UNIT if special == "unit" else 0)
        ref, bound = acc, e_acc + R.TINY
        if special == "unit":
            ref = (acc.clamp(-1, 1) + 1) / 2
            bound = e_acc / 2 + R.R_F32_OUT + R.TINY
        of = torch.empty(NB, Cout, H, W, device="cuda")
    elif special == "depth":
        flags |= _lib.EPI_DEPTH
        ref = (acc.mean(dim=1, keepdim=True).clamp(-1, 1) + 1) / 2
        bound = e_acc.sum(dim=1, keepdim=True) / 6 + R.R_F32_OUT + R.TINY
        of = torch.empty(NB, 1, H, W, device="cuda")
    elif special == "normals":
        flags |= _lib.EPI_NORMALS
        c = acc.clamp(-1, 1)
        nrm = torch.norm(c, dim=1, keepdim=True).clamp(min=1e-6)
        ref = c / nrm
        # d(c / |c|) <= 2 |dc| / |c| (first order), plus a few fp32 roundings
        bound = 2 * e_acc.norm(dim=1, keepdim=True) / nrm + R.R_F32_OUT + R.TINY
        of = torch.empty(NB, 3, H, W, device="cuda")
    elif special == "sched":
        flags |= _lib.EPI_SCHED
        kx, kv, kz = 0.9, -0.37, 0.21
        sx = torch.randn(NB, H, W, Cout, device="cuda")
        sz = torch.randn(NB, H, W, Cout, device="cuda")
        model = acc.permute(0, 2, 3, 1)
        # the coefficients as the device holds them (fp32)
        kx64, kv64, kz64 = (float(torch.tensor(v, dtype=torch.float32)) for v in (kx, kv, kz))
        ref = kx64 * R.f64(sx) + kv64 * model + kz64 * R.f64(sz)
        bound = (abs(kv64) * e_acc.permute(0, 2, 3, 1)
                 + R.R_F32_OUT * (abs(kx64) * sx.abs() + abs(kv64) * model.abs() + abs(kz64) * sz.abs()).double()
                 + R.TINY)
        aux = torch.empty(NB, H, W, Cout, device="cuda")
        sched = dict(sched_x=sx, sched_z=sz, sched_k=_sched_k(kx, kv, kz), aux_out=aux)
        of = torch.empty(NB, H, W, Cout, device="cuda")
    ws = torch.empty(max(splits, 16) * NB * H * W * Cout, device="cuda") if (splits > 1 or block_n == 0) else None
    run = lambda: ops.conv2d_ex(x_in, wp, b, NB, H, W, Cin, Cout, kind=kind, x2=x2, Cin2=Cin2, Hsrc=Hs, Wsrc=Ws,
                                residual=r, out=of, flags=flags, scale=sc, block_n=block_n, splits=splits, ws=ws,
                                **sched)
    run()
    torch.cuda.synchronize()
    res = {}
    _check(res, "f32", of, ref, bound)
    if special == "sched":
        aux_ref = acc.permute(0, 2, 3, 1)
        _check(res, "aux", sched["aux_out"], aux_ref, e_acc.permute(0, 2, 3, 1) + R.TINY)
    if special is None and r is None:
        _c_acc(res, of, ref, K, absprod.permute(0, 2, 3, 1), sc, pre)
    res["ms"] = _timeit(run)
    res["tflops"] = 2.0 * NB * H * W * Cout * K / res["ms"] / 1e9
    return res


def case_sched_exact(NB, H, W, Cin, Cout):
    """EPI_SCHED with kz = 0 and no noise: out == kx x + kv (acc + b) bit for bit, and aux_out == the plain conv output
    (same 16-wide kernel). kx, kv are powers of two, so each product is exact whatever the compiler contracts."""
    import torch

    from marigold_b200 import _lib, ops

    x, wb, _, _, b, _ = _conv_inputs(NB, H, W, Cin, Cout, 0, 0, H, W, True, False, seed=5)
    x_in, wp = x.to(torch.bfloat16).contiguous(), ops.pack_conv_weight(wb)
    plain = torch.empty(NB, H, W, Cout, device="cuda")
    ops.conv2d_ex(x_in, wp, b, NB, H, W, Cin, Cout, out=plain, block_n=16)
    kx, kv = 0.5, -0.25
    sx = torch.randn(NB, H, W, Cout, device="cuda")
    out, aux = torch.empty_like(plain), torch.empty_like(plain)
    ops.conv2d_ex(x_in, wp, b, NB, H, W, Cin, Cout, out=out, flags=_lib.EPI_SCHED, sched_x=sx, sched_z=None,
                  sched_k=_sched_k(kx, kv, 0.0), aux_out=aux, block_n=0)
    torch.cuda.synchronize()
    want = sx * kx + plain * kv
    ok_out, ok_aux = bool(torch.equal(out, want)), bool(torch.equal(aux, plain))
    return {"ok": ok_out and ok_aux, "worst": 0.0 if ok_out and ok_aux else math.inf, "out_exact": ok_out,
            "aux_exact": ok_aux}


def attn_splits(NB, T, C):
    """Restatement of flash_attn64_splits (attn_tc.cu): the KV split the operator runs."""
    units, nkv, slots = ((T + 127) // 128) * (C // 64) * NB, (T + 63) // 64, 132 * 2
    best, best_t = 1, 1e30
    for s in range(1, 9):
        if s > 1 and nkv // s < 6:
            break
        t = ((units * s + slots - 1) // slots) * (nkv / s + 15.0) + (8.0 if s > 1 else 0.0)
        if t < best_t - 1e-9:
            best_t, best = t, s
    return best


def dominant_key(q, k, at, logit, scale, d, seed):
    """Make key `at` of every image the dominant one for every query: q gains a shared random +-1 direction u, key
    `at` becomes logit / (d scale) u, so that each query's logit for it is about `logit` (d: the dot product's length,
    the head dim) while the others keep their spread. q, k: [NB, T, C], changed in place."""
    import torch

    g = torch.Generator(device=q.device).manual_seed(seed)
    u = torch.randint(0, 2, (q.shape[-1],), device=q.device, generator=g).float() * 2 - 1
    q += u
    k[:, at] = logit / (d * scale) * u


def check_rows(T, block, seed, n_random=2048):
    """Query rows checked where the float64 reference of every row is out of reach: the first and the last block of
    `block` rows, the rows either side of every block boundary, the last 64 rows and n_random seeded rows."""
    import torch

    rows = set(range(min(block, T))) | set(range(max(0, (T - 1) // block * block), T)) | set(range(max(0, T - 64), T))
    for r0 in range(block, T, block):
        rows |= {r0 - 1, r0}
    g = torch.Generator().manual_seed(seed)
    rows |= set(torch.randint(0, T, (n_random,), generator=g).tolist())
    return torch.tensor(sorted(rows), dtype=torch.long)


# Above this many float64 probabilities (NB heads T^2) case_attn holds its reference to check_rows' rows only
_ATTN_WHOLE_P = 1 << 30


def case_attn(NB, T, C, qk_std=1.0, dominant=False, dominant_at=None):
    """dominant_at: index of a key made dominant for every query (dominant_key, logit 14)."""
    import torch

    from marigold_b200 import _lib, ops
    from tests import ops_ref as R

    g = torch.Generator(device="cuda").manual_seed(3)
    heads = C // 64
    q = torch.randn(NB * T, C, device="cuda", generator=g) * qk_std
    k = torch.randn(NB * T, C, device="cuda", generator=g) * qk_std
    v = torch.randn(NB * T, C, device="cuda", generator=g)
    if dominant and T > 7:
        # key 7 of every image is 6 x query 0: query 0's logit for it exceeds the others by ~48
        k.view(NB, T, C)[:, 7] = 6 * q.view(NB, T, C)[:, 0]
    if dominant_at is not None:
        dominant_key(q.view(NB, T, C), k.view(NB, T, C), dominant_at, 14.0, 0.125, 64, seed=T)
    qkv = torch.cat([q, k, v], 1).to(torch.bfloat16).contiguous()
    del q, k, v
    q64, k64, v64 = [R.f64(t).reshape(NB, T, heads, 64).permute(0, 2, 1, 3) for t in qkv.split(C, dim=1)]
    # the flash kernel takes queries in tiles of 128 rows
    rows = check_rows(T, 128, seed=T).cuda() if NB * heads * T * T > _ATTN_WHOLE_P else None
    if rows is None:
        p = torch.softmax((q64 @ k64.transpose(-1, -2)) * 0.125, dim=-1)
        ref = (p @ v64).permute(0, 2, 1, 3).reshape(NB * T, C)
        pv_abs = (p @ v64.abs()).permute(0, 2, 1, 3).reshape(NB * T, C)
        del p
    else:
        ref = torch.empty(NB, heads, len(rows), 64, dtype=torch.float64, device="cuda")
        pv_abs = torch.empty_like(ref)
        step = max(1, (1 << 26) // (NB * heads * T))
        for i in range(0, len(rows), step):
            rr = rows[i:i + step]
            p = torch.softmax((q64[:, :, rr] @ k64.transpose(-1, -2)) * 0.125, dim=-1)
            ref[:, :, i:i + step], pv_abs[:, :, i:i + step] = p @ v64, p @ v64.abs()
            del p
        ref, pv_abs = (t.permute(0, 2, 1, 3).reshape(NB * len(rows), C) for t in (ref, pv_abs))
    del q64, k64, v64
    lib = _lib.load()
    n0 = lib.mgb_launch_count()
    out = ops.flash_attn64(qkv, NB, T, C, 0.125)
    launches = lib.mgb_launch_count() - n0
    torch.cuda.synchronize()
    res = {"splits": attn_splits(NB, T, C), "launches": launches}
    if rows is not None:
        out = out.view(NB, T, C)[:, rows].reshape(NB * len(rows), C)
        res["rows_checked"] = len(rows)
    _check(res, "bf16", out, ref, R.attn_bound(ref, pv_abs))
    d = (out.double() - ref).abs()
    excess = (d - R.U_BF16 * ref.abs()).clamp(min=0) / (R.U_BF16 * pv_abs + R.TINY)
    res["c_p"] = float(excess.max().item())
    res["ok"] = res["ok"] and launches == (2 if res["splits"] > 1 else 1)
    res["ms"] = _timeit(lambda: ops.flash_attn64(qkv, NB, T, C, 0.125))
    res["tflops"] = 4.0 * NB * heads * T * T * 64 / res["ms"] / 1e9
    return res


def _norm_mag(x64, mean, rstd, gamma, beta):
    """Magnitudes an fp32 normalise + affine combines: |gamma| (|x - mean| + |mean| + 1) rstd + |beta|."""
    return gamma.abs() * ((x64 - mean).abs() + mean.abs() + 1.0 / rstd) * rstd + beta.abs()


# Above this many elements the float64 reference of the whole tensor would not fit beside it on the device: the statistics
# are then computed, and the outputs checked, for images 0, NB // 2 and NB - 1 only.
_GN_WHOLE_ELEMS = 1 << 27


def case_groupnorm(NB, HW, C, G, eps, silu, Cb=0, offset=0.5):
    import torch

    from marigold_b200 import ops
    from tests import ops_ref as R

    g = torch.Generator(device="cuda").manual_seed(4)
    Ct = C + Cb
    x = torch.randn(NB, HW, Ct, device="cuda", generator=g).mul_(2).add_(offset)
    gamma = torch.randn(Ct, device="cuda", generator=g)
    beta = torch.randn(Ct, device="cuda", generator=g)
    xa, xb = x[..., :C].contiguous(), (x[..., C:].contiguous() if Cb else None)
    ga, be = R.f64(gamma).reshape(G, Ct // G), R.f64(beta).reshape(G, Ct // G)
    run = lambda: ops.groupnorm_ex(xa, xb, gamma, beta, NB, HW, G, eps, silu, raw_copy=True)
    y, raw = run()
    torch.cuda.synchronize()
    res = {"raw_exact": True}
    images = range(NB) if NB * HW * Ct <= _GN_WHOLE_ELEMS else sorted({0, NB // 2, NB - 1})
    for i in images:
        # float64 statistics of image i alone (the kernel's are per image too)
        x64 = R.f64(x[i]).reshape(HW, G, Ct // G)
        mean = x64.mean(dim=(0, 2), keepdim=True)
        var = x64.var(dim=(0, 2), keepdim=True, unbiased=False)
        rstd = 1.0 / torch.sqrt(var + eps)
        t = ((x64 - mean) * rstd * ga + be)
        mag = _norm_mag(x64, mean, rstd, ga, be).reshape(HW, Ct)
        del x64
        t = t.reshape(HW, Ct)
        ref = R.silu64(t) if silu else t
        del t
        r = _check(res, f"bf16[{i}]", y[i], ref, R.bf16_bound(ref, mag * (R.SILU_GAIN if silu else 1.0)))
        r["index"] = (i,) + r["index"]
        del ref, mag
        res["raw_exact"] = res["raw_exact"] and bool(torch.equal(raw[i], x[i].to(torch.bfloat16)))
    res["images_checked"] = list(images)
    res["ok"] = res["ok"] and res["raw_exact"]
    del y, raw
    res["ms"] = _timeit(run)
    res["gbs"] = NB * HW * Ct * (4 + 2 + 2) / res["ms"] / 1e6
    return res


def case_xattn2(M, C, offset=0.2):
    import torch
    import torch.nn.functional as F

    from marigold_b200 import ops
    from tests import ops_ref as R

    H = C // 64
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(M, C, device="cuda", generator=g) * 1.5 + offset
    p = [torch.randn(C, device="cuda", generator=g) * s + o for s, o in ((0.3, 1.0), (0.3, 0.0), (0.3, 1.0), (0.3, 0.0))]
    G = (torch.randn(H, C, device="cuda", generator=g) / C ** 0.5 * 4).to(torch.bfloat16)
    U = (torch.randn(H, C, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    c1 = torch.randn(C, device="cuda", generator=g) * 0.5
    GU = torch.stack([G, U]).contiguous()
    x64, G64, U64 = R.f64(x), R.f64(G), R.f64(U)
    p64 = [R.f64(t) for t in p]
    mu = x64.mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(x64.var(1, keepdim=True, unbiased=False) + 1e-5)
    z = F.layer_norm(x64, (C,), p64[0], p64[1], 1e-5)
    zmag = _norm_mag(x64, mu, rs, p64[0], p64[1])
    w = torch.sigmoid(0.125 * z @ G64.t())
    yf = x64 + R.f64(c1) + w @ U64
    # y sums x, c1 and H gated rows; the gates' logits carry LN2's and the fp32 dot's errors (|sigmoid'| <= 1/4)
    ymag = x64.abs() + R.f64(c1).abs() + w @ U64.abs() + 0.25 * 0.125 * (zmag @ G64.abs().t()) @ U64.abs()
    mu3 = yf.mean(1, keepdim=True)
    rs3 = 1.0 / torch.sqrt(yf.var(1, keepdim=True, unbiased=False) + 1e-5)
    af = F.layer_norm(yf, (C,), p64[2], p64[3], 1e-5)
    amag = _norm_mag(yf, mu3, rs3, p64[2], p64[3]) + p64[2].abs() * rs3 * (ymag + ymag.mean(1, keepdim=True))
    run = lambda: ops.xattn2(x, p[0], p[1], p[2], p[3], GU, c1, H, 0.125)
    y, a = run()
    torch.cuda.synchronize()
    res = {}
    _check(res, "y", y, yf, R.bf16_bound(yf, ymag))
    _check(res, "a", a, af, R.bf16_bound(af, amag))
    res["ms"] = _timeit(run)
    return res


def case_layernorm(M, C, offset=-1.0):
    import torch
    import torch.nn.functional as F

    from marigold_b200 import ops
    from tests import ops_ref as R

    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(M, C, device="cuda", generator=g) * 3 + offset
    gamma = torch.randn(C, device="cuda", generator=g)
    beta = torch.randn(C, device="cuda", generator=g)
    x64 = R.f64(x)
    ref = F.layer_norm(x64, (C,), R.f64(gamma), R.f64(beta), 1e-5)
    mu = x64.mean(1, keepdim=True)
    rs = 1.0 / torch.sqrt(x64.var(1, keepdim=True, unbiased=False) + 1e-5)
    run = lambda: ops.layernorm(x, gamma, beta)
    out = run()
    torch.cuda.synchronize()
    res = {}
    _check(res, "bf16", out, ref, R.bf16_bound(ref, _norm_mag(x64, mu, rs, R.f64(gamma), R.f64(beta))))
    res["ms"] = _timeit(run)
    return res


def _exact(res, key, out, ref):
    import torch

    res[key] = bool(torch.equal(out, ref))
    res["ok"] = res.get("ok", True) and res[key]
    res["worst"] = max(res.get("worst", 0.0), 0.0 if res[key] else math.inf)


def case_s2d(NB, H, W, C):
    import torch

    from marigold_b200 import ops

    x = torch.randn(NB, H, W, C, device="cuda")
    out = ops.space_to_depth(x)
    # odd sizes: planes hold ceil(H/2) x ceil(W/2) entries, zero where the source pixel does not exist
    xp = torch.nn.functional.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    ref = torch.stack([xp[:, a::2, b::2] for a in (0, 1) for b in (0, 1)], dim=1).to(torch.bfloat16)
    res = {}
    _exact(res, "exact", out, ref)
    return res


def case_upsample(NB, H, W, C, crop=False):
    import torch

    from marigold_b200 import ops

    x = torch.randn(NB, H, W, C, device="cuda")
    Ho, Wo = (2 * H - 1, 2 * W - 1) if crop else (2 * H, 2 * W)
    out = ops.upsample2x(x, Ho, Wo)
    # F.interpolate(size=(Ho, Wo), mode="nearest") as diffusers' Upsample2D does with upsample_size
    ref = torch.nn.functional.interpolate(x.permute(0, 3, 1, 2), size=(Ho, Wo), mode="nearest")
    res = {}
    _exact(res, "exact", out, ref.permute(0, 2, 3, 1).to(torch.bfloat16))
    return res


def case_softmax_rows(M, n, ld, std=3.0):
    import torch

    from marigold_b200 import ops
    from tests import ops_ref as R

    g = torch.Generator(device="cuda").manual_seed(6)
    s = torch.randn(M, ld, device="cuda", generator=g) * std
    s[:, n:] = float("nan")          # never read
    p = ops.softmax_rows(s, n)
    torch.cuda.synchronize()
    s64 = R.f64(s[:, :n])
    ref = torch.softmax(s64, dim=1)
    # bf16 rounding, plus fp32 exp (argument rounding grows with |s - max|) and the fp32 row sum of n terms
    dist = (s64.max(dim=1, keepdim=True).values - s64)
    bound = ref * (R.U_BF16 + R.softmax_rel(n, dist, ref)) + R.TINY
    res = {}
    _check(res, "bf16", p[:, :n], ref, bound)
    _exact(res, "pad_zero", p[:, n:], torch.zeros_like(p[:, n:]))
    return res


def case_transpose(M, N, ld):
    import torch

    from marigold_b200 import ops

    x = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    y = ops.transpose_bf16(x, ld)
    ref = torch.zeros(N, ld, dtype=torch.bfloat16, device="cuda")
    ref[:, :M] = x.t()
    res = {}
    _exact(res, "exact", y, ref)
    return res
