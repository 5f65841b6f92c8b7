"""One image on several ranks (`-m gpu`): the attentions' query rows split over the ranks (mgb_set_row_split).

- the flash attention on ranges of query blocks writes the whole launch's rows bit for bit, and no others;
- virtual ranks in one process: every exchange of an unsplit call is recorded through the hook at world 1, then each
  rank r of G runs the call with an exchange that checks r's rows against the recording and fills in the rest: encode,
  DDIM and LCM denoising, and the depth, normals and 2-target IID decodes give the unsplit call's bits;
- two and three processes on the one GPU under gloo, the split forced below its threshold: every rank's maps equal the
  one-process batch_size=1 call's;
- a handle whose split was cleared sizes, plans and graphs its work as one that never had it; errors."""
import os
import socket

import numpy as np
import pytest
import torch

from marigold_b200 import ops, parallel
from marigold_b200._lib import MgbError
from tests.helpers import arena_plan, attn_blocks, engine_from_oracle, oracle_models, synthetic_image

pytestmark = pytest.mark.gpu

NUM_SMS = 132


def _splits(NB, T, C):
    """flash_attn64_splits (csrc/attn_tc.cu), restated to pick a case that runs split-KV."""
    units, nkv, slots = -(-T // 128) * (C // 64) * NB, -(-T // 64), NUM_SMS * 2
    best, best_t = 1, 1e30
    for s in range(1, 9):
        if s > 1 and nkv // s < 6:
            break
        t = -(-(units * s) // slots) * (nkv / s + 15.0) + (8.0 if s > 1 else 0.0)
        if t < best_t - 1e-9:
            best, best_t = s, t
    return best


# ---- flash attention on query-block ranges ------------------------------------------------------------------------

@pytest.mark.parametrize("T,C", [(2304, 320), (2304, 1280), (9216, 320), (9216, 640), (9216, 1280), (190512, 320),
                                 (190512, 640), (381024, 320)])
def test_flash_attention_block_ranges(T, C):
    g = torch.Generator(device="cuda").manual_seed(T + C)
    qkv = (torch.randn(T, 3 * C, device="cuda", generator=g) * 2).to(torch.bfloat16)
    full = ops.flash_attn64(qkv, 1, T, C, 0.125)
    nqb = -(-T // 128)
    if (T, C) == (2304, 320):
        assert _splits(1, T, C) > 1               # the split-KV path with its combine pass
    for G in (2, 3, 8):
        chunk = parallel.row_split_chunk(T, G) // 128
        joined = torch.full_like(full, -1, dtype=torch.int16).view(torch.bfloat16)       # NaN everywhere
        owners = 0
        for r in range(G):
            b0, b1 = min(nqb, r * chunk), min(nqb, (r + 1) * chunk)
            out = torch.full_like(full, -1, dtype=torch.int16).view(torch.bfloat16)
            ops.flash_attn64_blocks(qkv, 1, T, C, 0.125, b0, b1, out=out)
            rows = parallel.row_split_rows(T, r, G)
            assert (rows.start, rows.stop) == (min(T, 128 * b0), min(T, 128 * b1))
            assert torch.equal(out[rows.start:rows.stop], full[rows.start:rows.stop]), (G, r)
            untouched = torch.cat([out[:rows.start], out[rows.stop:]]).view(torch.int16)
            assert bool((untouched == -1).all()), (G, r)        # no other row written
            joined[rows.start:rows.stop] = out[rows.start:rows.stop]
            owners += b1 > b0
        assert torch.equal(joined, full), G
        if T == 2304 and G == 8:
            assert owners < G                     # ranks that own no block


def test_flash_attention_block_range_errors():
    qkv = torch.zeros(300, 3 * 64, dtype=torch.bfloat16, device="cuda")
    out = torch.full((300, 64), -1, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    ops.flash_attn64_blocks(qkv, 1, 300, 64, 0.125, 2, 2, out=out)                         # empty: nothing written
    torch.cuda.synchronize()
    assert bool((out.view(torch.int16) == -1).all())
    for b0, b1 in ((0, 4), (2, 1), (-1, 1)):
        with pytest.raises(MgbError, match="query blocks"):
            ops.flash_attn64_blocks(qkv, 1, 300, 64, 0.125, b0, b1, out=out)


# ---- virtual ranks in one process ---------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def depth_eng():
    unet, vae, text = oracle_models("tiny")
    eng = engine_from_oracle(unet, vae, text)
    yield eng
    eng.set_row_split()
    eng.close()


@pytest.fixture(scope="module")
def iid_eng():
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
    eng.set_text_embedding(text)
    yield eng
    eng.set_row_split()
    eng.close()


def _unet_attn_shapes(eng, lh, lw):
    """(T, C) of the UNet step's 16 attentions in execution order (csrc/net.cu unet_forward)."""
    ch, L = eng.cfg.unet_block_channels, eng.cfg.unet_layers_per_block
    hs, ws = [lh], [lw]
    for _ in range(3):
        hs.append((hs[-1] + 1) // 2)
        ws.append((ws[-1] + 1) // 2)
    down = [(hs[i] * ws[i], ch[i]) for i in range(3) for _ in range(L)]
    mid = [(hs[3] * ws[3], ch[3])]
    up = [(hs[3 - i] * ws[3 - i], ch[3 - i]) for i in range(1, 4) for _ in range(L + 1)]
    return down + mid + up


def _schedule(eng, lcm, steps):
    from marigold_b200.schedulers import DDIMScheduler, LCMScheduler

    s = LCMScheduler() if lcm else DDIMScheduler()
    s.set_timesteps(steps)
    kx, kv, kz = s.coefficients()
    eng.set_schedule(s.timesteps, kx, kv, kz)


def _workloads(eng, H, W, n_targets):
    """name -> (callable, [(T, C)] of its exchanges in order)."""
    g = torch.Generator().manual_seed(H * W)
    rgb = (synthetic_image(max(H, W), seed=3)[:, :, :H, :W].float() / 255 * 2 - 1).cuda().contiguous()
    lh, lw = H // 8, W // 8
    ct = 4 * n_targets
    lat = torch.randn(1, 4, lh, lw, generator=g).cuda()
    z0 = torch.randn(1, ct, lh, lw, generator=g).cuda()
    sn = torch.randn(3, 1, ct, lh, lw, generator=g).cuda()
    tgt = torch.randn(1, ct, lh, lw, generator=g).cuda()
    vae_c = eng.cfg.vae_block_channels[3]
    T = lh * lw
    unet = _unet_attn_shapes(eng, lh, lw)

    def denoise(lcm, steps, noise):
        def run():
            _schedule(eng, lcm, steps)
            return eng.denoise(lat, z0, noise)
        return run, unet * steps

    w = {"encode": (lambda: eng.encode(rgb), [(T, vae_c)]),
         "ddim": denoise(False, 2, None),
         "lcm": denoise(True, 4, sn)}
    if n_targets == 1:
        w["decode_depth"] = (lambda: eng.decode(lat, 0), [(T, vae_c)])
        w["decode_normals"] = (lambda: eng.decode(lat, 1), [(T, vae_c)])
    else:
        w["decode_iid"] = (lambda: torch.cat([eng.decode(tgt[:, 4 * i:4 * i + 4].contiguous(), 3)
                                              for i in range(n_targets)], 1), [(T, vae_c)] * n_targets)
    return w


def _check_virtual_ranks(eng, workloads):
    """Each workload at world 1 through the hook (recording every exchange), then as every rank r of G in 2, 3, 8 with
    an exchange that checks r's rows against the recording and fills in the rest: the unsplit call's bits each time."""
    for name, (run, shapes) in workloads.items():
        eng.set_row_split()
        ref = run().clone()
        recorded = []
        eng.set_row_split(0, 1, lambda buf, r, g: recorded.append(buf.clone()))
        assert torch.equal(run(), ref), name                         # world 1: one rank computes every row
        assert len(recorded) == len(shapes), name
        for G in (2, 3, 8):
            for rank in range(G):
                k = [0]
                bad = []

                def exchange(buf, r, g):
                    T, C = shapes[k[0]]
                    rec = recorded[k[0]]
                    k[0] += 1
                    assert (r, g) == (rank, G) and buf.numel() == g * parallel.row_split_chunk(T, g) * C * 2
                    rows = parallel.row_split_rows(T, r, g)
                    lo, hi = rows.start * C * 2, rows.stop * C * 2
                    if not torch.equal(buf[lo:hi], rec[lo:hi]):
                        bad.append(k[0] - 1)
                    buf[:lo] = rec[:lo]
                    buf[hi:T * C * 2] = rec[hi:T * C * 2]

                eng.set_row_split(rank, G, exchange)
                out = run()
                assert not bad, (name, G, rank, bad)
                assert k[0] == len(shapes), (name, G, rank)
                assert torch.equal(out, ref), (name, G, rank)
        eng.set_row_split()


@pytest.mark.parametrize("H,W", [(480, 640), (472, 344)])
@pytest.mark.parametrize("model", ["depth", "iid2"])
def test_virtual_ranks_are_the_unsplit_call(request, model, H, W):
    eng = request.getfixturevalue("depth_eng" if model == "depth" else "iid_eng")
    _check_virtual_ranks(eng, _workloads(eng, H, W, 1 if model == "depth" else 2))


@pytest.mark.parametrize("force_rows", [128, 384])
def test_virtual_ranks_with_vae_row_blocks(depth_eng, force_rows):
    """The VAE attention in row blocks that do not line up with the ranks' shares (large photos run it so): 4800 tokens
    in blocks of 384 rows against shares of 1664 rows at G = 3, and of 640 at G = 8."""
    eng = depth_eng
    w = {k: v for k, v in _workloads(eng, 480, 640, 1).items() if k in ("encode", "decode_depth")}
    default = {k: run().clone() for k, (run, _) in w.items()}
    try:
        assert attn_blocks(eng, 1, 60 * 80, force_rows=force_rows)[0] == force_rows
        for k, (run, _) in w.items():
            assert torch.equal(run(), default[k]), k                   # row blocks never change the bits
        _check_virtual_ranks(eng, w)
    finally:
        attn_blocks(eng, 1, 60 * 80)


# ---- unchanged paths and errors -----------------------------------------------------------------------------------


def test_cleared_split_leaves_plans_bytes_and_graphs(depth_eng):
    eng = depth_eng
    fresh = engine_from_oracle(*oracle_models("tiny"))
    try:
        shapes = [(0, 60, 80), (1, 480, 640), (2, 60, 80), (0, 43, 59), (2, 43, 59)]
        want = [[a.tolist() for a in arena_plan(fresh, op, 1, d0, d1)] for op, d0, d1 in shapes]
        want_ws = [fresh.workspace_bytes(1, 480, 640), fresh.workspace_bytes(4, 472, 344)]
        eng.set_row_split(1, 3, lambda buf, r, g: None)
        assert eng.workspace_bytes(1, 480, 640) > 0   # sized for this rank's share
        eng.set_row_split()
        assert [[a.tolist() for a in arena_plan(eng, op, 1, d0, d1)] for op, d0, d1 in shapes] == want
        assert [eng.workspace_bytes(1, 480, 640), eng.workspace_bytes(4, 472, 344)] == want_ws
        # a denoise launches what the captured step graph holds, as before, after a row-split call
        lat, z0 = torch.randn(1, 4, 60, 80, device="cuda"), torch.randn(1, 4, 60, 80, device="cuda")
        _schedule(eng, False, 3)
        _schedule(fresh, False, 3)
        counts = []
        for e in (fresh, eng):
            e.denoise(lat, z0)                        # captures the step graph
            torch.cuda.synchronize()
            n0 = e.lib.mgb_launch_count()
            e.denoise(lat, z0)
            torch.cuda.synchronize()
            counts.append(e.lib.mgb_launch_count() - n0)
        # A split call that needs more workspace than the handle holds grows it, which drops the captured graph (its
        # addresses move); the next unsplit call captures it again. Once the workspace fits both, a split call leaves
        # the unsplit shape's graph as it is: the unsplit denoise after it replays the graph, with no capture.
        for _ in range(2):
            held = eng.held_bytes()
            eng.set_row_split(0, 2, lambda buf, r, g: None)
            eng.denoise(lat, z0)                      # eager, no capture
            eng.set_row_split()
            torch.cuda.synchronize()
            grew = eng.held_bytes() != held
            n0 = eng.lib.mgb_launch_count()
            out = eng.denoise(lat, z0)
            torch.cuda.synchronize()
            if not grew:
                assert eng.lib.mgb_launch_count() - n0 == counts[0] == counts[1]
            assert torch.equal(out, fresh.denoise(lat, z0))
        assert not grew                               # the second pass ran on the held workspace
    finally:
        fresh.close()


def test_row_split_errors(depth_eng):
    eng = depth_eng
    for rank, world in ((2, 2), (-1, 2), (0, 0)):
        with pytest.raises(MgbError, match="set_row_split"):
            eng.set_row_split(rank, world, lambda buf, r, g: None)
    lat = torch.randn(2, 4, 16, 16, device="cuda")
    _schedule(eng, False, 2)
    eng.set_row_split(0, 2, lambda buf, r, g: None)
    torch.cuda.synchronize()
    n0 = eng.lib.mgb_launch_count()
    for call in (lambda: eng.decode(lat, 0), lambda: eng.encode(torch.zeros(2, 3, 128, 128, device="cuda")),
                 lambda: eng.denoise(lat, lat), lambda: eng.unet_step(lat, lat.clone(), 0)):
        with pytest.raises(MgbError, match="one image per call"):
            call()
    assert eng.lib.mgb_launch_count() == n0       # refused before any launch

    def failing(buf, r, g):
        raise RuntimeError("exchange down")

    eng.set_row_split(0, 2, failing)
    with pytest.raises(MgbError, match="exchange down"):
        eng.decode(lat[:1], 0)
    eng.set_row_split()
    a = eng.decode(lat[:1], 0)
    fresh = engine_from_oracle(*oracle_models("tiny"))
    try:
        assert torch.equal(a, fresh.decode(lat[:1], 0))
    finally:
        fresh.close()


# ---- two and three processes on the one GPU (gloo) -----------------------------------------------------------------

IID_PROPS = {"target_names": ["albedo", "shading"], "albedo": {"prediction_space": "srgb"},
             "shading": {"prediction_space": "linear", "up_to_scale": True}}


def _pipes(n_targets):
    from marigold_b200.engine import Engine, EngineConfig
    from marigold_b200.pipeline import MarigoldDepthPipeline, MarigoldIIDPipeline
    from marigold_b200.schedulers import DDIMScheduler

    if n_targets == 1:
        unet, vae, text = oracle_models("tiny")
        return MarigoldDepthPipeline(engine_from_oracle(unet, vae, text), DDIMScheduler(), text,
                                     default_denoising_steps=2, default_processing_resolution=0)
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
    return MarigoldIIDPipeline(eng, DDIMScheduler(), text, target_properties=IID_PROPS, default_denoising_steps=2,
                               default_processing_resolution=0)


def _calls():
    """(name, n_targets, image, kwargs): E = 1 at native resolution (odd latent 43 x 59)."""
    img = synthetic_image(480, seed=9)[:, :, :344, :472].contiguous()
    z = torch.randn(1, 4, 43, 59, generator=torch.Generator().manual_seed(4))
    z2 = torch.randn(1, 8, 43, 59, generator=torch.Generator().manual_seed(5))
    return [("depth", 1, img, dict(noise=z)), ("depth_list", 1, [img], dict(noise=[z])),
            ("depth_gen", 1, img, dict(generator=torch.Generator().manual_seed(6))), ("iid", 2, img, dict(noise=z2))]


def _maps(out):
    """The output's arrays, flat: of each image of a list, its depth map or its targets' maps."""
    if isinstance(out, list):
        return [m for o in out for m in _maps(o)]
    if hasattr(out, "depth_np"):
        return [out.depth_np]
    return [e.array for e in out.entries]


def _worker(rank, world_size, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    parallel.ROW_SPLIT_MIN_TOKENS = 0                # forced: these latents are far below the threshold
    exchanges = []
    try:
        res = {}
        pipes = {1: _pipes(1), 2: _pipes(2)}
        for p in pipes.values():
            p.engine.set_row_split = _counting(p.engine.set_row_split, exchanges)
        for name, nt, img, kw in _calls():
            n0 = len(exchanges)
            res[name] = (_maps(pipes[nt](img, ensemble_size=1, **kw)), len(exchanges) - n0)
        q.put((rank, res, None))
    except Exception as e:  # noqa: BLE001
        q.put((rank, None, repr(e)))
    finally:
        dist.destroy_process_group()


def _counting(set_row_split, log):
    def wrapped(rank=0, world=1, exchange=None):
        if exchange is None:
            return set_row_split()

        def counted(buf, r, g):
            log.append(r)
            exchange(buf, r, g)
        return set_row_split(rank, world, counted)
    return wrapped


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world_size", [2, 3])
def test_processes_on_one_gpu_match_the_single_call(world_size):
    import torch.multiprocessing as mp

    want = {}
    pipes = {1: _pipes(1), 2: _pipes(2)}
    for name, nt, img, kw in _calls():
        want[name] = _maps(pipes[nt](img, ensemble_size=1, batch_size=1, **kw))
    for p in pipes.values():
        p.engine.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world_size, port, q)) for r in range(world_size)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=600) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    # exchanges per call: one encode, 16 per UNet step (2 steps), one decode per target
    n_exch = {"depth": 34, "depth_list": 34, "depth_gen": 34, "iid": 35}
    for rank, got, err in res:
        assert err is None, (rank, err)
        for name, (maps, n) in got.items():
            assert n == n_exch[name], (rank, name, n)
            assert len(maps) == len(want[name]) and all(np.array_equal(a, b) for a, b in zip(maps, want[name])), \
                (rank, name)
