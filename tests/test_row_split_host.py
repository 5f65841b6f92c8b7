"""Host logic of the row split (CPU): the chunk geometry, the decision rule, and under gloo at world sizes 2 and 3 on a
stub engine: every rank runs a one-job call (single or list) row-split and ends with the same maps, groups of several
jobs keep their member sharding, and the ranks agree on the split before any exchange."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from marigold_b200 import parallel
from tests.helpers import GB, FakeEngine, _expected, _images, _pipe, _run


def test_chunk_geometry():
    for T in (1, 127, 128, 129, 2304, 2537, 4800, 190512, 762048):
        for G in (1, 2, 3, 7, 8):
            chunk = parallel.row_split_chunk(T, G)
            assert chunk % 128 == 0 and G * chunk >= T and (G * chunk - T) < G * 128
            assert (chunk - 128) * G < -(-T // 128) * 128          # the fewest whole blocks that cover T
            rows = [parallel.row_split_rows(T, r, G) for r in range(G)]
            assert [i for rg in rows for i in rg] == list(range(T))
            assert all(len(rg) == 0 or rg.start == r * chunk for r, rg in enumerate(rows))
    # 18 blocks over 8 ranks: 3 each, the last two ranks own none
    assert [len(parallel.row_split_rows(2304, r, 8)) for r in range(8)] == [384] * 6 + [0, 0]


def test_decision_rule():
    assert parallel.ROW_SPLIT_MIN_TOKENS == 96 * 96                 # 768 x 768, the measured crossover
    assert parallel.row_split_rule(1, 3024, 4032, 2)
    assert parallel.row_split_rule(1, 768, 768, 8)
    assert not parallel.row_split_rule(1, 640, 480, 8)             # below the threshold
    assert not parallel.row_split_rule(1, 3024, 4032, 1)           # one rank
    assert not parallel.row_split_rule(2, 3024, 4032, 2)           # several jobs: member sharding
    assert not parallel.row_split_rule(1, 768, 768, 8, min_tokens=200_000)
    assert not parallel.row_split_rule(1, 768, 760, 8, min_tokens=96 * 96)     # latent 96 x 95
    assert parallel.row_split_rule(1, 775, 775, 2, min_tokens=96 * 96)         # floor(775 / 8) = 96


class SplitEngine(FakeEngine):
    """FakeEngine with the row-split hook: each encode, denoise and decode with the split installed runs one exchange of
    a buffer whose chunk r holds r + 1, and logs whether every chunk came back filled."""

    def __init__(self):
        super().__init__()
        self.split = None

    def set_row_split(self, rank=0, world=1, exchange=None):
        self.split = None if exchange is None else (rank, world, exchange)

    def _exchange(self):
        if self.split is None:
            return
        rank, world, fn = self.split
        buf = torch.zeros(world * 4, dtype=torch.uint8)
        buf[rank * 4:(rank + 1) * 4] = rank + 1
        fn(buf, rank, world)
        self.log.append(("exchange", torch.equal(buf, torch.arange(1, world + 1, dtype=torch.uint8).repeat_interleave(4))))

    def encode(self, rgb):
        self._exchange()
        return super().encode(rgb)

    def denoise(self, rl, z, sn=None):
        self._exchange()
        out = super().denoise(rl, z, sn)
        self.log[-1] = ("split" if self.split else "shard",) + self.log[-1][1:]
        return out

    def decode(self, t, mode):
        self._exchange()
        return super().decode(t, mode)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world_size, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    torch.cuda.mem_get_info = lambda device=None: (70 * GB, 80 * GB)
    parallel.ROW_SPLIT_MIN_TOKENS = 48             # 8 x 6 latent tokens and more
    try:
        res = {}
        agree = parallel.agree_batch_sizes
        # ---- the single call
        pipe = _pipe()
        pipe.engine = SplitEngine()
        log = pipe.engine.log
        parallel.agree_batch_sizes = lambda sizes, device=None: (log.append(("agree", list(sizes))), agree(sizes))[1]
        img = _images([(48, 64)])[0]
        z = torch.randn(1, 4, 6, 8, generator=torch.Generator().manual_seed(1))
        bs, split = pipe._member_batch(img, 0, 1, 0)
        rgb = img.float() / 255 * 2 - 1
        out = pipe._infer_members(rgb, 1, 2, bs, None, z, None, 0, split)
        res["single"] = bs == 1 and split and torch.equal(out, _expected(img, z, None))
        res["single_log"] = [e[0] for e in log]
        res["single_filled"] = all(e[1] for e in log if e[0] == "exchange")
        # a call below the threshold keeps member sharding: no agreement, no exchange
        pipe.engine.log.clear()
        small = _images([(40, 40)])[0]
        assert pipe._member_batch(small, 0, 1, 0) == (1, False)
        out = pipe._infer_members(small.float() / 255 * 2 - 1, 1, 2, 1, None, torch.zeros(1, 4, 5, 5), None, 0)
        res["small"] = [e[0] for e in log]
        # ---- a call that passed the split's agreement and then failed leaves nothing behind: the next call, E = 3,
        # shards its members and every rank finishes all three maps
        pipe = _pipe()
        pipe.engine = SplitEngine()
        finished = []
        pipe._finish = lambda preds, *a, **k: finished.append(preds)
        real_preprocess = pipe._preprocess

        def failing(im, pr, rs):
            raise AssertionError("bad input")

        pipe._preprocess = failing
        try:
            pipe(img, denoising_steps=2, ensemble_size=1, processing_res=0, noise=z)
            res["failed_call"] = False
        except AssertionError:
            res["failed_call"] = True
        pipe._preprocess = real_preprocess
        z3 = torch.randn(3, 4, 6, 8, generator=torch.Generator().manual_seed(2))
        pipe(img, denoising_steps=2, ensemble_size=3, processing_res=0, noise=z3)
        res["after_failure"] = len(finished) == 1 and torch.equal(finished[0], _expected(img, z3, None)) and \
            not any(e[0] in ("split", "exchange") for e in pipe.engine.log)
        # ---- a list: group (64, 64) has 3 jobs (member sharding), group (48, 80) one (row split)
        pipe = _pipe()
        pipe.engine = SplitEngine()
        log = pipe.engine.log
        sizes = [(64, 64), (48, 80), (64, 64), (64, 64)]
        images = _images(sizes)
        zs = [torch.randn(1, 4, h // 8, w // 8, generator=torch.Generator().manual_seed(i)) for i, (h, w) in
              enumerate(sizes)]
        got = _run(pipe, images, 1, 2, 0, noise=zs)
        res["list"] = all(torch.equal(got[i], _expected(images[i], zs[i], None)) for i in range(len(sizes)))
        res["list_log"] = [e for e in log if e[0] != "finish"]
        q.put((rank, res, None))
    except Exception as e:  # noqa: BLE001
        q.put((rank, None, repr(e)))
    finally:
        parallel.agree_batch_sizes = agree
        dist.destroy_process_group()


@pytest.mark.parametrize("world_size", [2, 3])
def test_ranks_gloo(world_size):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world_size, port, q)) for r in range(world_size)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=180) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    for rank, r, err in res:
        assert err is None, (rank, err)
        assert r["single"] and r["list"] and r["single_filled"], (rank, r)
        assert r["failed_call"] and r["after_failure"], (rank, r)
        # agreed before the first exchange; encode, denoise and decode each exchange once, on every rank
        assert r["single_log"][0] == "agree" and r["single_log"][1:] == ["exchange", "encode", "exchange", "split",
                                                                         "exchange"], r["single_log"]
        assert "agree" not in r["small"] and "exchange" not in r["small"]
        log = r["list_log"]
        assert log[0] == ("agree", [parallel.slots_per_rank(3, world_size), 1, 0, 1])   # sizes, then split flags
        # the 3-job group: this rank's jobs of today's sharding, no exchange; then the one-job group on every rank
        shard = [e for e in log if e[0] == "shard"]
        assert sum(e[1][0] for e in shard) == len(range(rank, 3, world_size))
        split = log[log.index(next(e for e in log if e[0] == "split")) - 3:]
        assert [e[0] for e in split] == ["exchange", "encode", "exchange", "split", "exchange"]
        assert all(e[1] for e in log if e[0] == "exchange")
