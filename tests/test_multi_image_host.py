"""Host logic of list calls (CPU): the job partition, rounds and their gathers (gloo, world sizes 2 and 3), the batch-size
agreement, the open-image bound, size groups and the per-image noise draws; and the whole list driver
(_MarigoldBase._infer_list) on a stub engine whose member maps are a known function of their image and noise."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from marigold_b200 import parallel
from marigold_b200.pipeline import find_batch_size, noise_draw_batches, select_list_batch_size, size_groups
from tests.helpers import GB, StubEngine, _expected, _images, _pipe, _run


def test_rounds_partition_the_jobs():
    for n_jobs in (1, 3, 9, 10, 30, 160):
        for G in (1, 2, 3, 8):
            for bs in (1, 2, 4, 16):
                seen = []
                for r in range(parallel.num_rounds(n_jobs, bs, G)):
                    mine_all = []
                    for rank in range(G):
                        jobs, mine = parallel.round_jobs(n_jobs, bs, r, rank, G)
                        assert jobs == list(range(r * G * bs, min((r + 1) * G * bs, n_jobs)))
                        assert len(mine) <= bs and all(k % G == rank for k in mine)
                        mine_all += mine
                    assert sorted(mine_all) == jobs
                    seen += jobs
                assert seen == list(range(n_jobs))
    # a one-image list: each rank's jobs are member_indices
    for E in (1, 3, 10):
        for G in (2, 8):
            bs = parallel.slots_per_rank(E, G)
            assert parallel.num_rounds(E, bs, G) == 1
            for rank in range(G):
                assert parallel.round_jobs(E, bs, 0, rank, G)[1] == parallel.member_indices(E, rank, G)


def test_open_images_is_the_most_a_round_spans():
    for E in (1, 2, 3, 10):
        for G in (1, 2, 3):
            for bs in (1, 2, 4, 16):
                for n_images in (1, 2, 5, 40):
                    n_jobs = n_images * E
                    L = G * bs
                    most = max(len({k // E for k in range(s, min(s + L, n_jobs))}) for s in range(n_jobs))
                    assert parallel.open_images(bs, E, G, n_images) >= most
                    if n_jobs >= L + E:          # long enough for the worst alignment to occur
                        assert parallel.open_images(bs, E, G, n_images) == most


def test_size_groups_and_noise_draws():
    assert size_groups([(128, 128), (96, 160), (128, 128), (96, 160), (64, 64)]) == \
        [((128, 128), [0, 2]), ((96, 160), [1, 3]), ((64, 64), [4])]
    assert size_groups([]) == []
    assert noise_draw_batches(10, 0, 480, 640) == [10]
    assert noise_draw_batches(20, 0, 1024, 768) == [8, 8, 4]
    assert noise_draw_batches(3, 2, 128, 128) == [2, 1]
    assert noise_draw_batches(4, 4, 128, 128) == [4]
    assert noise_draw_batches(10, 0, 768, 768, world_size=3) == [10]
    for E in (1, 5, 16, 17):
        assert sum(noise_draw_batches(E, 0, 768, 768)) == E


def test_list_batch_reserves_the_open_images(monkeypatch):
    import marigold_b200.pipeline as P

    # everything fits: find_batch_size's 16 at 768 px
    assert select_list_batch_size(StubEngine(per_member=GB), 160, 768, 768, 10, 1, 16, free_bytes=70 * GB) == 16
    # workspace 1 + B GB; each open image reserves r. 12..16 slots span 3 images of 10 members, 2..11 span 2: with
    # 1 + 11 + 2 r free, 11 is the largest batch that fits beside its own reserve
    r = 4 * GB
    monkeypatch.setattr(P, "call_reserve_bytes", lambda h, w, E, c: r)
    free = GB + 11 * GB + 2 * r
    eng = StubEngine(per_member=GB)
    assert select_list_batch_size(eng, 160, 768, 768, 10, 1, 16, free_bytes=free) == 11
    assert select_list_batch_size(eng, 160, 768, 768, 10, 1, 16, free_bytes=free - 1) == 10
    # a one-image group reserves one image, like the single call
    assert select_list_batch_size(eng, 10, 768, 768, 10, 1, 1, free_bytes=GB + 10 * GB + r) == 10
    # under 2 ranks a round spans 2 bs jobs: 5 slots per rank span 2 images, 6 span 3
    assert select_list_batch_size(eng, 80, 768, 768, 10, 1, 16, world_size=2, free_bytes=GB + 5 * GB + 2 * r) == 5
    assert select_list_batch_size(eng, 80, 768, 768, 10, 1, 16, world_size=2, free_bytes=GB + 6 * GB + 3 * r) == 6
    # an explicit batch is taken as given beside its reserve, or refused
    assert select_list_batch_size(eng, 160, 768, 768, 10, 1, 16, batch_size=4, free_bytes=free) == 4
    with pytest.raises(ValueError, match="beside the call's own"):
        select_list_batch_size(eng, 160, 768, 768, 10, 1, 16, batch_size=16, free_bytes=free)
    with pytest.raises(ValueError, match="needs"):
        select_list_batch_size(eng, 160, 768, 768, 10, 1, 16, free_bytes=GB + r)


# ---- the list driver on a stub engine ------------------------------------------------------------------------------


@pytest.fixture(autouse=True)
def _free_memory(monkeypatch):
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (70 * GB, 80 * GB))


def _single_draws(E, bs, shape, steps, lcm, g):
    """What the single call draws from g for one image at world size 1: per batch z0, then the step noise."""
    zs, ss = [], []
    for b in noise_draw_batches(E, bs, 8 * shape[1], 8 * shape[2]):
        zs.append(torch.randn((b,) + shape, generator=g))
        if lcm and steps > 1:
            ss.append(torch.stack([torch.randn((b,) + shape, generator=g) for _ in range(steps - 1)]))
    return torch.cat(zs), (torch.cat(ss, dim=1) if ss else None)


@pytest.mark.parametrize("lcm", [False, True])
@pytest.mark.parametrize("E,bs", [(3, 4), (4, 4), (1, 0), (5, 2), (3, 1)])
def test_driver_members_noise_and_finishing(E, bs, lcm):
    sizes = [(64, 64), (48, 80), (64, 64), (64, 64), (48, 80)]
    images = _images(sizes)
    steps = 3
    pipe = _pipe(lcm=lcm)
    got = _run(pipe, images, E, steps, bs, generator=torch.Generator().manual_seed(11))
    # the shared generator is drawn from in list order, each image what the single call draws
    g = torch.Generator().manual_seed(11)
    for i, (h, w) in enumerate(sizes):
        z, sn = _single_draws(E, bs, (4, h // 8, w // 8), steps, lcm, g)
        assert torch.equal(got[i], _expected(images[i], z, sn)), f"image {i}"
    # batches: group (64, 64) first, then (48, 80); only each group's last batch is smaller
    shapes = [s for op, *s in pipe.engine.log if op == "denoise"]
    for (h, w), idx in size_groups(sizes):
        b = bs if bs else find_batch_size(len(idx) * E, max(h, w), torch.float32)
        n = len(idx) * E
        want = [(min(b, n - s), 4, h // 8, w // 8) for s in range(0, n, b)]
        assert [s[0] for s in shapes[:len(want)]] == want
        shapes = shapes[len(want):]
    # each image is encoded once and finished right after the batch that holds its last member
    log = pipe.engine.log
    assert sum(1 for e in log if e[0] == "encode") == len(images)
    batches = [k for k, e in enumerate(log) if e[0] == "denoise"]
    finishes = {e[1]: k for k, e in enumerate(log) if e[0] == "finish"}
    order = [i for _, idx in size_groups(sizes) for i in idx]
    jobs = [(i, m) for i in order for m in range(E)]
    b_of_job, pos = [], 0
    for (h, w), idx in size_groups(sizes):
        b = bs if bs else find_batch_size(len(idx) * E, max(h, w), torch.float32)
        n = len(idx) * E
        b_of_job += [pos + j // b for j in range(n)]
        pos += -(-n // b)
    for i in order:
        last = max(b for (j, _), b in zip(jobs, b_of_job) if j == i)
        assert batches[last] < finishes[i], f"image {i} finished before its last batch"
        if last + 1 < len(batches):
            assert finishes[i] < batches[last + 1], f"image {i} finished late"


def test_driver_per_image_generators_and_explicit_noise():
    sizes = [(64, 64)] * 3
    images = _images(sizes)
    E, steps = 3, 4
    z = [torch.randn(E, 4, 8, 8, generator=torch.Generator().manual_seed(i)) for i in range(3)]
    sn = [torch.randn(steps - 1, E, 4, 8, 8, generator=torch.Generator().manual_seed(10 + i)) for i in range(3)]
    got = _run(_pipe(lcm=True), images, E, steps, 4, noise=z, step_noise=sn)
    for i in range(3):
        assert torch.equal(got[i], _expected(images[i], z[i], sn[i]))
    got = _run(_pipe(lcm=True), images, E, steps, 4, generator=[torch.Generator().manual_seed(20 + i) for i in range(3)])
    for i in range(3):
        zi, si = _single_draws(E, 4, (4, 8, 8), steps, True, torch.Generator().manual_seed(20 + i))
        assert torch.equal(got[i], _expected(images[i], zi, si))
    with pytest.raises(ValueError, match="noise"):
        _run(_pipe(), images, E, 2, 4, noise=z[:2])
    with pytest.raises(AssertionError, match="image 1"):
        _run(_pipe(), images, E, 2, 4, noise=[z[0], z[1][:2], z[2]])


# ---- several ranks (gloo) ------------------------------------------------------------------------------------------

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world_size, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    torch.cuda.mem_get_info = lambda device=None: (70 * GB, 80 * GB)        # this process's stand-in for a device
    try:
        res = {}
        # MIN agreement: every rank proposes its own value per group
        res["agree"] = parallel.agree_batch_sizes([8 + rank, 16 - rank, 3])
        # round gathers: job k's map is filled with k + 1; 11 jobs at bs 2 leave ranks without a job in the last round
        ok = True
        for n_jobs, bs in ((11, 2), (3, 2), (12, 2), (7, 1)):
            for r in range(parallel.num_rounds(n_jobs, bs, world_size)):
                jobs, mine = parallel.round_jobs(n_jobs, bs, r, rank, world_size)
                local = torch.stack([torch.full((1, 2, 3), k + 1.0) for k in mine]) if mine else torch.empty(0, 1, 2, 3)
                out = parallel.gather_round(local, bs, len(jobs))
                ok &= out.shape[0] == len(jobs) and all(bool((out[j] == k + 1).all()) for j, k in enumerate(jobs))
        res["gather"] = ok
        # the whole driver: every rank gets every image's maps, equal to the single-process result
        sizes = [(64, 64), (48, 80), (64, 64), (64, 64)]
        images = _images(sizes)
        E = 3
        z = [torch.randn(E, 4, h // 8, w // 8, generator=torch.Generator().manual_seed(i)) for i, (h, w) in
             enumerate(sizes)]
        got = _run(_pipe(), images, E, 2, 2, noise=z)
        res["driver"] = all(torch.equal(got[i], _expected(images[i], z[i], None)) for i in range(len(sizes)))
        # a shared generator: the full [E, ...] draw per image, in list order, on every rank
        got = _run(_pipe(), images, E, 2, 2, generator=torch.Generator().manual_seed(5))
        g = torch.Generator().manual_seed(5)
        res["shared"] = all(torch.equal(got[i], _expected(images[i], torch.randn(E, 4, h // 8, w // 8, generator=g), None))
                            for i, (h, w) in enumerate(sizes))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world_size", [2, 3])
def test_ranks_gloo(world_size):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world_size, port, q)) for r in range(world_size)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, r in res:
        assert r["agree"] == [8, 16 - (world_size - 1), 3]
        assert r["gather"] and r["driver"] and r["shared"], (rank, r)
