"""One engine handle over its life: the device memory it owns is all released by close(), its cached CUDA graph of a
UNet step follows the buffers it captured, and a call rejected for its arguments leaves the handle as it was."""
import pytest
import torch

from tests.helpers import engine_from_oracle, live_device_bytes, oracle_models

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def models():
    return oracle_models("tiny")


def _ddim(eng, n):
    from marigold_b200.schedulers import DDIMScheduler

    s = DDIMScheduler()
    s.set_timesteps(n)
    eng.set_schedule(s.timesteps, *s.coefficients())


def _latents(seed=3):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(2, 4, 16, 16, generator=g).cuda(), torch.randn(2, 4, 16, 16, generator=g).cuda()


def _image(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 3, S, S, generator=g) * 2 - 1).cuda()


def test_close_releases_every_buffer_the_handle_allocated(models):
    from marigold_b200.ensemble import ensemble_depth

    ends = []
    for cycle in range(2):
        start = live_device_bytes()
        eng = engine_from_oracle(*models)
        for n in (4, 10, 4):
            _ddim(eng, n)
        eng.encode(_image(1, 64, 10 + cycle))
        lat = eng.encode(_image(2, 128, 20 + cycle))          # a larger image: the workspace grows
        x = eng.denoise(lat, _latents(30 + cycle)[1])          # the first step captures the graph, later ones replay it
        depth = eng.decode(x, 0)
        ensemble_depth(torch.cat([depth, depth.flip(-1), depth.flip(-2)]), engine=eng)   # E = 3: the ensemble scratch
        torch.cuda.synchronize()
        assert live_device_bytes() > start
        eng.close()
        ends.append(live_device_bytes())
        assert ends[-1] == start, f"cycle {cycle}: {ends[-1] - start} bytes still held after close()"
    assert ends[0] == ends[1]


def test_step_graph_is_rebuilt_when_a_captured_buffer_moves(models):
    eng = engine_from_oracle(*models)
    _ddim(eng, 4)
    rgb, x = _latents()
    a = eng.denoise(rgb, x)
    before = live_device_bytes()
    eng.encode(_image(2, 256, 5))                              # the arena is reallocated, larger
    assert live_device_bytes() > before
    _ddim(eng, 10)
    _ddim(eng, 4)                                              # sched_k and the bias table are reallocated
    b = eng.denoise(rgb, x)
    eng.close()
    fresh = engine_from_oracle(*models)
    _ddim(fresh, 4)
    c = fresh.denoise(rgb, x)
    fresh.close()
    assert torch.equal(a, b)
    assert torch.equal(a, c)


def test_rejected_calls_leave_the_handle_as_it_was(models):
    from marigold_b200._lib import MgbError

    eng = engine_from_oracle(*models)
    _ddim(eng, 4)
    rgb, x = _latents()
    a = eng.denoise(rgb, x)
    with pytest.raises(MgbError):
        eng.set_text_embedding(torch.randn(1, 3, models[2].shape[-1]))   # the kernel takes the empty prompt's 2 tokens
    assert torch.equal(eng.denoise(rgb, x), a)
    with pytest.raises(MgbError):
        eng.set_schedule([], [], [], [])                                 # n = 0
    assert torch.equal(eng.denoise(rgb, x), a)
    eng.close()
