"""Member batch selection with the call's own tensors reserved (CPU): select_batch_size's reserve_bytes against the stub
engine of test_native_res_host.py, and the reserve the pipelines pass for a shape, task and ensemble size."""
import pytest
import torch

from marigold_b200.pipeline import (MarigoldDepthPipeline, MarigoldIIDPipeline, MarigoldNormalsPipeline,
                                    call_reserve_bytes, find_batch_size, select_batch_size)
from tests.helpers import GB, StubEngine


def test_zero_reserve_is_the_default():
    for free in (62 * GB, 70 * GB, 1000 * GB):
        a = select_batch_size(StubEngine(per_member=20 * GB), 10, 3000, 4000, free_bytes=free)
        assert select_batch_size(StubEngine(per_member=20 * GB), 10, 3000, 4000, free_bytes=free, reserve_bytes=0) == a


def test_reserve_lowers_the_batch():
    # 1 + 3 * 20 = 61 GB fits 62 GB; with 2 GB reserved only 1 + 2 * 20 = 41 does
    eng = StubEngine(per_member=20 * GB)
    assert select_batch_size(eng, 10, 3000, 4000, free_bytes=62 * GB, reserve_bytes=2 * GB) == 2
    assert eng.asked == [8, 7, 6, 5, 4, 3, 2]
    # held workspace still counts as available
    eng = StubEngine(per_member=20 * GB, held=20 * GB)
    assert select_batch_size(eng, 10, 3000, 4000, free_bytes=62 * GB, reserve_bytes=2 * GB) == 3
    # the table value is kept where it fits beside the reserve
    eng = StubEngine(per_member=4 * GB)
    assert select_batch_size(eng, 10, 768, 768, free_bytes=70 * GB, reserve_bytes=10 * GB) == \
        find_batch_size(10, 768, torch.float32)


def test_reserve_refuses_what_no_longer_fits():
    eng = StubEngine(per_member=50 * GB, held=GB)
    assert select_batch_size(eng, 1, 4032, 6048, free_bytes=79 * GB) == 1          # 51 of 80 GB
    with pytest.raises(ValueError, match=f"a batch of 1 member at 4032 x 6048 needs {51 * GB} bytes of device "
                                         f"workspace, but {50 * GB} bytes are available beside the call's own "
                                         f"{30 * GB}"):
        select_batch_size(eng, 1, 4032, 6048, free_bytes=79 * GB, reserve_bytes=30 * GB)
    with pytest.raises(ValueError, match="needs"):
        select_batch_size(StubEngine(per_member=50 * GB), 1, 4032, 6048, batch_size=1, free_bytes=79 * GB,
                          reserve_bytes=30 * GB)


def test_call_reserve_bytes():
    P = 6048 * 4032
    assert call_reserve_bytes(4032, 6048, 10, 1) == 4 * P * 25          # depth: 2.4 GB
    assert call_reserve_bytes(4032, 6048, 10, 3) == 4 * P * 69          # normals: 6.7 GB
    assert 6.7e9 < call_reserve_bytes(4032, 6048, 10, 3) < 6.8e9


class _Cfg:
    unet_out_channels = 8


class _Eng(StubEngine):
    cfg = _Cfg()
    device = "cpu"

    def set_text_embedding(self, t):
        pass


@pytest.mark.parametrize("cls,ch", [(MarigoldDepthPipeline, 1), (MarigoldNormalsPipeline, 3), (MarigoldIIDPipeline, 6)])
def test_member_batch_reserves_the_call_members(cls, ch, monkeypatch):
    """_member_batch passes call_reserve_bytes for the processing size, the task's channels and E."""
    import marigold_b200.pipeline as P

    seen = {}

    def fake_select(engine, n, h, w, batch_size=0, free_bytes=None, reserve_bytes=0):
        seen.update(n=n, h=h, w=w, reserve=reserve_bytes)
        return 1

    monkeypatch.setattr(P, "select_batch_size", fake_select)
    kw = {"target_properties": {"target_names": ["albedo", "shading"]}} if cls is MarigoldIIDPipeline else {}
    pipe = cls(_Eng(per_member=GB), None, None, **kw)
    img = torch.zeros(1, 3, 4032, 6048, dtype=torch.uint8)
    assert pipe._member_batch(img, 0, 10, 0) == (1, False)
    assert seen == {"n": 10, "h": 4032, "w": 6048, "reserve": call_reserve_bytes(4032, 6048, 10, ch)}
