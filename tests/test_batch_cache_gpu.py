"""Member batch selection against torch's caching allocator (`-m gpu`): memory that torch keeps cached for tensors
already freed is not free to the engine's workspace, which comes from the driver. select_batch_size hands the cache
back where the call would otherwise be refused, and only there."""
import gc

import pytest
import torch

from tests.helpers import engine_from_oracle, oracle_models

pytestmark = pytest.mark.gpu


def test_cached_memory_is_handed_back_before_a_refusal():
    from marigold_b200.pipeline import select_batch_size

    gc.collect()
    torch.cuda.empty_cache()
    eng = engine_from_oracle(*oracle_models("tiny"))
    try:
        h = w = 2048
        need = eng.workspace_bytes(1, h, w)
        free0 = torch.cuda.mem_get_info()[0]
        assert 0 < need < free0 // 2, (need, free0)
        # a fits without the cache: it is left alone
        filler = torch.empty(free0 - 2 * need, dtype=torch.uint8, device="cuda")
        del filler
        cached = torch.cuda.memory_reserved()
        assert select_batch_size(eng, 1, h, w) == 1
        assert torch.cuda.memory_reserved() == cached
        # fits only with the cache handed back
        torch.cuda.empty_cache()
        filler = torch.empty(torch.cuda.mem_get_info()[0] - need // 2, dtype=torch.uint8, device="cuda")
        del filler
        free = torch.cuda.mem_get_info()[0]
        assert free + eng.held_bytes() < need
        with pytest.raises(ValueError):
            select_batch_size(eng, 1, h, w, free_bytes=free)
        assert select_batch_size(eng, 1, h, w) == 1
        assert torch.cuda.mem_get_info()[0] + eng.held_bytes() >= need
        assert torch.isfinite(eng.decode(torch.randn(1, 4, h // 8, w // 8, device="cuda"), 0)).all()
    finally:
        eng.close()
        torch.cuda.empty_cache()
