"""Member batch selection at native resolution (CPU): select_batch_size against a stub engine and a stub free-memory
value, and the processing size the pipelines take it at. The 32-bit counts of the VAE graph at the supported maximum,
restated from shapes."""
import pytest
import torch

from marigold_b200.pipeline import MAX_PIXELS, _processing_size, find_batch_size, select_batch_size
from tests.helpers import GB, StubEngine


@pytest.mark.parametrize("E,h,w", [(1, 768, 768), (10, 768, 576), (16, 768, 768), (10, 1024, 1024), (64, 1024, 768)])
def test_table_value_kept_where_it_fits(E, h, w):
    eng = StubEngine(per_member=4 * GB)
    assert select_batch_size(eng, E, h, w, free_bytes=70 * GB) == find_batch_size(E, max(h, w), torch.float32)
    assert eng.asked == [find_batch_size(E, max(h, w), torch.float32)]      # one dry run when the table value fits


def test_lowered_to_the_largest_batch_that_fits():
    eng = StubEngine(per_member=20 * GB)
    # 8 from the table above 768 px; 1 + 3 * 20 = 61 GB fits 62 GB, 4 members would need 81
    assert select_batch_size(eng, 10, 3000, 4000, free_bytes=62 * GB) == 3
    assert eng.asked == [8, 7, 6, 5, 4, 3]
    # what the engine already holds counts as available: it is freed before the workspace grows
    assert select_batch_size(StubEngine(per_member=20 * GB, held=20 * GB), 10, 3000, 4000, free_bytes=62 * GB) == 4


def test_one_member_that_does_not_fit_raises_with_the_bytes():
    eng = StubEngine(per_member=90 * GB, held=GB)
    with pytest.raises(ValueError, match=f"a batch of 1 member at 3000 x 4000 needs {91 * GB} bytes of device "
                                         f"workspace, but {80 * GB} bytes are available"):
        select_batch_size(eng, 10, 3000, 4000, free_bytes=79 * GB)
    assert eng.asked == [8, 7, 6, 5, 4, 3, 2, 1]


def test_explicit_batch_size_is_checked_not_lowered():
    eng = StubEngine(per_member=20 * GB)
    assert select_batch_size(eng, 10, 3000, 4000, batch_size=2, free_bytes=62 * GB) == 2
    with pytest.raises(ValueError, match=f"a batch of 4 members at 3000 x 4000 needs {81 * GB} bytes"):
        select_batch_size(eng, 10, 3000, 4000, batch_size=4, free_bytes=62 * GB)
    # a batch larger than the members runs them all at once: checked at the member count
    assert select_batch_size(StubEngine(per_member=20 * GB), 2, 3000, 4000, batch_size=8, free_bytes=62 * GB) == 2


def test_past_the_supported_maximum():
    with pytest.raises(ValueError, match=f"supported maximum of {MAX_PIXELS} pixels"):
        select_batch_size(StubEngine(per_member=GB), 1, 8192, 8200, free_bytes=1000 * GB)
    # above it in a batch of 8 but not alone: lowered until it is within the maximum and fits
    assert select_batch_size(StubEngine(per_member=GB), 8, 4032, 6048, free_bytes=1000 * GB) == 2


def test_processing_size():
    assert _processing_size(3024, 4032, 0) == (3024, 4032)
    assert _processing_size(3024, 4032, 768) == (576, 768)
    assert _processing_size(3000, 4000, 768) == (576, 768)


def test_32bit_counts_at_the_supported_maximum():
    """Restated from shapes (csrc/net.h kMaxPixels): pixels and GEMM rows of one call, per-row sizes and grid dimensions
    stay 32-bit; element counts do not, and the kernels index them with 64-bit arithmetic."""
    INT_MAX, GRID_YZ = 2**31 - 1, 65535
    px = MAX_PIXELS
    assert px <= INT_MAX                                   # GEMM / conv rows (GemmParams.M), GroupNorm HW, epilogue hw
    T = px // 64                                           # latent tokens of the VAE attention
    Tp = (T + 63) // 64 * 64
    assert (Tp + 31) // 32 <= GRID_YZ                      # transpose_bf16 grid.y
    assert (T + 63) // 64 <= GRID_YZ                       # score GEMM n tiles (block_n >= 64 at N >= 64)
    assert 8448 * Tp > INT_MAX                             # a score block of one wave's rows: softmax rows at size_t offsets
    assert px * 256 > INT_MAX                              # full-resolution 256-channel decoder tensors: size_t indices
    # at 12 MP the decoder's 256-channel tensors already pass 2^31 elements
    assert 4000 * 3000 * 256 > INT_MAX
