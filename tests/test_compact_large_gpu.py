"""GPU: stream compaction from 2^30 rows on, where the one-pass kernel's 30-bit look-back counts would overflow and the
count -> scan -> scatter form takes over."""
import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.slow]


def test_compact_points_beyond_2_pow_30_rows(cuda, gsx_lib):
    """All rows survive: the count is n, xyz comes out unchanged and the row index is arange(n).  Peak use is about
    34 GiB (xyz in and out, the mask, the index and the arange it is compared with)."""
    import torch
    from gsx.pipeline import compact
    if torch.cuda.mem_get_info(cuda)[0] < 40 * 2**30:
        pytest.skip("needs 40 GiB of free device memory")
    n = 2**30 + 2048
    gen = torch.Generator(device=cuda).manual_seed(7)
    xyz = torch.rand(n, 3, device=cuda, generator=gen)
    mask = torch.ones(n, dtype=torch.bool, device=cuda)
    x, o, idx, m = compact(mask, xyz, None, None)
    assert o is None and m == n
    assert torch.equal(x, xyz)
    del x, xyz, mask
    assert torch.equal(idx, torch.arange(n, dtype=torch.int32, device=cuda))
