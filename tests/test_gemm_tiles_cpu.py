"""The shape helpers of tests/test_gemm_tiles_gpu.py, checked without a GPU: the shapes built for each N-tile width select
that width under gemm_tc.cu:dispatch_bn's rule on an H100 SXM (132 SMs) and an H100 PCIe (114 SMs)."""
import pytest

from tests.test_gemm_tiles_gpu import BATCHES, WIDTHS, qkv_width, rows_for_width, tile_width


def _tiles(M, N, bn):
    return ((M + 127) // 128) * ((N + bn - 1) // bn)


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("N", [1024, 1000])
@pytest.mark.parametrize("width", WIDTHS)
def test_rows_for_width_selects_the_width(width, N, sms):
    M = rows_for_width(width, N, sms)
    assert tile_width(M, N, sms) == width
    # dispatch_bn's conditions, written out once more
    wide = _tiles(M, N, 256) >= sms
    mid = _tiles(M, N, 128) >= sms // 2
    assert (width == 256) == wide and (width == 128) == (mid and not wide) and (width == 64) == (not mid)
    # the tile loop of the persistent kernel runs more than once for the wide tiles
    assert width == 64 or _tiles(M, N, width) > sms
    # B = 3 batches whose boundaries fall inside row tiles; a partial last row tile
    assert M % BATCHES == 0 and (M // BATCHES) % 64 != 0 and M % 128 != 0


def test_tile_width_mirrors_dispatch_bn():
    # hand-counted: 34 x 4 = 136 >= 132 tiles of 256; 21 x 8 = 168 >= 66 tiles of 128; 8 x 8 = 64 < 66
    assert tile_width(128 * 33 + 77, 1024, 132) == 256
    assert tile_width(128 * 20 + 5, 1000, 132) == 128
    assert tile_width(128 * 8, 1024, 132) == 64
    assert tile_width(128 * 8, 1024, 114) == 128  # 64 >= 57: the same M selects a wider tile on 114 SMs
    assert tile_width(10 ** 6, 200, 132) == 128 and tile_width(10 ** 6, 96, 132) == 64  # N < 256 / N < 128 caps it
    assert [qkv_width(d) for d in (3072, 512, 384, 192)] == [256, 256, 128, 64]
