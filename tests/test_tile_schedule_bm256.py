"""The tile walk of igemm_kernel on 256-row tiles: half as many M tiles, the same index arithmetic (test_tile_schedule.walk).
The geometries are the 32x32 UNet level at batch 8 (one wave), forced launches of more than one wave, and the multi-tile rows of
test_igemm_bm256_gpu, on 132 SMs."""
import itertools

import pytest

from test_tile_schedule import walk

# (M tiles of 256 rows, N tiles of 160 columns)
CASES = [(128, 2), (32, 4), (128, 4), (10, 17), (18, 2), (1, 1)]


@pytest.mark.parametrize("tiles_m,tiles_n", CASES)
def test_bm256_walk_covers_every_tile_once_at_132_sms(tiles_m, tiles_n):
    ctas = min(132, tiles_m * tiles_n)
    seen = [(m, n) for _, m, n, _ in walk(ctas, tiles_m, tiles_n, 1)]
    assert sorted(seen) == sorted(itertools.product(range(tiles_m), range(tiles_n)))


def test_bm256_multi_tile_rows_change_the_n_tile():
    from test_igemm_coverage_gpu import multi_tile_n_change
    from test_igemm_bm256_gpu import CASES as ROWS, geometry
    for c in ROWS:
        if c["walk"]:
            tm, tn = geometry(c)
            assert multi_tile_n_change(min(tm * tn, 132), tm, tn, 1), c["id"]
