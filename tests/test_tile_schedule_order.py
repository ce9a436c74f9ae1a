"""Host-side model of both tile walks of igemm_kernel: M-fast (the M tile index changes fastest) and N-fast (the N tile index
changes fastest, single-pass launches only), with the incremental index arithmetic the producer and the consumers share, and the
rule in run_igemm that picks between them.  Every output tile is visited exactly once, by exactly one CTA, in either order, and
the LayerNorm row prefetch of the consumers always names the M tile of the tile the CTA runs next."""
import itertools
from collections import defaultdict

import pytest

from test_tile_schedule import walk as walk_m_fast


def walk(num_ctas, tiles_m, tiles_n, ksplit, n_fast):
    """Yields (cta, m_idx, n_idx, ks, m_next) as igemm_kernel computes them; m_next is the M tile the LayerNorm prefetch requests
    after the index update (None after the CTA's last tile)."""
    assert not (n_fast and ksplit > 1)
    num_tiles = tiles_m * tiles_n * ksplit
    units_f = tiles_n if n_fast else tiles_m
    step_f, step_s = num_ctas % units_f, num_ctas // units_f
    for cta in range(num_ctas):
        unit_f, unit_s = cta % units_f, cta // units_f
        t = cta
        while t < num_tiles:
            m_idx = unit_s if n_fast else unit_f
            n_idx, ks = (unit_f if n_fast else unit_s), 0
            if ksplit > 1:
                n_idx, ks = unit_s % tiles_n, unit_s // tiles_n
            unit_f += step_f
            unit_s += step_s
            if unit_f >= units_f:
                unit_f -= units_f
                unit_s += 1
            m_next = (unit_s if n_fast else unit_f) if t + num_ctas < num_tiles else None
            yield cta, m_idx, n_idx, ks, m_next
            t += num_ctas


def n_fast_rule(M, a_chan, N, Ktot, ksplit, tiles_n):
    """run_igemm: N-fast when the launch is single-pass, has several N tiles and A (M output pixels x the channels of every A
    map) outweighs W (N x Ktot)"""
    return ksplit == 1 and tiles_n > 1 and M * a_chan > N * Ktot


# (M tiles, N tiles, ksplit) at 132 SMs: the 64x64 level's ff-down / proj_out (256 x 2), its 3x3 convs at BN 160 (256 x 2) and
# 64 (256 x 5), GEGLU (256 x 10), the 256-row 32x32 level (32 x 4, one wave) and forced multi-wave 256-row launches (128 x 4,
# 10 x 17), the coverage rows (10 x 17, 24 x 9, 32 x 17) and small grids
CASES = [(256, 2, 1), (256, 5, 1), (256, 10, 1), (32, 4, 1), (128, 4, 1), (10, 17, 1), (24, 9, 1), (32, 17, 1), (128, 3, 1),
         (5, 3, 1), (1, 2, 1), (300, 3, 1), (7, 1, 1)]


@pytest.mark.parametrize("n_fast", [0, 1])
@pytest.mark.parametrize("tiles_m,tiles_n,ksplit", CASES)
def test_both_orders_cover_every_tile_once_at_132_sms(tiles_m, tiles_n, ksplit, n_fast):
    ctas = min(132, tiles_m * tiles_n * ksplit)
    seen = [(m, n, k) for _, m, n, k, _ in walk(ctas, tiles_m, tiles_n, ksplit, n_fast)]
    assert sorted(seen) == sorted(itertools.product(range(tiles_m), range(tiles_n), range(ksplit)))


@pytest.mark.parametrize("sms,tiles_m,tiles_n,ksplit", [(148, 256, 2, 1), (120, 4, 5, 6), (148, 4, 5, 7), (74, 3, 37, 1),
                                                        (132, 256, 10, 1), (2, 1, 2, 1)])
def test_m_fast_walk_is_the_walk_it_replaces(sms, tiles_m, tiles_n, ksplit):
    ctas = min(sms, tiles_m * tiles_n * ksplit)
    got = [(c, m, n, k) for c, m, n, k, _ in walk(ctas, tiles_m, tiles_n, ksplit, 0)]
    assert got == list(walk_m_fast(ctas, tiles_m, tiles_n, ksplit))


@pytest.mark.parametrize("n_fast", [0, 1])
@pytest.mark.parametrize("tiles_m,tiles_n,ksplit", CASES)
def test_ln_prefetch_names_the_next_tile(tiles_m, tiles_n, ksplit, n_fast):
    ctas = min(132, tiles_m * tiles_n * ksplit)
    seq = defaultdict(list)
    for cta, m, _n, _k, m_next in walk(ctas, tiles_m, tiles_n, ksplit, n_fast):
        seq[cta].append((m, m_next))
    for s in seq.values():
        assert [nxt for _, nxt in s[:-1]] == [m for m, _ in s[1:]] and s[-1][1] is None


def waves_of_each_m_tile(tiles_m, tiles_n, n_fast, sms=132):
    """{M tile: the waves (the k-th tile of a CTA runs in wave k) in which some CTA runs one of its tiles}"""
    k_of, out = defaultdict(int), defaultdict(set)
    for cta, m, _n, _k, _ in walk(min(sms, tiles_m * tiles_n), tiles_m, tiles_n, 1, n_fast):
        out[m].add(k_of[cta])
        k_of[cta] += 1
    return out


def test_n_fast_reads_each_a_band_in_one_wave_on_the_64x64_ff_down():
    """ff-down of the 64x64 level (256 M tiles x 2 N tiles): N-fast, both N tiles of an M tile run in the same wave, so its A rows
    are read from HBM once; M-fast, N tile 1 of every M tile runs in a later wave than N tile 0."""
    assert all(len(w) == 1 for w in waves_of_each_m_tile(256, 2, 1).values())
    assert all(len(w) == 2 for w in waves_of_each_m_tile(256, 2, 0).values())


def test_n_fast_walk_changes_the_n_tile_within_a_cta_on_the_geglu_shape():
    seq = [n for cta, _, n, _, _ in walk(132, 256, 10, 1, 1) if cta == 0]
    assert len(seq) >= 19 and set(seq) == {0, 2, 4, 6, 8}       # 132 % 10 == 2


@pytest.mark.parametrize("desc,M,a_chan,N,Ktot,ksplit,tiles_n,want", [
    ("ff-down 64x64", 32768, 1280, 320, 1280, 1, 2, True),
    ("proj_out 64x64", 32768, 320, 320, 320, 1, 2, True),
    ("GEGLU 64x64", 32768, 320, 2560, 320, 1, 10, True),
    ("3x3 conv 960 -> 320 + skip, 64x64", 32768, 960 + 960, 320, 9 * 960 + 960, 1, 2, True),
    ("3x3 conv 320 -> 320, 64x64", 32768, 320, 320, 9 * 320, 1, 2, True),
    ("to_k of a 77-token context", 616, 768, 320, 768, 1, 3, True),
    ("split-K 8x8 conv", 512, 1280, 1280, 9 * 1280, 4, 8, False),
    ("one N tile", 32768, 320, 64, 320, 1, 1, False),
    ("W outweighs A", 1200, 256, 4192, 200, 1, 17, False),
])
def test_order_rule(desc, M, a_chan, N, Ktot, ksplit, tiles_n, want):
    assert n_fast_rule(M, a_chan, N, Ktot, ksplit, tiles_n) == want, desc
