"""Host-side model of igemm.cu's persistent tile scheduler (the producer, MMA and epilogue roles must walk the SAME
(m, n, k-split) sequence, each with its own incremental arithmetic).  Pure Python mirror of the index updates in
igemm_kernel: every output tile is visited exactly once, by exactly one CTA, in the grid-strided M-fast order."""
import itertools

import pytest


def walk(num_ctas, unitsM, tilesN, ksplit):
    """Yields (cta, m_idx, n_idx, ks) exactly as the producer / epilogue loops of igemm_kernel compute them (CTAS == 1)."""
    num_tiles = unitsM * tilesN * ksplit
    for cta in range(num_ctas):
        t_first, t_step, t_end = cta, num_ctas, num_tiles
        step_m, step_r = t_step % unitsM, t_step // unitsM
        unit_m, rest = t_first % unitsM, t_first // unitsM
        t = t_first
        while t < t_end:
            m_idx = unit_m
            n_idx, ks = rest, 0
            if ksplit > 1:
                n_idx, ks = rest % tilesN, rest // tilesN
            unit_m += step_m
            rest += step_r
            if unit_m >= unitsM:
                unit_m -= unitsM
                rest += 1
            # the MMA role only needs the k-split index: (t / unitsM) / tilesN
            assert ks == ((t // unitsM) // tilesN if ksplit > 1 else 0)
            yield cta, m_idx, n_idx, ks
            t += t_step


CASES = [(148, 256, 2, 1), (148, 256, 4, 1), (148, 64, 10, 1), (148, 16, 5, 1), (37, 7, 1, 1), (120, 4, 5, 6),
         (148, 4, 5, 7), (2, 1, 2, 1), (148, 1024, 1, 1), (74, 3, 37, 1), (148, 300, 3, 1)]


@pytest.mark.parametrize("sms,unitsM,tilesN,ksplit", CASES)
def test_default_order_covers_every_tile_once(sms, unitsM, tilesN, ksplit):
    ctas = min(sms, unitsM * tilesN * ksplit)
    seen = [(m, n, k) for _, m, n, k in walk(ctas, unitsM, tilesN, ksplit)]
    assert sorted(seen) == sorted(itertools.product(range(unitsM), range(tilesN), range(ksplit)))


def test_strided_walk_changes_the_n_tile_every_other_tile_on_the_geglu_shape():
    tiles = list(walk(132, 256, 10, 1))
    seq = [n for cta, _, n, _ in tiles if cta == 0]
    assert sum(1 for a, b in zip(seq, seq[1:]) if a != b) >= len(seq) // 2 - 1          # 20 tiles, ~10 table reloads


# the instantiations run_igemm can launch: (BN, epilogue MODE)
IGEMM_INSTANTIATIONS = [(bn, mode) for bn in (64, 128, 160, 256) for mode in (0, 3, 5, 7)] + [(256, 4), (256, 6)]


def test_igemm_coverage_table_reaches_every_instantiation_with_a_multi_tile_walk():
    """test_igemm_coverage_gpu.CASES: every instantiation has a row in which, on 132 SMs, some CTA runs two or more tiles on
    different N tiles, with an M tail, a K tail and (except GEGLU, whose N is a multiple of 256) a partial last N tile.  A new
    instantiation without such a row fails here."""
    from test_igemm_coverage_gpu import CASES, multi_tile_n_change, tile_geometry
    assert len(IGEMM_INSTANTIATIONS) == 18
    for bn, mode in IGEMM_INSTANTIATIONS:
        rows = [c for c in CASES if (c["bn"], c["mode"]) == (bn, mode) and c["walk"]]
        assert rows, f"no multi-tile case for BN {bn} mode {mode}"
        for c in rows:
            tm, tn, ks, _ = tile_geometry(c)
            assert multi_tile_n_change(min(tm * tn * ks, 132), tm, tn, ks), f"{c['id']}: no CTA changes its N tile on 132 SMs"
        assert any(c["kind"] != "conv" and c["M"] % 128 and c["K"] % 64 and (c["N"] % bn or mode in (4, 6)) for c in rows), \
            f"BN {bn} mode {mode}: no multi-tile case with M, K and N tails"
    assert {(c["bn"], c["mode"]) for c in CASES if c["bn"]} <= set(IGEMM_INSTANTIATIONS)
