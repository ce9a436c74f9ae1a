"""Host-side model of igemm.cu's persistent tile scheduler (the producer, MMA and epilogue roles must walk the SAME
(m, n, k-split) sequence, each with its own incremental arithmetic).  Pure Python mirror of the index updates in
igemm_kernel: every output tile is visited exactly once, by exactly one CTA, in both the default (M-fast) and the opt-in
N-fast order, and the N-fast order keeps a CTA on one N tile whenever grid % tilesN == 0 (the host-side condition)."""
import itertools

import pytest


def walk(num_ctas, unitsM, tilesN, ksplit, nfast, chunked=False):
    """Yields (cta, m_idx, n_idx, ks) exactly as the producer / epilogue loops of igemm_kernel compute them (CTAS == 1).
    chunked: every CTA walks a contiguous range of ceil(tiles / CTAs) tiles instead of the grid-strided sequence."""
    num_tiles = unitsM * tilesN * ksplit
    per_cta = -(-num_tiles // num_ctas)
    for cta in range(num_ctas):
        t_first, t_step = (cta * per_cta, 1) if chunked else (cta, num_ctas)
        t_end = min(num_tiles, t_first + per_cta) if chunked else num_tiles
        step_m, step_r = t_step % unitsM, t_step // unitsM
        unit_m, rest = t_first % unitsM, t_first // unitsM
        nf_step_n, nf_step_m = (t_step % tilesN, t_step // tilesN) if nfast else (0, 0)
        nf_n, nf_m = (t_first % tilesN, t_first // tilesN) if nfast else (0, 0)
        t = t_first
        while t < t_end:
            m_idx = nf_m if nfast else unit_m
            n_idx, ks = (nf_n if nfast else rest), 0
            if ksplit > 1:
                n_idx, ks = rest % tilesN, rest // tilesN
            nf_n += nf_step_n
            nf_m += nf_step_m
            if nfast and nf_n >= tilesN:
                nf_n -= tilesN
                nf_m += 1
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
    seen = [(m, n, k) for _, m, n, k in walk(ctas, unitsM, tilesN, ksplit, nfast=False)]
    assert sorted(seen) == sorted(itertools.product(range(unitsM), range(tilesN), range(ksplit)))


@pytest.mark.parametrize("sms,unitsM,tilesN,ksplit", [c for c in CASES if c[3] == 1 and c[2] > 1])
def test_nfast_order_covers_every_tile_once_and_pins_the_n_tile(sms, unitsM, tilesN, ksplit):
    ctas = min(sms, unitsM * tilesN)
    tiles = list(walk(ctas, unitsM, tilesN, 1, nfast=True))
    assert sorted((m, n) for _, m, n, _ in tiles) == sorted(itertools.product(range(unitsM), range(tilesN)))
    if ctas % tilesN == 0:      # the only case in which run_igemm turns N-fast on
        per_cta = {}
        for cta, _, n, _ in tiles:
            per_cta.setdefault(cta, set()).add(n)
        assert all(len(v) == 1 for v in per_cta.values()), "a CTA must keep its N tile (bias tile cached in shared memory)"
        # and the N tiles of one M tile run in the same wave: neighbouring CTAs, same iteration
        first_wave = [(m, n) for cta, m, n, _ in tiles if cta < tilesN]
        assert {m for m, _ in first_wave[:1]} == {0}


@pytest.mark.parametrize("sms,unitsM,tilesN,ksplit", [c for c in CASES if c[3] == 1])
def test_chunked_order_covers_every_tile_once_and_rarely_changes_the_n_tile(sms, unitsM, tilesN, ksplit):
    """p.chunked: contiguous tile ranges.  Same coverage; a CTA sees at most ceil(range / unitsM) + 1 distinct N tiles, where the
    strided walk changes its N tile every unitsM / CTAs tiles (GEGLU at the 64x64 level: 256 M tiles x 10 N tiles on 148 CTAs)."""
    ctas = min(sms, unitsM * tilesN)
    tiles = list(walk(ctas, unitsM, tilesN, 1, nfast=False, chunked=True))
    assert sorted((m, n) for _, m, n, _ in tiles) == sorted(itertools.product(range(unitsM), range(tilesN)))
    per = -(-unitsM * tilesN // ctas)
    changes = {}
    last = {}
    for cta, _, n, _ in tiles:
        if cta in last and last[cta] != n:
            changes[cta] = changes.get(cta, 0) + 1
        last[cta] = n
    assert max(changes.values(), default=0) <= -(-per // unitsM), "a contiguous range crosses at most range / unitsM N-tile boundaries"


def test_strided_walk_changes_the_n_tile_every_other_tile_on_the_geglu_shape():
    tiles = list(walk(132, 256, 10, 1, nfast=False))
    seq = [n for cta, _, n, _ in tiles if cta == 0]
    assert sum(1 for a, b in zip(seq, seq[1:]) if a != b) >= len(seq) // 2 - 1          # 20 tiles, ~10 table reloads
    seq_c = [n for cta, _, n, _ in walk(132, 256, 10, 1, nfast=False, chunked=True) if cta == 0]
    assert sum(1 for a, b in zip(seq_c, seq_c[1:]) if a != b) == 0


# the instantiations run_igemm can launch: (BN, epilogue MODE)
IGEMM_INSTANTIATIONS = [(bn, mode) for bn in (64, 128, 160, 256) for mode in (0, 1, 3, 5, 7)] + [(256, 2), (256, 4), (256, 6)]


def test_igemm_coverage_table_reaches_every_instantiation_with_a_multi_tile_walk():
    """test_igemm_coverage_gpu.CASES: every instantiation has a row in which, on 132 SMs, some CTA runs two or more tiles on
    different N tiles, with an M tail, a K tail and (except GEGLU, whose N is a multiple of 256) a partial last N tile.  A new
    instantiation without such a row fails here."""
    from test_igemm_coverage_gpu import CASES, multi_tile_n_change, tile_geometry
    assert len(IGEMM_INSTANTIATIONS) == 23
    for bn, mode in IGEMM_INSTANTIATIONS:
        rows = [c for c in CASES if (c["bn"], c["mode"]) == (bn, mode) and c["walk"]]
        assert rows, f"no multi-tile case for BN {bn} mode {mode}"
        for c in rows:
            tm, tn, ks, _ = tile_geometry(c)
            assert multi_tile_n_change(min(tm * tn * ks, 132), tm, tn, ks), f"{c['id']}: no CTA changes its N tile on 132 SMs"
        assert any(c["kind"] != "conv" and c["M"] % 128 and c["K"] % 64 and (c["N"] % bn or mode in (2, 4, 6)) for c in rows), \
            f"BN {bn} mode {mode}: no multi-tile case with M, K and N tails"
    assert {(c["bn"], c["mode"]) for c in CASES if c["bn"]} <= set(IGEMM_INSTANTIATIONS)
