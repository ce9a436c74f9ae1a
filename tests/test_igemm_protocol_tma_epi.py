"""Protocol model of igemm_kernel's TMA-store epilogues (modes 3-7, igemm.cu), run on the CPU.

In these modes the accumulator never leaves the registers: after a tile's last product retires (wgmma_wait<0>) each warp runs
the epilogue on its own 16 rows and stores them through four 1 KB staging boxes with TMA stores, and the producer (warp 8) runs
ahead into the next tile gated only by the empty barriers of the ring.  The two warpgroups meet only where the bias / LayerNorm
tables in shared memory are reloaded (a barrier before and after the reload, when the N tile changes).  Same simulator as
tests/test_attention_protocol.py (random interleavings, random latencies, in-order products per warpgroup); checks that

  * a ring stage is never refilled while a product still reads it, and every product reads the k-block it expects;
  * the epilogue reads the accumulator only once every product of the tile has retired;
  * the tables are read only when they hold the tile's N tile, and are rewritten only once nobody reads them;
  * a staging box is rewritten only after the TMA store issued from it has read it (bulk wait_group.read), and no store still
    reads shared memory when its warp exits.

tests/test_igemm_protocol.py models modes 0-2, whose accumulator is parked in shared memory that aliases the ring.  The mutation
tests below drop each wait of the kernel in turn and require the model to catch it."""
import pytest

from test_attention_protocol import AsyncQueue, MBar, NamedBar, Sim, delay, wait

SLOTS = 4          # staging boxes per warp
MUTATIONS = ("no_empty_wait", "no_full_wait", "no_wgmma_wait1", "no_wgmma_wait0", "no_table_sync_before", "no_table_sync_after",
             "no_wait_read", "no_final_wait")


def simulate_tma_epi(seed, ntiles, kblocks, STAGES, nchunks, n_every=2, mutate=None):
    """One persistent CTA over `ntiles` tiles of `kblocks` k-blocks; the N tile (and so the tables) changes every `n_every`
    tiles; every warp stores `nchunks` 32-column chunks per tile."""
    assert mutate is None or mutate in MUTATIONS
    sim = Sim(seed)
    NG, WPG = 2, 4
    full, empty = [MBar(1) for _ in range(STAGES)], [MBar(NG * WPG) for _ in range(STAGES)]
    epi_bar = NamedBar(NG)                                          # bar.sync 1, 256 over both warpgroups
    stage_data, stage_busy = [None] * STAGES, [0] * STAGES          # (tile, kb) held by a stage; products reading it
    kb_done = [0] * NG
    aqs = [AsyncQueue() for _ in range(NG)]
    table = dict(n=None, writers=set(), readers=0)                  # sbias / slnx: N tile held, groups that wrote their part
    warps = [dict(slot=0, boxes=[None] * SLOTS, stores=[], exited=False) for _ in range(NG * WPG)]
    live = dict(consumers=NG)

    def n_tile(t):
        return t // n_every

    def producer():
        stage, phase = 0, 0
        for t in range(ntiles):
            for kb in range(kblocks):
                if mutate != "no_empty_wait":
                    yield wait(empty[stage], phase ^ 1)
                assert stage_busy[stage] == 0, "smem stage refilled while a product still reads it"
                yield from delay(sim)
                stage_data[stage] = (t, kb)
                full[stage].arrive()                                   # TMA complete_tx
                stage += 1
                if stage == STAGES:
                    stage, phase = 0, phase ^ 1

    def store_unit():
        """the TMA unit: reads each warp's stores from its staging boxes in issue order, then completes them"""
        while True:
            busy = [w for w in warps if w["stores"]]
            if not busy:
                if live["consumers"] == 0:
                    return
                yield None
                continue
            w = sim.rng.choice(busy)
            st = w["stores"][0]
            yield from delay(sim)
            if not st["read"]:
                assert not w["exited"], "a TMA store reads the staging box of a warp that has exited"
                assert w["boxes"][st["slot"]] == st["data"], "staging box rewritten before the TMA store issued from it read it"
                st["read"] = True
            else:
                w["stores"].pop(0)                                     # the bulk group completes

    def sync_groups():
        g0 = epi_bar.gen
        epi_bar.arrive()
        yield lambda g0=g0: epi_bar.gen != g0

    def consumer(g):
        aq = aqs[g]
        stage, phase = 0, 0
        for it in range(ntiles):
            if it == 0 or n_tile(it) != n_tile(it - 1):                # table reload, uniform over both groups
                if mutate != "no_table_sync_before":
                    yield from sync_groups()                           # the previous tile's readers are done
                assert table["readers"] == 0, "table rewritten while an epilogue still reads it"
                if table["n"] != n_tile(it):
                    table["n"], table["writers"] = n_tile(it), set()
                yield from delay(sim)
                table["writers"].add(g)
                if mutate != "no_table_sync_after":
                    yield from sync_groups()                           # both groups' parts are written
            kb_done[g] = 0
            prev = None
            for kb in range(kblocks):
                if mutate != "no_full_wait":
                    yield wait(full[stage], phase)

                def start(it=it, kb=kb, stage=stage):
                    assert stage_data[stage] == (it, kb), f"product of tile {it} k-block {kb} reads a stage holding {stage_data[stage]}"
                    stage_busy[stage] += 1

                def end(stage=stage):
                    stage_busy[stage] -= 1
                    kb_done[g] += 1
                aq.issue(start, end)
                if prev is not None:                                   # wgmma_wait<1>: the previous k-block's product retired
                    if mutate != "no_wgmma_wait1":
                        yield aq.drained(1)
                    for _ in range(WPG):
                        yield from delay(sim, 1)
                        empty[prev].arrive()
                prev = stage
                stage += 1
                if stage == STAGES:
                    stage, phase = 0, phase ^ 1
            if mutate != "no_wgmma_wait0":
                yield aq.drained(0)                                    # wgmma_wait<0>
            for _ in range(WPG):
                yield from delay(sim, 1)
                empty[prev].arrive()
            # epilogue from the registers: each warp, chunk by chunk
            for w in range(WPG):
                W = warps[g * WPG + w]
                for c in range(nchunks):
                    assert kb_done[g] == kblocks, f"group {g} reads the accumulator of tile {it} after {kb_done[g]} of {kblocks} products"
                    assert table["n"] == n_tile(it) and len(table["writers"]) == NG, \
                        f"epilogue of tile {it} reads the tables of N tile {table['n']} (written by {sorted(table['writers'])})"
                    table["readers"] += 1
                    yield from delay(sim, 1)
                    table["readers"] -= 1
                    if mutate != "no_wait_read":                       # bulk_wait_read<SLOTS - 1> (lane 0), then __syncwarp
                        yield lambda W=W: sum(not s["read"] for s in W["stores"]) <= SLOTS - 1
                    data = (it, g, w, c)
                    W["boxes"][W["slot"]] = data                       # stmatrix into the box, fence.proxy.async
                    W["stores"].append(dict(slot=W["slot"], data=data, read=False))   # TMA store + commit_group
                    W["slot"] = (W["slot"] + 1) % SLOTS
        for w in range(WPG):                                           # bulk_wait<0> before the CTA may exit
            W = warps[g * WPG + w]
            if mutate != "no_final_wait":
                yield lambda W=W: not W["stores"]
            W["exited"] = True
        aq.closed = True
        live["consumers"] -= 1

    sim.spawn(producer())
    sim.spawn(store_unit())
    for g in range(NG):
        sim.spawn(consumer(g))
        sim.spawn(sim.async_unit(aqs[g]))
    sim.run()


CHUNKS = {4: 8, 5: 5, 6: 4, 8: 2}          # STAGES -> 32-column chunks per warp (BN 256, 160, 128, 64)


@pytest.mark.parametrize("STAGES", [4, 5, 6, 8])
@pytest.mark.parametrize("ntiles,kblocks", [(1, 1), (1, 9), (3, 5), (4, 2), (5, 1), (6, 3), (4, 12)])
def test_tma_epilogue_protocol(STAGES, ntiles, kblocks):
    for seed in range(12):
        simulate_tma_epi(seed, ntiles, kblocks, STAGES, CHUNKS[STAGES])


@pytest.mark.parametrize("mutate", MUTATIONS)
def test_model_catches_each_missing_wait(mutate):
    caught = 0
    for seed in range(40):
        for kblocks in (1, 2):          # one k-block: the mainloop no longer hides a missing table barrier; two: a stage release
            try:
                simulate_tma_epi(seed, 6, kblocks, 4, 3, n_every=1, mutate=mutate)
            except AssertionError:
                caught += 1
    assert caught >= 8, f"only {caught}/80 interleavings expose the mutation {mutate}"
