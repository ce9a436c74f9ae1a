"""Protocol model of the d_head <= 80 attention kernels, whose consumer warps issue the TMA loads (attention.cu, TMA_WARP false).

attention_kernel<DK, DVP, BKV, KV_STAGES, false> (two or three stages) has no producer warp: lane 0 of warp 0 loads Q and
refills the K ring, lane 0 of warp 4 refills the V^T ring.  Both load the first KV_STAGES - 1 tiles up front; in iteration j each loads tile
j + KV_STAGES - 1 into the stage of tile j - 1, right after issuing its warpgroup's S_j product, once that stage's empty barrier
(count 8: one arrival per consumer warp of both warpgroups) has completed the phase of tile j - 1.  So warpgroup 0 waits for
warpgroup 1 only to release K stages, and warpgroup 1 waits for warpgroup 0 only to release V^T stages.  The loads complete
asynchronously, in any order, on the full barriers (one arrival each).

Same simulator as tests/test_attention_protocol.py (random interleavings, random latencies, in-order products per warpgroup),
which models the kernel with a producer warp (d_head 160).  Checks, at every access, that

  * a stage is refilled only once both warpgroups' products on its previous tile have retired and every warp released it;
  * no load is in flight into a stage while a product reads it, and every product reads the tile it wants;
  * nobody passes an mbarrier wait early through parity aliasing (a wait that passes a lap early fails the first check);
  * the run terminates (no deadlock, no livelock), under random interleavings and with either warpgroup tiles behind.

The mutation tests change one thing of the kernel each and require the model to catch it.
"""
import pytest

from test_attention_protocol import AsyncQueue, MBar, Sim, delay, wait

MUTATIONS = ("no_empty_wait", "stale_parity", "count_4")


def simulate_consumer_tma(seed, ntiles, ST, mutate=None, jitter=3, slow=None):
    """One CTA of the 256-thread kernel.  slow: index of the warpgroup whose softmax runs four times longer (None: neither).
    mutate (self-checks of the checker):
      'no_empty_wait' a refill is issued without waiting for the stage's empty barrier;
      'stale_parity'  from the second lap on, the empty wait uses the parity of the lap before (passes one phase early);
      'count_4'       the empty barriers count 4 arrivals (one warpgroup's) instead of 8."""
    assert mutate is None or mutate in MUTATIONS
    sim = Sim(seed)
    NG, WPG = 2, 4
    q_full = MBar(1)
    k_full, v_full = [MBar(1) for _ in range(ST)], [MBar(1) for _ in range(ST)]
    k_empty = [MBar(WPG if mutate == "count_4" else NG * WPG) for _ in range(ST)]
    v_empty = [MBar(WPG if mutate == "count_4" else NG * WPG) for _ in range(ST)]
    q_loaded = [False]
    held = {"k": [None] * ST, "v": [None] * ST}         # tile held by each stage
    busy = {"k": [0] * ST, "v": [0] * ST}               # products currently reading the stage
    released = {"k": [[0] * ntiles for _ in range(NG)], "v": [[0] * ntiles for _ in range(NG)]}   # warp releases per tile
    inflight = []                                       # issued TMA loads: (ring, stage, tile)
    S = [dict(tile=None) for _ in range(NG)]
    P = [dict(tile=None, busy=0) for _ in range(NG)]
    pv_retired = [-1] * NG
    aqs = [AsyncQueue() for _ in range(NG)]
    live = dict(consumers=NG)
    full = {"k": k_full, "v": v_full}
    empty = {"k": k_empty, "v": v_empty}

    def tma_unit():
        """completes the issued loads in random order, each after a random latency"""
        while inflight or live["consumers"]:
            if not inflight:
                yield lambda: inflight or not live["consumers"]
                continue
            ring, st, t = inflight.pop(sim.rng.randrange(len(inflight)))
            yield from delay(sim)
            if ring == "q":
                q_loaded[0] = True
                q_full.arrive()
                continue
            assert busy[ring][st] == 0, f"{ring.upper()} tile {t} lands in stage {st} while a product reads it"
            held[ring][st] = t
            full[ring][st].arrive()

    def load(ring, t):
        """the elected lane: wait until the stage's previous tile t - ST is released, then issue tile t"""
        st = t % ST
        parity = ((t // ST) & 1) ^ 1
        if mutate == "stale_parity" and t >= ST:
            parity ^= 1
        if mutate != "no_empty_wait":
            yield wait(empty[ring][st], parity)
        if t >= ST:
            for g in range(NG):
                assert released[ring][g][t - ST] == WPG, \
                    f"{ring.upper()} stage {st} refilled with tile {t} before warpgroup {g} released tile {t - ST}"
        assert busy[ring][st] == 0, f"{ring.upper()} stage {st} refilled while a product reads it"
        assert not any(r == ring and s == st for r, s, _ in inflight), f"two loads in flight into {ring.upper()} stage {st}"
        inflight.append((ring, st, t))

    def release(ring, g, st, j):
        for _ in range(WPG):                            # each warp: __syncwarp, lane 0 arrives
            yield from delay(sim)
            released[ring][g][j] += 1
            empty[ring][st].arrive()

    def consumer(g):
        aq = aqs[g]
        ring = "k" if g == 0 else "v"
        softmax_steps = jitter * (4 if slow == g else 1)
        if g == 0:                                      # warp 0: Q and the first ST - 1 K tiles
            inflight.append(("q", None, None))
        for t in range(min(ST - 1, ntiles)):
            yield from load(ring, t)
        yield wait(q_full, 0)
        for j in range(ntiles):
            st, ph = j % ST, (j // ST) & 1
            yield wait(k_full[st], ph)

            def s_start(j=j, st=st):
                assert q_loaded[0], "S product before Q arrived"
                assert held["k"][st] == j, f"S_{g}({j}) reads a K stage holding tile {held['k'][st]}"
                busy["k"][st] += 1
                S[g]["tile"] = None

            def s_end(j=j, st=st):
                busy["k"][st] -= 1
                S[g]["tile"] = j
            aq.issue(s_start, s_end)
            if j + ST - 1 < ntiles:                      # under the S product: refill the stage of tile j - 1
                yield from load(ring, j + ST - 1)
            yield aq.drained(0)                          # wgmma_wait<0>
            yield from release("k", g, st, j)
            assert S[g]["tile"] == j, f"group {g} read S registers holding tile {S[g]['tile']} instead of {j}"
            yield from delay(sim, softmax_steps)         # masking, row max, lazy rescale, P
            assert P[g]["busy"] == 0, f"group {g} writes P({j}) while PV({P[g]['tile']}) still reads the registers"
            P[g]["tile"] = j
            yield wait(v_full[st], ph)

            def pv_start(j=j, st=st):
                assert held["v"][st] == j, f"PV_{g}({j}) reads a V stage holding tile {held['v'][st]}"
                assert P[g]["tile"] == j, f"PV_{g}({j}) reads P of tile {P[g]['tile']}"
                busy["v"][st] += 1
                P[g]["busy"] += 1

            def pv_end(j=j, st=st):
                busy["v"][st] -= 1
                P[g]["busy"] -= 1
                pv_retired[g] = j
            aq.issue(pv_start, pv_end)
            yield aq.drained(0)
            yield from release("v", g, st, j)
        assert pv_retired[g] == ntiles - 1, f"epilogue of group {g} read O before the last PV retired"
        aq.closed = True
        live["consumers"] -= 1

    for g in range(NG):
        sim.spawn(consumer(g))
        sim.spawn(sim.async_unit(aqs[g]))
    sim.spawn(tma_unit())
    sim.run()


@pytest.mark.parametrize("slow", [None, 0, 1])
@pytest.mark.parametrize("stages", [2, 3, 4])
@pytest.mark.parametrize("ntiles", [1, 2, 3, 4, 5, 8, 32])
def test_consumer_tma_protocol(ntiles, stages, slow):
    """both warpgroups share every stage and each refills one ring, so with either one tiles behind the other the
    releases of both have to be counted right, and neither may wait on the other in a cycle"""
    for seed in range(25 if ntiles < 32 else 5):
        simulate_consumer_tma(seed, ntiles, stages, slow=slow)


@pytest.mark.parametrize("mutate", MUTATIONS)
def test_model_catches_each_mutation(mutate):
    caught = 0
    for seed in range(60):
        try:
            simulate_consumer_tma(seed, 12, 3, mutate=mutate, jitter=12, slow=seed % 2)
        except AssertionError:
            caught += 1
    assert caught >= 10, f"only {caught}/60 interleavings expose the mutation {mutate}: the model lost its teeth"
