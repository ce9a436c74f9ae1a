"""Protocol model of the attention kernel's warp-role synchronisation (attention.cu), run on the CPU.

attention_kernel<DK, DVP, BKV, KV_STAGES> coordinates a TMA producer warp and two consumer warpgroups (64 query rows each)
through 1-bit-parity mbarriers: K / V^T tiles arrive through two rings (k_full / v_full, one TMA arrival each) and are
released by all eight consumer warps (k_empty / v_empty, count 8).  Each warpgroup issues its products asynchronously
(wgmma.mma_async): S = Q K_j^T reads the K stage and writes the S registers, O += P V_j reads the V stage and the P registers.
A missing wgmma.wait_group, a release by the wrong number of warps or a wrong parity is a hang or silent corruption on the
GPU.  This test replays the kernel's sequence of waits / arrives / issues under thousands of random interleavings and random
latencies and checks, at every access, that:

  * a K / V stage is not refilled before every product that reads it has retired, and every product reads the tile it wants;
  * the softmax reads S_j only once the product that writes it has retired;
  * P_j is not written while PV_{j-1} may still read the P registers;
  * nobody passes an mbarrier wait early through parity aliasing; the run terminates (no deadlock).

It knows nothing about arithmetic — only about who may touch what, when.  tests/test_igemm_protocol_tma_epi.py reuses the
simulator.
"""
import random

import pytest


class MBar(object):
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0, "more arrivals than the barrier expects in one phase"
        if self.pending == 0:
            self.phase ^= 1
            self.pending = self.count

    def done(self, parity):          # mbarrier.try_wait.parity: has the phase with this parity completed?
        return self.phase != parity


class NamedBar(object):
    def __init__(self, warps):
        self.warps, self.n, self.gen = warps, 0, 0

    def arrive(self):
        self.n += 1
        assert self.n <= self.warps, "named barrier over-subscribed"
        if self.n == self.warps:
            self.n, self.gen = 0, self.gen + 1


class AsyncQueue(object):
    """One warpgroup's wgmma groups: (start_fn, end_fn) products that retire in issue order."""

    def __init__(self):
        self.q, self.issued, self.retired, self.closed = [], 0, 0, False

    def issue(self, start, end):
        self.q.append((start, end))
        self.issued += 1

    def drained(self, upto=0):       # wgmma.wait_group upto: at most `upto` products still pending
        return lambda: self.issued - self.retired <= upto


class Sim(object):
    """Agents are generators; they yield a predicate (block until true) or None (just a scheduling point)."""

    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.agents = []

    def spawn(self, gen):
        self.agents.append([gen, None])

    def async_unit(self, aq):
        """retires the products of one warpgroup in order, each after a random latency"""
        while True:
            if not aq.q:
                if aq.closed:
                    return
                yield None
                continue
            start, end = aq.q[0]
            start()                                   # product starts reading its operands
            for _ in range(self.rng.randint(0, 3)):
                yield None
            end()                                     # product retires
            aq.q.pop(0)
            aq.retired += 1

    def run(self, limit=300_000):
        steps = 0
        while self.agents:
            ready = [ag for ag in self.agents if ag[1] is None or ag[1]()]
            assert ready, "deadlock: every live role is blocked"
            ag = self.rng.choice(ready)
            try:
                ag[1] = next(ag[0])
            except StopIteration:
                self.agents.remove(ag)
            steps += 1
            assert steps < limit, "livelock (roles spin without progress)"


def delay(sim, hi=3):
    for _ in range(sim.rng.randint(0, hi)):
        yield None


def wait(bar, parity):
    return lambda: bar.done(parity)


# ---------------------------------------------------------------------------------------------------------------------
# attention_kernel<DK, DVP, BKV, KV_STAGES>: warp 8 = TMA producer, warps 0-7 = two consumer warpgroups
# ---------------------------------------------------------------------------------------------------------------------
def simulate_attention(seed, ntiles, ST, mutate=None, jitter=3, skewed=False):
    """One CTA: the producer and the two consumer warpgroups, each owning one 64-row query tile of the CTA's 128 rows.
    skewed: warpgroup 1's softmax phase runs up to four times longer than warpgroup 0's, so one group is tiles behind the
    other on the shared K / V stages.  jitter = longest softmax phase of a tile in scheduling steps.
    mutate (self-checks of the checker), each one wait or release of the real kernel changed:
      'no_s_free'     the group uses its scores and frees the K stage without waiting for the S product (no wgmma_wait<0>);
      'no_pv_wait'    the group writes the next P and frees the V stage without waiting for the PV product;
      'k_release_g0'  the K stage is released by warpgroup 0's warps only (k_empty count 4);
      'surplus_pass'  one warp of warpgroup 0 arrives twice on k_empty (one arrival more per phase than the barrier counts);
      'single_p_full' PV is issued behind the k_full wait alone, as if K and V^T completed on a single full barrier;
      'no_last_wait'  the last tile's PV product is not waited for before the epilogue reads O."""
    sim = Sim(seed)
    NG, WPG = 2, 4
    q_full = MBar(1)
    k_full, v_full = [MBar(1) for _ in range(ST)], [MBar(1) for _ in range(ST)]
    k_empty = [MBar(WPG if mutate == "k_release_g0" else NG * WPG) for _ in range(ST)]
    v_empty = [MBar(NG * WPG) for _ in range(ST)]
    q_loaded = [False]
    kst, vst = [None] * ST, [None] * ST            # tile held by each K / V stage
    kbusy, vbusy = [0] * ST, [0] * ST              # products currently reading the stage
    S = [dict(tile=None) for _ in range(NG)]       # tile whose scores sit in the group's S registers
    P = [dict(tile=None, busy=0) for _ in range(NG)]
    pv_retired = [-1] * NG
    aqs = [AsyncQueue() for _ in range(NG)]

    def tma():
        yield from delay(sim)
        q_loaded[0] = True
        q_full.arrive()
        for j in range(ntiles):
            st, ph = j % ST, (j // ST) & 1
            yield wait(k_empty[st], ph ^ 1)
            assert kbusy[st] == 0, "K stage refilled while a product reads it"
            yield from delay(sim)
            kst[st] = j
            k_full[st].arrive()
            yield wait(v_empty[st], ph ^ 1)
            assert vbusy[st] == 0, "V stage refilled while a product reads it"
            yield from delay(sim)
            vst[st] = j
            v_full[st].arrive()

    def consumer(g):
        aq = aqs[g]
        softmax_steps = jitter * (4 if (skewed and g == 1) else 1)
        yield wait(q_full, 0)
        for j in range(ntiles):
            st, ph = j % ST, (j // ST) & 1
            last = j == ntiles - 1
            yield wait(k_full[st], ph)

            def s_start(j=j, st=st):
                assert q_loaded[0], "S product before Q arrived"
                assert kst[st] == j, f"S_{g}({j}) reads a K stage holding tile {kst[st]}"
                kbusy[st] += 1
                S[g]["tile"] = None

            def s_end(j=j, st=st):
                kbusy[st] -= 1
                S[g]["tile"] = j
            aq.issue(s_start, s_end)
            if mutate != "no_s_free":
                yield aq.drained(0)                       # wgmma_wait<0>
            if not (mutate == "k_release_g0" and g == 1):
                for w in range(WPG):                      # each warp: __syncwarp, lane 0 arrives
                    yield from delay(sim)
                    k_empty[st].arrive()
                    if mutate == "surplus_pass" and g == 0 and w == 0:
                        k_empty[st].arrive()
            assert S[g]["tile"] == j, f"group {g} read S registers holding tile {S[g]['tile']} instead of {j}"
            yield from delay(sim, softmax_steps)          # masking, row max, lazy rescale of O
            assert P[g]["busy"] == 0, f"group {g} writes P({j}) while PV({P[g]['tile']}) still reads the registers"
            P[g]["tile"] = j
            if mutate != "single_p_full":
                yield wait(v_full[st], ph)

            def pv_start(j=j, st=st):
                assert vst[st] == j, f"PV_{g}({j}) reads a V stage holding tile {vst[st]}"
                assert P[g]["tile"] == j, f"PV_{g}({j}) reads P of tile {P[g]['tile']}"
                vbusy[st] += 1
                P[g]["busy"] += 1

            def pv_end(j=j, st=st):
                vbusy[st] -= 1
                P[g]["busy"] -= 1
                pv_retired[g] = j
            aq.issue(pv_start, pv_end)
            if mutate != "no_pv_wait" and not (mutate == "no_last_wait" and last):
                yield aq.drained(0)
            for _ in range(WPG):
                yield from delay(sim)
                v_empty[st].arrive()
        assert pv_retired[g] == ntiles - 1, f"epilogue of group {g} read O before the last PV retired"
        aq.closed = True

    sim.spawn(tma())
    for g in range(NG):
        sim.spawn(consumer(g))
        sim.spawn(sim.async_unit(aqs[g]))
    sim.run()


def _caught(mutation, runs=100, ntiles=6, **kw):
    caught = 0
    for seed in range(runs):
        try:
            simulate_attention(seed, ntiles, 2, mutate=mutation, jitter=12, **kw)
        except AssertionError:
            caught += 1
    return caught


@pytest.mark.parametrize("stages", [1, 2, 3])
@pytest.mark.parametrize("ntiles", [1, 2, 3, 5, 8, 32])
def test_wgmma_attention_protocol(ntiles, stages):
    for seed in range(40 if ntiles < 32 else 8):
        simulate_attention(seed, ntiles, stages)


@pytest.mark.parametrize("skewed", [True, False])
@pytest.mark.parametrize("ntiles", [1, 2, 3, 4, 7, 32])
def test_two_tile_kernel_protocol(ntiles, skewed):
    """the CTA's two 64-row query tiles (one per warpgroup) share every K / V stage; with skewed=True one group runs tiles
    behind the other, so the stage releases of both groups have to be counted right"""
    for seed in range(40 if ntiles < 32 else 6):
        simulate_attention(seed, ntiles, 3, skewed=skewed)
        simulate_attention(seed + 1000, ntiles, 2, skewed=skewed)


@pytest.mark.parametrize("mutation", ["no_s_free", "no_pv_wait", "k_release_g0", "surplus_pass"])
def test_two_tile_model_self_check(mutation):
    """each mutation removes one wait / changes one release of the real kernel: the model must notice"""
    # (a surplus arrival per phase releases a stage early once the surplus adds up to a whole warpgroup: run 24 tiles)
    caught = _caught(mutation, ntiles=24 if mutation == "surplus_pass" else 6, skewed=(mutation in ("k_release_g0", "surplus_pass")))
    assert caught >= 10, f"only {caught}/100 interleavings expose the '{mutation}' bug: the model lost its teeth"


@pytest.mark.parametrize("mutation", ["single_p_full", "no_last_wait"])
def test_the_model_catches_the_hazards_it_was_written_for(mutation):
    """V^T must be waited for on its own barrier, and the epilogue must wait for the last PV product"""
    caught = _caught(mutation, runs=300)
    assert caught >= 10, f"only {caught}/300 interleavings expose the '{mutation}' bug: the model lost its teeth"
