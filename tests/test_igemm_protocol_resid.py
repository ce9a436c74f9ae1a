"""Protocol model of the residual path of igemm_kernel's TMA-store epilogues (modes 3 and 7, igemm.cu), run on the CPU.

A warp's residual enters through the staging boxes its output leaves from: lane 0 TMA-loads the residual of a 32-column chunk
into the box the chunk will be stored from, completing on that box's mbarrier.  The first kBoxes chunks of a tile are requested
under the tile's mainloop, after a bulk wait_group.read that shows the previous tile's stores have read every box; chunk
j - 1 + kBoxes is requested at chunk j into the box of chunk j - 1, after the same wait.  The epilogue waits on the box's
mbarrier, reads the residual (ldmatrix), writes the output over it (stmatrix) and stores the box.  Same simulator as
tests/test_attention_protocol.py (random interleavings; TMA loads complete in any order, stores in issue order).  Checks that

  * a residual load never overwrites a box before the store issued from it has read it;
  * the epilogue reads a box only once it holds the residual of that very chunk;
  * a store reads the output it was issued for;
  * with the output written in place over the residual, every residual element is read before its output is stored.

The mutation tests drop each wait of the protocol in turn and require the model to catch it."""
import pytest

from test_attention_protocol import MBar, Sim, delay, wait

MUTATIONS = ("no_read_wait_first", "no_read_wait_next", "no_resid_wait")


def simulate_resid(seed, ntiles, nchunks, boxes, nwarps=2, mutate=None):
    """`nwarps` epilogue warps over `ntiles` tiles of `nchunks` 32-column chunks each (kMB * ochunks), `boxes` staging boxes per
    warp (kBoxes: 4 on 128-row tiles, 2 on 256-row ones)"""
    assert mutate is None or mutate in MUTATIONS
    sim = Sim(seed)
    glob = {}                                                          # (warp, tile, chunk) -> "resid" / "out" (in place)
    warps = [dict(boxes=[None] * boxes, bars=[MBar(1) for _ in range(boxes)], stores=[], loads=[], done=False)
             for _ in range(nwarps)]

    def request(W, w, t, j, b):
        W["loads"].append(dict(box=b, key=(w, t, j)))

    def read_wait(W):
        return lambda: all(s["read"] for s in W["stores"])           # cp.async.bulk.wait_group.read 0

    def tma_unit():
        """completes residual loads in any order and reads / completes each warp's stores in issue order"""
        while True:
            work = [("load", W) for W in warps if W["loads"]] + [("store", W) for W in warps if W["stores"]]
            if not work:
                if all(W["done"] for W in warps):
                    return
                yield None
                continue
            kind, W = sim.rng.choice(work)
            yield from delay(sim)
            if kind == "load":
                ld = W["loads"].pop(sim.rng.randrange(len(W["loads"])))
                assert all(s["read"] for s in W["stores"] if s["box"] == ld["box"]), \
                    "residual load overwrites a staging box before the store issued from it has read it"
                assert glob.get(ld["key"]) == "resid", "residual read after its output was stored over it"
                W["boxes"][ld["box"]] = ("resid",) + ld["key"]
                W["bars"][ld["box"]].arrive()                          # complete_tx
            else:
                st = W["stores"][0]
                if not st["read"]:
                    assert W["boxes"][st["box"]] == st["data"], "a store reads a box that no longer holds its output"
                    st["read"] = True
                else:
                    W["stores"].pop(0)
                    glob[st["data"][1:]] = "out"

    def epilogue(w):
        W = warps[w]
        slot, phase = 0, [0] * boxes
        for t in range(ntiles):
            for j in range(nchunks):
                glob[(w, t, j)] = "resid"
            yield from delay(sim, 2)                                   # the first k-block's products are issued
            if mutate != "no_read_wait_first":
                yield read_wait(W)
            for j in range(min(boxes, nchunks)):
                request(W, w, t, j, (slot + j) % boxes)
            yield from delay(sim)                                      # rest of the mainloop
            for j in range(nchunks):
                b = slot
                if mutate != "no_resid_wait":
                    yield wait(W["bars"][b], phase[b])
                phase[b] ^= 1
                assert W["boxes"][b] == ("resid", w, t, j), f"chunk {j} of tile {t} reads box {b} holding {W['boxes'][b]}"
                yield from delay(sim, 1)                               # ldmatrix, the adds
                if j >= 1 and j - 1 + boxes < nchunks:
                    if mutate != "no_read_wait_next":
                        yield read_wait(W)
                    request(W, w, t, j - 1 + boxes, (slot + boxes - 1) % boxes)
                data = ("out", w, t, j)
                W["boxes"][b] = data                                   # stmatrix, fence.proxy.async
                W["stores"].append(dict(box=b, data=data, read=False))
                slot = (slot + 1) % boxes
        yield lambda: not W["stores"] and not W["loads"]               # bulk_wait<0> before the CTA exits
        W["done"] = True

    sim.spawn(tma_unit())
    for w in range(nwarps):
        sim.spawn(epilogue(w))
    sim.run()


# (chunks per tile, boxes): BN 64 / 128 / 160 / 256 on 128-row tiles (4 boxes), BN 160 on 256-row tiles (2 boxes, 2 x 5 chunks)
SHAPES = [(2, 4), (4, 4), (5, 4), (8, 4), (10, 2), (1, 4), (1, 2)]


@pytest.mark.parametrize("nchunks,boxes", SHAPES)
@pytest.mark.parametrize("ntiles", [1, 2, 5])
def test_residual_box_protocol(ntiles, nchunks, boxes):
    for seed in range(20):
        simulate_resid(seed, ntiles, nchunks, boxes)


@pytest.mark.parametrize("mutate", MUTATIONS)
def test_model_catches_each_missing_residual_wait(mutate):
    caught = 0
    for seed in range(40):
        for nchunks, boxes in ((5, 4), (10, 2)):
            try:
                simulate_resid(seed, 4, nchunks, boxes, mutate=mutate)
            except AssertionError:
                caught += 1
    assert caught >= 8, f"only {caught}/80 interleavings expose the mutation {mutate}"
