"""Top-k / nucleus cuts of the text sampler, CPU side: the fp64 restatement (oracle/text_filter_oracle.py) against what the
reference's top_k_top_p_filtering kept (tests/golden/text_filter.npz), and the argument checks of vdb_textdec_sample_filtered
and optimus_vae_next.decode_ids, which must reject bad cuts before any launch."""
import math
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
NEAR = 1e-5


def test_restatement_reproduces_the_reference_kept_sets():
    """Same count, same tokens above the boundary, same number of ties kept at it.  A case may differ only when the reference's
    fp32 exclusive mass at its last kept or first removed token lies within 1e-5 of top_p (fp32 cumsum against fp64 sums)."""
    from oracle.make_text_filter_golden import TEMPERATURE, TOP_K, TOP_P, filter_rows
    from oracle.text_filter_oracle import filter_keep_mask, scaled_logits
    gold = dict(np.load(os.path.join(GOLD, "text_filter.npz")))
    assert tuple(gold["top_k"]) == TOP_K and tuple(gold["top_p"]) == TOP_P and tuple(gold["temperature"]) == TEMPERATURE
    rows = filter_rows()
    np.testing.assert_array_equal(rows.double().sum(-1).numpy(), gold["row_sum"])     # the rows are the ones the fixture saw
    exempt, cases = [], 0
    for r in range(rows.shape[0]):
        for t, temp in enumerate(TEMPERATURE):
            l = scaled_logits(rows[r], temp)
            for a, k in enumerate(TOP_K):
                for b, p in enumerate(TOP_P):
                    cases += 1
                    keep = filter_keep_mask(l, k, p)
                    v = torch.tensor(gold["boundary"][r, a, b, t])
                    got = (int(keep.sum()), int((keep & (l > v)).nonzero().sum()), int((keep & (l == v)).sum()), float(l[keep].min()))
                    want = (int(gold["kept"][r, a, b, t]), int(gold["above_index_sum"][r, a, b, t]), int(gold["ties_kept"][r, a, b, t]),
                            float(v))
                    if got != want:
                        p32 = float(np.float32(p))
                        near = min(abs(float(gold["excl_last"][r, a, b, t]) - p32), abs(float(gold["excl_next"][r, a, b, t]) - p32))
                        assert 0.0 < p < 1.0 and near < NEAR, (r, k, p, temp, got, want)
                        exempt.append((r, k, p, temp, got[0] - want[0]))
    print(f"[textfilter] restatement == reference on {cases - len(exempt)} of {cases} cases; {len(exempt)} exempt "
          f"(boundary within {NEAR} of top_p), at top_p {sorted(set(e[2] for e in exempt))}")
    assert sum(1 for e in exempt if e[2] != 0.999) <= 4, exempt


def test_top_k_ties_and_a_dominant_token_in_the_fixture():
    """The planted cases: ties at the 40th value keep 44 tokens, a tie at the max keeps 2 under top_k=1, and a token whose
    probability alone exceeds top_p is kept alone."""
    from oracle.make_text_filter_golden import TOP_K, TOP_P
    gold = dict(np.load(os.path.join(GOLD, "text_filter.npz")))
    k40, k1 = TOP_K.index(40), TOP_K.index(1)
    assert (gold["kept"][4, k40, TOP_P.index(0.0)] == 44).all() and (gold["ties_kept"][4, k40, TOP_P.index(0.0)] == 8).all()
    assert (gold["kept"][4, k1, TOP_P.index(0.0)] == 2).all()
    assert (gold["kept"][6, :, 1:] == 1).all()


def test_filtered_entry_point_checks_arguments_before_launch():
    """Every call here is refused before a launch (the fake addresses are never touched)."""
    from vdb200._lib import lib
    x, out, step = 0x10000, 0x30000, 0x40000

    def sample(R=4, V=50260, temp=1.0, top_k=40, top_p=0.9, seed=x, logits=x):
        return lib.vdb_textdec_sample_filtered(logits, R, V, V, temp, top_k, top_p, seed, None, 32, None, 0, out, 33, out, out, step,
                                               50259, 30, None, None)
    for kw, msg in ((dict(top_k=-1), b"top_k"), (dict(top_p=math.nan), b"top_p"), (dict(top_p=-0.1), b"top_p"),
                    (dict(top_p=1.5), b"top_p"), (dict(top_p=math.inf), b"top_p"), (dict(R=17), b"R <= 16"),
                    (dict(temp=0.0), b"temperature"), (dict(seed=None), b"seed"), (dict(seed=x + 4), b"8-byte aligned"),
                    (dict(logits=None), b"null"), (dict(V=60000), b"53248")):
        assert sample(**kw) == 1 and msg in lib.vdb_last_error(), (kw, lib.vdb_last_error())


def test_decode_ids_rejects_bad_cuts_before_launch():
    from lib.model_zoo.optimus import optimus_vae_next
    m = optimus_vae_next(decoder=dict(config=dict(n_layer=2)))
    z = torch.zeros(2, 768)                                    # on the CPU: a check after the first launch would fail otherwise
    for kw in (dict(top_k=-1), dict(top_k=1.5), dict(top_k=True), dict(top_k="40"), dict(top_p=math.nan), dict(top_p=math.inf),
               dict(top_p=-0.1), dict(top_p=1.01), dict(top_p="0.9"), dict(top_p=None)):
        with pytest.raises(ValueError, match="top_k" if "top_k" in kw else "top_p"):
            m.decode_ids(z, **kw)
        with pytest.raises(ValueError):
            m.decode(z, **kw)
