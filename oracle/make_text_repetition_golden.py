"""TEST INFRASTRUCTURE ONLY. Writes tests/golden/text_repetition.npz from Hugging Face's own RepetitionPenaltyLogitsProcessor and
NoRepeatNGramLogitsProcessor (transformers.generation.logits_process), run on the CPU over seeded fp32 logits and token histories.

    python oracle/make_text_repetition_golden.py

Per case (penalty, n, s) the fixture holds the logits after the penalty processor and then (n > 0) the n-gram processor, given
the histories tokens[:, :s + 1].  The logits hold positive, negative, +0 / -0, subnormal and large values (+-3e38 times 3 overflows
to -inf); the histories hold repeated ids and overlapping n-gram occurrences, and s runs below, at and above n - 1.  HF refuses ids
outside [0, V), so the fixture has none; ignoring them is this project's own rule, tested against the numpy oracle alone.  The
generator asserts that oracle/text_repetition_oracle.process reproduces every case bitwise.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
V, W = 48, 33                                   # vocabulary, token row width (the decoder's 33 token slots)
PENALTY = (1.0, 0.5, 1.2, 3.0)
NGRAM = (0, 1, 2, 3, 4, 30)
STEP = (0, 1, 2, 3, 5, 17, 28, 29, 31)
SPECIAL = (0.0, -0.0, 3e38, -3e38, 1e-40, -1e-40, 1e30, -1e30, 1.0, -1.0)    # the logits of ids 0 .. 9 in every row
ROW_NAMES = ("uniform ids", "ids below 4", "one id repeated", "period 2", "period 3 with breaks", "ids below 2")


def inputs():
    """(fp32 logits [6, V], int64 tokens [6, W]), deterministic from a numpy generator (see ROW_NAMES)."""
    rng = np.random.default_rng(2024)
    logits = (rng.standard_normal((len(ROW_NAMES), V)) * 3).astype(np.float32)
    logits[:, :len(SPECIAL)] = np.array(SPECIAL, dtype=np.float32)
    tok = np.stack([rng.integers(0, V, W), rng.integers(0, 4, W), np.full(W, 5), np.resize([7, 9], W), np.resize([1, 2, 3], W),
                    rng.integers(0, 2, W)]).astype(np.int64)
    tok[4, [8, 19]] = [11, 4]                   # breaks in the period-3 row
    return logits, tok


def hf_process(logits, tokens, s, penalty, n):
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    ids = torch.from_numpy(tokens[:, :s + 1]).long()
    x = RepetitionPenaltyLogitsProcessor(float(penalty))(ids, torch.from_numpy(logits.copy()))
    if n > 0:
        x = NoRepeatNGramLogitsProcessor(n)(ids, x)
    return x.numpy()


def main():
    sys.path.insert(0, ROOT)
    from oracle.text_repetition_oracle import process
    logits, tokens = inputs()
    cases, out = [], []
    for p in PENALTY:
        for n in NGRAM:
            for s in STEP:
                want = hf_process(logits, tokens, s, p, n)
                got = process(logits, tokens, s, None, p, n)
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (p, n, s)
                cases.append((p, n, s))
                out.append(want)
    c = np.array(cases)
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "text_repetition.npz")
    np.savez_compressed(path, logits=logits, tokens=tokens, penalty=c[:, 0].astype(np.float64), ngram=c[:, 1].astype(np.int64),
                        step=c[:, 2].astype(np.int64), out=np.stack(out))
    print(f"oracle == HF bitwise on {len(cases)} cases; wrote {path}, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
