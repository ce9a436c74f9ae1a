"""TEST INFRASTRUCTURE ONLY. numpy fp32 restatement of the text decoder's repetition logits processors (vdb_textdec_repetition;
the "Repetition" paragraph of lib/model_zoo/optimus.py's docstring): Hugging Face's RepetitionPenaltyLogitsProcessor and
NoRepeatNGramLogitsProcessor on the history h = tokens[r, 0 .. s], with ids outside [0, V) ignored and finished rows untouched.

process: the edit of one step's logits.  has_repeated_ngram: whether a token row holds some n-gram twice.
processed_pick / processed_beam_search: the sampler's and the beam search's oracles (text_filter_oracle, text_beam_oracle) run on
processed logits.
"""
import numpy as np
import torch

from oracle.text_beam_oracle import beam_search
from oracle.text_filter_oracle import filter_keep_mask, filtered_pick, scaled_logits


def banned_tokens(h, n):
    """The ids the no-repeat n-gram rule bans after history h (a list): h[j + n - 1] for every j <= s - n + 1 whose n - 1
    tokens equal the last n - 1 tokens of h (s = len(h) - 1).  n = 1 bans every token of h; none while len(h) < n."""
    s = len(h) - 1
    tail = h[s - n + 2:] if n > 1 else []
    return [h[j + n - 1] for j in range(0, s - n + 2) if h[j:j + n - 1] == tail]


def process(logits, tokens, s, done, penalty, n):
    """fp32 logits [R, V], int tokens [R, >= s + 1], step s, done [R] (nonzero: left as it is; None: no row finished), penalty
    (1: off), n (0: off) -> the edited copy, fp32 [R, V].  Each distinct id v of h = tokens[r, :s + 1] in [0, V) gets
    l < 0 ? l * p : l / p in fp32 (p rounded to fp32), then every banned id in [0, V) gets -inf."""
    out = np.array(logits, dtype=np.float32, copy=True)
    R, V = out.shape
    p = np.float32(penalty)
    for r in range(R):
        if done is not None and done[r]:
            continue
        h = [int(t) for t in tokens[r, :s + 1]]
        row = out[r]
        if p != np.float32(1.0):
            for v in dict.fromkeys(h):                       # distinct ids, each once
                if 0 <= v < V:
                    with np.errstate(over="ignore"):         # fp32 overflow to +-inf is part of the arithmetic
                        row[v] = row[v] * p if row[v] < 0 else row[v] / p
        if n > 0:
            for v in banned_tokens(h, n):
                if 0 <= v < V:
                    row[v] = -np.inf
    return out


def has_repeated_ngram(row, n):
    """True when some n consecutive tokens of row occur twice (overlapping occurrences count)."""
    row = [int(t) for t in row]
    grams = [tuple(row[i:i + n]) for i in range(len(row) - n + 1)]
    return len(set(grams)) != len(grams)


def processed_pick(raw, history, s, penalty, n, temperature, top_k, top_p, u):
    """The sampler's pick at step s from one row's raw fp32 logits [V] and its tokens (>= s + 1): processed, scaled by
    temperature, cut by top_k / top_p, then text_filter_oracle.filtered_pick with the uniforms u -> (picks, distances to a CDF
    step, scaled processed logits).  A -inf token weighs 0, as in the kernel: it is never the pick."""
    l = scaled_logits(process(np.asarray(raw)[None], np.asarray(history)[None], s, None, penalty, n)[0], temperature)
    keep = filter_keep_mask(l, top_k, top_p) & torch.isfinite(l)
    pick, near = filtered_pick(l, keep, u)
    return pick, near, l


def processed_beam_search(raw_logits_fn, n_latents, K, bos, eos, max_len, temperature, penalty, n, length_penalty=1.0,
                          on_step=None):
    """text_beam_oracle.beam_search over processed logits: raw_logits_fn(s, tokens [R, s + 1]) gives every row's raw fp32 logits
    of step s; each row is processed with its own history before the beam step (a finished beam's row is never read)."""
    fn = lambda s, hist: process(raw_logits_fn(s, hist), hist, s, None, penalty, n)
    return beam_search(fn, n_latents, K, bos, eos, max_len, temperature, length_penalty, on_step=on_step)
