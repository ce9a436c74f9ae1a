"""TEST INFRASTRUCTURE ONLY. fp64 CPU restatement of the text decoder's beam search (vdb_textdec_beam_step, optimus.py's module
docstring).  The reference names beam search (optimus_vae.decode(z, 'beam', K), reference optimus.py:196-213) but its GPT-2 has
no beam_search_decode, so there is nothing of the reference's to match: this implements the specification the kernels do.

beam_step: one step over given fp32 logits, on a BeamState of n latents x K beams (rows latent * K + beam).
beam_search: a whole decode over a logits callback, then the final ranking by S / n ** length_penalty.
"""
import math
from dataclasses import dataclass

import numpy as np


def log_softmax64(logits, temperature):
    """fp32 logits [R, V] -> fp64 log softmax(logits / temperature), the division, max, exp, sum and log all in fp64."""
    x = np.asarray(logits, dtype=np.float32).astype(np.float64) / float(np.float32(temperature))
    m = x.max(-1, keepdims=True)
    return x - (m + np.log(np.exp(x - m).sum(-1, keepdims=True)))


@dataclass
class BeamState:
    tokens: np.ndarray      # int [R, W], token 0 = <BOS>
    src: np.ndarray         # int [R, T], the KV cache's slot-to-row table
    scores: np.ndarray      # fp64 [R]
    done: np.ndarray        # bool [R]
    lengths: np.ndarray     # int [R]

    @staticmethod
    def start(n, K, bos, eos, width=33, slots=32, nsteps=28):
        """The state before step 0: <BOS> then eos padding, beam 0 of each latent at score 0 and the others at -inf."""
        R = n * K
        tokens = np.full((R, width), eos, dtype=np.int64)
        tokens[:, 0] = bos
        scores = np.full(R, -np.inf)
        scores[::K] = 0.0
        return BeamState(tokens, np.repeat(np.arange(R)[:, None], slots, 1), scores, np.zeros(R, bool),
                         np.full(R, nsteps + 1, dtype=np.int64))

    def copy(self):
        return BeamState(self.tokens.copy(), self.src.copy(), self.scores.copy(), self.done.copy(), self.lengths.copy())


def _key(c):
    """sort key of a candidate (score, parent, token): higher score, then lower parent, then lower token first"""
    return (-c[0], c[1], c[2])


def beam_step(st, logits, K, s, eos, max_len, temperature=1.0):
    """One step s on a copy of st -> (new state, trace [R, 3] of (parent beam, token or -1, score), margins).
    margins: per latent, the smallest relative score gap between consecutive candidates among the K + 1 best, over the pairs
    that are not exact ties (exact ties are settled by the tie rule; a gap this small is a near-tie fp64 rounding could flip)."""
    logp = log_softmax64(logits, temperature)
    R = st.scores.shape[0]
    new = st.copy()
    trace = np.zeros((R, 3))
    margins = []
    V = logp.shape[1]
    for n0 in range(0, R, K):
        cands = []
        for b in range(K):
            r = n0 + b
            if st.done[r]:
                cands.append((st.scores[r], b, -1))
                continue
            sc = st.scores[r] + logp[r]
            # the latent's K + 1 best can hold at most the row's K + 1 best under the same order: an exact pre-filter
            keep = np.lexsort((np.arange(V), -sc))[:K + 1]
            cands += [(sc[v], b, int(v)) for v in keep]
        cands.sort(key=_key)
        top = cands[:K + 1]
        gaps = [abs(a[0] - c[0]) / max(abs(a[0]), abs(c[0]), 1.0) for a, c in zip(top, top[1:])
                if a[0] != c[0] and math.isfinite(a[0]) and math.isfinite(c[0])]
        margins.append(min(gaps) if gaps else math.inf)
        for j, (sc, p, v) in enumerate(cands[:K]):
            place(new, st, n0 + j, n0 + p, v, sc, s, eos, max_len)
            trace[n0 + j] = (p, v, sc)
    return new, trace, margins


def place(new, st, r, pr, v, sc, s, eos, max_len):
    """new beam r of step s <- parent row pr of st extended by token v (-1: pr finished, carried as itself), score sc"""
    new.tokens[r, :s + 2] = st.tokens[pr, :s + 2]
    new.src[r, :s] = st.src[pr, :s]
    new.src[r, s] = pr
    new.scores[r], new.done[r], new.lengths[r] = sc, True, st.lengths[pr]
    if v >= 0:
        new.tokens[r, s + 1] = v
        if v == eos:
            new.lengths[r] = s + 2
        elif s + 1 >= max_len - 2:
            new.tokens[r, s + 2] = eos
            new.lengths[r] = s + 3
        else:
            new.done[r] = False


def scored_tokens(length, max_len):
    """tokens a finished hypothesis of this length was scored on: a chosen <eos> counts, the forced one (length max_len) not"""
    return min(length - 1, max_len - 2)


def rank_final(st, K, max_len, length_penalty=1.0):
    """-> per latent, [(ids, score, normalized score)] of its K beams, best normalized score first, ties to the lower beam."""
    out = []
    for n0 in range(0, st.scores.shape[0], K):
        beams = []
        for j in range(K):
            r = n0 + j
            L = int(st.lengths[r])
            beams.append((st.tokens[r, :L].copy(), st.scores[r], st.scores[r] / scored_tokens(L, max_len) ** length_penalty))
        out.append([beams[j] for j in sorted(range(K), key=lambda j: (-beams[j][2], j))])
    return out


def beam_search(logits_fn, n, K, bos, eos, max_len, temperature=1.0, length_penalty=1.0, on_step=None):
    """A whole beam-search decode: logits_fn(s, tokens [R, s+1]) -> fp32 logits [R, V] of every row's next token (rows
    latent * K + beam, the history as the state holds it).  Runs steps 0 .. max_len - 3, stopping once every beam is finished.
    on_step(s, logits, new state, trace, margins) sees each step.  -> (rank_final's list, final state)."""
    st = BeamState.start(n, K, bos, eos, width=max_len + 1, slots=max_len, nsteps=max_len - 2)
    for s in range(max_len - 2):
        logits = logits_fn(s, st.tokens[:, :s + 1])
        st2, trace, margins = beam_step(st, logits, K, s, eos, max_len, temperature)
        if on_step is not None:
            on_step(s, logits, st2, trace, margins)
        st = st2
        if st.done.all():
            break
    return rank_final(st, K, max_len, length_penalty), st
