"""Optimus text VAE on vdb200 kernels — reference lib/model_zoo/optimus.py:662-688, 729-763 (optimus_vae_next.encode / decode)
over BertForLatentConnector_XX (optimus_models/optimus_bert.py:1348-1437) and GPT2ForLatentConnector_XX
(optimus_models/optimus_gpt2.py:813-994, 1025-1082), configs/model/optimus.yaml.

encode(texts) turns sentences into text latents z_mu [n, 768] (`net.vae_encode(texts, which='text')`, `net.ctx_encode(texts,
which='vae_text')`).  The BERT encoder is built only when the module is given an `encoder` config.  Its 12 post-LN layers (LayerNorm
eps 1e-12, erf GELU) run on the same kernels as the CLIP towers: ops.gemm, ops.layernorm and the flash attention, here with one key
count per sentence (vdb_attention_varlen_bf16) in place of the reference's -10000 padding mask.  The pooler (tanh of a dense layer on
the [CLS] row) and the z_mu half of `linear` run as two weight-streaming GEMVs on the [CLS] rows, 16 sentences at a time.
The WordPiece tokenizer is written from the behaviour of the reference's: the sentence is lowercased first (optimus.py:731, although
the vocabulary is cased and do_lower_case is false, so accents are kept), BERT's basic tokenizer drops control characters, spaces out
CJK characters, splits on whitespace and splits off every punctuation character, then greedy longest-match WordPiece with `##`
continuations gives the pieces ([UNK] for a word over 100 characters or with no match); they are cut to max_length and framed by
[CLS] ... [SEP].  Differences from the reference's encode, all deliberate:
  - bf16 weights and activations with fp32 accumulation and fp32 LayerNorm statistics (the pooler and head read fp32 rows);
  - the padding mask is a hard mask (exactly what -10000 gives in fp32);
  - a bare `str` raises TypeError: the reference would iterate over its characters and encode each one as a sentence;
  - a sentence of whitespace only encodes as [CLS] [SEP], like the empty one.  The reference's tokenizer turns it into one of its
    special tokens, picked by the iteration order of a Python set of strings, which changes with the process's hash seed.

decode(z) turns text latents [n, 768] into strings, the last call of app.py's i2t / t2t flows (`net.vae_decode(x, which='text')`).
GPT-2 (LayerNorm eps 1e-5, tanh GELU, Conv1D weights [in, out], attention scale 1/8) runs one token at a time for all n rows as one
batch, with the latent injected twice: `transformer.linear` maps z to one slice per layer that is both key and value of position 0,
and `transformer.linear_emb` is added to every token embedding (positions start at 1).  The LM head is tied to `wte`.

Differences from the reference, all deliberate:
  - the reference decodes each latent alone and re-runs the whole prefix at every token; here every row advances one token per step
    over a KV cache, and a row that has finished keeps its tokens frozen while the others continue;
  - the draw of token s+1 of row r is an inverse-CDF pick of softmax(logits / temperature) with a Philox4x32-10 uniform at counter
    (r, s), keyed by one 64-bit seed taken from torch's default CPU generator per decode() call: `torch.manual_seed` fixes the text,
    but the tokens are not those torch.multinomial would draw;
  - by default (top_k=0, top_p=0.0) the full softmax is sampled.  The reference's top_k_top_p_filtering(top_p=1.0) removes nothing
    in exact arithmetic but, in fp32, can cut a tail whose sorted cumulative sum rounds above 1.0 (probability mass of order 1e-6);
    top_p=1.0 here samples the full softmax too;
  - decode(z, top_k=..., top_p=...) applies the reference's top-k and nucleus cuts (optimus.py:690-719) in the sampling kernel,
    inside the captured step graph; top_k=1 is greedy decoding.  The probabilities the nucleus cut sums are fp64-exact fixed-point
    integers rather than an fp32 cumsum, and tied tokens at the nucleus boundary are taken in vocabulary order (the reference's
    unstable sort leaves their order open); see vdb_textdec_sample_filtered;
  - the reference's 29th forward pass, whose draw is always overwritten with <EOS>, is skipped;
  - weights are bf16 (packed at load); the residual stream, attention, logits and the sampler's sums are fp32 / fp64.

Beam search: decode(z, num_beams=K) (and decode_ids, decode_beams) stands in for the reference's optimus_vae.decode(z, 'beam', K)
(optimus.py:196-213), whose beam_search_decode does not exist in its GPT-2, so the definition here is the specification
(vdb_textdec_beam_step; oracle/text_beam_oracle.py implements the same):
  - each latent gets K beams, rows latent * K + beam of one batch; each starts as <BOS> with the latent's memory and embedding
    offset; at step 0 only beam 0 is live (the others start at score -inf), so the first step does not make K copies of one
    hypothesis;
  - a hypothesis' score is the sum over its chosen tokens of log softmax(logits / temperature), computed in fp64 from the fp32
    logits (the division, max, exp, sum and log);
  - candidates at step s: every live beam b crossed with every token v, scored S_b + logp_b(v), and every finished beam as itself
    with its score unchanged; the K best become the new beams, ties to the lower parent beam, then the lower token id;
  - a candidate whose token is <EOS> is finished; a live beam whose token s+1 lands on max_len - 2 without <EOS> gets <EOS>
    appended unscored (the sampler's rule above) and is finished; a latent is done when all K beams are (live scores only fall);
  - final ranking by S / n ** length_penalty, n the scored tokens (a chosen <EOS> counts, a forced one does not; length_penalty 0
    ranks by the raw sum), ties to the lower beam index.  K = 1 picks the argmax, the lowest token id among equal maxima: the
    tokens of greedy decoding (top_k=1), which differs only at an exact tie for the maximum, where it draws among the tied tokens.
The KV cache is not moved when beams are reordered: each physical (row, slot) is written once, and the indexed attention reads
slot j of beam r from row src[r, j], a table the beam step permutes with the token rows.  A step streams the weights once for all
n * K rows (the GEMV is one 16-row tile), so n * K <= 16 rows run together; more latents are split into groups of 16 // K,
decoded one after the other, each group re-streaming the weights.
"""
import json
import math
import numbers
import os
import unicodedata

import torch
import torch.nn as nn

from lib.model_zoo.common.get_model import register
from .diffusion_utils import PackedModule, bf16, f32, require_cuda

symbol = 'optimus'

PAD_ID, BOS_ID, EOS_ID = 50257, 50258, 50259     # added in the order <PAD>, <BOS>, <EOS> after GPT-2's 50257 tokens (optimus.py:30-34)
MAX_LENGTH = 30                                   # optimus.py:756 (max_length=30)
CACHE_SLOTS = 32                                  # token slots of the KV cache (a sequence holds at most MAX_LENGTH - 1 inputs)
# Steps per captured graph between two host reads of the all-done flags.  A step of the full-size decoder streams ~247 MB of weights
# (>= 74 us at 3.35 TB/s); a host read of the flags costs one device sync plus a graph launch, a few tens of us.  A chunk of 4
# caps the steps that run after every row has finished at 3 and the syncs of a full-length decode (28 steps) at 7.
STEPS_PER_CHECK = 4
DEFAULT_VOCAB_FILE = 'lib/model_zoo/optimus_models/vocab/gpt2-vocab.json'   # relative to the reference's tree, where app.py runs
DEFAULT_BERT_VOCAB_FILE = 'lib/model_zoo/optimus_models/vocab/bert-base-cased-vocab.txt'
ENC_MAX_POSITIONS = 512                           # BERT's position table; [CLS] and [SEP] take two of them
ENC_HEAD_ROWS = 16                                # [CLS] rows per pooler / z_mu GEMV launch (vdb_textdec_gemv's row limit)


def _ops():
    from vdb200 import ops
    return ops


def _check_cuts(top_k, top_p):
    """-> (int top_k, float top_p) of the sampler's top-k / nucleus cuts, or ValueError."""
    if isinstance(top_k, bool) or not isinstance(top_k, numbers.Integral) or top_k < 0:
        raise ValueError(f"optimus_vae_next: top_k must be an int >= 0 (0: no top-k cut), got {top_k!r}")
    if isinstance(top_p, bool) or not isinstance(top_p, numbers.Real) or not math.isfinite(top_p) or not 0.0 <= top_p <= 1.0:
        raise ValueError(f"optimus_vae_next: top_p must be a finite float in [0, 1] (0 or 1: no nucleus cut), got {top_p!r}")
    return int(top_k), float(top_p)


MAX_BEAMS = 16                                    # the rows of one token step (vdb_textdec_beam_step's K limit)


def _check_beams(num_beams, length_penalty, top_k, top_p):
    """-> (int num_beams, float length_penalty), or ValueError; beam search takes no top-k / nucleus cut."""
    if isinstance(num_beams, bool) or not isinstance(num_beams, numbers.Integral) or not 0 <= num_beams <= MAX_BEAMS:
        raise ValueError(f"optimus_vae_next: num_beams must be an int in [0, {MAX_BEAMS}] (0: sampling), got {num_beams!r}")
    if isinstance(length_penalty, bool) or not isinstance(length_penalty, numbers.Real) or not math.isfinite(length_penalty):
        raise ValueError(f"optimus_vae_next: length_penalty must be a finite float, got {length_penalty!r}")
    if num_beams and (top_k != 0 or top_p != 0.0):
        raise ValueError("optimus_vae_next: beam search (num_beams >= 1) takes no top_k / top_p cut")
    return int(num_beams), float(length_penalty)


class VocabularyMissingError(RuntimeError):
    pass


# ---------------------------------------------------------------------------------------------------------- detokenizer
def _byte_to_char():
    """GPT-2's reversible byte <-> printable-character table: printable Latin-1 bytes stand for themselves, every other byte b is
    the character 256 + (its rank among the non-printable bytes)."""
    keep = list(range(ord('!'), ord('~') + 1)) + list(range(0xA1, 0xAC + 1)) + list(range(0xAE, 0xFF + 1))
    table, extra = {}, 0
    for b in range(256):
        if b in keep:
            table[b] = chr(b)
        else:
            table[b] = chr(256 + extra)
            extra += 1
    return table


_CLEANUP = ((' .', '.'), (' ?', '?'), (' !', '!'), (' ,', ','), (" ' ", "'"), (" n't", "n't"), (" 'm", "'m"), (" do not", " don't"),
            (" 's", "'s"), (" 've", "'ve"), (" 're", "'re"))


class GPT2Detokenizer(object):
    """ids -> text as the reference's GPT2Tokenizer.decode(ids, clean_up_tokenization_spaces=True) with <PAD> / <BOS> / <EOS> added:
    byte-level tokens are joined and decoded as UTF-8 with errors='replace', each added token contributes " " + its text, then the
    tokenizer's clean-up replacements run.  The vocabulary (gpt2-vocab.json) is read on first use."""
    ADDED = {PAD_ID: '<PAD>', BOS_ID: '<BOS>', EOS_ID: '<EOS>'}

    def __init__(self, vocab_file=DEFAULT_VOCAB_FILE):
        self.vocab_file = vocab_file
        self._id_to_bytes = None

    def _load(self):
        if self._id_to_bytes is None:
            if not os.path.isfile(self.vocab_file):
                raise VocabularyMissingError(
                    f"GPT-2 vocabulary '{self.vocab_file}' not found (cwd {os.getcwd()}): the text decoder needs the Optimus "
                    "gpt2-vocab.json to turn token ids into text; set the text VAE's vocab_file, or call decode_ids() for the ids")
            with open(self.vocab_file, encoding='utf-8') as fh:
                enc = json.load(fh)
            char_to_byte = {c: b for b, c in _byte_to_char().items()}
            self._id_to_bytes = {i: bytes(char_to_byte[c] for c in tok) for tok, i in enc.items()}
        return self._id_to_bytes

    def decode(self, ids):
        table = self._load()
        parts, run = [], bytearray()
        for i in ids:
            i = int(i)
            if i in self.ADDED:
                if run:
                    parts.append(run.decode('utf-8', errors='replace'))
                    run = bytearray()
                parts.append(' ' + self.ADDED[i])
            else:
                run += table[i]
        if run:
            parts.append(run.decode('utf-8', errors='replace'))
        text = ''.join(parts)
        for a, b in _CLEANUP:
            text = text.replace(a, b)
        return text

    def sentence(self, ids):
        """optimus.py:759-762: decode, drop the first and last words (<BOS>, <EOS>), join with single spaces."""
        return ' '.join(self.decode(ids).split()[1:-1])


# ---------------------------------------------------------------------------------------------------------- WordPiece tokenizer
def _bert_whitespace(ch):
    return ch in ' \t\n\r' or unicodedata.category(ch) == 'Zs'


def _bert_control(ch):
    return ch not in '\t\n\r' and unicodedata.category(ch).startswith('C')


def _bert_punctuation(ch):
    cp = ord(ch)   # every non-alphanumeric ASCII symbol counts, as well as Unicode's P* categories
    return 33 <= cp <= 47 or 58 <= cp <= 64 or 91 <= cp <= 96 or 123 <= cp <= 126 or unicodedata.category(ch).startswith('P')


_CJK_RANGES = ((0x4E00, 0x9FFF), (0x3400, 0x4DBF), (0x20000, 0x2A6DF), (0x2A700, 0x2B73F), (0x2B740, 0x2B81F), (0x2B820, 0x2CEAF),
               (0xF900, 0xFAFF), (0x2F800, 0x2FA1F))    # the CJK Unified Ideographs blocks BERT isolates (not kana / hangul)


def _bert_cjk(ch):
    cp = ord(ch)
    return any(lo <= cp <= hi for lo, hi in _CJK_RANGES)


class BertWordPieceTokenizer(object):
    """sentence -> BERT ids as optimus_vae_next.encode tokenizes (optimus.py:731-737): lowercase, basic tokenization, greedy
    longest-match WordPiece, [CLS] ... [SEP].  The vocabulary (one piece per line, id = line number) is read on first use."""
    CLS, SEP, UNK = '[CLS]', '[SEP]', '[UNK]'
    MAX_WORD_CHARS = 100

    def __init__(self, vocab_file=DEFAULT_BERT_VOCAB_FILE):
        self.vocab_file = vocab_file
        self._vocab = None

    def _load(self):
        if self._vocab is None:
            if not os.path.isfile(self.vocab_file):
                raise VocabularyMissingError(
                    f"BERT vocabulary '{self.vocab_file}' not found (cwd {os.getcwd()}): the text encoder needs the Optimus "
                    "bert-base-cased-vocab.txt to turn text into token ids; set the text VAE's tokenizer_encoder vocab_file, or "
                    "call encode_ids() with ids")
            vocab = {}
            with open(self.vocab_file, encoding='utf-8') as fh:
                for i, line in enumerate(fh):
                    vocab[line.rstrip('\n')] = i
            self._vocab = vocab
        return self._vocab

    @staticmethod
    def basic_tokens(text):
        """BERT's basic tokenizer without case folding: drop NUL / U+FFFD / control characters, whitespace -> ' ', spaces around
        CJK ideographs, split on whitespace, then every punctuation character becomes a token of its own."""
        chars = []
        for ch in text:
            if ch in '\x00\ufffd' or _bert_control(ch):
                continue
            if _bert_whitespace(ch):
                chars.append(' ')
            elif _bert_cjk(ch):
                chars += [' ', ch, ' ']
            else:
                chars.append(ch)
        out = []
        for word in ''.join(chars).split():
            run = ''
            for ch in word:
                if _bert_punctuation(ch):
                    if run:
                        out.append(run)
                    out.append(ch)
                    run = ''
                else:
                    run += ch
            if run:
                out.append(run)
        return out

    def wordpieces(self, word):
        vocab = self._load()
        if len(word) > self.MAX_WORD_CHARS:
            return [self.UNK]
        pieces, start = [], 0
        while start < len(word):
            end = len(word)
            while end > start:
                piece = word[start:end] if start == 0 else '##' + word[start:end]
                if piece in vocab:
                    break
                end -= 1
            if end == start:                 # no piece of the vocabulary starts here: the whole word is unknown
                return [self.UNK]
            pieces.append(piece)
            start = end
        return pieces

    def tokenize(self, sentence):
        return [p for w in self.basic_tokens(sentence.lower()) for p in self.wordpieces(w)]

    def encode(self, sentence, max_length=77):
        """-> [CLS] id, the ids of the first max_length pieces, [SEP] id."""
        vocab = self._load()
        unk = vocab.get(self.UNK)
        ids = [vocab.get(p, unk) for p in self.tokenize(sentence)[:max_length]]
        return [vocab[self.CLS]] + ids + [vocab[self.SEP]]


# ---------------------------------------------------------------------------------------------------------- modules (key layout)
class _Conv1D(nn.Module):
    def __init__(self, nf, nx):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(nx, nf).normal_(std=0.02))   # [in, out]
        self.bias = nn.Parameter(torch.zeros(nf))


class _Attention(nn.Module):
    def __init__(self, nx, n_ctx):
        super().__init__()
        self.register_buffer("bias", torch.tril(torch.ones(n_ctx, n_ctx)).view(1, 1, n_ctx, n_ctx))   # kept so checkpoints load
        self.c_attn = _Conv1D(3 * nx, nx)
        self.c_proj = _Conv1D(nx, nx)


class _MLP(nn.Module):
    def __init__(self, n_state, nx):
        super().__init__()
        self.c_fc = _Conv1D(n_state, nx)
        self.c_proj = _Conv1D(nx, n_state)


class _Block(nn.Module):
    def __init__(self, n_ctx, nx, eps):
        super().__init__()
        self.ln_1 = nn.LayerNorm(nx, eps=eps)
        self.attn = _Attention(nx, n_ctx)
        self.ln_2 = nn.LayerNorm(nx, eps=eps)
        self.mlp = _MLP(4 * nx, nx)


class _GPT2Model(nn.Module):
    def __init__(self, vocab_size, n_positions, n_ctx, n_embd, n_layer, eps, latent_size):
        super().__init__()
        self.wte = nn.Embedding(vocab_size, n_embd)
        self.wpe = nn.Embedding(n_positions, n_embd)
        self.h = nn.ModuleList([_Block(n_ctx, n_embd, eps) for _ in range(n_layer)])
        self.ln_f = nn.LayerNorm(n_embd, eps=eps)
        self.linear = nn.Linear(latent_size, n_embd * n_layer, bias=False)
        self.linear_emb = nn.Linear(latent_size, n_embd, bias=False)
        for m in self.modules():      # GPT2PreTrainedModel._init_weights (optimus_gpt2.py:845-857)
            if isinstance(m, (nn.Linear, nn.Embedding)):
                m.weight.data.normal_(mean=0.0, std=0.02)


class GPT2LatentDecoder(nn.Module):
    """GPT2ForLatentConnector_XX with latent_as_gpt_emb = latent_as_gpt_memory = True: `transformer.*` and the tied `lm_head`."""

    def __init__(self, config, latent_size=768):
        super().__init__()
        c = dict(config)
        self.n_layer, self.n_embd, self.n_head = int(c['n_layer']), int(c['n_embd']), int(c['n_head'])
        self.vocab_size, self.eps = int(c['vocab_size']), float(c.get('layer_norm_epsilon', 1e-5))
        if self.n_embd != 64 * self.n_head:
            raise NotImplementedError("the decode attention kernel needs d_head == 64")
        self.transformer = _GPT2Model(self.vocab_size, int(c['n_positions']), int(c['n_ctx']), self.n_embd, self.n_layer, self.eps,
                                      int(c.get('latent_size', latent_size)))
        self.lm_head = nn.Linear(self.n_embd, self.vocab_size, bias=False)
        self.lm_head.weight = self.transformer.wte.weight                # tie_weights (optimus_gpt2.py:1063-1068)


OPTIMUS_GPT2_CONFIG = dict(      # configs/model/optimus.yaml: optimus_gpt2_decoder (inference-relevant fields)
    vocab_size=50260, n_positions=1024, n_ctx=1024, n_embd=768, n_layer=12, n_head=12, layer_norm_epsilon=1e-5, latent_size=768)

OPTIMUS_BERT_CONFIG = dict(      # configs/model/optimus.yaml: optimus_bert_encoder (inference-relevant fields)
    vocab_size=28996, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
    max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, hidden_act='gelu')


class _Dense(nn.Module):
    """nn.Linear's parameters with BERT's init (normal 0.02, zero bias)"""

    def __init__(self, nin, nout, bias=True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(nout, nin).normal_(std=0.02))
        self.bias = nn.Parameter(torch.zeros(nout)) if bias else None


class _BertEmbeddings(nn.Module):
    def __init__(self, c):
        super().__init__()
        D = c['hidden_size']
        self.word_embeddings = nn.Embedding(c['vocab_size'], D)
        self.position_embeddings = nn.Embedding(c['max_position_embeddings'], D)
        self.token_type_embeddings = nn.Embedding(c['type_vocab_size'], D)
        self.LayerNorm = nn.LayerNorm(D, eps=c['layer_norm_eps'])
        for e in (self.word_embeddings, self.position_embeddings, self.token_type_embeddings):
            e.weight.data.normal_(std=0.02)


class _BertSelfAttention(nn.Module):
    def __init__(self, D):
        super().__init__()
        self.query, self.key, self.value = _Dense(D, D), _Dense(D, D), _Dense(D, D)


class _BertAddNorm(nn.Module):   # BertSelfOutput / BertOutput: LayerNorm(dense(x) + residual)
    def __init__(self, nin, D, eps):
        super().__init__()
        self.dense = _Dense(nin, D)
        self.LayerNorm = nn.LayerNorm(D, eps=eps)


class _BertAttention(nn.Module):
    def __init__(self, D, eps):
        super().__init__()
        self.self = _BertSelfAttention(D)
        self.output = _BertAddNorm(D, D, eps)


class _BertIntermediate(nn.Module):
    def __init__(self, D, F):
        super().__init__()
        self.dense = _Dense(D, F)


class _BertLayer(nn.Module):
    def __init__(self, c):
        super().__init__()
        D, F, eps = c['hidden_size'], c['intermediate_size'], c['layer_norm_eps']
        self.attention = _BertAttention(D, eps)
        self.intermediate = _BertIntermediate(D, F)
        self.output = _BertAddNorm(F, D, eps)


class _BertLayers(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.layer = nn.ModuleList([_BertLayer(c) for _ in range(c['num_hidden_layers'])])


class _BertPooler(nn.Module):
    def __init__(self, D):
        super().__init__()
        self.dense = _Dense(D, D)


class BertLatentEncoder(nn.Module):
    """BertForLatentConnector_XX's parameters (`embeddings.*`, `encoder.layer.i.*`, `pooler.dense`, `linear` [2 * latent, 768])."""

    def __init__(self, config, latent_size=768):
        super().__init__()
        c = dict(config)
        self.hidden, self.n_head = int(c['hidden_size']), int(c['num_attention_heads'])
        self.eps = float(c['layer_norm_eps'])
        if self.hidden != 64 * self.n_head:
            raise NotImplementedError("the encoder's varlen attention kernel needs d_head == 64")
        if c.get('hidden_act', 'gelu') != 'gelu':
            raise NotImplementedError(f"BERT hidden_act '{c['hidden_act']}': only the erf GELU is built")
        self.embeddings = _BertEmbeddings(c)
        self.encoder = _BertLayers(c)
        self.pooler = _BertPooler(self.hidden)
        self.linear = _Dense(self.hidden, 2 * latent_size, bias=False)


class _State(object):
    """Device buffers of one batch size: fixed addresses, so captured step graphs can be replayed on later decode() calls."""

    def __init__(self, dec, R, device):
        D, L, V = dec.n_embd, dec.n_layer, dec.vocab_size
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.R = R
        self.h, self.emb, self.a = z(R, D), z(R, D), z(R, D)
        self.qkv, self.m, self.mem = z(R, 3 * D), z(R, 4 * D), z(R, L * D)
        self.logits = z(R, V)
        self.kc = z(L, R, dec.n_head, CACHE_SLOTS, 64)
        self.vc = z(L, R, dec.n_head, CACHE_SLOTS, 64)
        self.tokens = z(R, CACHE_SLOTS + 1, dt=torch.int32)
        self.forced = z(R, CACHE_SLOTS + 1, dt=torch.int32)
        self.uniforms = z(R, CACHE_SLOTS, dt=torch.float64)
        self.done, self.lengths = z(R, dt=torch.int32), z(R, dt=torch.int32)
        self.step, self.seed = z(1, dt=torch.int32), z(1, dt=torch.int64)
        self.record = z(CACHE_SLOTS, R, V)
        # beam search: slot-to-row table of the KV cache, fp64 scores, the per-row candidates, the per-step (parent, token, score)
        self.src = z(R, CACHE_SLOTS, dt=torch.int32)
        self.scores = z(R, dt=torch.float64)
        self.cand_tok, self.cand_logp = z(R * MAX_BEAMS, dt=torch.int32), z(R * MAX_BEAMS, dt=torch.float64)
        self.trace = z(CACHE_SLOTS, R, 3, dt=torch.float64)
        self.graphs = {}


@register('optimus_vae_next')
class optimus_vae_next(PackedModule):
    """Same state-dict layout as the reference's optimus_vae_next: the decoder (`decoder.transformer.*`, `decoder.lm_head.weight`
    tied to `wte`, the persistent `h.i.attn.bias` masks) and, when an `encoder` config is given, the BERT encoder (`encoder.*`).
    Without one, a checkpoint's `encoder.*` keys are absorbed by strict=False and encode() raises NotImplementedError."""

    def __init__(self, decoder=None, tokenizer_decoder=None, encoder=None, tokenizer_encoder=None, args=None, vocab_file=None):
        super().__init__()
        dcfg = dict(decoder.get('args', decoder)) if decoder is not None else {}
        config = dict(OPTIMUS_GPT2_CONFIG)
        config.update(dict(dcfg.get('config', {})))
        self.decoder = GPT2LatentDecoder(config, latent_size=dcfg.get('latent_size', 768))
        if vocab_file is None and tokenizer_decoder is not None:
            vocab_file = dict(tokenizer_decoder.get('args', tokenizer_decoder)).get('vocab_file')
        self.tokenizer_decoder = GPT2Detokenizer(vocab_file or DEFAULT_VOCAB_FILE)
        self.nz = int(config['latent_size'])
        self.eos_token_id, self.pad_token_id = EOS_ID, PAD_ID
        self.tokenizer_encoder = None
        if encoder is not None:
            ecfg = dict(encoder.get('args', encoder))
            bert = dict(OPTIMUS_BERT_CONFIG)
            bert.update(dict(ecfg.get('config', {})))
            self.encoder = BertLatentEncoder(bert, latent_size=ecfg.get('latent_size', self.nz))
            bert_vocab = None
            if tokenizer_encoder is not None:
                bert_vocab = dict(tokenizer_encoder.get('args', tokenizer_encoder)).get('vocab_file')
            self.tokenizer_encoder = BertWordPieceTokenizer(bert_vocab or DEFAULT_BERT_VOCAB_FILE)

    def get_device(self):
        return self.decoder.transformer.wte.weight.device

    # ------------------------------------------------------------------ encoder
    def _pack_encoder(self):
        e = self.encoder
        D = e.hidden
        emb = e.embeddings
        layers = []
        for lyr in e.encoder.layer:
            a, ao, io, oo = lyr.attention.self, lyr.attention.output, lyr.intermediate, lyr.output
            wo = ao.dense.weight.detach().float()
            layers.append(dict(
                wqk=bf16(torch.cat([a.query.weight.detach(), a.key.weight.detach()], 0)),
                bqk=f32(torch.cat([a.query.bias.detach(), a.key.bias.detach()], 0)),
                wv=bf16(a.value.weight),
                # the rows of P sum to 1 over the visible keys, so P (V + 1 b_v^T) = P V + b_v: the V bias moves through dense
                wo=bf16(wo), bo=(ao.dense.bias.detach().float() + wo @ a.value.bias.detach().float()).contiguous(),
                ln1=(f32(ao.LayerNorm.weight), f32(ao.LayerNorm.bias)),
                w1=bf16(io.dense.weight), b1=f32(io.dense.bias),
                w2=bf16(oo.dense.weight), b2=f32(oo.dense.bias),
                ln2=(f32(oo.LayerNorm.weight), f32(oo.LayerNorm.bias))))
        # token type ids are always 0 here: token_type_embeddings[0] rides in the position table
        pos = (emb.position_embeddings.weight.detach().float() + emb.token_type_embeddings.weight.detach().float()[0]).contiguous()
        return dict(layers=layers, word=f32(emb.word_embeddings.weight), pos=pos,
                    ln_emb=(f32(emb.LayerNorm.weight), f32(emb.LayerNorm.bias)),
                    w_pool=bf16(e.pooler.dense.weight), b_pool=f32(e.pooler.dense.bias),
                    w_mu=bf16(e.linear.weight[:e.linear.weight.shape[0] // 2]), heads=e.n_head, D=D, eps=e.eps)

    def _require_encoder(self):
        if getattr(self, 'encoder', None) is None:
            raise NotImplementedError("optimus_vae_next.encode needs the Optimus BERT encoder: build the text VAE with an `encoder` "
                                      "config (configs/model/optimus.yaml optimus_bert_encoder; VDB_TEXT_FLOWS=1 does)")

    @torch.no_grad()
    def encode_ids(self, ids, lengths):
        """BertForLatentConnector_XX.forward + linear(.).chunk(2)[0] on token rows: ids int64 [n, L] ([CLS] first, zero padded),
        lengths [n] = the ids of each row that are not padding.  -> z_mu fp32 [n, latent] on the module's device."""
        self._require_encoder()
        ops = _ops()
        dev = self.encoder.linear.weight.device
        ids = torch.as_tensor(ids).long()
        V = self.encoder.embeddings.word_embeddings.num_embeddings
        if ids.dim() != 2 or ids.numel() == 0 or int(ids.min()) < 0 or int(ids.max()) >= V:
            raise ValueError(f"optimus_vae_next.encode: need token ids [n, L] in [0, {V})")
        ids = ids.to(dev).contiguous()
        require_cuda(ids, "optimus_vae_next.encode")
        n, L = ids.shape
        lengths = [int(v) for v in lengths]
        if len(lengths) != n or not all(1 <= v <= L for v in lengths):
            raise ValueError(f"optimus_vae_next.encode: need 1 <= lengths[i] <= {L} for each of the {n} rows, got {lengths}")
        if L > ENC_MAX_POSITIONS:
            raise ValueError(f"optimus_vae_next.encode: at most {ENC_MAX_POSITIONS} tokens per row, got {L}")
        p = self.packed()["enc"]
        D, H = p["D"], p["heads"]
        Lp = (L + 7) // 8 * 8
        kv_len = torch.tensor(lengths, dtype=torch.int32).to(dev)      # one copy per call, shared by every layer
        x = ops.clip_text_embed(ids, p["word"], p["pos"], Lp).view(n * Lp, D)    # word + position (+ type 0); pad rows zero
        x = ops.layernorm(x, *p["ln_emb"], eps=p["eps"])
        o = torch.zeros(n * Lp, D, dtype=torch.bfloat16, device=dev)
        for lp in p["layers"]:
            qk = ops.gemm(x, lp["wqk"], bias=lp["bqk"])                                   # [n*Lp, 2D]: q | k
            vt = ops.gemm(lp["wv"], x)                                                    # [D, n*Lp] = V^T (bias folded into bo)
            ops.attention(qk, qk, vt, o, n, H, Lp, Lp, D // H, scale=(D // H) ** -0.5, q_col0=0, k_col0=D,
                          q_bstride=Lp, kv_bstride=Lp, kv_len=kv_len)
            x = ops.layernorm(ops.gemm(o, lp["wo"], bias=lp["bo"], resid=x), *lp["ln1"], eps=p["eps"])
            h = ops.gemm(x, lp["w1"], bias=lp["b1"], act=ops.ACT_GELU)
            x = ops.layernorm(ops.gemm(h, lp["w2"], bias=lp["b2"], resid=x), *lp["ln2"], eps=p["eps"])
        cls = ops.to_f32(x).view(n, Lp * D)[:, :D]                                       # the [CLS] rows, row stride Lp * D
        pooled = torch.empty(n, D, dtype=torch.float32, device=dev)
        z = torch.empty(n, p["w_mu"].shape[0], dtype=torch.float32, device=dev)
        for r0 in range(0, n, ENC_HEAD_ROWS):
            r1 = min(n, r0 + ENC_HEAD_ROWS)
            ops.textdec_gemv(cls[r0:r1], p["w_pool"], pooled[r0:r1], bias=p["b_pool"], act=ops.ACT_TANH)
            ops.textdec_gemv(pooled[r0:r1], p["w_mu"], z[r0:r1])
        return z

    def tokenize(self, text, max_length=77):
        """-> (ids int64 [n, 2 + longest], lengths): the rows optimus_vae_next.encode feeds BERT (optimus.py:730-738)."""
        self._require_encoder()
        if isinstance(text, str):
            raise TypeError("optimus_vae_next.encode takes a list of sentences, not a str (the reference would encode every "
                            "character of it as a sentence of its own)")
        if not 0 <= int(max_length) <= ENC_MAX_POSITIONS - 2:
            raise ValueError(f"optimus_vae_next.encode: max_length must be in [0, {ENC_MAX_POSITIONS - 2}], got {max_length}")
        rows = [self.tokenizer_encoder.encode(s, max_length=int(max_length)) for s in text]
        if not rows:
            raise ValueError("optimus_vae_next.encode: no sentences")
        ids = torch.zeros(len(rows), max(len(r) for r in rows), dtype=torch.long)
        for i, r in enumerate(rows):
            ids[i, :len(r)] = torch.tensor(r, dtype=torch.long)
        return ids, [len(r) for r in rows]

    @torch.no_grad()
    def encode(self, text, max_length=77):
        """optimus_vae_next.encode (optimus.py:729-743): z_mu [n, latent] of a list of sentences, in the parameters' dtype."""
        ids, lengths = self.tokenize(text, max_length=max_length)
        return self.encode_ids(ids, lengths).to(self.encoder.linear.weight.dtype)

    # ------------------------------------------------------------------ decoder
    def _pack(self):
        packed = self._pack_decoder()
        if getattr(self, 'encoder', None) is not None:
            packed["enc"] = self._pack_encoder()
        return packed

    def _pack_decoder(self):
        t = self.decoder.transformer
        layers = []
        for blk in t.h:
            layers.append(dict(
                ln1=(f32(blk.ln_1.weight), f32(blk.ln_1.bias), blk.ln_1.eps),
                w_attn=bf16(blk.attn.c_attn.weight.t()), b_attn=f32(blk.attn.c_attn.bias),
                w_aproj=bf16(blk.attn.c_proj.weight.t()), b_aproj=f32(blk.attn.c_proj.bias),
                ln2=(f32(blk.ln_2.weight), f32(blk.ln_2.bias), blk.ln_2.eps),
                w_fc=bf16(blk.mlp.c_fc.weight.t()), b_fc=f32(blk.mlp.c_fc.bias),
                w_mproj=bf16(blk.mlp.c_proj.weight.t()), b_mproj=f32(blk.mlp.c_proj.bias)))
        return dict(layers=layers, lnf=(f32(t.ln_f.weight), f32(t.ln_f.bias), t.ln_f.eps),
                    wte32=f32(t.wte.weight), wpe32=f32(t.wpe.weight), lm_head=bf16(self.decoder.lm_head.weight),
                    w_lin=bf16(t.linear.weight), w_emb=bf16(t.linear_emb.weight))

    def _state(self, R, device):
        states = self.__dict__.setdefault('_states', {})
        key = (str(device), R)
        if key not in states:
            states[key] = _State(self.decoder, R, device)
        return states[key]

    def invalidate_packed(self):
        super().invalidate_packed()
        self.__dict__['_states'] = {}        # captured graphs hold the old weight addresses

    # ------------------------------------------------------------------ one token step (5 launches per layer + 4)
    def _step(self, st, p, temperature, eos, max_len, mode, record, top_k=0, top_p=0.0, num_beams=0):
        ops = _ops()
        dec = self.decoder
        D = dec.n_embd
        ops.textdec_embed(st.tokens, st.step, p["wte32"], p["wpe32"], st.emb, st.h, pos_offset=1)
        for i, L in enumerate(p["layers"]):
            ops.textdec_gemv(st.h, L["w_attn"], st.qkv, bias=L["b_attn"], ln=L["ln1"])
            if num_beams:
                ops.textdec_attention_indexed(st.qkv, st.mem[:, i * D:(i + 1) * D], st.kc[i], st.vc[i], st.src, st.step, st.a,
                                              scale=0.125)
            else:
                ops.textdec_attention(st.qkv, st.mem[:, i * D:(i + 1) * D], st.kc[i], st.vc[i], st.step, st.a, scale=0.125)
            ops.textdec_gemv(st.a, L["w_aproj"], st.h, bias=L["b_aproj"], accumulate=True)
            ops.textdec_gemv(st.h, L["w_fc"], st.m, bias=L["b_fc"], ln=L["ln2"], act=ops.ACT_GELU_TANH)
            ops.textdec_gemv(st.m, L["w_mproj"], st.h, bias=L["b_mproj"], accumulate=True)
        ops.textdec_gemv(st.h, p["lm_head"], st.logits, ln=p["lnf"])
        if num_beams:
            ops.textdec_beam_step(st.logits, num_beams, st.tokens, st.src, st.scores, st.done, st.lengths, st.step, st.cand_tok,
                                  st.cand_logp, temperature=temperature, eos=eos, max_len=max_len,
                                  record=st.record if record else None, trace=st.trace if record else None)
        else:
            ops.textdec_sample(st.logits, st.tokens, st.done, st.lengths, st.step, temperature=temperature,
                               seed=st.seed if mode == "seed" else None, uniforms=st.uniforms if mode == "uniforms" else None,
                               forced=st.forced if mode == "forced" else None, eos=eos, max_len=max_len,
                               record=st.record if record else None, top_k=top_k, top_p=top_p)
        ops.add_int(st.step, 1)

    @torch.no_grad()
    def _run(self, z, temperature, eos, pre_scale=1.0, max_len=MAX_LENGTH, nsteps=None, mode="seed", uniforms=None, forced=None,
             record=False, graph=True, top_k=0, top_p=0.0, num_beams=0):
        """mode "beam" (num_beams >= 1) decodes the n latents of z as rows latent * num_beams + beam, n * num_beams <= 16."""
        top_k, top_p = _check_cuts(top_k, top_p)
        require_cuda(z, "optimus_vae_next.decode")
        if z.dim() != 2 or z.shape[1] != self.nz:
            raise ValueError(f"optimus_vae_next: expected latents [n, {self.nz}], got {tuple(z.shape)}")
        K = int(num_beams) if mode == "beam" else 0
        R = z.shape[0] * max(K, 1)
        if not 1 <= R <= 16:
            raise ValueError(f"optimus_vae_next: decodes 1 to 16 latents per call, got {R}" if not K else
                             f"optimus_vae_next: beam search runs n * num_beams <= 16 rows per call, got {z.shape[0]} x {K}")
        ops = _ops()
        p = self.packed()
        st = self._state(R, z.device)
        nsteps = max_len - 2 if nsteps is None else nsteps
        if nsteps > CACHE_SLOTS:
            raise ValueError(f"optimus_vae_next: at most {CACHE_SLOTS} steps")
        # per-call state: latent projections (the memory slices and the embedding offset), tokens, flags, seed
        zs = z.float() * float(pre_scale)
        zs = (zs.repeat_interleave(K, 0) if K else zs).contiguous()
        ops.textdec_gemv(zs, p["w_emb"], st.emb)
        ops.textdec_gemv(zs, p["w_lin"], st.mem)
        init = torch.full((R, CACHE_SLOTS + 1), eos, dtype=torch.int32)
        init[:, 0] = BOS_ID
        if mode == "forced":
            init[:, :forced.shape[1]] = forced.cpu()
        st.tokens.copy_(init)
        st.done.zero_()
        st.lengths.fill_(nsteps + 1)
        st.step.zero_()
        if mode == "seed":
            st.seed.copy_(torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64))
        elif mode == "uniforms":
            st.uniforms.zero_()
            st.uniforms[:, :uniforms.shape[1]].copy_(uniforms)
        elif mode == "beam":
            scores = torch.full((R,), -math.inf, dtype=torch.float64)
            scores[::K] = 0.0                     # only beam 0 of each latent is live at step 0
            st.scores.copy_(scores)
            st.src.copy_(torch.arange(R, dtype=torch.int32)[:, None].expand(R, CACHE_SLOTS))
        else:
            st.forced.zero_()
            st.forced[:, :forced.shape[1]].copy_(forced)
        key = (float(temperature), int(eos), int(max_len), mode, bool(record), top_k, top_p, K)
        s = 0
        while s < nsteps:
            n = min(STEPS_PER_CHECK, nsteps - s)
            g = st.graphs.get(key) if graph and n == STEPS_PER_CHECK else None
            if g is not None:
                g.replay()
            else:
                for _ in range(n):
                    self._step(st, p, temperature, eos, max_len, mode, record, top_k, top_p, K)
                if graph and n == STEPS_PER_CHECK and key not in st.graphs:
                    # the chunk just ran eagerly (kernels configured, caches warm); capture one for the later chunks
                    torch.cuda.current_stream().synchronize()
                    step_before = st.step.clone()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        for _ in range(n):
                            self._step(st, p, temperature, eos, max_len, mode, record, top_k, top_p, K)
                    st.step.copy_(step_before)        # capture does not execute, but keep the counter exactly as the eager chunk left it
                    st.graphs[key] = g
            s += n
            if mode != "forced" and bool(st.done.cpu().all()):
                break
        return st, s

    def _beam_group(self, z, num_beams, temperature, pre_scale, eos, length_penalty, record=False, graph=True):
        """Beam search of n latents with n * num_beams <= 16 -> (per latent, its num_beams (ids, score, normalized score) best
        first; the state; the steps run)."""
        st, ran = self._run(z, temperature, eos, pre_scale=pre_scale, mode="beam", record=record, graph=graph, num_beams=num_beams)
        tokens, lengths, scores = st.tokens.cpu(), st.lengths.cpu().tolist(), st.scores.cpu().tolist()
        out = []
        for i in range(z.shape[0]):
            beams = []
            for j in range(num_beams):
                r = i * num_beams + j
                n = min(lengths[r] - 1, MAX_LENGTH - 2)   # scored tokens: a forced final <EOS> has none
                beams.append((tokens[r, :lengths[r]].long(), scores[r], scores[r] / n ** length_penalty))
            out.append([beams[j] for j in sorted(range(num_beams), key=lambda j: (-beams[j][2], j))])
        return out, st, ran

    @torch.no_grad()
    def decode_beams(self, z, num_beams, temperature=1.0, pre_scale=1.0, length_penalty=1.0, eos_token=EOS_ID, graph=True):
        """Beam search (see the module docstring): for each latent, its num_beams final hypotheses as (ids int64 CPU tensor from
        <BOS> to <EOS>, score = summed fp64 log-probability, score / n ** length_penalty), best normalized score first.
        num_beams latents' worth of rows run per token step, at most 16: more latents are decoded in groups of 16 // num_beams,
        one after the other, each re-streaming the weights."""
        num_beams, length_penalty = _check_beams(num_beams, length_penalty, 0, 0.0)
        if num_beams < 1:
            raise ValueError(f"optimus_vae_next.decode_beams: num_beams must be >= 1, got {num_beams}")
        require_cuda(z, "optimus_vae_next.decode")
        if z.dim() != 2 or z.shape[0] < 1:
            raise ValueError(f"optimus_vae_next: expected latents [n, {self.nz}], got {tuple(z.shape)}")
        per = MAX_BEAMS // num_beams
        out = []
        for i0 in range(0, z.shape[0], per):
            out += self._beam_group(z[i0:i0 + per], num_beams, temperature, pre_scale, int(eos_token), length_penalty,
                                    graph=graph)[0]
        return out

    @torch.no_grad()
    def decode_ids(self, z, temperature=1.0, eos_token=EOS_ID, pre_scale=1.0, uniforms=None, return_logits=False, graph=True,
                   top_k=0, top_p=0.0, num_beams=0, length_penalty=1.0):
        """Sampled token rows, each an int64 CPU tensor starting with <BOS> and (unless eos_token never occurs and is never forced)
        ending with eos_token, length <= 30.  uniforms (fp64 [n, >=28]) replaces the Philox draws; return_logits also returns the
        fp32 logits of every step that ran, [steps, n, 50260] on the device.  top_k > 0 keeps the top_k most likely tokens (ties
        included), 0 < top_p < 1 the nucleus of mass top_p (optimus.py:690-719); the defaults sample the full softmax.
        num_beams >= 1: each latent's best beam-search hypothesis instead (decode_beams; no cuts, uniforms or logits)."""
        num_beams, length_penalty = _check_beams(num_beams, length_penalty, top_k, top_p)
        if num_beams:
            if uniforms is not None or return_logits:
                raise ValueError("optimus_vae_next: beam search takes no uniforms and returns no logits")
            return [b[0][0] for b in self.decode_beams(z, num_beams, temperature=temperature, pre_scale=pre_scale,
                                                       length_penalty=length_penalty, eos_token=eos_token, graph=graph)]
        st, ran = self._run(z, temperature, int(eos_token), pre_scale=pre_scale, mode="uniforms" if uniforms is not None else "seed",
                            uniforms=uniforms, record=return_logits, graph=graph, top_k=top_k, top_p=top_p)
        tokens, lengths = st.tokens.cpu(), st.lengths.cpu()
        rows = [tokens[r, :int(lengths[r])].long() for r in range(st.R)]
        if return_logits:
            return rows, st.record[:ran].clone()
        return rows

    @torch.no_grad()
    def teacher_forced_logits(self, z, ids, graph=False):
        """fp32 logits [n, L, vocab] of every position of the given token rows (int64 [n, L], L <= 32), the product's kernels run
        step by step over the KV cache with the tokens forced instead of sampled."""
        ids = torch.as_tensor(ids)
        R, L = ids.shape
        st, ran = self._run(z, 1.0, -1, max_len=1 << 30, nsteps=L, mode="forced", forced=ids.to(torch.int32).to(z.device),
                            record=True, graph=graph)
        return st.record[:L].permute(1, 0, 2).contiguous()

    @torch.no_grad()
    def decode(self, z, temperature=1.0, pre_scale=1.0, top_k=0, top_p=0.0, num_beams=0, length_penalty=1.0):
        """optimus_vae_next.decode (optimus.py:746-763): one string per latent row; top_k / top_p / num_beams / length_penalty as
        in decode_ids (num_beams >= 1: the best beam-search hypothesis)."""
        rows = self.decode_ids(z, temperature=temperature, pre_scale=pre_scale, top_k=top_k, top_p=top_p, num_beams=num_beams,
                               length_penalty=length_penalty)
        return [self.tokenizer_decoder.sentence(r.tolist()) for r in rows]
