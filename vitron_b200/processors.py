"""fp32 statement of the vb200_logits_process contract (include/vitron_b200.h): the HF transformers 4.31 logits
processors that `generate` builds from repetition_penalty, no_repeat_ngram_size, min_length and min_new_tokens.

It is what a CPU-resident LlamaEngine runs in place of the kernel (such an engine runs no kernels of this library), and
the GPU tests compare the kernel with it. It restates, from transformers/generation/logits_process.py at v4.31.0:

- `RepetitionPenaltyLogitsProcessor`: `score = torch.gather(scores, 1, input_ids)`, `score = torch.where(score < 0,
  score * penalty, score / penalty)`, `scores.scatter_(1, input_ids, score)`. Gather then scatter: an id that occurs
  several times is penalised once. fp32, with a correctly rounded division.
- `NoRepeatNGramLogitsProcessor` with `_get_ngrams` / `_get_generated_ngrams` / `_calc_banned_ngram_tokens`: with
  cur_len = input_ids.shape[-1], nothing is banned while cur_len + 1 < n; otherwise every id that followed an earlier
  occurrence of the last n - 1 ids is set to -inf (n = 1: every id of the history).
- `MinLengthLogitsProcessor`: while cur_len < min_length, every EOS id is set to -inf.
- `MinNewTokensLengthLogitsProcessor(prompt_length_to_skip=input_len)`: while cur_len - input_len < min_new_tokens,
  every EOS id is set to -inf.

They apply in that order, the order of 4.31's `GenerationMixin._get_logits_processor`, which adds each one only when
repetition_penalty is not None and != 1.0, no_repeat_ngram_size > 0, and (with an EOS id) min_length > 0 /
min_new_tokens > 0. `check_settings` applies those rules and the constructors' ValueErrors.

A row's history is 4.31's `input_ids` row: the caller's raw input_ids row, all input_len columns (the -200 / -300 image
and region sentinels count as one position each, left-padding columns are included), followed by the row's generated
ids (for a beam, its own history: token j of row r is token_log[beam_src[r, P + j], j], as beam.running_ids reads it).

In greedy and sampled decoding the processors act on the raw fp32 logits (before the sampler's warpers); in beam search
and beam sampling on log_softmax(logits) (`logprobs=True`: beam.log_softmax64 rounded to fp32), before the running
beam score is added, so the beam scores accumulate processed scores as 4.31's do.

Stated divergences, in cases where 4.31 fails or indexes outside the vocabulary:
- Sentinel ids (< 0) are positions of the history but not vocabulary entries. The repetition penalty skips them (4.31's
  torch.gather raises on index -200, so `generate(images=..., repetition_penalty=...)` fails in the reference). N-gram
  matching compares them like any other id, but a sentinel is never banned (4.31's `scores[i, [-200]] = -inf` wraps
  around and bans vocabulary id V - 200).
- Ids outside [0, V), EOS ids included (e.g. eos_token_id=-1, which 4.31 would wrap to V - 1), are never penalised or
  banned.
"""
import struct

import numpy as np
import torch

PARAMS = struct.Struct("<fiiiii8i")   # vb_proc_params (56 bytes)
MAX_EOS = 8
MAX_HIST = 8192                      # staged history tokens per row: prompt buffer width + token_log width
MAX_N = 49152


def check_settings(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, eos_ids=()):
    """4.31's enable rules and constructor checks. Returns the settings with every disabled processor at its off value
    (penalty 1.0, sizes 0) and whether any processor is enabled."""
    rp, ng, ml, mn = 1.0, 0, 0, 0
    if repetition_penalty is not None and repetition_penalty != 1.0:
        if not isinstance(repetition_penalty, float) or not (repetition_penalty > 0):
            raise ValueError(f"`penalty` has to be a strictly positive float, but is {repetition_penalty}")
        rp = float(repetition_penalty)
    if no_repeat_ngram_size is not None and no_repeat_ngram_size > 0:
        if not isinstance(no_repeat_ngram_size, int):
            raise ValueError(f"`ngram_size` has to be a strictly positive integer, but is {no_repeat_ngram_size}")
        ng = int(no_repeat_ngram_size)
    has_eos = eos_ids is not None and len(eos_ids) > 0
    if min_length is not None and has_eos and min_length > 0:
        if not isinstance(min_length, int):
            raise ValueError(f"`min_length` has to be a non-negative integer, but is {min_length}")
        ml = int(min_length)
    if min_new_tokens is not None and has_eos and min_new_tokens > 0:
        if not isinstance(min_new_tokens, int):
            raise ValueError(f"`min_new_tokens` has to be a positive integer, but is {min_new_tokens}")
        mn = int(min_new_tokens)
    if has_eos and len(eos_ids) > MAX_EOS and (ml or mn):
        raise ValueError(f"at most {MAX_EOS} EOS ids are supported, got {len(eos_ids)}")
    settings = dict(repetition_penalty=rp, no_repeat_ngram_size=ng, min_length=ml, min_new_tokens=mn)
    return settings, (rp != 1.0 or ng > 0 or ml > 0 or mn > 0)


def pack_params(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, input_len=0,
                eos_ids=()):
    """vb_proc_params as a CPU uint8 tensor."""
    eos = [int(e) for e in eos_ids]
    if len(eos) > MAX_EOS:
        raise ValueError(f"at most {MAX_EOS} EOS ids are supported, got {len(eos)}")
    raw = PARAMS.pack(float(repetition_penalty), int(no_repeat_ngram_size), int(min_length), int(min_new_tokens),
                      int(input_len), len(eos), *(eos + [0] * (MAX_EOS - len(eos))))
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8)


def unpack_params(buf):
    v = PARAMS.unpack(bytes(buf.cpu().numpy().tobytes()))
    return dict(repetition_penalty=v[0], no_repeat_ngram_size=v[1], min_length=v[2], min_new_tokens=v[3],
                input_len=v[4], eos=list(v[6:6 + v[5]]))


def history(prompt_ids, input_len, r, t, token_log=None, beam_src=None, prompt_len=None):
    """Row r's history as a list of ints: prompt_ids[r, :input_len], then its t generated ids."""
    h = [int(x) for x in prompt_ids[r, :input_len].tolist()]
    if t > 0:
        if beam_src is not None:
            P = int(prompt_len[r])
            src = beam_src[r, P:P + t].long()
        else:
            src = torch.full((t,), r, dtype=torch.long)
        h += [int(x) for x in token_log[src, torch.arange(t)].tolist()]
    return h


def penalize(row, hist, penalty):
    """RepetitionPenaltyLogitsProcessor on one fp32 numpy row, in place: each distinct in-vocabulary id once."""
    V = row.shape[0]
    ids = np.unique(np.asarray([i for i in hist if 0 <= i < V], dtype=np.int64))
    if ids.size:
        s = row[ids]
        p = np.float32(penalty)
        with np.errstate(invalid="ignore", over="ignore"):
            row[ids] = np.where(s < 0, s * p, s / p)


def banned_ngram_tokens(hist, n):
    """_get_ngrams + _get_generated_ngrams: ids that followed an earlier occurrence of the last n - 1 ids."""
    cur_len = len(hist)
    if cur_len + 1 < n:
        return []
    ngrams = {}
    for ng in zip(*[hist[i:] for i in range(n)]):
        ngrams.setdefault(tuple(ng[:-1]), []).append(ng[-1])
    return ngrams.get(tuple(hist[cur_len + 1 - n:cur_len]), [])


def process(logits, params, prompt_ids, token_log=None, kv_len=None, prompt_len=None, beam_src=None, logprobs=False):
    """Same arguments as ops.logits_process, on host tensors: rows of fp32 logits processed in place (and returned)."""
    from .beam import log_softmax64
    prm = unpack_params(params)
    R, V = logits.shape
    prompt_ids, token_log, kv_len, prompt_len, beam_src = (None if x is None else x.cpu() for x in
                                                           (prompt_ids, token_log, kv_len, prompt_len, beam_src))
    rows = log_softmax64(logits).float() if logprobs else logits.detach().cpu().float()
    out = rows.numpy().copy()
    input_len = prm["input_len"]
    for r in range(R):
        t = int(kv_len[r]) - int(prompt_len[r]) if kv_len is not None else 0
        hist = history(prompt_ids, input_len, r, t, token_log, beam_src, prompt_len)
        cur_len = len(hist)
        if prm["repetition_penalty"] != 1.0:
            penalize(out[r], hist, prm["repetition_penalty"])
        if prm["no_repeat_ngram_size"] > 0:
            for tok in banned_ngram_tokens(hist, prm["no_repeat_ngram_size"]):
                if 0 <= tok < V:
                    out[r, tok] = -np.inf
        if (0 < prm["min_length"] and cur_len < prm["min_length"]) or \
                (0 < prm["min_new_tokens"] and cur_len - input_len < prm["min_new_tokens"]):
            for e in prm["eos"]:
                if 0 <= e < V:
                    out[r, e] = -np.inf
    logits.copy_(torch.from_numpy(out).to(logits.device))
    return logits
