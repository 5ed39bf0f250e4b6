"""float64 statement of the vb200_beam_advance contract (include/vitron_b200.h): one step of HF transformers 4.31
`beam_search` with `BeamSearchScorer` / `BeamHypotheses` for a decoder-only model, `do_sample=False` and no logits
processors, and the `finalize` that builds the returned sequences.

It is what a CPU-resident LlamaEngine runs for its beam step (such an engine runs no kernels of this library), and the
GPU tests compare the kernel with it. The rules, in order:

1. Initial beam scores are 0 for beam 0 and -1e9 for beams 1..k-1: step 0 picks from beam 0 only.
2. Each row's candidate scores are log_softmax(fp32 logits) + the row's beam score; NaN counts as -inf, and a row with no
   number above -inf scores -inf everywhere.
3. Per request the top 2k of the flat [k * V] scores are taken. Ties go to the lower flat index beam * V + token (a stated
   choice: torch's topk leaves tie order unspecified).
4. Candidates are walked in rank order: an EOS candidate (any id of eos) at rank < k becomes a finished hypothesis, at
   rank >= k it is skipped; any other candidate becomes the next beam until k beams are filled. If fewer than k are
   filled (possible only with several EOS ids), the missing beams continue their own row with pad and score -1e9, where
   4.31 raises.
5. A hypothesis scores sum_logprobs / L ** length_penalty, L = input_len + the tokens generated before the EOS: the
   reference's hyp.shape[-1], which counts the -200 image sentinel and left padding as one position each; length_penalty
   is carried as a double, as the Python float 4.31 uses. This is 4.31;
   later transformers releases divide by the generated length only (the two agree at length_penalty = 0).
6. Each request keeps its k best hypotheses; a better one evicts the lowest score (the earliest added among equals).
7. is_done follows 4.31 for early_stopping True, False and "never" (max_length = input_len + max_new_tokens). A done
   request's beams get pad, score 0 and themselves as parent from then on (4.31 points them at row 0; their content is
   never used).
8. finalize adds the running beams of unfinished requests as hypotheses, keeps the best num_return_sequences of each
   request (highest score, the latest added among equals, as 4.31's stable sort + pop), pads with pad and appends
   eos[0] (pad when there is no EOS id) where a hypothesis is shorter than the output, which is
   min(longest + 1, max_length) positions wide.

Beam sampling (vb200_beam_sample_advance, `generate(do_sample=True, num_beams=k)`) restates 4.31's
`GenerationMixin.beam_sample` and the `is_beam_sample_gen_mode` branch of `GenerationMixin.generate`
(transformers/generation/utils.py at v4.31.0). Rules 4-8 hold as above; rules 1-3 become, per search b, step t:

1s. Initial beam scores are 0 for every beam. 4.31's beam_sample initialises
        beam_scores = torch.zeros((batch_size, num_beams), dtype=torch.float, device=input_ids.device)
        beam_scores = beam_scores.view((batch_size * num_beams,))
    without beam_search's `beam_scores[:, 1:] = -1e9`: step 0 draws its 2k candidates from k identical live rows, so
    two beams may take the same token (ties in w go to the lower flat index, i.e. the lower beam).
2s. c = log_softmax(fp32 logits[r]) + beam_score[r] (`next_token_scores + beam_scores[:, None]`), then the logits warpers
    on the cumulative c ("intentionally applied after adding running beam scores"): TemperatureLogitsWarper w = c / T,
    TopKLogitsWarper(max(top_k, 2)) and TopPLogitsWarper(top_p, min_tokens_to_keep=2) (`_get_logits_warper` passes
    min_tokens_to_keep = 2 when num_beams > 1); removed entries become -inf. top_k None / 0 is off, as in the sampled
    path. Within a row top-k and top-p see w up to a constant, so they are vitron_b200.sampling's value-based cuts of
    the sampler (ties at a cut stay together) with "at least the 2 largest kept" added; 4.31 keeps the last 2 of its
    ascending sort, which differs only in tie order. w is an fp32 value, as in 4.31: a w below the fp32 range is -inf.
    Temperature compounds, |w_t| ~ (|s| + |w_{t-1}|) / T, so at T < 1 a long search's scores leave the fp32 range (at
    T = 0.2 after roughly 55 steps). 4.31 then raises (softmax of an all -inf row is NaN, and multinomial rejects it);
    here a search whose entries are all -inf has no draws, so by rule 4 its k beams continue their own rows with pad
    and score -1e9, and the next step's scores are finite again.
3s. `probs = softmax(w.view(B, k * V))`, `torch.multinomial(probs, 2k)` without replacement, then the drawn scores are
    sorted descending. The draw is stated as torch's own algorithm, an exponential race, in the log domain:
    key = w - log(-log U) over the entries with w > -inf; the 2k largest keys (ties to the lower flat index f = j * V +
    token) are the draws. U = (2 * (x >> 9) + 1) * 2^-24 in (0, 1), x = word f % 4 of Philox4x32-10(counter
    (t, b, f // 4, 1), key (seed low 32 bits, seed high 32 bits)). The draws are ranked by w, descending, ties to the
    lower flat index (torch.sort leaves tie order open), and go through rules 4-7 with w as the candidate score: the new
    beam scores and the hypotheses' sum_logprobs are warped scores. Entries whose fp32 probability underflows to 0
    (e.g. the pad beams of rule 4 at -1e9 next to live ones) rank after every positive one and are drawn in key order
    where 4.31 raises ("not enough non-negative category to sample"); fewer than 2k entries with w > -inf give fewer
    draws, handled as rule 4's missing beams.
5s. num_return_sequences = r runs r independent searches per prompt: 4.31 builds
    `BeamSearchScorer(batch_size=batch_size * num_return_sequences, ...)` and expands the input by
    `num_beams * num_return_sequences`, and finalize keeps each search's best hypothesis, so the output is [B * r, L]
    in request-major order (search b * r + i samples prompt b).
"""
import struct

import numpy as np
import torch

MAX_K = 16
MAX_EOS = 8
PARAMS = struct.Struct("<diiiii8i4x")   # vb_beam_params (64 bytes, length_penalty a double)
EARLY_STOPPING = {False: 0, True: 1, "never": 2}
_SEQ_STRIDE = 2 * MAX_K               # hypothesis insertion order: seq = t * 32 + rank (the kernel's hyp_seq)


def pack_params(length_penalty, early_stopping, pad_token_id, input_len, max_length, eos_ids):
    """vb_beam_params as a CPU uint8 tensor."""
    eos = [int(e) for e in eos_ids]
    if len(eos) > MAX_EOS:
        raise ValueError(f"at most {MAX_EOS} EOS ids are supported, got {len(eos)}")
    if early_stopping not in EARLY_STOPPING:
        raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
    raw = PARAMS.pack(float(length_penalty), EARLY_STOPPING[early_stopping], int(pad_token_id), int(input_len),
                      int(max_length), len(eos), *(eos + [0] * (MAX_EOS - len(eos))))
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8)


def unpack_params(buf):
    v = PARAMS.unpack(bytes(buf.cpu().numpy().tobytes()))
    es = {0: False, 1: True, 2: "never"}[v[1]]
    return dict(length_penalty=float(v[0]), early_stopping=es, pad=v[2], input_len=v[3], max_length=v[4],
                eos=list(v[6:6 + v[5]]))


def log_softmax64(logits):
    """Rule 2 without the beam score: float64 log-softmax of rows of fp32 logits, NaN as -inf."""
    l = logits.detach().cpu().float().double()
    l = torch.where(torch.isnan(l), torch.full_like(l, float("-inf")), l)
    mx = l.max(-1, keepdim=True).values
    out = l - mx - torch.log(torch.exp(l - mx).sum(-1, keepdim=True))
    return torch.where(mx == float("-inf"), torch.full_like(l, float("-inf")), out)


def top_candidates(scores, k):
    """Rule 3: scores float64 [k, V] -> list of (score, flat index) of the top 2k, best first."""
    s = scores.reshape(-1).numpy()
    flat = np.arange(s.shape[0])
    order = np.lexsort((flat, -s))[:2 * k]
    return [(float(s[i]), int(i)) for i in order]


class Hypotheses:
    """BeamHypotheses of one request, in the kernel's slot layout: entries are dicts (score, length, seq, ids)."""

    def __init__(self, k, length_penalty, early_stopping, max_length):
        self.k, self.lp, self.es, self.max_length = k, length_penalty, early_stopping, max_length
        self.slots = []

    def worst(self):
        return min(h["score"] for h in self.slots) if self.slots else 1e9

    def add(self, sum_logprobs, length, seq, ids=None):
        """Returns the slot the hypothesis went to, or None."""
        score = float(sum_logprobs) / float(length) ** self.lp
        if len(self.slots) >= self.k and not score > self.worst():
            return None
        h = dict(score=score, length=length, seq=seq, ids=ids)
        if len(self.slots) < self.k:
            self.slots.append(h)
            return len(self.slots) - 1
        slot = min(range(len(self.slots)), key=lambda s: (self.slots[s]["score"], self.slots[s]["seq"]))
        self.slots[slot] = h
        return slot

    def is_done(self, best_sum_logprobs, cur_len):
        if len(self.slots) < self.k:
            return False
        if self.es is True:
            return True
        length = self.max_length if (self.es == "never" and self.lp > 0.0) else cur_len
        return self.worst() >= float(best_sum_logprobs) / float(length) ** self.lp


def process(cands, k, V, hyps, t, prm):
    """Rules 4-7 for one request that is not done: cands from top_candidates, t tokens generated before this step.
    Returns (children [(parent beam, token, score)] * k, added [(slot, parent beam)], done)."""
    children, added = [], []
    eos = set(prm["eos"])
    for rank, (score, flat) in enumerate(cands):
        if len(children) == k:
            break
        j, tok = divmod(flat, V)
        if tok in eos:
            if rank >= k:
                continue
            slot = hyps.add(score, prm["input_len"] + t, t * _SEQ_STRIDE + rank)
            if slot is not None:
                added.append((slot, j))
        else:
            children.append((j, tok, score))
    while len(children) < k:
        children.append((len(children), prm["pad"], -1e9))
    return children, added, hyps.is_done(cands[0][0] if cands else float("-inf"), prm["input_len"] + t)


def beam_advance(logits, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count, hyp_ids,
                 next_src, positions, kv_len, token_log, prompt_len, logprobs=False):
    """Same arguments and bookkeeping as ops.beam_advance, on host tensors. logprobs=True: the rows already hold
    (processed) log-probabilities, vitron_b200.processors' logprobs output."""
    lsm = _logprobs(logits) if logprobs else log_softmax64(logits)

    def cands(b, r0, t):
        return top_candidates(lsm[r0:r0 + k] + beam_score[r0:r0 + k].double().cpu()[:, None], k)
    _advance(cands, logits.shape, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count,
             hyp_ids, next_src, positions, kv_len, token_log, prompt_len)


def _logprobs(rows):
    """Rows that already hold log-probabilities, as float64 (NaN as -inf)."""
    l = rows.detach().cpu().float().double()
    return torch.where(torch.isnan(l), torch.full_like(l, float("-inf")), l)


def warped_scores(logits, beam_score, temperature, logprobs=False):
    """Rule 2s up to the cuts: w = (log_softmax(logits) + beam_score) / T, float64 [R, V]; a w that fp32 cannot hold is
    -inf. logprobs=True: the rows are log-probabilities already."""
    lsm = _logprobs(logits) if logprobs else log_softmax64(logits)
    w = (lsm + beam_score.double().cpu()[:, None]) / float(temperature)
    return torch.where(torch.isinf(w.float()), torch.full_like(w, float("-inf")), w)


def warp_kept(w, top_k, top_p):
    """Rule 2s's cuts per row of w: (kept bool [R, V], near bool [R]: a top-p fraction within 1e-5 of top_p)."""
    from .sampling import sample_support
    kept, _, near = sample_support(w, 1.0, max(int(top_k), 2) if top_k > 0 else 0, float(top_p), min_keep=2)
    return kept & (w > float("-inf")), near


def gumbel(seed, t, b, flat):
    """Rule 3s's noise -log(-log U) of the flat indices `flat` (int array) of search b at step t, float64."""
    from .sampling import philox4x32_10
    flat = np.asarray(flat, dtype=np.uint64)
    ctr = np.stack([np.full_like(flat, t & 0xFFFFFFFF), np.full_like(flat, b), flat >> np.uint64(2),
                    np.ones_like(flat)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint64), ctr.shape[:-1] + (2,))
    x = np.take_along_axis(philox4x32_10(ctr, key), (flat & np.uint64(3)).astype(np.int64)[..., None], -1)[..., 0]
    u = (2.0 * (x >> np.uint64(9)).astype(np.float64) + 1.0) * 2.0 ** -24
    return -np.log(-np.log(u))


def sample_draws(w, kept, k, b, t, seed):
    """Rule 3s for one search: w / kept [k, V]. Returns (draws [(w, flat)] ranked by w, keys of every keyed entry
    sorted descending)."""
    V = w.shape[1]
    flat = np.nonzero(kept.reshape(-1).numpy())[0]
    if flat.size == 0:
        return [], np.zeros(0)
    key = w.reshape(-1).numpy()[flat] + gumbel(seed, t, b, flat)
    order = np.lexsort((flat, -key))
    drawn = [(float(w.reshape(-1)[f]), int(f)) for f in flat[order[:2 * k]]]
    drawn.sort(key=lambda c: (-c[0], c[1]))
    assert all(0 <= f < k * V for _, f in drawn)
    return drawn, key[order]


def beam_sample_advance(logits, k, params, sample_params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq,
                        hyp_count, hyp_ids, next_src, positions, kv_len, token_log, prompt_len, logprobs=False):
    """Same arguments and bookkeeping as ops.beam_sample_advance, on host tensors (logprobs as in beam_advance)."""
    from .ops import SAMPLE_PARAMS
    temperature, top_k, top_p, _, seed = SAMPLE_PARAMS.unpack(sample_params.cpu().numpy().tobytes())
    w = warped_scores(logits, beam_score, temperature, logprobs)
    kept, _ = warp_kept(w, top_k, top_p)

    def cands(b, r0, t):
        return sample_draws(w[r0:r0 + k], kept[r0:r0 + k], k, b, t, seed)[0]
    _advance(cands, logits.shape, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count,
             hyp_ids, next_src, positions, kv_len, token_log, prompt_len)


def _advance(cands_of, shape, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count,
             hyp_ids, next_src, positions, kv_len, token_log, prompt_len):
    """Rules 4-7 and the bookkeeping of one step; cands_of(b, r0, t) gives request b's ranked (score, flat) candidates."""
    prm = unpack_params(params)
    R, V = shape
    for b in range(R // k):
        r0 = b * k
        t, P = int(kv_len[r0]) - int(prompt_len[r0]), int(prompt_len[r0])
        if int(done[b]):
            children, added = [(c, prm["pad"], 0.0) for c in range(k)], []
        else:
            hyps = Hypotheses(k, prm["length_penalty"], prm["early_stopping"], prm["max_length"])
            hyps.slots = [dict(score=float(hyp_score[r0 + s]), length=int(hyp_len[r0 + s]), seq=int(hyp_seq[r0 + s]))
                          for s in range(int(hyp_count[b]))]
            children, added, is_done = process(cands_of(b, r0, t), k, V, hyps, t, prm)
            for s, h in enumerate(hyps.slots):
                hyp_score[r0 + s], hyp_len[r0 + s], hyp_seq[r0 + s] = h["score"], h["length"], h["seq"]
            hyp_count[b] = len(hyps.slots)
            if is_done:
                done[b] = 1
        for slot, j in added:            # generated ids of the new hypotheses, read through the parent's history
            w = beam_src[r0 + j, P:P + t].long()
            hyp_ids[r0 + slot, :t] = token_log[w, torch.arange(t)]
        hist = beam_src[[r0 + j for j, _, _ in children], P:P + t].clone()
        beam_src[r0:r0 + k, P:P + t] = hist
        for c, (j, tok, score) in enumerate(children):
            rr = r0 + c
            beam_score[rr], parent[rr], next_src[rr] = score, r0 + j, tok
            token_log[rr, t] = tok
            beam_src[rr, P + t] = rr
    positions.add_(1)
    kv_len.add_(1)


def running_ids(beam_src, token_log, prompt_len, t):
    """Generated ids [R, t] of every running beam: token j of row r was logged by row beam_src[r, P + j]."""
    R = beam_src.shape[0]
    cols = prompt_len.long()[:, None] + torch.arange(t)[None, :]
    w = torch.gather(beam_src.long(), 1, cols)
    return token_log[w, torch.arange(t)[None, :].expand(R, t)]


def finalize(hyps, done, running_scores, running, num_return_sequences, prm):
    """Rule 8. hyps: one Hypotheses per request (ids filled in); running: generated ids [B * k, t] with scores
    [B * k]. Returns the generated part [B * num_return_sequences, width] of the output, int64."""
    k = hyps[0].k if hyps else 1
    t = running.shape[1]
    best = []
    for b, h in enumerate(hyps):
        if not done[b]:
            for c in range(k):
                slot = h.add(float(running_scores[b * k + c]), prm["input_len"] + t, (1 << 40) + c)
                if slot is not None:
                    h.slots[slot]["ids"] = running[b * k + c]
        ranked = sorted(h.slots, key=lambda e: (e["score"], e["seq"]))
        best += [ranked.pop() for _ in range(num_return_sequences)]
    lengths = [e["length"] for e in best]
    width = min(max(lengths) + 1, prm["max_length"]) - prm["input_len"]
    end = prm["eos"][0] if prm["eos"] else prm["pad"]
    out = torch.full((len(best), width), int(prm["pad"]), dtype=torch.int64)
    for i, e in enumerate(best):
        n = e["length"] - prm["input_len"]
        out[i, :n] = torch.as_tensor(e["ids"][:n], dtype=torch.int64)
        if n < width:
            out[i, n] = end
    return out
