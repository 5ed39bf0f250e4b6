"""CPU (no GPU): the float64 statement of the beam-sampling step (vitron_b200.beam.beam_sample_advance) against a literal
transcription of transformers 4.31 `beam_sample` (torch.multinomial replaced by the same Gumbel keys), the statement's
draws against the exact without-replacement probabilities, argument validation of vb200_beam_sample_advance, and the host
logic of generate(do_sample=True, num_beams=k) on a CPU engine against the statement driven over the engine's logits."""
import itertools
import math
import random

import numpy as np
import pytest
import torch

from vitron_b200 import beam as E
from vitron_b200 import ops
from tests.test_beam_cpu import LiteralHyps, _ids, engine_logits_fn, lib, tiny_model  # noqa: F401 (lib: fixture)

NEG = float("-inf")


def sparams(temperature, top_k, top_p, seed):
    """The vb_sample_params generate() writes (LlamaEngine.set_sampling)."""
    return ops.sample_params(max(float(temperature), 1e-6), 0 if not top_k else int(top_k),
                             1.0 if top_p is None else float(top_p), seed)


def literal_beam_sample(model, prompts, k, r, max_new, T, top_k, top_p, lp, es, eos, pad, seed):
    """4.31 beam_sample + BeamSearchScorer read literally, in float64: warpers on the cumulative scores, a draw of 2k
    without replacement per search (the exponential race of torch.multinomial, with the statement's Philox keys), the
    draws sorted by warped score, then the scorer; r searches per prompt, each returning its best hypothesis."""
    n_in = len(prompts[0])
    max_length = n_in + max_new
    S = len(prompts) * r
    seqs = [list(prompts[s // r]) for s in range(S) for _ in range(k)]
    scores = torch.zeros(S * k, dtype=torch.float64)       # beam_sample: torch.zeros((batch_size, num_beams))
    hyps = [LiteralHyps(k, lp, es, max_length) for _ in range(S)]
    done = [False] * S
    for step in range(max_new):
        cur_len = n_in + step
        logits = torch.tensor([model(s) for s in seqs], dtype=torch.float32).double()
        V = logits.shape[1]
        nts = torch.log_softmax(logits, -1) + scores[:, None]
        nts = nts.masked_fill(torch.isinf(nts.float() / T), NEG)     # fp32 scores: below the range is -inf
        # _get_logits_warper(num_beams > 1): TemperatureLogitsWarper, TopKLogitsWarper / TopPLogitsWarper with
        # min_tokens_to_keep = 2, applied to the running scores
        if T != 1.0:
            nts = nts / T
        if top_k:
            kk = min(max(top_k, 2), V)
            nts = nts.masked_fill(nts < torch.topk(nts, kk)[0][..., -1, None], NEG)
        if top_p is not None and top_p < 1.0:
            sl, si = torch.sort(nts, descending=False)
            cum = sl.softmax(dim=-1).cumsum(dim=-1)
            rm = cum <= (1 - top_p)
            rm[..., -2:] = 0
            nts = nts.masked_fill(rm.scatter(1, si, rm), NEG)
        flat = nts.view(S, k * V)
        logp = torch.log_softmax(flat, -1)         # log of softmax(next_token_scores): the multinomial's weights
        new_seqs, new_scores = [], []
        for b in range(S):
            if done[b]:
                new_seqs += [seqs[b * k] + [pad] for _ in range(k)]
                new_scores += [0.0] * k
                continue
            idx = torch.nonzero(logp[b] > NEG).flatten().numpy()
            key = logp[b, idx].numpy() + E.gumbel(seed, step, b, idx)
            drawn = [int(f) for f in idx[np.lexsort((idx, -key))][:2 * k]]
            top = sorted(((float(flat[b, f]), f) for f in drawn), key=lambda c: (-c[0], c[1]))
            nxt = []
            for rank, (sc, f) in enumerate(top):
                j, tok = divmod(f, V)
                if tok in eos:
                    if rank >= k:
                        continue
                    hyps[b].add(seqs[b * k + j], sc)
                else:
                    nxt.append((seqs[b * k + j] + [tok], sc))
                if len(nxt) == k:
                    break
            while len(nxt) < k:
                nxt.append((seqs[b * k + len(nxt)] + [pad], -1e9))
            new_seqs += [s for s, _ in nxt]
            new_scores += [s for _, s in nxt]
            done[b] = done[b] or hyps[b].is_done(top[0][0] if top else NEG, cur_len)
        seqs, scores = new_seqs, torch.tensor(new_scores, dtype=torch.float32).double()   # an fp32 tensor in 4.31
        if all(done):
            break
    out = []
    for b in range(S):
        if not done[b]:
            for j in range(k):
                hyps[b].add(seqs[b * k + j], float(scores[b * k + j]))
        out.append(sorted(hyps[b].beams, key=lambda x: x[0]).pop()[1])
    width = min(max(len(s) for s in out) + 1, max_length)
    res = torch.full((len(out), width), pad, dtype=torch.int64)
    for i, s in enumerate(out):
        res[i, :len(s)] = torch.tensor(s)
        if len(s) < width:
            res[i, len(s)] = eos[0] if eos else pad
    return res


def statement_sample_search(step_logits, prompt_ids, prompt_lens, k, r, max_new, lp, es, eos, pad, sprm):
    """vitron_b200.beam.beam_sample_advance driven over host buffers laid out as a LlamaEngine's (r searches per prompt),
    then finalize keeping each search's best. step_logits(running generated ids [R, t] or None) -> fp32 logits [R, V]
    (or [B, V] at step 0)."""
    B, n_in = prompt_ids.shape
    Bs = B * r
    R, S = Bs * k, max(prompt_lens) + max_new + 1
    z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt)
    st = dict(beam_score=torch.zeros(R), parent=z(R),
              done=z(R), beam_src=z(R, S), hyp_score=z(R, dt=torch.float64), hyp_len=z(R), hyp_seq=z(R),
              hyp_count=z(R), hyp_ids=z(R, S, dt=torch.int64))
    P = torch.tensor(prompt_lens, dtype=torch.int32).repeat_interleave(r * k)
    book = dict(next_src=z(R), positions=P - 1, kv_len=P.clone(), token_log=z(R, S, dt=torch.int64), prompt_len=P)
    prm = dict(length_penalty=lp, early_stopping=es, pad=pad, input_len=n_in, max_length=n_in + max_new, eos=eos)
    params = E.pack_params(lp, es, pad, n_in, n_in + max_new, eos)
    E.beam_sample_advance(step_logits(None).repeat_interleave(r * k, 0), k, params, sprm, **st, **book)
    t = 1
    while t < max_new and not bool(st["done"][:Bs].all()):
        E.beam_sample_advance(step_logits(E.running_ids(st["beam_src"], book["token_log"], P, t)), k, params, sprm, **st,
                              **book)
        t += 1
    hyps = []
    for b in range(Bs):
        h = E.Hypotheses(k, lp, es, n_in + max_new)
        h.slots = [dict(score=float(st["hyp_score"][b * k + s]), length=int(st["hyp_len"][b * k + s]),
                        seq=int(st["hyp_seq"][b * k + s]), ids=st["hyp_ids"][b * k + s, :int(st["hyp_len"][b * k + s]) - n_in])
                   for s in range(int(st["hyp_count"][b]))]
        hyps.append(h)
    gen = E.finalize(hyps, st["done"][:Bs].tolist(), st["beam_score"],
                     E.running_ids(st["beam_src"], book["token_log"], P, t), 1, prm)
    return torch.cat([prompt_ids.repeat_interleave(r, 0), gen], 1)


def smooth_model(V, seed):
    """Logits of a sequence: a seeded continuous function of the whole sequence (no ties)."""
    def f(seq):
        rnd = random.Random(hash((seed, tuple(seq))))
        return [rnd.gauss(0.0, 2.0) for _ in range(V)]
    return f


# T != 1 compounds into the carried scores; top_k = 1 and a tiny top_p exercise the 2 kept entries
WARPS = [(1.0, None, None), (0.5, None, None), (1.7, 5, 0.9), (1.0, 1, None), (0.8, None, 1e-4), (0.3, 3, 0.5)]


@pytest.mark.parametrize("T, top_k, top_p", WARPS)
@pytest.mark.parametrize("k, r, es, lp, eos", [(2, 1, False, 1.0, [3]), (3, 2, True, 2.0, [3, 5]),
                                               (4, 2, "never", 0.0, [1, 2, 6]), (2, 3, "never", 1.5, [4])])
def test_statement_matches_literal_beam_sample(T, top_k, top_p, k, r, es, lp, eos):
    V, max_new, pad = 11, 7, 0
    prompts = [[4, 7, 8], [8, 8, 1]]
    for seed in (1, 2 ** 40 + 7):
        model = smooth_model(V, seed)
        want = literal_beam_sample(model, prompts, k, r, max_new, T, top_k, top_p, lp, es, eos, pad, seed)
        ids = torch.tensor(prompts)

        def step(gen):
            if gen is None:
                return torch.tensor([model(p) for p in prompts])
            return torch.tensor([model(prompts[row // (r * k)] + gen[row].tolist()) for row in range(gen.shape[0])])
        got = statement_sample_search(step, ids, [3, 3], k, r, max_new, lp, es, eos, pad, sparams(T, top_k, top_p, seed))
        assert torch.equal(got, want), (seed, got.tolist(), want.tolist())


def test_temperature_compounds_into_the_carried_scores():
    """Warping the cumulative scores (4.31) is not warping each step's log-probs: beam scores carry a 1 / T per step."""
    V, k = 6, 2
    lg = torch.randn((k, V), generator=torch.Generator().manual_seed(0))
    bs = torch.tensor([-1.0, -2.5])
    w = E.warped_scores(lg, bs, 0.5)
    assert torch.allclose(w, (E.log_softmax64(lg) + bs.double()[:, None]) / 0.5)
    kept, _ = E.warp_kept(w, 1, 1.0)
    assert kept.sum(1).tolist() == [2, 2]                  # top_k = 1 keeps 2 with beams
    kept, _ = E.warp_kept(w, 0, 1e-9)
    assert kept.sum(1).tolist() == [2, 2]                  # so does a tiny top_p
    kept, _ = E.warp_kept(torch.full((1, V), NEG, dtype=torch.float64), 0, 1.0)
    assert not bool(kept.any())                            # -inf is never drawn


def _exact_child_pairs(p, w, k):
    """Exact distribution of the first two children of step 0: 2k draws without replacement from the k identical live
    rows (flat probabilities p / k, warped scores w per row), ranked by (w descending, flat index ascending):
    {(flat a, flat b): probability}."""
    V = len(p)
    pf, wf = np.tile(p, k) / k, np.tile(w, k)
    rank = np.empty(k * V, dtype=np.int64)
    rank[np.lexsort((np.arange(k * V), -wf))] = np.arange(k * V)
    perms = np.array(list(itertools.permutations(range(k * V), 2 * k)), dtype=np.int64)
    pr, left = np.ones(len(perms)), np.ones(len(perms))
    for c in range(2 * k):
        pr *= pf[perms[:, c]] / left
        left -= pf[perms[:, c]]
    order = np.argsort(rank[perms], axis=1)[:, :2]
    top = np.take_along_axis(perms, order, 1)
    codes, inv = np.unique(top[:, 0] * k * V + top[:, 1], return_inverse=True)
    sums = np.bincount(inv.ravel(), weights=pr)
    return {(int(c) // (k * V), int(c) % (k * V)): float(q) for c, q in zip(codes, sums)}


def chi_square_pvalue(counts, probs, n):
    """Pearson chi-square of observed counts against probabilities, categories with expected count < 5 pooled."""
    from scipy.stats import chisquare
    obs, exp, po, pe = [], [], 0, 0.0
    for c, pr in probs.items():
        if pr * n >= 5:
            obs.append(counts.get(c, 0))
            exp.append(pr * n)
        else:
            po += counts.get(c, 0)
            pe += pr * n
    assert not set(counts) - set(probs)
    if pe > 0:
        obs.append(po)
        exp.append(pe)
    exp = np.asarray(exp) * (sum(obs) / sum(exp))
    return chisquare(obs, exp).pvalue


def first_step_case():
    V, k, T = 16, 2, 0.7
    lg = torch.randn((1, V), generator=torch.Generator().manual_seed(5)) * 1.5
    w = (E.log_softmax64(lg)[0] / T).numpy()
    p = np.exp(w - w.max())
    return lg, V, k, T, w, p / p.sum()


def test_chi_square_of_the_statements_first_step_draws():
    """Step 0 (both beams at 0, identical rows): the children the statement picks over many seeds follow the exact
    without-replacement probabilities over the two live rows."""
    lg, V, k, T, w, p = first_step_case()
    exact = _exact_child_pairs(p, w, k)
    ws = E.warped_scores(lg.repeat(k, 1), torch.zeros(k), T)
    kept, _ = E.warp_kept(ws, 0, 1.0)
    n, counts = 8000, {}
    for seed in range(n):
        d, _ = E.sample_draws(ws, kept, k, 0, 0, seed)
        c = (d[0][1], d[1][1])
        counts[c] = counts.get(c, 0) + 1
    assert chi_square_pvalue(counts, exact, n) > 1e-3


def overflow_case():
    """Two searches (k = 2, V = 6, T = 0.2) whose carried scores leave the fp32 range this step: search 0 entirely,
    search 1 in beam 0 only. Returns (logits, state, params, sample params)."""
    k, V, P, t = 2, 6, 4, 3
    R = 2 * k
    lg = torch.randn((R, V), generator=torch.Generator().manual_seed(2))
    z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt)
    st = dict(beam_score=torch.tensor([-1e38, -2e38, -3e38, -4.0]), parent=z(R), done=z(R), beam_src=z(R, 12),
              hyp_score=z(R, dt=torch.float64), hyp_len=z(R), hyp_seq=z(R), hyp_count=z(R), hyp_ids=z(R, 12, dt=torch.int64),
              next_src=z(R), positions=torch.full((R,), P + t - 1, dtype=torch.int32),
              kv_len=torch.full((R,), P + t, dtype=torch.int32), token_log=z(R, 12, dt=torch.int64),
              prompt_len=torch.full((R,), P, dtype=torch.int32))
    for r in range(R):
        st["beam_src"][r, P:P + t + 1] = r
    return lg, st, E.pack_params(1.0, False, 0, P, P + 8, [-1]), sparams(0.2, None, None, 9)


def test_scores_beyond_fp32_continue_with_pad():
    """Temperature compounds: scores that leave the fp32 range are -inf. A search with no entry above -inf has no
    draws, and its beams continue their own rows with pad and score -1e9 (4.31 raises there); a search with one such
    beam draws from its live row."""
    lg, st, prm, sp = overflow_case()
    E.beam_sample_advance(lg, 2, prm, sp, **st)
    assert st["parent"][:2].tolist() == [0, 1] and st["next_src"][:2].tolist() == [0, 0]
    assert st["beam_score"][:2].tolist() == [-1e9, -1e9] and st["token_log"][:2, 3].tolist() == [0, 0]
    assert st["parent"][2:].tolist() == [3, 3] and bool((st["beam_score"][2:] > -30).all())
    assert int(st["done"][0]) == 0 and st["kv_len"].tolist() == [8] * 4
    assert bool(torch.isinf(E.warped_scores(lg, torch.tensor([-1e38] * 4), 0.2)).all())


def test_beam_sample_advance_argument_validation_without_device(lib):
    import ctypes as C
    buf = (C.c_uint8 * (1 << 16))()
    p = C.addressof(buf)
    p += (-p) % 16
    ERR_ARG, ERR_WS, ERR_UNSUP = -1, -3, -4
    ws = lib.vb200_beam_workspace_size(8)
    assert ws >= 16384 + 8 * 32 * 12

    def call(logits=p, ld=64, B=2, k=4, n=64, params=p, sprm=p, token_log=p, workspace=p, wsb=ws, done=p, src_ld=64):
        return lib.vb200_beam_sample_advance(logits, ld, B, k, n, params, p, p, done, p, src_ld, p, p, p, p, p, 64, p, p,
                                             p, token_log, 64, p, workspace, wsb, sprm, None)
    assert call(sprm=None) == ERR_ARG
    assert call(logits=None) == ERR_ARG and call(params=None) == ERR_ARG and call(done=None) == ERR_ARG
    assert call(token_log=None) == ERR_ARG and call(B=0) == ERR_ARG and call(k=0) == ERR_ARG
    assert call(n=1, ld=1) == ERR_ARG and call(ld=32) == ERR_ARG and call(src_ld=0) == ERR_ARG
    assert call(k=17) == ERR_UNSUP and call(n=49153, ld=49153) == ERR_UNSUP and call(B=4097, k=1) == ERR_UNSUP
    assert call(workspace=None) == ERR_WS and call(wsb=ws - 1) == ERR_WS


def test_beam_sample_advance_wrapper_checks(lib):
    """ops.beam_sample_advance checks every state buffer as ops.beam_advance does, and the sampling buffer."""
    R, k, S = 4, 2, 16
    i32 = lambda n=R: torch.zeros(n, dtype=torch.int32)
    state = dict(beam_score=torch.zeros(R), parent=i32(), done=i32(), beam_src=torch.zeros((R, S), dtype=torch.int32),
                 hyp_score=torch.zeros(R, dtype=torch.float64), hyp_len=i32(), hyp_seq=i32(), hyp_count=i32(),
                 hyp_ids=torch.zeros((R, S), dtype=torch.int64), next_src=i32(), positions=i32(), kv_len=i32(),
                 token_log=torch.zeros((R, S), dtype=torch.int64), prompt_len=i32())
    logits, prm, sp = torch.zeros((R, 8)), E.pack_params(1.0, False, 0, 3, 9, [2]), sparams(1.0, None, None, 0)
    for name, t in dict(beam_score=torch.zeros(R, dtype=torch.float64), done=i32(R - 1),
                        beam_src=torch.zeros((R, S), dtype=torch.int64), prompt_len=torch.zeros(R, dtype=torch.int16)).items():
        with pytest.raises(ValueError, match=name):
            ops.beam_sample_advance(logits, k, prm, sp, **dict(state, **{name: t}))
    with pytest.raises(ValueError, match="sample_params"):
        ops.beam_sample_advance(logits, k, prm, sp[:16], **state)
    with pytest.raises(ValueError, match="sample_params"):
        ops.beam_sample_advance(logits, k, prm, sp.view(torch.int32), **state)


def _generate(model, ids, seed, **kw):
    torch.manual_seed(seed)
    return model.generate(ids, do_sample=True, **kw)


@pytest.mark.parametrize("k, r, T, top_k, top_p, es, lp", [(2, 1, 1.0, None, None, False, 1.0),
                                                           (3, 2, 0.6, 4, 0.9, True, 2.0),
                                                           (2, 3, 1.3, 1, None, "never", 0.5)])
def test_beam_sample_generate_matches_a_statement_search(monkeypatch, k, r, T, top_k, top_p, es, lp):
    """generate(do_sample=True, num_beams=k, num_return_sequences=r) on a CPU engine (one prefill, prompt pages forked
    to r * k rows, graph-less beam-sampling steps) equals the statement driven over the same engine's logits, with the
    seed generate draws from torch's CPU generator; it is reproducible under torch.manual_seed and independent of
    sync_every."""
    model, fx, _ = tiny_model(monkeypatch, max_batch=12)
    ids = _ids(2, 9, 4, fx["llm"]["vocab_size"])
    n = 6
    kw = dict(num_beams=k, num_return_sequences=r, temperature=T, top_k=top_k, top_p=top_p, early_stopping=es,
              length_penalty=lp, max_new_tokens=n, eos_token_id=-1)
    runs = [_generate(model, ids, 11, sync_every=s, **kw) for s in (4, 1)]
    assert torch.equal(runs[0], runs[1])
    torch.manual_seed(11)
    seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64)) & (2 ** 64 - 1)
    want = statement_sample_search(engine_logits_fn(model, ids), ids, [9, 9], k, r, n, lp, es, [-1], 0,
                                   sparams(T, top_k, top_p, seed))
    assert runs[0].shape == want.shape == (2 * r, 9 + n)
    assert torch.equal(runs[0], want), (runs[0].tolist(), want.tolist())
    if top_k != 1:   # (top_k = 1 keeps 2 entries per row: the 2k draws are the whole kept set, whatever the seed)
        assert not torch.equal(_generate(model, ids, 12, **kw), runs[0])   # another seed, another sample


def test_beam_sample_generate_eos_criteria_and_errors(monkeypatch):
    """EOS hypotheses end with EOS then pad and match the statement; stopping_criteria sees the running beams of all
    B * r searches; B * r * k rows over max_batch is a ValueError; greedy / beam / sampled calls are unchanged."""
    model, fx, _ = tiny_model(monkeypatch)
    ids = _ids(2, 7, 9, fx["llm"]["vocab_size"])
    base = _generate(model, ids, 3, num_beams=2, num_return_sequences=2, max_new_tokens=8, eos_token_id=-1)
    eos = int(base[0, 7 + 1])
    got = _generate(model, ids, 3, num_beams=2, num_return_sequences=2, max_new_tokens=8, eos_token_id=eos,
                    pad_token_id=0, sync_every=3)
    torch.manual_seed(3)
    seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64)) & (2 ** 64 - 1)
    want = statement_sample_search(engine_logits_fn(model, ids), ids, [7, 7], 2, 2, 8, 1.0, False, [eos], 0,
                                   sparams(1.0, None, None, seed))
    assert torch.equal(got, want)
    seen = []

    def crit(seq, scores):
        seen.append(tuple(seq.shape))
        return seq.shape[1] >= 7 + 3
    out = _generate(model, ids, 3, num_beams=2, num_return_sequences=2, max_new_tokens=8, eos_token_id=-1,
                    stopping_criteria=crit)
    assert seen[0] == (8, 8) and seen[-1] == (8, 10) and out.shape == (4, 7 + 4)
    with pytest.raises(ValueError, match="max_batch"):
        _generate(model, ids, 0, num_beams=3, num_return_sequences=2, max_new_tokens=4)
    greedy = model.generate(ids, max_new_tokens=5, eos_token_id=-1)
    assert torch.equal(model.generate(ids, num_beams=1, max_new_tokens=5, eos_token_id=-1), greedy)
    sampled = _generate(model, ids, 5, num_beams=1, max_new_tokens=5, eos_token_id=-1, temperature=0.7)
    assert torch.equal(_generate(model, ids, 5, max_new_tokens=5, eos_token_id=-1, temperature=0.7), sampled)


def test_beam_sample_steps_need_start_beam():
    from vitron_b200.llama import LlamaEngine
    eng = LlamaEngine(dict(hidden_size=16, intermediate_size=32, num_hidden_layers=1, num_attention_heads=2, vocab_size=10),
                      "cpu", max_batch=2, max_seq_len=64)
    with pytest.raises(RuntimeError, match="start_beam"):
        eng.decode_steps(2, 1, sampled="beam_sample")


def test_gumbel_noise_layout():
    """U = (2 * (x >> 9) + 1) * 2^-24 lies in (0, 1); word f % 4 of counter (t, b, f // 4, 1)."""
    from vitron_b200.sampling import philox4x32_10
    f = np.arange(12)
    g = E.gumbel(77, 3, 5, f)
    x = philox4x32_10([3, 5, 2, 1], [77, 0])[1]       # flat index 9 = word 1 of group 2
    u = (2.0 * (int(x) >> 9) + 1.0) * 2.0 ** -24
    assert 0.0 < u < 1.0 and g[9] == -math.log(-math.log(u))
    assert np.isfinite(g).all() and len(set(g.tolist())) == 12
