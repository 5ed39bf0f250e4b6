"""CPU (no GPU): the fp32 statement of the logits processors (vitron_b200/processors.py) against a literal restatement of
HF transformers 4.31's processors and against the installed transformers classes, its two stated divergences, the
argument checks of vb200_logits_process / ops.logits_process without a device, and generate(repetition_penalty=...,
no_repeat_ngram_size=..., min_length=..., min_new_tokens=...) on a CPU engine in all four decoding modes against a
4.31-style loop over the same engine's logits."""
import functools

import numpy as np
import pytest
import torch

from vitron_b200 import beam as BE
from vitron_b200 import ops
from vitron_b200 import processors as E
from vitron_b200 import sampling
from tests.test_beam_cpu import _ids, engine_logits_fn, lib, statement_search, tiny_model  # noqa: F401 (lib: fixture)
from tests.test_beam_sample_cpu import sparams, statement_sample_search

INF = float("inf")


# ------------------------------------------------------------------ transformers 4.31, read literally
def _get_ngrams(ngram_size, prev_input_ids, num_hypos):
    generated_ngrams = [{} for _ in range(num_hypos)]
    for idx in range(num_hypos):
        gen_tokens = prev_input_ids[idx].tolist()
        generated_ngram = generated_ngrams[idx]
        for ngram in zip(*[gen_tokens[i:] for i in range(ngram_size)]):
            prev_ngram_tuple = tuple(ngram[:-1])
            generated_ngram[prev_ngram_tuple] = generated_ngram.get(prev_ngram_tuple, []) + [ngram[-1]]
    return generated_ngrams


def _get_generated_ngrams(banned_ngrams, prev_input_ids, ngram_size, cur_len):
    start_idx = cur_len + 1 - ngram_size
    ngram_idx = tuple(prev_input_ids[start_idx:cur_len].tolist())
    return banned_ngrams.get(ngram_idx, [])


def _calc_banned_ngram_tokens(ngram_size, prev_input_ids, num_hypos, cur_len):
    if cur_len + 1 < ngram_size:
        return [[] for _ in range(num_hypos)]
    generated_ngrams = _get_ngrams(ngram_size, prev_input_ids, num_hypos)
    return [_get_generated_ngrams(generated_ngrams[i], prev_input_ids[i], ngram_size, cur_len) for i in range(num_hypos)]


def literal_431(input_ids, scores, input_len, repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0,
                min_new_tokens=0, eos=()):
    """_get_logits_processor's list applied in order: RepetitionPenalty, NoRepeatNGram, MinLength, MinNewTokensLength."""
    scores = scores.clone()
    if repetition_penalty is not None and repetition_penalty != 1.0:
        score = torch.gather(scores, 1, input_ids)
        score = torch.where(score < 0, score * repetition_penalty, score / repetition_penalty)
        scores.scatter_(1, input_ids, score)
    if no_repeat_ngram_size is not None and no_repeat_ngram_size > 0:
        banned = _calc_banned_ngram_tokens(no_repeat_ngram_size, input_ids, scores.shape[0], input_ids.shape[-1])
        for i, banned_tokens in enumerate(banned):
            scores[i, banned_tokens] = -INF
    if min_length > 0 and eos:
        if input_ids.shape[-1] < min_length:
            for i in eos:
                scores[:, i] = -INF
    if min_new_tokens > 0 and eos:
        if input_ids.shape[-1] - input_len < min_new_tokens:
            for i in eos:
                scores[:, i] = -INF
    return scores


def assert_same_scores(got, want):
    """Same -inf entries exactly; elsewhere within one fp32 rounding (4.31 divides by a Python scalar, which torch may
    evaluate as a multiplication by its reciprocal; the statement divides with correct rounding)."""
    assert torch.equal(torch.isneginf(got), torch.isneginf(want))
    fin = torch.isfinite(want)
    torch.testing.assert_close(got[fin], want[fin], rtol=1.2e-7, atol=0)


def run_statement(scores, prompt, gen, **settings):
    """processors.process over host buffers laid out as an engine's: prompt [R, n_in], gen [R, t]."""
    R, n_in = prompt.shape
    t = gen.shape[1]
    eos = settings.pop("eos", ())
    token_log = torch.zeros((R, t + 4), dtype=torch.int64)
    token_log[:, :t] = gen
    P = torch.full((R,), 50, dtype=torch.int32)
    prm = E.pack_params(input_len=n_in, eos_ids=eos, **settings)
    out = scores.clone()
    if t == 0:
        return E.process(out, prm, prompt.to(torch.int32))
    return E.process(out, prm, prompt.to(torch.int32), token_log=token_log, kv_len=P + t, prompt_len=P)


SETTINGS = [dict(repetition_penalty=1.3), dict(repetition_penalty=0.7), dict(no_repeat_ngram_size=1),
            dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=3), dict(no_repeat_ngram_size=9),
            dict(min_length=12, eos=[2, 5, 7]), dict(min_new_tokens=3, eos=[5, 2]),
            dict(repetition_penalty=1.2, no_repeat_ngram_size=2, min_length=10, min_new_tokens=2, eos=[1, 3])]


@pytest.mark.parametrize("settings", SETTINGS, ids=lambda s: "-".join(f"{k}{v}" for k, v in s.items()))
@pytest.mark.parametrize("t", [0, 1, 4])
def test_statement_matches_literal_431(settings, t):
    """Each processor alone and combined, on histories with repeated ids and n-grams (a small vocabulary), raw fp32
    logits and log-probabilities; t = 0 is the first generated token, cur_len + 1 < n the n-gram boundary."""
    g = torch.Generator().manual_seed(t)
    V, R, n_in = 11, 6, 7
    for trial in range(4):
        prompt = torch.randint(0, V, (R, n_in), generator=g)
        gen = torch.randint(0, V, (R, t), generator=g)
        scores = torch.randn((R, V), generator=g) * 3
        if trial == 3:
            scores = BE.log_softmax64(scores).float()
        ids = torch.cat([prompt, gen], 1)
        s = dict(settings)
        want = literal_431(ids, scores, n_in, eos=s.get("eos", ()), **{k: v for k, v in s.items() if k != "eos"})
        got = run_statement(scores, prompt, gen, **s)
        assert_same_scores(got, want)


def test_ngram_boundary_and_sizes():
    """cur_len + 1 < n bans nothing; n = cur_len + 1 matches an empty set of windows; n = 1 bans the whole history."""
    h = [4, 1, 4, 1, 4]
    assert E.banned_ngram_tokens(h, 7) == [] and E.banned_ngram_tokens(h, 6) == []
    assert sorted(set(E.banned_ngram_tokens(h, 1))) == [1, 4]
    assert E.banned_ngram_tokens(h, 2) == [1, 1]          # 4 was followed by 1 twice
    assert E.banned_ngram_tokens(h, 3) == [1]             # the last 2-gram (1, 4) was followed by 1
    for n in range(1, 8):
        want = _calc_banned_ngram_tokens(n, torch.tensor([h]), 1, len(h))[0]
        assert E.banned_ngram_tokens(h, n) == want


def test_repetition_penalty_applies_once_per_distinct_id():
    row = np.array([2.0, -2.0, 3.0, 0.0], dtype=np.float32)
    E.penalize(row, [0, 0, 0, 1, 1, 3], 2.0)
    assert row.tolist() == [1.0, -4.0, 3.0, 0.0]
    row = np.array([1.0, 1.0, 1.0], dtype=np.float32)
    E.penalize(row, [1], 3.0)
    assert row[1] == np.float32(1.0) / np.float32(3.0)     # correctly rounded division


def test_statement_matches_installed_transformers():
    """The transformers classes installed here (without sentinels in the history)."""
    lp = pytest.importorskip("transformers.generation.logits_process")
    g = torch.Generator().manual_seed(3)
    V, R, n_in, t = 13, 5, 6, 5
    prompt = torch.randint(0, V, (R, n_in), generator=g)
    gen = torch.randint(0, V, (R, t), generator=g)
    ids = torch.cat([prompt, gen], 1)
    scores = torch.randn((R, V), generator=g) * 2

    def mk(cls, *a):
        try:
            return cls(*a)
        except TypeError:
            return cls(*a, device="cpu")
    cases = [(dict(repetition_penalty=1.4), [lp.RepetitionPenaltyLogitsProcessor(1.4)]),
             (dict(no_repeat_ngram_size=2), [lp.NoRepeatNGramLogitsProcessor(2)]),
             (dict(no_repeat_ngram_size=1), [lp.NoRepeatNGramLogitsProcessor(1)]),
             (dict(min_length=n_in + t + 1, eos=[3, 8]), [mk(lp.MinLengthLogitsProcessor, n_in + t + 1, [3, 8])]),
             (dict(min_new_tokens=t + 1, eos=[4]), [mk(lp.MinNewTokensLengthLogitsProcessor, n_in, t + 1, [4])]),
             (dict(min_new_tokens=t, eos=[4]), [mk(lp.MinNewTokensLengthLogitsProcessor, n_in, t, [4])])]
    for settings, procs in cases:
        want = scores.clone()
        for p in procs:
            want = p(ids, want)
        assert_same_scores(run_statement(scores, prompt, gen, **settings), want)


def test_divergences_on_sentinels():
    """4.31's gather raises on the -200 image sentinel, and its n-gram ban wraps it to V - 200; the statement skips the
    sentinel in the penalty and never bans it, while matching it like any other id."""
    V = 300
    prompt = torch.tensor([[1, -200, 5, 7, -200]])
    gen = torch.tensor([[9]])
    ids = torch.cat([prompt, gen], 1)
    scores = torch.randn((1, V), generator=torch.Generator().manual_seed(0))
    with pytest.raises((RuntimeError, IndexError)):
        literal_431(ids, scores, 5, repetition_penalty=1.5)
    got = run_statement(scores, prompt, gen, repetition_penalty=1.5)
    changed = torch.nonzero(got[0] != scores[0]).flatten().tolist()
    assert changed == [1, 5, 7, 9]
    prompt2 = torch.tensor([[5, -200, 7, 5]])
    lit2 = literal_431(prompt2, scores, 4, no_repeat_ngram_size=2)
    assert bool(torch.isneginf(lit2[0, V - 200]))                       # 5 was followed by -200
    got2 = run_statement(scores, prompt2, torch.zeros((1, 0), dtype=torch.long), no_repeat_ngram_size=2)
    assert torch.isneginf(got2[0]).sum() == 0                            # the sentinel is never banned
    prompt3 = torch.tensor([[-200, 5, 6, -200]])
    got3 = run_statement(scores, prompt3, torch.zeros((1, 0), dtype=torch.long), no_repeat_ngram_size=2)
    assert torch.nonzero(torch.isneginf(got3[0])).flatten().tolist() == [5]   # matched through the sentinel


def test_check_settings_follows_431():
    on = lambda **kw: E.check_settings(**kw)[1]
    assert not on() and not on(repetition_penalty=None) and not on(no_repeat_ngram_size=-3)
    assert not on(min_length=5) and not on(min_new_tokens=5)            # no EOS id: not added
    assert on(min_length=5, eos_ids=[2]) and on(repetition_penalty=1.01) and on(no_repeat_ngram_size=1)
    for kw in (dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=2),
               dict(no_repeat_ngram_size=2.0), dict(min_length=2.5, eos_ids=[1]), dict(min_new_tokens=1.5, eos_ids=[1])):
        with pytest.raises(ValueError):
            E.check_settings(**kw)
    with pytest.raises(ValueError, match="EOS"):
        E.pack_params(eos_ids=list(range(9)))
    buf = E.pack_params(1.5, 3, 7, 2, 11, [4, 9])
    assert buf.numel() == 56 and E.unpack_params(buf) == dict(repetition_penalty=1.5, no_repeat_ngram_size=3,
                                                              min_length=7, min_new_tokens=2, input_len=11, eos=[4, 9])


# ------------------------------------------------------------------ C entry point and wrapper without a device
def test_logits_process_argument_validation_without_device(lib):
    import ctypes as C
    buf = (C.c_uint8 * (1 << 16))()
    p = C.addressof(buf)
    p += (-p) % 16
    ERR_ARG, ERR_UNSUP = -1, -4

    def call(logits=p, ld=64, rows=2, n=64, params=p, prompt=p, prompt_ld=64, token_log=p, log_stride=64, beam_src=None,
             src_ld=0, kv_len=p, prompt_len=p, logprobs=0):
        return lib.vb200_logits_process(logits, ld, rows, n, params, prompt, prompt_ld, token_log, log_stride, beam_src,
                                        src_ld, kv_len, prompt_len, logprobs, None)
    assert call(logits=None) == ERR_ARG and call(params=None) == ERR_ARG and call(prompt=None) == ERR_ARG
    assert call(rows=0) == ERR_ARG and call(n=0) == ERR_ARG and call(ld=32) == ERR_ARG and call(prompt_ld=0) == ERR_ARG
    assert call(kv_len=None) == ERR_ARG and call(prompt_len=None) == ERR_ARG     # both or neither
    assert call(token_log=None) == ERR_ARG and call(log_stride=0) == ERR_ARG
    assert call(beam_src=p, src_ld=0) == ERR_ARG and call(beam_src=p, src_ld=64, kv_len=None, prompt_len=None) == ERR_ARG
    assert call(n=49153, ld=49153) == ERR_UNSUP
    assert call(prompt_ld=4096, log_stride=4097) == ERR_UNSUP


def test_logits_process_wrapper_checks(lib):
    R, S = 4, 16
    logits, prm = torch.zeros((R, 8)), E.pack_params(1.5)
    prompt = torch.zeros((R, S), dtype=torch.int32)
    i32 = torch.zeros(R, dtype=torch.int32)
    tl = torch.zeros((R, S), dtype=torch.int64)
    for kw, match in ((dict(params=prm[:40]), "params"), (dict(params=prm.view(torch.int32)), "params"),
                      (dict(prompt_ids=prompt.long()), "prompt_ids"), (dict(prompt_ids=prompt[:2]), "prompt_ids"),
                      (dict(kv_len=i32), "prompt_len"), (dict(kv_len=i32, prompt_len=i32.long()), "prompt_len"),
                      (dict(kv_len=i32, prompt_len=i32, token_log=tl.int()), "token_log"),
                      (dict(kv_len=i32, prompt_len=i32, token_log=tl, beam_src=tl), "beam_src"),
                      (dict(logits=logits.double()), "fp32")):
        args = dict(dict(logits=logits, params=prm, prompt_ids=prompt), **kw)
        with pytest.raises(ValueError, match=match):
            ops.logits_process(**args)


# ------------------------------------------------------------------ generate on a CPU engine
PROC = dict(repetition_penalty=1.8, no_repeat_ngram_size=2, min_new_tokens=3)


def _proc_step(step_logits, ids, settings, eos, logprobs, k=1):
    """The reference's logits: the engine's full-recompute logits of every running sequence, through the literal 4.31
    processors on input_ids = prompt + generated ids (after log_softmax in the beam modes)."""
    n_in = ids.shape[1]

    def step(gen):
        raw = step_logits(gen)
        rows = BE.log_softmax64(raw).float() if logprobs else raw.float()
        run = ids if gen is None else torch.cat([ids.repeat_interleave(gen.shape[0] // ids.shape[0], 0), gen], 1)
        return literal_431(run, rows, n_in, eos=eos, **settings)
    return step


def _greedy_or_sample_reference(model, ids, n, settings, eos, sprm=None):
    step = _proc_step(engine_logits_fn(model, ids), ids, settings, eos, False)
    gen = None
    for t in range(n):
        scores = step(gen)
        if sprm is None:
            tok = torch.argmax(scores, -1)
        else:
            T, top_k, top_p, _, seed = ops.SAMPLE_PARAMS.unpack(sprm.numpy().tobytes())
            tok, _ = sampling.sample_reference(scores, T, top_k, top_p, seed, t)
        gen = tok[:, None] if gen is None else torch.cat([gen, tok[:, None]], 1)
    return torch.cat([ids, gen], 1)


def _seed(s):
    torch.manual_seed(s)
    return int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64)) & (2 ** 64 - 1)


def _finished(seq, n_in, eos, pad):
    """generate's output of a full-length run: pad after each row's first EOS, cut after the last row's first EOS when
    every row has one."""
    out, ends = seq.clone(), []
    for row in out:
        hit = [j for j in range(n_in, row.shape[0]) if int(row[j]) in eos]
        ends.append(hit[0] if hit else None)
        if hit:
            row[hit[0] + 1:] = pad
    return out if None in ends else out[:, :max(ends) + 1]


@pytest.mark.parametrize("settings", [PROC, dict(repetition_penalty=0.6, no_repeat_ngram_size=1),
                                      dict(no_repeat_ngram_size=3, min_length=13)])
def test_greedy_and_sampled_generate_match_a_431_loop(monkeypatch, settings):
    """EOS is the first token the unprocessed greedy call picks for row 0, so the minimum-length rules change the
    output; the reference runs every step and then pads after EOS as generate does."""
    model, fx, _ = tiny_model(monkeypatch)
    V = fx["llm"]["vocab_size"]
    ids = _ids(2, 9, 4, V)
    n = 7
    eos = [int(model.generate(ids, max_new_tokens=1, eos_token_id=-1)[0, 9]), 2]
    got = model.generate(ids, max_new_tokens=n, eos_token_id=eos, pad_token_id=0, sync_every=3, **settings)
    want = _finished(_greedy_or_sample_reference(model, ids, n, settings, eos), 9, eos, 0)
    assert torch.equal(got, want), (got.tolist(), want.tolist())
    if settings.get("no_repeat_ngram_size") == 1:
        for r in got.tolist():
            assert len(set(r[9:])) == len(r) - 9 and not set(r[9:]) & set(r[:9])
    torch.manual_seed(7)
    got_s = model.generate(ids, do_sample=True, temperature=0.8, top_k=20, max_new_tokens=n, eos_token_id=eos,
                           pad_token_id=0, **settings)
    want_s = _greedy_or_sample_reference(model, ids, n, settings, eos, sparams(0.8, 20, None, _seed(7)))
    assert torch.equal(got_s, _finished(want_s, 9, eos, 0)), (got_s.tolist(), want_s.tolist())


def test_processors_do_not_leak_between_calls(monkeypatch):
    model, fx, _ = tiny_model(monkeypatch)
    ids = _ids(2, 9, 4, fx["llm"]["vocab_size"])
    plain = model.generate(ids, max_new_tokens=6, eos_token_id=-1)
    pen = model.generate(ids, max_new_tokens=6, eos_token_id=-1, repetition_penalty=3.0, no_repeat_ngram_size=1)
    assert not torch.equal(plain, pen)
    assert torch.equal(model.generate(ids, max_new_tokens=6, eos_token_id=-1), plain)
    assert not model.engine.proc_on


@pytest.mark.parametrize("sample", [False, True])
def test_beam_generate_matches_a_431_loop(monkeypatch, sample):
    """Beam search / beam sampling: the processors act on log_softmax before the beam scores are added, at every step
    including the first; the reference drives the beam statement over literally processed log-probabilities."""
    model, fx, _ = tiny_model(monkeypatch, max_batch=12)
    V = fx["llm"]["vocab_size"]
    ids = _ids(2, 9, 4, V)
    n, k, r = 6, 3, 2
    settings = dict(repetition_penalty=1.5, no_repeat_ngram_size=2, min_length=9 + 3)
    eos = [int(_ids(2, 9, 4, V)[1, 2])]
    kw = dict(num_beams=k, max_new_tokens=n, eos_token_id=eos, pad_token_id=0, **settings)
    if sample:
        kw.update(do_sample=True, num_return_sequences=r, temperature=0.9)
        torch.manual_seed(5)
    got = model.generate(ids, **kw)
    step = _proc_step(engine_logits_fn(model, ids), ids, settings, eos, True)
    monkeypatch.setattr(BE, "beam_advance", functools.partial(BE.beam_advance, logprobs=True))
    monkeypatch.setattr(BE, "beam_sample_advance", functools.partial(BE.beam_sample_advance, logprobs=True))
    if sample:
        want = statement_sample_search(step, ids, [9, 9], k, r, n, 1.0, False, eos, 0, sparams(0.9, None, None, _seed(5)))
    else:
        want = statement_search(step, ids, [9, 9], k, n, 1.0, False, eos, 0, 1)
    assert torch.equal(got, want), (got.tolist(), want.tolist())


def test_generate_argument_validation(monkeypatch):
    model, fx, _ = tiny_model(monkeypatch)
    ids = _ids(1, 5, 4, fx["llm"]["vocab_size"])
    for kw in (dict(repetition_penalty=0.0), dict(repetition_penalty=2), dict(no_repeat_ngram_size=2.0),
               dict(min_new_tokens=1.5, eos_token_id=2), dict(min_length=3.0, eos_token_id=2)):
        with pytest.raises(ValueError):
            model.generate(ids, max_new_tokens=2, **kw)
    # disabled by 4.31's rules: no error, no processors
    out = model.generate(ids, max_new_tokens=3, eos_token_id=-1, repetition_penalty=None, no_repeat_ngram_size=-1)
    assert out.shape == (1, 8) and not model.engine.proc_on
