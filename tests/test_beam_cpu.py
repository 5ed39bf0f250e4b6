"""CPU (no GPU): the float64 statement of the beam step (vitron_b200/beam.py) against a literal HF-4.31-style beam search,
argument validation of vb200_beam_advance / vb200_attn_decode_rope_beam, and the host logic of generate(num_beams=k) on a
CPU engine (kernels replaced by torch statements; the beam-indirect attention by the one below) against beam searches
driven directly over the oracle's LlamaCPU and installed transformers."""
import heapq
import math
import os
import random

import pytest
import torch

from vitron_b200 import beam as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16 = torch.bfloat16


# ------------------------------------------------------------------ the statement against a literal search
class LiteralHyps:
    """transformers 4.31 BeamHypotheses, as a list in insertion order."""

    def __init__(self, k, lp, es, max_length):
        self.k, self.lp, self.es, self.max_length, self.beams, self.worst = k, lp, es, max_length, [], 1e9

    def add(self, hyp, s):
        score = s / (len(hyp) ** self.lp)
        if len(self.beams) < self.k or score > self.worst:
            self.beams.append((score, list(hyp)))
            if len(self.beams) > self.k:
                ranked = sorted([(sc, i) for i, (sc, _) in enumerate(self.beams)])
                del self.beams[ranked[0][1]]
                self.worst = ranked[1][0]
            else:
                self.worst = min(score, self.worst)

    def is_done(self, best, cur_len):
        if len(self.beams) < self.k:
            return False
        if self.es is True:
            return True
        if self.es is False or self.lp <= 0.0:
            return self.worst >= best / cur_len ** self.lp
        return self.worst >= best / self.max_length ** self.lp


def literal_search(model, prompts, k, max_new, lp, es, eos, pad, nrs):
    """4.31 beam_search + BeamSearchScorer read literally: Python floats, heapq over every (beam, token) candidate."""
    n_in = len(prompts[0])
    max_length = n_in + max_new
    seqs = [list(p) for p in prompts for _ in range(k)]
    scores = [0.0 if j == 0 else -1e9 for _ in prompts for j in range(k)]
    hyps = [LiteralHyps(k, lp, es, max_length) for _ in prompts]
    done = [False] * len(prompts)
    for step in range(max_new):
        cur_len = n_in + step
        new_seqs, new_scores = [], []
        for b in range(len(prompts)):
            if done[b]:
                new_seqs += [seqs[b * k] + [pad] for _ in range(k)]
                new_scores += [0.0] * k
                continue
            cand = []
            for j in range(k):
                row = model(seqs[b * k + j])
                logz = math.log(sum(math.exp(v - max(row)) for v in row)) + max(row)
                for tok, v in enumerate(row):
                    cand.append((-(v - logz + scores[b * k + j]), j * len(row) + tok))
            top = heapq.nsmallest(2 * k, cand)
            nxt = []
            for rank, (neg, flat) in enumerate(top):
                j, tok = divmod(flat, len(row))
                if tok in eos:
                    if rank >= k:
                        continue
                    hyps[b].add(seqs[b * k + j], -neg)
                else:
                    nxt.append((seqs[b * k + j] + [tok], -neg))
                if len(nxt) == k:
                    break
            while len(nxt) < k:   # 4.31 raises here; the stated rule continues the beam's own row with pad
                nxt.append((seqs[b * k + len(nxt)] + [pad], -1e9))
            new_seqs += [s for s, _ in nxt]
            new_scores += [s for _, s in nxt]
            done[b] = done[b] or hyps[b].is_done(-top[0][0], cur_len)
        seqs, scores = new_seqs, new_scores
        if all(done):
            break
    out = []
    for b in range(len(prompts)):
        if not done[b]:
            for j in range(k):
                hyps[b].add(seqs[b * k + j], scores[b * k + j])
        ranked = sorted(hyps[b].beams, key=lambda x: x[0])
        out += [ranked.pop()[1] for _ in range(nrs)]
    width = min(max(len(s) for s in out) + 1, max_length)
    res = torch.full((len(out), width), pad, dtype=torch.int64)
    for i, s in enumerate(out):
        res[i, :len(s)] = torch.tensor(s)
        if len(s) < width:
            res[i, len(s)] = eos[0]
    return res


def statement_search(step_logits, prompt_ids, prompt_lens, k, max_new, lp, es, eos, pad, nrs):
    """The beam step of vitron_b200.beam driven over host buffers laid out as a LlamaEngine's, then finalize.
    step_logits(running generated ids [R, t] or None for step 0) -> fp32 logits [R, V] (or [B, V] at step 0)."""
    B, n_in = prompt_ids.shape
    R, S = B * k, max(prompt_lens) + max_new + 1
    z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt)
    st = dict(beam_score=torch.tensor([0.0 if j == 0 else -1e9 for _ in range(B) for j in range(k)]), parent=z(R),
              done=z(R), beam_src=z(R, S), hyp_score=z(R, dt=torch.float64), hyp_len=z(R), hyp_seq=z(R),
              hyp_count=z(R), hyp_ids=z(R, S, dt=torch.int64))
    P = torch.tensor(prompt_lens, dtype=torch.int32).repeat_interleave(k)
    book = dict(next_src=z(R), positions=P - 1, kv_len=P.clone(), token_log=z(R, S, dt=torch.int64), prompt_len=P)
    prm = dict(length_penalty=lp, early_stopping=es, pad=pad, input_len=n_in, max_length=n_in + max_new, eos=eos)
    params = E.pack_params(lp, es, pad, n_in, n_in + max_new, eos)
    E.beam_advance(step_logits(None).repeat_interleave(k, 0), k, params, **st, **book)
    t = 1
    while t < max_new and not bool(st["done"][:B].all()):
        E.beam_advance(step_logits(E.running_ids(st["beam_src"], book["token_log"], P, t)), k, params, **st, **book)
        t += 1
    hyps = []
    for b in range(B):
        h = E.Hypotheses(k, lp, es, n_in + max_new)
        h.slots = [dict(score=float(st["hyp_score"][b * k + s]), length=int(st["hyp_len"][b * k + s]),
                        seq=int(st["hyp_seq"][b * k + s]), ids=st["hyp_ids"][b * k + s, :int(st["hyp_len"][b * k + s]) - n_in])
                   for s in range(int(st["hyp_count"][b]))]
        hyps.append(h)
    gen = E.finalize(hyps, st["done"][:B].tolist(), st["beam_score"], E.running_ids(st["beam_src"], book["token_log"], P, t),
                     nrs, prm)
    return torch.cat([prompt_ids.repeat_interleave(nrs, 0), gen], 1)


def toy_model(V, seed):
    """Logits of a sequence: a seeded function of the whole sequence on a half-integer grid (ties everywhere)."""
    def f(seq):
        rnd = random.Random(hash((seed, tuple(seq))))
        return [rnd.randint(-6, 6) * 0.5 for _ in range(V)]
    return f


@pytest.mark.parametrize("es", [False, True, "never"])
@pytest.mark.parametrize("lp", [0.0, 1.0, 2.0])
@pytest.mark.parametrize("k, eos", [(2, [3]), (3, [3, 5]), (4, [1, 2, 6])])
def test_statement_matches_literal_search(es, lp, k, eos):
    V, max_new, pad, nrs = 9, 7, 0, min(2, k)
    prompts = [[4, 7, 8], [8, 8, 1], [2, 2, 2]]
    for seed in range(4):
        model = toy_model(V, seed)
        want = literal_search(model, prompts, k, max_new, lp, es, eos, pad, nrs)
        ids = torch.tensor(prompts)

        def step(gen):
            if gen is None:
                return torch.tensor([model(p) for p in prompts])
            return torch.tensor([model(prompts[r // k] + gen[r].tolist()) for r in range(gen.shape[0])])
        got = statement_search(step, ids, [3] * 3, k, max_new, lp, es, eos, pad, nrs)
        assert torch.equal(got, want), (seed, got.tolist(), want.tolist())


def test_statement_rules():
    """Ties go to the lower flat index; EOS at rank >= k is skipped; NaN counts as -inf; eviction and is_done."""
    s = torch.tensor([[0.0, 1.0, 1.0], [1.0, 0.5, float("-inf")]], dtype=torch.float64)
    assert E.top_candidates(s, 2) == [(1.0, 1), (1.0, 2), (1.0, 3), (0.5, 4)]
    l = E.log_softmax64(torch.tensor([[float("nan"), 0.0, 0.0], [float("-inf")] * 3]))
    assert l[0, 0] == float("-inf") and abs(float(l[0, 1]) - math.log(0.5)) < 1e-15 and bool((l[1] == float("-inf")).all())
    prm = dict(eos=[2], pad=0, input_len=4, length_penalty=1.0)
    h = E.Hypotheses(2, 1.0, False, 10)
    ch, added, done = E.process([(-1.0, 2), (-2.0, 1), (-3.0, 5), (-4.0, 4)], 2, 3, h, 1, prm)
    assert [c[:2] for c in ch] == [(0, 1), (1, 1)] and added == [(0, 0)] and not done   # flat 5: EOS at rank 2
    assert h.slots[0]["score"] == -1.0 / 5
    h2 = E.Hypotheses(1, 1.0, False, 10)
    ch, added, _ = E.process([(-1.0, 0), (-2.0, 2)], 1, 3, h2, 0, prm)   # EOS (token 2) at rank 1 >= k: skipped
    assert added == [] and ch == [(0, 0, -1.0)]
    h3 = E.Hypotheses(2, 1.0, False, 10)
    assert h3.add(-1.0, 2, 0) == 0 and h3.add(-1.0, 2, 1) == 1
    assert h3.add(-1.0, 2, 2) is None                      # not better than the worst
    assert h3.add(-0.5, 2, 3) == 0                         # evicts the earliest of the equal lowest
    assert h3.is_done(-10.0, 5) and not h3.is_done(0.0, 5)


def test_done_requests_are_padded():
    """A request that is done gets pad tokens and score 0 on every later step, and its output ends in EOS then pad."""
    model = toy_model(9, 1)
    out = literal_search(model, [[1, 2, 3]], 2, 12, 1.0, True, [3, 4, 5], 0, 1)
    ids = torch.tensor([[1, 2, 3]])
    got = statement_search(lambda g: torch.tensor([model([1, 2, 3])] if g is None else
                                                  [model([1, 2, 3] + g[r].tolist()) for r in range(g.shape[0])]),
                           ids, [3], 2, 12, 1.0, True, [3, 4, 5], 0, 1)
    assert torch.equal(got, out)
    assert got.shape[1] < 3 + 12 and int(got[0, -1]) in (3, 0)


# ------------------------------------------------------------------ C entry points without a device
@pytest.fixture(scope="module")
def lib():
    from vitron_b200 import _lib, build
    build.build()
    return _lib.load()


def test_beam_advance_argument_validation_without_device(lib):
    import ctypes as C
    buf = (C.c_uint8 * (1 << 16))()
    p = C.addressof(buf)
    p += (-p) % 16
    ERR_ARG, ERR_WS, ERR_UNSUP = -1, -3, -4
    ws = lib.vb200_beam_workspace_size(8)
    assert ws >= 16384 + 8 * 32 * 8

    def call(logits=p, ld=64, B=2, k=4, n=64, params=p, src_ld=64, hyp_ld=64, log_stride=64, token_log=p, workspace=p,
             wsb=ws, done=p):
        return lib.vb200_beam_advance(logits, ld, B, k, n, params, p, p, done, p, src_ld, p, p, p, p, p, hyp_ld, p, p, p,
                                      token_log, log_stride, p, workspace, wsb, None)
    assert call(logits=None) == ERR_ARG
    assert call(params=None) == ERR_ARG
    assert call(done=None) == ERR_ARG
    assert call(token_log=None) == ERR_ARG
    assert call(B=0) == ERR_ARG
    assert call(k=0) == ERR_ARG
    assert call(n=1, ld=1) == ERR_ARG                          # a beam step needs two tokens
    assert call(ld=32) == ERR_ARG                              # row stride shorter than a row
    assert call(src_ld=0) == ERR_ARG and call(hyp_ld=0) == ERR_ARG and call(log_stride=0) == ERR_ARG
    assert call(k=17) == ERR_UNSUP
    assert call(n=49153, ld=49153) == ERR_UNSUP
    assert call(B=4097, k=1) == ERR_UNSUP
    assert call(workspace=None) == ERR_WS
    assert call(wsb=ws - 1) == ERR_WS


def test_attn_decode_rope_beam_argument_validation_without_device(lib):
    import ctypes as C
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf)
    p += (-p) % 16
    ERR_ARG, ERR_UNSUP = -1, -4

    def call(beam_src=p, src_ld=1024, gen_start=p, table=p, head_dim=128, max_kv_len=1024):
        return lib.vb200_attn_decode_rope_beam(p, 3 * 4 * 128, table, p, p, p, 16, p, beam_src, src_ld, gen_start, p,
                                               512, 2, 4, head_dim, 64, max_kv_len, 0.1, p, 4096, None)
    assert call(beam_src=None) == ERR_ARG
    assert call(gen_start=None) == ERR_ARG
    assert call(table=None) == ERR_ARG
    assert call(src_ld=512) == ERR_ARG                         # the indirection must cover every key
    assert call(head_dim=64) == ERR_UNSUP                      # head_dim 128 only, as attn_decode_rope


# ------------------------------------------------------------------ generate(num_beams=k) host logic
def attn_decode_rope_beam(qkv, table, k_pages, v_pages, block_table, kv_len, beam_src, gen_start, n_heads, head_dim,
                          page_size, max_kv_len, scale=None, out=None):
    """Torch statement of vb200_attn_decode_rope_beam: attn_decode_rope with key j >= gen_start[b] read from the pages
    of row beam_src[b, j]."""
    B = qkv.shape[0]
    half = head_dim // 2
    scale = head_dim ** -0.5 if scale is None else scale
    x = qkv[:, :3 * n_heads * head_dim].float().view(B, 3, n_heads, head_dim)
    cos = torch.cat([table[:, :half], table[:, :half]], -1)[:, None]
    sin = torch.cat([table[:, half:], table[:, half:]], -1)[:, None]
    rot = lambda t: torch.cat([-t[..., half:], t[..., :half]], -1)
    q = (x[:, 0] * cos + rot(x[:, 0]) * sin).to(BF16).float()
    k = (x[:, 1] * cos + rot(x[:, 1]) * sin).to(BF16)
    v = x[:, 2].to(BF16)
    for b in range(B):
        slot = int(kv_len[b]) - 1
        page = int(block_table[b, slot // page_size])
        k_pages[page, :, slot % page_size] = k[b]
        v_pages[page, :, slot % page_size] = v[b]
    res = torch.empty((B, n_heads * head_dim), dtype=BF16) if out is None else out
    for b in range(B):
        n, g = int(kv_len[b]), int(gen_start[b])
        rows = [b if j < g else int(beam_src[b, j]) for j in range(n)]
        pages = [int(block_table[r, j // page_size]) for j, r in enumerate(rows)]
        kk = torch.stack([k_pages[p, :, j % page_size] for j, p in enumerate(pages)], 1).float()
        vv = torch.stack([v_pages[p, :, j % page_size] for j, p in enumerate(pages)], 1).float()
        p = torch.softmax(torch.einsum("hd,hnd->hn", q[b], kk) * scale, -1)
        res[b] = torch.einsum("hn,hnd->hd", p, vv).reshape(-1).to(BF16)
    return res


def tiny_model(monkeypatch, max_batch=8):
    from oracle.weights import seeded_state_dict
    from vitron_b200 import ops
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    from tests import cpu_ops_emulator
    cpu_ops_emulator.install(monkeypatch)
    monkeypatch.setattr(ops, "attn_decode_rope_beam", attn_decode_rope_beam)
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "vitron_llm_tiny.pt"), weights_only=False)
    vit = dict(fx["vit"], hidden_act="gelu")
    cfg = VitronConfig(llm=fx["llm"], vision=VisionConfig(**vit), video=None, tokenizer_model_max_length=4096)
    model = VitronLlamaForCausalLM(cfg, "cpu", max_batch=max_batch, max_seq_len=256)
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    model.load_state_dict(sd)
    return model, fx, sd


def _ids(B, S, seed, V):
    return torch.randint(3, V, (B, S), generator=torch.Generator().manual_seed(seed))


def _llm_sd(sd):
    return {k: v.float() for k, v in sd.items() if k.startswith("model.layers") or k.startswith("model.embed")
            or k in ("model.norm.weight", "lm_head.weight")}


def engine_logits_fn(model, ids):
    """Full recompute through the engine's own prefill (same kernels' statements as the decode step): the logits the
    beam search of the engine sees, for the statement driver."""
    eng, emb = model.engine, model.model.embed_tokens

    def step(gen):
        seqs = ids if gen is None else torch.cat([ids.repeat_interleave(gen.shape[0] // ids.shape[0], 0), gen], 1)
        return eng.prefill(emb(seqs)).float()
    return step


@pytest.mark.parametrize("k, nrs, es, lp", [(2, 1, False, 1.0), (3, 2, True, 2.0), (4, 4, "never", 0.0)])
def test_beam_generate_matches_a_statement_search(monkeypatch, k, nrs, es, lp):
    """generate(num_beams=k) on a CPU engine (one prefill, forked prompt pages, beam-indirect decode, graph-less beam
    steps) equals the statement driven over the same engine's logits of every running beam, recomputed from scratch
    by a prefill each step."""
    model, fx, sd = tiny_model(monkeypatch)
    ids = _ids(2, 9, 4, fx["llm"]["vocab_size"])
    n = 6
    got = model.generate(ids, num_beams=k, num_return_sequences=nrs, early_stopping=es, length_penalty=lp,
                         max_new_tokens=n, eos_token_id=-1, sync_every=4)
    want = statement_search(engine_logits_fn(model, ids), ids, [9, 9], k, n, lp, es, [-1], 0, nrs)
    assert got.shape == want.shape == (2 * nrs, 9 + n)
    assert torch.equal(got, want), (got.tolist(), want.tolist())


def test_beam_generate_matches_a_search_over_the_oracle(monkeypatch):
    """The same against the statement driven over the fp32 oracle (LlamaCPU, full recompute per step). The engine
    computes in bf16, so beams may part where two candidates are within bf16 rounding; this fixture's margins hold."""
    from oracle import restate_llm as R
    model, fx, sd = tiny_model(monkeypatch)
    ids = _ids(2, 9, 4, fx["llm"]["vocab_size"])
    k, n = 2, 6
    got = model.generate(ids, num_beams=k, max_new_tokens=n, eos_token_id=-1)
    ref = R.LlamaCPU(_llm_sd(sd), fx["llm"])
    emb = _llm_sd(sd)["model.embed_tokens.weight"]

    def step(gen):
        seqs = ids if gen is None else torch.cat([ids.repeat_interleave(k, 0), gen], 1)
        return ref.prefill(emb[seqs]).float()
    want = statement_search(step, ids, [9, 9], k, n, 1.0, False, [-1], 0, 1)
    assert torch.equal(got, want), (got.tolist(), want.tolist())


def test_beam_generate_eos_sync_chunks_and_criteria(monkeypatch):
    """EOS hypotheses end the output with EOS then pad; the result does not depend on sync_every; stopping_criteria
    sees the running beams [B * k, input_len + t] and stops the search."""
    model, fx, sd = tiny_model(monkeypatch)
    V = fx["llm"]["vocab_size"]
    ids = _ids(2, 7, 9, V)
    base = model.generate(ids, num_beams=3, max_new_tokens=8, eos_token_id=-1)
    eos = int(base[0, 7 + 1])                      # the best beam's second token: some beam reaches it early
    runs = [model.generate(ids, num_beams=3, num_return_sequences=2, max_new_tokens=8, eos_token_id=eos, pad_token_id=0,
                           sync_every=s) for s in (1, 3, 16)]
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2])
    want = statement_search(engine_logits_fn(model, ids), ids, [7, 7], 3, 8, 1.0, False, [eos], 0, 2)
    assert torch.equal(runs[0], want)
    assert bool((runs[0][:, 7:] == eos).any())
    seen = []

    def crit(seq, scores):
        seen.append(tuple(seq.shape))
        return seq.shape[1] >= 7 + 3
    got = model.generate(ids, num_beams=3, max_new_tokens=8, eos_token_id=-1, stopping_criteria=crit)
    assert seen[0] == (6, 8) and seen[-1] == (6, 10) and got.shape == (2, 7 + 4)


def test_beam_generate_against_transformers(monkeypatch):
    """length_penalty = 0 (where 4.31 and the installed transformers agree): generate(num_beams=k) equals
    transformers' LlamaForCausalLM.generate(num_beams=k) built locally from the same weights; so does the statement
    driven over that model's own logits."""
    transformers = pytest.importorskip("transformers")
    model, fx, sd = tiny_model(monkeypatch)
    c = fx["llm"]
    hf_cfg = transformers.LlamaConfig(vocab_size=c["vocab_size"], hidden_size=c["hidden_size"],
                                      intermediate_size=c["intermediate_size"], num_hidden_layers=c["num_hidden_layers"],
                                      num_attention_heads=c["num_attention_heads"], rms_norm_eps=1e-5, rope_theta=10000.0,
                                      max_position_embeddings=256, tie_word_embeddings=False, pad_token_id=0,
                                      bos_token_id=1, eos_token_id=2)
    hf = transformers.LlamaForCausalLM(hf_cfg).eval()
    missing, unexpected = hf.load_state_dict(_llm_sd(sd), strict=False)
    assert not [m for m in missing if "rotary" not in m] and not unexpected
    ids = _ids(2, 8, 5, c["vocab_size"])
    n, k = 6, 3
    with torch.no_grad():
        want = hf.generate(ids, attention_mask=torch.ones_like(ids), num_beams=k, num_return_sequences=2, do_sample=False,
                           length_penalty=0.0, early_stopping=False, max_new_tokens=n, min_new_tokens=0,
                           eos_token_id=2, pad_token_id=0)

        def step(gen):
            seqs = ids if gen is None else torch.cat([ids.repeat_interleave(k, 0), gen], 1)
            return hf(seqs).logits[:, -1].float()
        stmt = statement_search(step, ids, [8, 8], k, n, 0.0, False, [2], 0, 2)
    assert torch.equal(stmt, want), (stmt.tolist(), want.tolist())
    got = model.generate(ids, num_beams=k, num_return_sequences=2, length_penalty=0.0, max_new_tokens=n, eos_token_id=2,
                         pad_token_id=0)
    assert torch.equal(got, want), (got.tolist(), want.tolist())


def test_num_beams_one_is_greedy_and_value_errors(monkeypatch):
    model, fx, _ = tiny_model(monkeypatch, max_batch=4)
    ids = _ids(2, 9, 4, fx["llm"]["vocab_size"])
    greedy = model.generate(ids, max_new_tokens=5, eos_token_id=-1)
    assert torch.equal(model.generate(ids, num_beams=1, max_new_tokens=5, eos_token_id=-1), greedy)
    with pytest.raises(ValueError, match="num_return_sequences"):
        model.generate(ids, num_beams=2, num_return_sequences=3, max_new_tokens=5)
    with pytest.raises(ValueError, match="max_batch"):
        model.generate(ids, num_beams=3, max_new_tokens=5)
    assert model.generate(ids, num_beams=2, max_new_tokens=5, eos_token_id=-1).shape == (2, 14)


def test_fork_shares_full_pages_and_frees_once():
    from vitron_b200.llama import LlamaConfig, PagedKVCache
    cfg = LlamaConfig(hidden_size=16, intermediate_size=32, num_hidden_layers=2, num_attention_heads=2, vocab_size=10)
    c = PagedKVCache(cfg, max_batch=6, max_seq_len=256, device="cpu")
    total = len(c._free)
    c.reserve(0, 130)
    c.reserve(1, 64)
    c.pages[:, :, c._owned[0][2], :, :2] = 7.0
    c.fork([130, 64], 3)
    for j in range(3):
        assert c._owned[j][:2] == c._owned[0][:2]            # request 0: two full pages shared
        assert len(c._owned[j]) == 3 and bool((c.pages[:, :, c._owned[j][2], :, :2] == 7.0).all())
        assert c._owned[3 + j] == c._owned[3]                 # request 1: one full page, no partial page
    assert len({c._owned[j][2] for j in range(3)}) == 3
    assert len(c._free) == total - (2 + 3 + 1)
    for s in range(6):
        c.release(s)
    assert sorted(c._free) == list(range(total))


def test_beam_advance_wrapper_checks_every_state_buffer(lib):
    """ops.beam_advance rejects a state buffer of the wrong dtype, length or layout before anything is launched."""
    from vitron_b200 import ops
    R, k, S = 4, 2, 16
    i32 = lambda n=R: torch.zeros(n, dtype=torch.int32)
    state = dict(beam_score=torch.zeros(R), parent=i32(), done=i32(), beam_src=torch.zeros((R, S), dtype=torch.int32),
                 hyp_score=torch.zeros(R, dtype=torch.float64), hyp_len=i32(), hyp_seq=i32(), hyp_count=i32(),
                 hyp_ids=torch.zeros((R, S), dtype=torch.int64), next_src=i32(), positions=i32(), kv_len=i32(),
                 token_log=torch.zeros((R, S), dtype=torch.int64), prompt_len=i32())
    logits, prm = torch.zeros((R, 8)), E.pack_params(1.0, False, 0, 3, 9, [2])
    bad = dict(beam_score=torch.zeros(R, dtype=torch.float64), hyp_score=torch.zeros(R), parent=torch.zeros(R, dtype=torch.int64),
               done=i32(R - 1), hyp_len=torch.zeros((R, 1), dtype=torch.int32), hyp_seq=torch.zeros(2 * R, dtype=torch.int32)[::2],
               hyp_count=torch.zeros(R), next_src=torch.zeros(R, dtype=torch.int64), positions=i32(1),
               kv_len=torch.zeros(R, dtype=torch.int64), prompt_len=torch.zeros(R, dtype=torch.int16),
               beam_src=torch.zeros((R, S), dtype=torch.int64), hyp_ids=torch.zeros((R, S), dtype=torch.int32),
               token_log=torch.zeros((R - 1, S), dtype=torch.int64))
    for name, t in bad.items():
        with pytest.raises(ValueError, match=name):
            ops.beam_advance(logits, k, prm, **dict(state, **{name: t}))
    with pytest.raises(ValueError, match="params"):
        ops.beam_advance(logits, k, prm[:56], **state)


def test_beam_steps_need_start_beam():
    from vitron_b200.llama import LlamaEngine
    eng = LlamaEngine(dict(hidden_size=16, intermediate_size=32, num_hidden_layers=1, num_attention_heads=2, vocab_size=10),
                      "cpu", max_batch=2, max_seq_len=64)
    with pytest.raises(RuntimeError, match="start_beam"):
        eng.decode_steps(2, 1, sampled="beam")
    with pytest.raises(RuntimeError, match="start_beam"):
        eng.beam_advance(torch.zeros((2, 10)))


def test_length_penalty_is_carried_as_a_double():
    for lp in (0.6, 1.1, 1.0 / 3.0):
        assert E.unpack_params(E.pack_params(lp, "never", 0, 5, 9, [2]))["length_penalty"] == lp
    assert E.PARAMS.size == 64
