"""GPU: the logits processors' kernel (vb200_logits_process) against the fp32 statement in vitron_b200/processors.py, and
generate(repetition_penalty=..., no_repeat_ngram_size=..., min_length=..., min_new_tokens=...) through the CUDA-graphed
decode step in greedy, sampled, beam-search and beam-sampling modes."""
import os

import pytest
import torch

from vitron_b200 import processors as E
from tests.test_beam_gpu import MIDSIZE, _model

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(R, V, g, beam):
    """Rows of logits (a NaN entry, a row of NaNs) and histories with duplicates, sentinels, pad columns and, for beam
    rows, generated ids read through beam_src. Prompts draw from a small id range so that n-grams repeat."""
    n_in, P, t = 29, 300, 9
    S = P + t + 8
    lg = torch.randn((R, V), generator=g) * 4
    lg[0, 1] = float("nan")
    if R > 2:
        lg[2] = float("nan")
    hi = min(V, 6)
    prompt = torch.randint(0, hi, (R, n_in), generator=g, dtype=torch.int32)
    prompt[:, 3] = -200                                  # the image sentinel
    prompt[::2, :4] = 0                                  # left padding (pad id 0)
    prompt[1::3, 7] = -300                               # a region sentinel
    token_log = torch.randint(0, hi, (R, S), generator=g)
    token_log[:, 2] = V - 1
    beam_src = None
    if beam:
        k = 4 if R % 4 == 0 else 1
        beam_src = torch.zeros((R, S), dtype=torch.int32)
        for r in range(R):
            b0 = (r // k) * k
            beam_src[r, P:P + t] = torch.randint(b0, b0 + k, (t,), generator=g, dtype=torch.int32)
    kv_len = torch.full((R,), P + t, dtype=torch.int32)
    kv_len[0] = P                                         # a row with nothing generated yet
    return lg, prompt, token_log, beam_src, kv_len, torch.full((R,), P, dtype=torch.int32), n_in


SETTINGS = [dict(repetition_penalty=1.3), dict(repetition_penalty=0.6), dict(no_repeat_ngram_size=1),
            dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=4), dict(min_length=45, eos=[2, 5, 0]),
            dict(min_new_tokens=4, eos=[3]),
            dict(repetition_penalty=1.1, no_repeat_ngram_size=3, min_length=30, min_new_tokens=8, eos=[1, 4])]


@pytest.mark.parametrize("V", [37, 32000, 49152])
@pytest.mark.parametrize("R", [1, 8, 32])
def test_kernel_matches_statement(cuda, V, R):
    """Raw mode is bit-identical to the statement. In LOGPROBS mode the entries the processors change are exactly the
    statement's, and the values agree within |d| <= 4e-6 * (1 + |want|) (fp32 log-softmax on the device against the
    float64 one rounded to fp32, times a penalty <= 1.3). Without kv_len the row sees its prompt only."""
    from vitron_b200 import ops
    g = torch.Generator().manual_seed(V + R)
    for beam in (False, True):
        lg, prompt, tl, bs, kv, pl, n_in = _case(R, V, g, beam)
        for s in SETTINGS:
            s = dict(s)
            eos = s.pop("eos", ())
            prm = E.pack_params(input_len=n_in, eos_ids=eos, **s)
            off = E.pack_params(input_len=n_in, no_repeat_ngram_size=10 ** 6)
            for state in (dict(token_log=tl, kv_len=kv, prompt_len=pl, beam_src=bs), {}):
                dev = {n: v.to(cuda) for n, v in state.items() if v is not None}
                want = E.process(lg.clone(), prm, prompt, **state)
                got = ops.logits_process(lg.clone().to(cuda), prm.to(cuda), prompt.to(cuda), **dev).cpu()
                assert torch.equal(got.isnan(), want.isnan()), (beam, s)
                assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(want)), (beam, s)
                w_lp = E.process(lg.clone(), prm, prompt, logprobs=True, **state)
                g_lp = ops.logits_process(lg.clone().to(cuda), prm.to(cuda), prompt.to(cuda), logprobs=True, **dev).cpu()
                base_w = E.process(lg.clone(), off, prompt, logprobs=True, **state)
                base_g = ops.logits_process(lg.clone().to(cuda), off.to(cuda), prompt.to(cuda), logprobs=True,
                                            **dev).cpu()
                assert torch.equal(g_lp != base_g, w_lp != base_w), (beam, s)
                assert torch.equal(torch.isneginf(g_lp), torch.isneginf(w_lp))
                fin = torch.isfinite(w_lp)
                assert bool(((g_lp[fin] - w_lp[fin]).abs() <= 4e-6 * (1 + w_lp[fin].abs())).all()), (beam, s)


def _graph_free_reference(m, monkeypatch):
    """The same engine with every decode step un-graphed and processors.process applied to d_logits between the decode
    body and the advance kernel."""
    eng = m.engine
    monkeypatch.setattr(eng, "process_logits", lambda logits, step=False, beam=False: E.process(
        logits, eng.d_proc, eng.d_proc_prompt[:logits.shape[0]], logprobs=beam,
        **(dict(token_log=eng.token_log[:logits.shape[0]], kv_len=eng.d_len[:logits.shape[0]],
                prompt_len=eng.d_prompt[:logits.shape[0]],
                **(dict(beam_src=eng.beam["beam_src"][:logits.shape[0]]) if beam else {})) if step else {})))
    real = type(eng).decode_steps
    monkeypatch.setattr(eng, "decode_steps", lambda B, n, use_graph=True, sampled=False: real(eng, B, n, False, sampled))


MODES = {"greedy": dict(), "sample": dict(do_sample=True, temperature=0.8, top_p=0.95),
         "beam": dict(num_beams=4), "beam_sample": dict(do_sample=True, num_beams=4, temperature=0.9)}
PROC_A = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=6)
PROC_B = dict(repetition_penalty=0.8, no_repeat_ngram_size=2, min_length=120)


@pytest.mark.parametrize("mode", list(MODES))
def test_graphed_generate_matches_ungraphed_statement(cuda, mode, monkeypatch):
    """Tokens of the graphed decode with processors equal the un-graphed engine with the statement in place of the
    kernel; new settings replay the same graphs; inactive processors (an n-gram size above any history) run the
    kernel and change no token; processors off capture the graphs of before, with one launch less."""
    B, NEW = 2, 14
    m, _ = _model(MIDSIZE, B * 2, cuda, 96, NEW)
    V = MIDSIZE["vocab_size"]
    ids = torch.randint(3, 40, (B, 96), generator=torch.Generator().manual_seed(9)).to(cuda)   # repeats in the prompt
    eos = int(torch.randint(3, V, (), generator=torch.Generator().manual_seed(1)))

    def run(**kw):
        torch.manual_seed(4)
        return m.generate(ids, max_new_tokens=NEW, eos_token_id=eos, pad_token_id=0, sync_every=5, **MODES[mode], **kw)
    plain = run()
    plain_launches = m.engine.launches_per_step
    inactive = run(no_repeat_ngram_size=10 ** 4)
    assert torch.equal(inactive, plain)
    assert m.engine.launches_per_step == plain_launches + 1
    got_a = run(**PROC_A)
    n_graphs = len(m.engine._graphs)
    got_b = run(**PROC_B)
    assert len(m.engine._graphs) == n_graphs            # new settings, same graph
    assert not torch.equal(got_a, plain)
    assert torch.equal(run(), plain)                    # settings do not leak into the next call
    with monkeypatch.context() as mp:
        _graph_free_reference(m, mp)
        want_a, want_b = run(**PROC_A), run(**PROC_B)
    assert torch.equal(got_a, want_a), (got_a.tolist(), want_a.tolist())
    assert torch.equal(got_b, want_b), (got_b.tolist(), want_b.tolist())


def test_no_repeat_unigrams_with_greedy(cuda):
    B, NEW = 2, 24
    m, _ = _model(MIDSIZE, B, cuda, 64, NEW)
    ids = torch.randint(3, MIDSIZE["vocab_size"], (B, 64), generator=torch.Generator().manual_seed(2)).to(cuda)
    out = m.generate(ids, max_new_tokens=NEW, eos_token_id=-1, no_repeat_ngram_size=1).cpu()
    for row in out.tolist():
        gen = row[64:]
        assert len(gen) == NEW and len(set(gen)) == NEW and not set(gen) & set(row[:64])


def test_full_model_generate_with_images(cuda, monkeypatch):
    """generate(images=..., repetition_penalty=1.3, min_new_tokens=4) on the golden tiny model, whose input_ids hold the
    -200 image sentinel (4.31 fails there), matches the un-graphed reference loop."""
    from oracle.weights import seeded_state_dict
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "vitron_llm_tiny.pt"), weights_only=False)
    vit = dict(fx["vit"], hidden_act="gelu")
    cfg = VitronConfig(llm=fx["llm"], vision=VisionConfig(**vit), video=None, tokenizer_model_max_length=4096)
    m = VitronLlamaForCausalLM(cfg, cuda, max_batch=16, max_seq_len=256)
    m.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"]))
    g = fx["gen_img"]
    ids = g["input_ids"].to(cuda)
    assert bool((ids == -200).any())
    imgs = [i.to(cuda) for i in g["images"]]
    eos = int(m.generate(ids, images=imgs, regions=g["regions"], max_new_tokens=1, eos_token_id=-1)[0, -1])

    def run(**kw):
        return m.generate(ids, images=imgs, regions=g["regions"], max_new_tokens=10, eos_token_id=eos, pad_token_id=0,
                          repetition_penalty=1.3, min_new_tokens=4, **kw)
    outs = {n: run(**kw) for n, kw in (("greedy", {}), ("beam", dict(num_beams=3)))}
    with monkeypatch.context() as mp:
        _graph_free_reference(m, mp)
        for n, kw in (("greedy", {}), ("beam", dict(num_beams=3))):
            assert torch.equal(outs[n], run(**kw)), n
    assert int(outs["greedy"][0, ids.shape[1]]) != eos
