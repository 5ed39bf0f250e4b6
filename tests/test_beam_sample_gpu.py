"""GPU: the beam-sampling step (vb200_beam_sample_advance) against the float64 statement in vitron_b200/beam.py, a
chi-square test of its draws, and beam sampling through the CUDA-graphed decode step of the engine and of generate()."""
import os

import pytest
import torch

from vitron_b200 import beam as E
from tests.test_beam_gpu import MIDSIZE, STATE, _case, _model
from tests.test_beam_sample_cpu import _exact_child_pairs, chi_square_pvalue, first_step_case, overflow_case, sparams

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _unpack(sp):
    from vitron_b200.ops import SAMPLE_PARAMS
    T, top_k, top_p, _, seed = SAMPLE_PARAMS.unpack(sp.cpu().numpy().tobytes())
    return T, top_k, top_p, seed


def _near(lg, st, k, sp):
    """Searches whose outcome fp32 device arithmetic may legitimately change: a row's top-p fraction within 1e-5 of
    top_p, the statement's keys at ranks 2k - 1 and 2k (the draw boundary), or two adjacent drawn warped scores, closer
    than 1e-5 * (1 + |value|) without being equal."""
    T, top_k, top_p, seed = _unpack(sp)
    w = E.warped_scores(lg, st["beam_score"], T)
    kept, near_p = E.warp_kept(w, top_k, top_p)
    t = int(st["kv_len"][0]) - int(st["prompt_len"][0])
    near = set()
    close = lambda a, b: a != b and abs(a - b) < 1e-5 * (1 + abs(a))
    for b in range(lg.shape[0] // k):
        rows = slice(b * k, (b + 1) * k)
        drawn, keys = E.sample_draws(w[rows], kept[rows], k, b, t, seed)
        if bool(near_p[rows].any()) or (len(keys) > 2 * k and close(keys[2 * k - 1], keys[2 * k])) or \
                any(close(drawn[i][0], drawn[i + 1][0]) for i in range(len(drawn) - 1)):
            near.add(b)
    return near


SETTINGS = [(1.0, None, None), (0.7, 50, 0.9), (1.5, 1, None), (0.5, None, 0.05), (2.0, 5, 0.99)]


@pytest.mark.parametrize("V", [37, 32000, 49152])
@pytest.mark.parametrize("T, top_k, top_p", SETTINGS)
def test_beam_sample_advance_matches_statement(cuda, V, T, top_k, top_p):
    """Mid-search states (ties, a NaN entry, a NaN row, stored hypotheses, a done search) and step-0 states (every beam
    at 0): tokens, parents, history and hypothesis store equal the statement wherever no fp32 near-tie decides them;
    scores agree within fp32 rounding; repeats are bit-identical."""
    from vitron_b200 import ops
    g = torch.Generator().manual_seed(V + int(T * 10))
    skipped = total = 0
    for k in (2, 4, 16):
        for step0 in (False, True):
            B = 3
            lg, st, prm = _case(B, k, V, g)
            if V > 20:
                lg[k + 1] = float("nan")                     # a row with no number
            if step0:
                st["beam_score"] = torch.zeros(B * k)
            sp = sparams(T, top_k, top_p, int(torch.randint(0, 2 ** 62, (), generator=g)) * 3)
            want = {n: t.clone() for n, t in st.items()}
            E.beam_sample_advance(lg, k, prm, sp, **want)
            outs = []
            for _ in range(2):
                dev = {n: t.to(cuda) for n, t in st.items()}
                ops.beam_sample_advance(lg.to(cuda), k, prm.to(cuda), sp.to(cuda), **dev)
                outs.append({n: t.cpu() for n, t in dev.items()})
            for n in STATE:
                assert torch.equal(outs[0][n], outs[1][n]), (k, n)
            got, skip = outs[0], _near(lg, st, k, sp)
            total += B
            skipped += len(skip)
            for b in range(B):
                if b in skip:
                    continue
                rows = slice(b * k, (b + 1) * k)
                for n in ("parent", "next_src", "beam_src", "token_log", "positions", "kv_len", "hyp_len", "hyp_seq"):
                    assert torch.equal(got[n][rows], want[n][rows]), (k, step0, b, n)
                assert int(got["done"][b]) == int(want["done"][b]) and int(got["hyp_count"][b]) == int(want["hyp_count"][b])
                torch.testing.assert_close(got["beam_score"][rows], want["beam_score"][rows], rtol=2e-6, atol=1e-5)
                torch.testing.assert_close(got["hyp_score"][rows], want["hyp_score"][rows], rtol=2e-6, atol=1e-6)
                for s in range(int(want["hyp_count"][b])):
                    L = int(want["hyp_len"][b * k + s]) - 12
                    assert torch.equal(got["hyp_ids"][b * k + s, :L], want["hyp_ids"][b * k + s, :L]), (k, b, s)
    print(f"searches decided by a near-tie and skipped: {skipped} of {total}")
    assert skipped <= total // 4, (skipped, total)


def test_chi_square_of_the_kernels_draws(cuda):
    """Step 0 (every beam at 0) of 1024 searches with the same logits (each search its own Philox counters), 8 seeds:
    the children the kernel picks follow the exact without-replacement probabilities over the k live rows; the
    statement picks the same children."""
    from vitron_b200 import ops
    lg1, V, k, T, w, p = first_step_case()
    exact = _exact_child_pairs(p, w, k)
    B, S = 1024, 8
    R = B * k
    counts, n = {}, 0
    for seed in range(S):
        st = dict(beam_score=torch.zeros(R), parent=torch.zeros(R, dtype=torch.int32),
                  done=torch.zeros(R, dtype=torch.int32), beam_src=torch.zeros((R, 8), dtype=torch.int32),
                  hyp_score=torch.zeros(R, dtype=torch.float64), hyp_len=torch.zeros(R, dtype=torch.int32),
                  hyp_seq=torch.zeros(R, dtype=torch.int32), hyp_count=torch.zeros(R, dtype=torch.int32),
                  hyp_ids=torch.zeros((R, 8), dtype=torch.int64), next_src=torch.zeros(R, dtype=torch.int32),
                  positions=torch.full((R,), 2, dtype=torch.int32), kv_len=torch.full((R,), 3, dtype=torch.int32),
                  token_log=torch.zeros((R, 8), dtype=torch.int64), prompt_len=torch.full((R,), 3, dtype=torch.int32))
        prm, sp = E.pack_params(1.0, False, 0, 3, 8, [-1]), sparams(T, None, None, seed)
        lg = lg1.repeat(R, 1)
        dev = {nm: t.to(cuda) for nm, t in st.items()}
        ops.beam_sample_advance(lg.to(cuda), k, prm.to(cuda), sp.to(cuda), **dev)
        tok, par = dev["next_src"].cpu().view(B, k), dev["parent"].cpu().view(B, k) - (torch.arange(B) * k)[:, None]
        for b in range(B):
            c = (int(par[b, 0]) * V + int(tok[b, 0]), int(par[b, 1]) * V + int(tok[b, 1]))
            counts[c] = counts.get(c, 0) + 1
        n += B
        if seed == 0:
            want = {nm: t.clone() for nm, t in st.items()}
            E.beam_sample_advance(lg, k, prm, sp, **want)
            assert torch.equal(want["next_src"], dev["next_src"].cpu())
    assert chi_square_pvalue(counts, exact, n) > 1e-3


def test_scores_beyond_fp32_continue_with_pad(cuda):
    """A search whose scores leave the fp32 range has no draws and continues with pad at -1e9, bit for bit as the
    statement; a search with one such beam draws from its live row."""
    from vitron_b200 import ops
    lg, st, prm, sp = overflow_case()
    want = {n: t.clone() for n, t in st.items()}
    E.beam_sample_advance(lg, 2, prm, sp, **want)
    dev = {n: t.to(cuda) for n, t in st.items()}
    ops.beam_sample_advance(lg.to(cuda), 2, prm.to(cuda), sp.to(cuda), **dev)
    for n in STATE:
        if n in ("beam_score", "hyp_score"):
            torch.testing.assert_close(dev[n].cpu(), want[n], rtol=2e-6, atol=1e-5)
        else:
            assert torch.equal(dev[n].cpu(), want[n]), n
    assert dev["beam_score"][:2].tolist() == [-1e9, -1e9]


def test_engine_beam_sample_steps_vs_statement(cuda):
    """Graphed beam-sampling steps (2 searches per prompt, ragged prompts) equal the statement's step over the engine's
    own logits; a new temperature / top-k / top-p / seed on replay takes effect without a recapture; the step has the
    beam-search step's launch count."""
    from vitron_b200 import ops
    k, r, NEW, B = 3, 2, 8, 2
    m, _ = _model(MIDSIZE, B * 2, cuda, 777, NEW)
    eng, V, R = m.engine, MIDSIZE["vocab_size"], B * r * k
    lens = [777, 764]
    ids = torch.randint(3, V, (B, 777), generator=torch.Generator().manual_seed(7)).to(cuda)
    emb = m.model.embed_tokens(ids)
    prm = E.pack_params(1.0, False, 0, 777, 777 + NEW, [-1])
    with torch.no_grad():
        eng.start_beam(eng.prefill(emb[:, :], lens), k, NEW, prm.to(cuda), searches=r)
        eng.decode_steps(R, 1, sampled="beam")
        beam_launches = eng.launches_per_step
        eng.set_sampling(0.8, 20, 0.95, 1234)
        lg0 = eng.prefill(emb, lens)
        eng.start_beam(lg0, k, NEW, prm.to(cuda), sample=True, searches=r)
        n_graphs, compared, skipped = None, 0, 0
        for t in range(1, NEW):
            if t == 4:                                   # new parameters, same graph
                eng.set_sampling(1.4, None, 0.8, 2 ** 50 + 3)
            before = {n: v[:R].cpu().clone() for n, v in eng.beam.items()}
            book = dict(next_src=eng.d_src[:R].cpu(), positions=eng.d_pos[:R].cpu(), kv_len=eng.d_len[:R].cpu(),
                        token_log=eng.token_log[:R].cpu(), prompt_len=eng.d_prompt[:R].cpu())
            eng.decode_steps(R, 1, sampled="beam_sample")
            if n_graphs is None:
                n_graphs = len(eng._graphs)
                assert eng.launches_per_step == beam_launches > 0
            assert len(eng._graphs) == n_graphs
            lg, sp = eng.d_logits[:R].cpu().clone(), eng.d_sample.cpu()
            want = {n: v.clone() for n, v in dict(before, **book).items()}
            E.beam_sample_advance(lg, k, prm, sp, **want)
            skip = _near(lg, dict(before, **book), k, sp)
            for b in range(B * r):
                if b in skip:
                    skipped += 1
                    continue
                rows = slice(b * k, (b + 1) * k)
                assert torch.equal(eng.beam["parent"][rows].cpu(), want["parent"][rows]), (t, b)
                assert torch.equal(eng.d_src[rows].cpu(), want["next_src"][rows]), (t, b)
                assert torch.equal(eng.beam["beam_src"][rows].cpu(), want["beam_src"][rows]), (t, b)
                torch.testing.assert_close(eng.beam["beam_score"][rows].cpu(), want["beam_score"][rows], rtol=2e-6,
                                           atol=1e-5)
                compared += 1
    print(f"searches compared {compared}, skipped at a near-tie {skipped}")
    assert compared >= 3 * skipped and compared > 0
    runs = []
    for s in (16, 3):
        torch.manual_seed(5)
        runs.append(m.generate(ids, do_sample=True, temperature=0.9, top_p=0.95, num_beams=k, num_return_sequences=r,
                               max_new_tokens=NEW, eos_token_id=-1, sync_every=s))
    assert runs[0].shape == (B * r, 777 + NEW) and torch.equal(runs[0], runs[1])


def test_full_model_beam_sample_generate_with_images(cuda):
    """generate(images=..., do_sample=True, num_beams=3, num_return_sequences=2) on the golden tiny model: reproducible
    under torch.manual_seed, [B * 2, input_len + gen_len], prompt ids first; the sampled and beam-search calls on the
    same model are unchanged by it."""
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
    imgs = [i.to(cuda) for i in g["images"]]

    def run(**kw):
        torch.manual_seed(3)
        return m.generate(ids, images=imgs, regions=g["regions"], max_new_tokens=10, eos_token_id=-1, **kw)
    beam_before = run(num_beams=4, num_return_sequences=2)
    outs = [run(do_sample=True, temperature=0.7, top_p=0.9, num_beams=3, num_return_sequences=2) for _ in range(2)]
    assert torch.equal(outs[0], outs[1])
    assert outs[0].shape == (2 * ids.shape[0], ids.shape[1] + 10)
    assert torch.equal(outs[0][:, :ids.shape[1]], ids.repeat_interleave(2, 0))
    assert torch.equal(run(num_beams=4, num_return_sequences=2), beam_before)
