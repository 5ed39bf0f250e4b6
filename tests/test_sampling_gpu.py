"""GPU: the device sampler (vb200_sample_advance) against the float64 statement of its contract in
vitron_b200/sampling.py, its distribution, and sampled generation through the CUDA-graphed decode step."""
import pytest
import torch

from vitron_b200 import sampling as E

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _logits(B, V, g):
    lg = torch.randn((B, V), generator=g) * 3
    if V > 20:
        lg[:, 5] = lg[:, 9]                              # a planted tie
        lg[:, 17] = lg.max(1).values                     # a tie at the maximum
        lg[0, 3] = float("nan")
    if B > 32:
        lg[32] = float("nan")                            # no number in the row: token 0
    return lg


@pytest.mark.parametrize("V", [37, 1000, 32000, 32001, 32002])
def test_sample_advance_matches_reference(cuda, V):
    """Every token equals the float64 reference except where the reference's draw (or top-p cut) is within 1e-5 of a
    boundary; those differing tokens must be under 1 % of the rows. The bookkeeping equals argmax_advance's on the same
    state."""
    from vitron_b200 import ops
    g = torch.Generator().manual_seed(V)
    rows = differing = 0
    for B in (1, 8, 33):
        lg = _logits(B, V, g)
        lg_d = lg.to(cuda)                               # row stride V: odd V rows are not 16-byte aligned
        plen = torch.randint(5, 50, (B,), generator=g, dtype=torch.int32)
        kvl = plen + torch.randint(0, 40, (B,), generator=g, dtype=torch.int32)
        pos = torch.randint(10, 100, (B,), generator=g, dtype=torch.int32)
        steps = (kvl - plen).numpy()
        for T in (1e-6, 0.2, 1.0, 5.0):
            for k in (0, 1, 40, V + 5):
                for p in (1.0, 0.0, 0.5, 0.95):
                    seed = int(torch.randint(0, 2 ** 62, (), generator=g))
                    params = ops.sample_params(T, k, p, seed).to(cuda)
                    st = [t.to(cuda) for t in (pos, kvl, plen)] + [torch.zeros((B, 64), dtype=torch.int64, device=cuda)]
                    src = torch.full((B,), -1, dtype=torch.int32, device=cuda)
                    tok = ops.sample_advance(lg_d, params, None, next_src=src, positions=st[0], kv_len=st[1],
                                             token_log=st[3], prompt_len=st[2]).cpu()
                    # T, top_p as the kernel reads them (fp32)
                    t32, p32 = float(torch.tensor(T, dtype=torch.float32)), float(torch.tensor(p, dtype=torch.float32))
                    ref, near = E.sample_reference(lg, t32, k, p32, seed, steps)
                    bad = (tok != ref) & ~near
                    assert not bool(bad.any()), (B, T, k, p, bad.nonzero().flatten().tolist(), tok[bad].tolist(), ref[bad].tolist())
                    rows += B
                    differing += int((tok != ref).sum())
                    # same state through argmax_advance on one-hot logits of the sampled tokens: identical outputs
                    one_hot = torch.zeros((B, V), device=cuda)
                    one_hot[torch.arange(B), tok.to(cuda)] = 1.0
                    st2 = [t.to(cuda) for t in (pos, kvl, plen)] + [torch.zeros((B, 64), dtype=torch.int64, device=cuda)]
                    src2 = torch.full((B,), -1, dtype=torch.int32, device=cuda)
                    idx2 = ops.argmax_advance(one_hot, torch.empty((B,), dtype=torch.int64, device=cuda), next_src=src2,
                                              positions=st2[0], kv_len=st2[1], token_log=st2[3], prompt_len=st2[2])
                    assert torch.equal(idx2.cpu(), tok) and torch.equal(src, src2)
                    for a, b in zip(st, st2):
                        assert torch.equal(a, b)
    assert differing < 0.01 * rows, (differing, rows)


def test_sample_distribution_chi_square(cuda):
    """65,536 rows of the same V = 37 logits (the row index is part of the Philox counter) with top-p active: the
    counts follow the renormalised kept distribution and nothing outside the kept set is drawn."""
    from scipy.stats import chisquare
    from vitron_b200 import ops
    V, N, T, top_p = 37, 65536, 0.8, 0.9
    g = torch.Generator().manual_seed(3)
    lg = torch.randn((1, V), generator=g)
    tok = ops.sample_advance(lg.expand(N, V).contiguous().to(cuda), ops.sample_params(T, 0, top_p, 0xC0FFEE).to(cuda))
    kept, p, _ = E.sample_support(lg, float(torch.tensor(T, dtype=torch.float32)), 0,
                                  float(torch.tensor(top_p, dtype=torch.float32)))
    kept, p = kept[0], p[0]
    assert 3 <= int(kept.sum()) < V
    counts = torch.bincount(tok.cpu(), minlength=V)
    assert int(counts[~kept].sum()) == 0
    expected = (p[kept] / p.sum() * N).numpy()
    pv = chisquare(counts[kept].double().numpy(), expected).pvalue
    assert pv > 1e-4, pv


MIDSIZE = dict(hidden_size=512, intermediate_size=1408, num_hidden_layers=4, num_attention_heads=4, vocab_size=2000,
               rms_norm_eps=1e-5, rope_theta=10000.0)
VICUNA_4L = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=4, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)


@pytest.mark.parametrize("cfg, B", [(MIDSIZE, 3), (VICUNA_4L, 8), (VICUNA_4L, 17)], ids=["midsize-B3", "vicuna4l-B8", "vicuna4l-B17"])
def test_sampled_graphed_decode(cuda, cfg, B):
    """Graphed sampled decode, one token at a time, against the reference sampler on each step's logits; top_k = 1 is
    greedy; generate() is reproducible under torch.manual_seed across sync chunks and seed-dependent; a forced EOS pads
    its row; the sampled step has as many launches as the greedy one. B = 8 runs the GEMV decode path, B = 17 the GEMM."""
    from oracle.weights import seeded_state_dict
    from vitron_b200 import ops, param_shapes as PS
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    vc = VitronConfig(llm=cfg, vision=None, video=None, tokenizer_model_max_length=4096)
    S, NEW = 48, 12
    m = VitronLlamaForCausalLM(vc, cuda, max_batch=B, max_seq_len=S + 2 * NEW)
    if cfg is MIDSIZE:
        sd = seeded_state_dict(PS.llama_shapes(vc.llm), 3)
    else:
        sd = PS.random_state_dict(PS.vitron_shapes(vc), cuda, seed=0)
    m.load_state_dict(sd)
    del sd
    eng, V = m.engine, cfg["vocab_size"]
    ids = torch.randint(3, V, (B, S), generator=torch.Generator().manual_seed(B)).to(cuda)
    emb = m.model.embed_tokens(ids)

    with torch.no_grad():
        # greedy reference ids
        eng.start_decode(ops.argmax_rows(eng.prefill(emb)), NEW)
        eng.decode_steps(B, NEW - 1)
        greedy = eng.token_log[:B, :NEW].clone()
        launches_greedy = eng.launches_per_step
        # sampled, stepped one token at a time: each token is the reference sampler on that step's logits with (seed, t)
        seed, differing = 0x5EED0123456789AB, 0
        for T, k, p in ((0.7, 50, 0.9), (1.0, None, None)):
            eng.set_sampling(T, k, p, seed)
            t32 = float(torch.tensor(T, dtype=torch.float32))
            p32 = 1.0 if p is None else float(torch.tensor(p, dtype=torch.float32))
            logits0 = eng.prefill(emb)
            first = ops.sample_advance(logits0, eng.d_sample).cpu()
            ref, near = E.sample_reference(logits0, t32, k or 0, p32, seed, 0)
            assert not bool(((first != ref) & ~near).any())
            differing += int((first != ref).sum())
            eng.start_decode(first.to(cuda), NEW)
            for t in range(1, NEW):
                eng.decode_steps(B, 1, sampled=True)
                got = eng.token_log[:B, t].cpu()
                ref, near = E.sample_reference(eng.d_logits[:B], t32, k or 0, p32, seed, t)
                assert not bool(((got != ref) & ~near).any()), (T, k, p, t, got.tolist(), ref.tolist())
                differing += int((got != ref).sum())
        assert differing <= 0.01 * 2 * NEW * B, differing
        assert eng.launches_per_step == launches_greedy > 0
        # top_k = 1 keeps only the maximum: the greedy ids exactly
        eng.set_sampling(1.0, 1, None, 99)
        eng.start_decode(ops.sample_advance(eng.prefill(emb), eng.d_sample), NEW)
        eng.decode_steps(B, NEW - 1, sampled=True)
        assert torch.equal(eng.token_log[:B, :NEW], greedy)

    runs = []
    for s, chunk in ((7, 16), (7, 3), (8, 16)):
        torch.manual_seed(s)
        runs.append(m.generate(ids, do_sample=True, temperature=1.0, max_new_tokens=NEW, eos_token_id=-1, sync_every=chunk))
    assert runs[0].shape == (B, S + NEW)
    assert torch.equal(runs[0], runs[1])
    assert not torch.equal(runs[0], runs[2])
    assert torch.equal(m.generate(ids, do_sample=True, top_k=1, max_new_tokens=NEW, eos_token_id=-1)[:, S:], greedy)
    eos = int(runs[0][0, S])
    torch.manual_seed(7)
    got = m.generate(ids, do_sample=True, temperature=1.0, max_new_tokens=NEW, eos_token_id=eos, pad_token_id=0)
    assert int(got[0, S]) == eos and bool((got[0, S + 1:] == 0).all())
