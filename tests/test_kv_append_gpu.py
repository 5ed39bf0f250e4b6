"""GPU: paged prefill attention (vb200_attention_paged) against an fp32 reference over the gathered pages, and
`LlamaEngine.append` / `forward(past_key_values=...)` against a prefill of the whole sequence and the fp32 oracle."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q_START = [0, 1, 63, 64, 65, 700, 2047]
Q_LEN = [1, 2, 17, 64, 128, 129, 768]


def _rnd(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(BF16)


def _close(a, b, atol, rtol, what=""):
    err = (a.float() - b.float()).abs()
    bad = (err > atol + rtol * b.float().abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


def _paged_case(dev, B, H, starts, lens, seed):
    """Pages in shuffled order, q as the q third of fused qkv rows."""
    P, D = 64, 128
    Sq = max(lens)
    max_pages = (max(s + n for s, n in zip(starts, lens)) + P - 1) // P
    num_pages = B * max_pages + 3
    perm = torch.randperm(num_pages, generator=torch.Generator().manual_seed(seed))
    table = perm[:B * max_pages].view(B, max_pages).to(torch.int32).to(dev)
    kp = _rnd((num_pages, H, P, D), dev, seed + 1)
    vp = _rnd((num_pages, H, P, D), dev, seed + 2)
    qkv = _rnd((B * Sq, 3 * H * D), dev, seed + 3)
    q = qkv.view(B, Sq, 3, H, D)[:, :, 0]
    return q, kp, vp, table


def _paged_ref(q, kp, vp, table, starts, lens):
    B, Sq, H, D = q.shape
    out = torch.zeros((B, Sq, H, D), dtype=torch.float32, device=q.device)
    for b in range(B):
        s0, n = starts[b], lens[b]
        T = s0 + n
        pages = table[b, :(T + 63) // 64].long()
        k = kp[pages].permute(1, 0, 2, 3).reshape(H, -1, D)[:, :T].float()
        v = vp[pages].permute(1, 0, 2, 3).reshape(H, -1, D)[:, :T].float()
        s = torch.einsum("qhd,hkd->hqk", q[b, :n].float(), k) / math.sqrt(D)
        allowed = torch.arange(T, device=q.device)[None, :] <= (s0 + torch.arange(n, device=q.device))[:, None]
        s = s.masked_fill(~allowed[None], float("-inf"))
        out[b, :n] = torch.einsum("hqk,hkd->qhd", s.softmax(-1), v)
    return out


def _cases(B):
    if B == 1:                                       # every (q_start, q_len) pair
        return [([s], [n]) for s in Q_START for n in Q_LEN]
    g = torch.Generator().manual_seed(B)
    out = []
    for _ in range(4):                               # ragged rows
        si = torch.randint(0, len(Q_START), (B,), generator=g).tolist()
        li = torch.randint(0, len(Q_LEN), (B,), generator=g).tolist()
        out.append(([Q_START[i] for i in si], [Q_LEN[i] for i in li]))
    out.append(([Q_START[i % 7] for i in range(B)], [Q_LEN[(i + 3) % 7] for i in range(B)]))
    out.append(([700] * B, [17] * B))                # short chunk over a long past: split over the keys
    return out


@pytest.mark.parametrize("B", [1, 3, 8])
def test_attention_paged_against_fp32(cuda, B):
    from vitron_b200 import _lib, ops
    lib = _lib.load()
    H = {1: 32, 3: 16, 8: 8}[B]                      # chunks of <= 128 queries split over the keys at each B
    paths = set()
    for ci, (starts, lens) in enumerate(_cases(B)):
        q, kp, vp, table = _paged_case(cuda, B, H, starts, lens, 100 * B + ci)
        qs = torch.tensor(starts, dtype=torch.int32, device=cuda)
        ql = torch.tensor(lens, dtype=torch.int32, device=cuda)
        max_kv = max(s + n for s, n in zip(starts, lens))
        paths.add(lib.vb200_attention_paged_workspace_size(B, H, q.shape[1], 128, max_kv) > 0)
        out = ops.attention_paged(q, kp, vp, table, qs, ql, max_kv)
        ref = _paged_ref(q, kp, vp, table, starts, lens)
        what = f"B={B} q_start={starts} q_len={lens}"
        for b in range(B):
            _close(out[b, :lens[b]], ref[b, :lens[b]], 2e-2, 2e-2, what)
            assert out[b, lens[b]:].abs().max().item() == 0 if lens[b] < q.shape[1] else True, what
        assert torch.equal(ops.attention_paged(q, kp, vp, table, qs, ql, max_kv), out), what   # bit-identical
    assert paths == {False, True}, paths               # both the split and the unsplit path ran
    assert ops.attention_watchdog()[0] == 0


MIDSIZE = dict(hidden_size=512, intermediate_size=1408, num_hidden_layers=4, num_attention_heads=4, vocab_size=2000,
               rms_norm_eps=1e-5, rope_theta=10000.0)
VICUNA_4L = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=4, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)


def _engine(cfg, dev, max_batch, max_seq_len, nf4=False):
    from vitron_b200 import param_shapes as PS
    from vitron_b200.llama import LlamaConfig, LlamaEngine
    sd = PS.random_state_dict(PS.llama_shapes(LlamaConfig.from_any(cfg)), dev, seed=1)
    g = torch.Generator(device=dev).manual_seed(2)
    for k in list(sd):
        if "layernorm" in k or k == "model.norm.weight":
            sd[k] = (1 + 0.2 * torch.rand(sd[k].shape, generator=g, device=dev)).to(sd[k].dtype)
    return LlamaEngine(cfg, dev, max_batch=max_batch, max_seq_len=max_seq_len).load_state_dict(sd, nf4=nf4)


def _oracle_chunk_logits(eng, cfg, ids, P):
    """fp32 LlamaCPU (torch.cat KV cache) on the engine's reference-named weights: prefill P, then the chunk."""
    from oracle import restate_llm as R
    sd = {k: v.float() for k, v in eng.state_dict().items()}
    ref = R.LlamaCPU(sd, cfg)
    ref.kv = [None] * cfg["num_hidden_layers"]
    E = sd["model.embed_tokens.weight"]
    with torch.device(ids.device):                   # the oracle's RoPE tables and causal masks on the weights' device
        ref._layers(E[ids[:, :P]], 0)
        h = ref._layers(E[ids[:, P:]], P)
    return F.linear(R.rms_norm(h, sd["model.norm.weight"], cfg["rms_norm_eps"]), sd["lm_head.weight"])


def _check_engine(eng, cfg, dev, B, P, S):
    V = cfg["vocab_size"]
    ids = torch.randint(3, V, (B, P + S), generator=torch.Generator().manual_seed(B * 1000 + S)).to(dev)
    E = eng.embed
    with torch.no_grad():
        full = eng.prefill(E[ids], all_logits=True)[:, P:].clone()
        eng.prefill(E[ids[:, :P]])
        got = eng.append(E[ids[:, P:]], [S] * B).clone()
        oracle = _oracle_chunk_logits(eng, cfg, ids, P)
    scale = oracle.abs().max().item()
    assert (got - full).abs().max().item() <= 0.05 * scale, (B, P, S)
    assert (got - oracle).abs().max().item() <= 0.05 * scale, (B, P, S)
    assert (full - oracle).abs().max().item() <= 0.05 * scale, (B, P, S)
    top2 = oracle.topk(2, -1).values
    decisive = (top2[..., 0] - top2[..., 1]) > 0.05 * scale
    assert torch.equal(got.argmax(-1)[decisive], oracle.argmax(-1)[decisive]), (B, P, S)
    # ragged chunk rows (padding slots are skipped by the K/V scatter, padded queries give zeros)
    lens = [max(1, S - 3 * b) for b in range(B)]
    with torch.no_grad():
        eng.prefill(E[ids[:, :P]])
        rag = eng.append(E[ids[:, P:]], lens).clone()
        ref = eng.prefill(E[ids], [P + n for n in lens], all_logits=True)[:, P:]
    for b, n in enumerate(lens):
        assert (rag[b, :n] - ref[b, :n]).abs().max().item() <= 0.05 * scale, (B, P, S, b)
    return int(decisive.sum())


@pytest.mark.parametrize("nf4", [False, True], ids=["bf16", "nf4"])
def test_engine_append_midsize(cuda, nf4):
    eng = _engine(MIDSIZE, cuda, 8, 256, nf4)
    assert eng.nf4 == nf4
    decisive = sum(_check_engine(eng, MIDSIZE, cuda, B, P, S) for B, P, S in ((1, 100, 1), (8, 64, 37), (3, 130, 120)))
    assert decisive > 0                              # the greedy check compared some tokens


@pytest.mark.parametrize("nf4", [False, True], ids=["bf16", "nf4"])
def test_engine_append_vicuna_layers(cuda, nf4):
    eng = _engine(VICUNA_4L, cuda, 8, 1024, nf4)
    decisive = sum(_check_engine(eng, VICUNA_4L, cuda, B, 768, S) for B in (1, 8) for S in (1, 32, 256))
    assert decisive > 0                              # the greedy check compared some tokens


def _tiny_model(dev):
    from oracle.weights import seeded_state_dict
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "vitron_llm_tiny.pt"), weights_only=False)
    vit = dict(fx["vit"], hidden_act="gelu")
    cfg = VitronConfig(llm=fx["llm"], vision=VisionConfig(**vit), tokenizer_model_max_length=4096)
    m = VitronLlamaForCausalLM(cfg, dev, max_batch=4, max_seq_len=256)
    m.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"]))
    return m, fx


def test_model_image_then_text_chunk(cuda):
    m, fx = _tiny_model(cuda)
    imgs = [i.to(cuda) for i in fx["img"]["images"]]
    ids = torch.tensor([[1, 116, 90, -200, 98, 171, 39, 44, 12, 7],
                        [1, 256, -200, 74, 301, 5, 88, 9, 60, 61]], device=cuda)
    with torch.no_grad():
        full = m.forward(input_ids=ids, images=imgs).logits
        lens = m._last_lens
        pre = m.forward(input_ids=ids[:, :6], images=imgs, use_cache=True)
        past = pre.past_key_values
        suf = m.forward(input_ids=ids[:, 6:], attention_mask=torch.ones((2, past.seq_len + 4), device=cuda),
                        past_key_values=past)
    assert suf.past_key_values.lens == lens == [n + 4 for n in past.lens]
    scale = full.abs().max().item()
    for b in range(2):
        got = torch.cat([pre.logits[b, :past.lens[b]], suf.logits[b]])
        assert (got - full[b, :lens[b]]).abs().max().item() <= 0.05 * scale, b


def test_generate_after_appends_matches_fresh_model(cuda):
    fresh, _ = _tiny_model(cuda)
    used, _ = _tiny_model(cuda)
    ids = torch.randint(3, 320, (2, 12), generator=torch.Generator().manual_seed(0)).to(cuda)
    with torch.no_grad():
        past = used.forward(input_ids=ids[:, :5], use_cache=True).past_key_values
        past = used.forward(input_ids=ids[:, 5:9], past_key_values=past).past_key_values
        used.forward(input_ids=ids[:, 9:], past_key_values=past)
        a = used.generate(ids, max_new_tokens=8, eos_token_id=-1)
        b = fresh.generate(ids, max_new_tokens=8, eos_token_id=-1)
    assert torch.equal(a, b)
