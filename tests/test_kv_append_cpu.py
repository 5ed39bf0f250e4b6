"""CPU (no GPU): incremental `forward(past_key_values=...)` host logic. The kernels are replaced by the torch statements of
tests/cpu_ops_emulator.py plus the statement of vb200_attention_paged below; the model runs on the golden tiny LLM
(tests/golden/vitron_llm_tiny.pt) and is compared with its own single forward and with oracle/restate_llm.py::LlamaCPU
run as a prefill plus multi-token chunks. The kernel itself is checked on the GPU (test_kv_append_gpu.py)."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16 = torch.bfloat16


def attention_paged(q, k_pages, v_pages, block_table, q_start, q_len, max_kv_len, scale=None, out=None):
    """Statement of vb200_attention_paged: query i of row b sees cache keys j <= q_start[b] + i; rows i >= q_len[b] = 0."""
    B, Sq, H, D = q.shape
    P = k_pages.shape[2]
    scale = D ** -0.5 if scale is None else scale
    o = torch.zeros((B, Sq, H, D), dtype=BF16)
    for b in range(B):
        s0, n = int(q_start[b]), int(q_len[b])
        T = s0 + n
        assert T <= max_kv_len
        pages = block_table[b, :(T + P - 1) // P].long()
        kk = k_pages[pages].permute(1, 0, 2, 3).reshape(H, -1, D)[:, :T].float()
        vv = v_pages[pages].permute(1, 0, 2, 3).reshape(H, -1, D)[:, :T].float()
        s = torch.einsum("qhd,hkd->hqk", q[b, :n].float(), kk) * scale
        allowed = torch.arange(T)[None, :] <= (s0 + torch.arange(n))[:, None]
        s = s.masked_fill(~allowed[None], float("-inf"))
        o[b, :n] = torch.einsum("hqk,hkd->qhd", s.softmax(-1), vv).to(BF16)
    if out is not None:
        out.copy_(o)
        return out
    return o


@pytest.fixture
def fx():
    return torch.load(os.path.join(ROOT, "tests", "golden", "vitron_llm_tiny.pt"), weights_only=False)


@pytest.fixture
def model(monkeypatch, fx):
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200 import ops
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    cpu_ops_emulator.install(monkeypatch)
    monkeypatch.setattr(ops, "attention_paged", attention_paged)
    vit = dict(fx["vit"], hidden_act="gelu")
    cfg = VitronConfig(llm=fx["llm"], vision=VisionConfig(**vit), tokenizer_model_max_length=4096)
    m = VitronLlamaForCausalLM(cfg, "cpu", max_batch=4, max_seq_len=256)
    m.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"]))
    return m


def _ids(B, S, seed, V=320):
    return torch.randint(3, V, (B, S), generator=torch.Generator().manual_seed(seed))


def _close(got, ref, inf=0.01, l2=0.01):
    got, ref = got.float(), ref.float()
    e_inf = ((got - ref).abs().max() / (ref.abs().max() + 1e-6)).item()
    e_l2 = ((got - ref).norm() / (ref.norm() + 1e-6)).item()
    assert e_inf < inf and e_l2 < l2, (e_inf, e_l2)


def test_chunked_forward_equals_full_forward_and_oracle(model, fx):
    from oracle import restate_llm as R
    from oracle.weights import seeded_state_dict
    ids = _ids(2, 21, 0)
    full = model.forward(input_ids=ids).logits
    out = model.forward(input_ids=ids[:, :9], use_cache=True)
    assert out.past_key_values.lens == [9, 9] and out.past_key_values.seq_len == 9
    logits = [out.logits]
    past = out.past_key_values
    for a, b in ((9, 10), (10, 16), (16, 21)):          # one-token and multi-token chunks
        o = model.forward(input_ids=ids[:, a:b], past_key_values=past, attention_mask=torch.ones((2, b)), use_cache=True)
        assert o.logits.shape == (2, b - a, 320)
        logits.append(o.logits)
        past = o.past_key_values
    assert past.lens == [21, 21]
    chunked = torch.cat(logits, 1)
    _close(chunked, full)

    # LlamaCPU with its torch.cat cache, run as the same prefill + chunks
    sd = {k: v.float() for k, v in seeded_state_dict(fx["shapes"], fx["seed"]).items()}
    ref = R.LlamaCPU(sd, fx["llm"])
    ref.kv = [None] * fx["llm"]["num_hidden_layers"]
    hs = [ref._layers(sd["model.embed_tokens.weight"][ids[:, a:b]], a) for a, b in ((0, 9), (9, 10), (10, 16), (16, 21))]
    h = R.rms_norm(torch.cat(hs, 1), sd["model.norm.weight"], 1e-5)
    _close(chunked, F.linear(h, sd["lm_head.weight"]), 0.05, 0.04)


def test_left_padded_ragged_rows(model):
    ids = _ids(3, 18, 1)
    am = torch.ones((3, 18), dtype=torch.long)
    am[0, :4] = 0                                     # left padding: rows cache 8, 12 and 10 prefix tokens
    am[2, :2] = 0
    full = model.forward(input_ids=ids, attention_mask=am).logits
    pre = model.forward(input_ids=ids[:, :12], attention_mask=am[:, :12], use_cache=True)
    assert pre.past_key_values.lens == [8, 12, 10]
    suf = model.forward(input_ids=ids[:, 12:], attention_mask=am, past_key_values=pre.past_key_values)
    assert suf.past_key_values.lens == [14, 18, 16]
    got = torch.cat([pre.logits, suf.logits], 1)
    valid = am.bool()
    _close(got[valid], full[valid])
    assert got[~valid].abs().max() == 0


def test_image_inside_a_chunk(model, fx):
    """Rows of the chunk expand to different lengths (one image vs two): right-padded internally, logits in the layout a
    single forward produces."""
    imgs = [fx["img"]["images"][0], fx["img"]["images"][1], fx["img"]["images"][0]]
    ids = torch.tensor([[1, 116, 90, -200, 98, 171, 39],
                        [1, 256, -200, 74, -200, 301, 5]])
    labels = ids.clone().masked_fill(ids < 0, -100)
    full = model.forward(input_ids=ids, images=imgs, labels=labels)
    lens = model._last_lens
    pre = model.forward(input_ids=ids[:, :2], use_cache=True)
    suf = model.forward(input_ids=ids[:, 2:], attention_mask=torch.ones((2, 7)), past_key_values=pre.past_key_values,
                        images=imgs, labels=labels[:, 2:])
    n_img = (full.logits.shape[1] - 5) // 2           # rows of one image's features (row 1, the longest, holds two)
    assert lens == [7 - 1 + n_img, 7 - 2 + 2 * n_img]
    assert suf.past_key_values.lens == lens and suf.logits.shape[1] == lens[1] - 2
    for b in range(2):
        _close(torch.cat([pre.logits[b], suf.logits[b, :lens[b] - 2]]), full.logits[b, :lens[b]])
    assert suf.logits[0, lens[0] - 2:].abs().max() == 0                # right padding of the shorter row
    assert suf.loss is not None and math.isfinite(float(suf.loss))


def test_branching_and_stale_handles(model):
    ids = _ids(2, 20, 2)
    h = model.forward(input_ids=ids[:, :10], use_cache=True).past_key_values
    a = model.forward(input_ids=ids[:, 10:14], past_key_values=h)
    b = model.forward(input_ids=ids[:, 14:20], past_key_values=h)       # branch: overwrites a's positions
    ref = model.forward(input_ids=torch.cat([ids[:, :10], ids[:, 14:20]], 1)).logits[:, 10:]
    with pytest.raises(ValueError, match="stale"):                    # the reference forward above reset the cache
        model.forward(input_ids=ids[:, :1], past_key_values=b.past_key_values)
    _close(b.logits, ref)

    h = model.forward(input_ids=ids[:, :10], use_cache=True).past_key_values
    a = model.forward(input_ids=ids[:, 10:14], past_key_values=h).past_key_values
    b = model.forward(input_ids=ids[:, 14:16], past_key_values=h).past_key_values   # below a's length: a is stale
    with pytest.raises(ValueError, match="stale"):
        model.forward(input_ids=ids[:, :1], past_key_values=a)
    with pytest.raises(ValueError, match="stale"):
        a[0]
    c = model.forward(input_ids=ids[:, 16:17], past_key_values=b)     # b and h are still intact
    assert c.past_key_values.lens == [13, 13]
    model.forward(input_ids=ids[:, 16:17], past_key_values=h)
    model.forward(input_ids=ids[:, :3])                                # forward without past: every handle stale
    with pytest.raises(ValueError, match="stale"):
        model.forward(input_ids=ids[:, :1], past_key_values=h)
    h = model.forward(input_ids=ids[:, :10], use_cache=True).past_key_values
    model.generate(ids[:, :4], max_new_tokens=2)
    with pytest.raises(ValueError, match="stale"):
        model.forward(input_ids=ids[:, :1], past_key_values=h)
    assert model.forward(input_ids=ids[:, :4]).past_key_values is None          # use_cache unset: unchanged


def test_append_without_use_cache_still_invalidates_overwritten_handles(model):
    """Scoring candidates from one prefix with use_cache=False writes their K/V all the same: a handle whose positions
    such an append overwrote is stale."""
    ids = _ids(2, 20, 9)
    h = model.forward(input_ids=ids[:, :10], use_cache=True).past_key_values
    a = model.forward(input_ids=ids[:, 10:14], past_key_values=h).past_key_values
    out = model.forward(input_ids=ids[:, 16:18], past_key_values=h, use_cache=False)
    assert out.past_key_values is None
    with pytest.raises(ValueError, match="stale"):
        model.forward(input_ids=ids[:, 14:15], past_key_values=a)
    model.forward(input_ids=ids[:, 18:19], past_key_values=h, use_cache=False)     # h itself stays intact
    ref = model.forward(input_ids=torch.cat([ids[:, :10], ids[:, 16:18]], 1)).logits[:, 10:]
    _close(out.logits, ref)


def test_attention_paged_wrapper_requires_contiguous_block_table():
    from vitron_b200 import build, ops
    build.build()
    pages = torch.zeros((4, 2, 64, 128), dtype=BF16)
    q = torch.zeros((2, 4, 2, 128), dtype=BF16)
    table = torch.zeros((2, 8), dtype=torch.int32)
    rows = torch.zeros((2,), dtype=torch.int32)
    with pytest.raises(ValueError, match="block_table"):        # a column slice: row stride 8, 4 real columns
        ops.attention_paged(q, pages, pages, table[:, :4], rows, rows, 4)


def test_mask_tuple_and_capacity_errors(model):
    ids = _ids(2, 12, 3)
    h = model.forward(input_ids=ids[:, :8], attention_mask=torch.tensor([[1] * 8, [0] * 2 + [1] * 6]),
                      use_cache=True).past_key_values
    assert h.lens == [8, 6]
    ok = torch.tensor([[1] * 12, [0] * 2 + [1] * 10])
    bad_chunk = ok.clone()
    bad_chunk[1, -1] = 0
    bad_past = torch.ones((2, 12), dtype=torch.long)
    for m in (bad_chunk, bad_past, ok[:, :11], ok[:1]):
        with pytest.raises(ValueError, match="attention_mask"):
            model.forward(input_ids=ids[:, 8:], attention_mask=m, past_key_values=h)
    k, v = model.forward(input_ids=ids[:, 8:], attention_mask=ok, past_key_values=h).past_key_values[0]
    with pytest.raises(ValueError, match="PagedPast"):
        model.forward(input_ids=ids[:, 8:], past_key_values=((k, v), (k, v)))
    h = model.forward(input_ids=ids[:, :8], use_cache=True).past_key_values
    with pytest.raises(ValueError, match="exceeds the KV cache capacity"):
        model.forward(input_ids=_ids(2, 250, 4), past_key_values=h)


def test_handle_layers_and_past_len(model):
    ids = _ids(2, 70, 5)
    am = torch.ones((2, 70), dtype=torch.long)
    am[1, :5] = 0
    past = model.forward(input_ids=ids, attention_mask=am, use_cache=True).past_key_values
    cfg = model.engine.cfg
    assert len(past) == cfg.num_hidden_layers and past.lens == [70, 65]
    assert past[-1][-1].shape[-2] == 70 == model._past_len(past)
    k, v = past[-1]
    assert k.shape == v.shape == (2, cfg.num_attention_heads, 70, cfg.head_dim)
    assert v[1, :, 65:].abs().max() == 0 and v[1, :, :65].abs().max() > 0
    # the gathered keys are the cached (RoPE-rotated) ones: the first row's key 66 sits on its second page
    cache = model.engine.cache
    page = cache._owned[0][66 // cache.page_size]
    assert torch.equal(k[0, :, 66], cache.k(cfg.num_hidden_layers - 1)[page, :, 66 % cache.page_size])


def test_generate_after_appends_matches_fresh_model(model, fx):
    ids = _ids(2, 10, 6)
    want = model.generate(ids, max_new_tokens=4, eos_token_id=-1)
    h = model.forward(input_ids=ids[:, :6], use_cache=True).past_key_values
    model.forward(input_ids=ids[:, 6:], past_key_values=h)
    assert torch.equal(model.generate(ids, max_new_tokens=4, eos_token_id=-1), want)


def test_engine_append_rejects_bad_lengths(model):
    eng = model.engine
    eng.prefill(eng.embed[_ids(2, 5, 7)])
    with pytest.raises(ValueError):
        eng.append(eng.embed[_ids(2, 3, 8)], [3, 4])                   # chunk length past the chunk
    with pytest.raises(ValueError):
        eng.append(eng.embed[_ids(2, 3, 8)], [3, 0])
    assert eng.append(eng.embed[_ids(2, 3, 8)], [3, 2], all_logits=False).shape == (2, 320)


def test_attention_paged_argument_validation():
    from vitron_b200 import _lib, build
    build.build()
    lib = _lib.load()
    F_ = 16                                            # a non-null, 16-byte aligned stand-in pointer (never dereferenced)
    args = dict(q=F_, q_sb=3 * 128 * 32 * 8, q_ss=3 * 128 * 32, q_sh=128, k=F_, v=F_, num_pages=64, bt=F_, max_pages=8,
                qs=F_, ql=F_, out=F_, o_sb=128 * 32 * 8, o_ss=128 * 32, o_sh=128, B=2, H=32, Sq=8, hd=128, page=64,
                max_kv=512, scale=0.088, ws=None, wsb=0, stream=None)

    def call(**kw):
        a = dict(args, **kw)
        return lib.vb200_attention_paged(*a.values())
    for null in ("q", "k", "v", "bt", "qs", "ql", "out"):
        assert call(**{null: None}) == -1, null
    assert call(B=0) == -1 and call(Sq=0) == -1 and call(num_pages=0) == -1
    assert call(max_kv=513) == -1                      # past the block table (8 pages of 64)
    assert call(q_ss=100) == -1 and call(o_sh=-8) == -1 and call(q=F_ + 2) == -1
    assert call(hd=64, q_sh=64, o_sh=64) == -4 and call(page=32, max_kv=256) == -4
    assert lib.vb200_attention_paged_workspace_size(1, 32, 128, 128, 896) > 0          # 32 CTAs: split over the keys
    assert lib.vb200_attention_paged_workspace_size(8, 32, 128, 128, 896) == 0         # 256 CTAs: unsplit
    assert lib.vb200_attention_paged_workspace_size(1, 32, 128, 64, 896) == 0
