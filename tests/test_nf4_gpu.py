"""GPU: the NF4 kernels (csrc/gemv_nf4.cu) against the statement of vitron_b200/nf4.py, and an NF4 engine against a bf16
engine that holds the same W_eff. Everything is compared with W_eff, never with the unquantised weights."""
import pytest
import torch

from vitron_b200 import nf4

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
VICUNA_SHAPES = [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008)]


def _weight(n, k, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return nf4.quantize((torch.randn((n, k), generator=g, device=dev) * 0.02).to(BF16))


@pytest.mark.parametrize("n, k", VICUNA_SHAPES + [(200, 192), (37, 64)])
def test_dequant_bit_identical(cuda, n, k):
    from vitron_b200 import ops
    w = _weight(n, k, cuda, n + k)
    ks = torch.rand((k,), device=cuda) + 0.5
    assert torch.equal(ops.nf4_dequant(w), nf4.dequantize(w).to(BF16))
    assert torch.equal(ops.nf4_dequant(w, ks), (nf4.dequantize(w) * ks[None, :]).to(BF16))


@pytest.mark.parametrize("n, k", VICUNA_SHAPES + [(1000, 4096), (2000, 1408)])
@pytest.mark.parametrize("m", [1, 8, 9, 16, 17, 32])
def test_gemm_nf4_against_w_eff(cuda, m, n, k):
    from vitron_b200 import ops
    w = _weight(n, k, cuda, 7 * n + k)
    g = torch.Generator(device=cuda).manual_seed(m)
    x = torch.randn((m, k), generator=g, device=cuda).to(BF16)
    ks = (torch.rand((k,), generator=g, device=cuda) + 0.5).contiguous()
    weff = nf4.dequantize(w)
    glu = n == 22016
    n_out = n // 2 if glu else n
    bias = (torch.randn((n,), generator=g, device=cuda) * 0.1).to(BF16)
    res = torch.randn((m, n_out), generator=g, device=cuda).to(BF16)

    def ref(xs, rms, use_bias, use_res):
        v = xs.float() @ weff.t()
        if rms:
            v = v * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + 1e-5)
        if use_bias:
            v = v + bias.float()
        if glu:
            blk = v.reshape(m, n // 32, 2, 16)
            v = torch.nn.functional.silu(blk[:, :, 0].reshape(m, -1)) * blk[:, :, 1].reshape(m, -1)
        if use_res:
            v = v + res.float()
        return v

    xk = (x.float() * ks[None, :]).to(BF16)       # the kernel rounds X * kscale to bf16 before the products
    cases = [dict(), dict(rms=True, kscale=True), dict(bias=True, res=True), dict(rms=True, res=True, fp32=True, kscale=True)]
    for cs in cases:
        got = ops.gemm(x, w, glu=ops.GLU_SWIGLU if glu else ops.GLU_NONE, rms_eps=1e-5 if cs.get("rms") else 0.0,
                       bias=bias if cs.get("bias") else None, residual=res if cs.get("res") else None,
                       out_fp32=bool(cs.get("fp32")), kscale=ks if cs.get("kscale") else None)
        want = ref(xk if cs.get("kscale") else x, cs.get("rms"), cs.get("bias"), cs.get("res"))
        assert got.dtype == (torch.float32 if cs.get("fp32") else BF16)
        err = (got.float() - want).abs().max().item()
        assert err <= 3e-2 * want.abs().max().item() + 2e-2, (cs, err)


def test_gemm_nf4_repeatable(cuda):
    from vitron_b200 import ops
    w = _weight(22016, 4096, cuda, 3)
    x = torch.randn((17, 4096), device=cuda).to(BF16)
    ks = torch.rand((4096,), device=cuda) + 0.5
    a = ops.gemm(x, w, glu=ops.GLU_SWIGLU, rms_eps=1e-5, kscale=ks)
    for _ in range(3):
        assert torch.equal(ops.gemm(x, w, glu=ops.GLU_SWIGLU, rms_eps=1e-5, kscale=ks), a)


MIDSIZE = dict(hidden_size=512, intermediate_size=1408, num_hidden_layers=4, num_attention_heads=4, vocab_size=2000,
               rms_norm_eps=1e-5, rope_theta=10000.0)
VICUNA_4L = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=4, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)


def _engines(cfg, dev, max_batch, max_seq_len):
    """An NF4 engine loaded from a seeded state dict (non-unit RMSNorm gains) and a bf16 engine holding its W_eff."""
    from vitron_b200 import param_shapes as PS
    from vitron_b200.llama import LlamaConfig, LlamaEngine
    sd = PS.random_state_dict(PS.llama_shapes(LlamaConfig.from_any(cfg)), dev, seed=1)
    g = torch.Generator(device=dev).manual_seed(2)
    for k in list(sd):
        if "layernorm" in k or k == "model.norm.weight":
            sd[k] = (1 + 0.2 * torch.rand(sd[k].shape, generator=g, device=dev)).to(sd[k].dtype)
    e4 = LlamaEngine(cfg, dev, max_batch=max_batch, max_seq_len=max_seq_len).load_state_dict(sd, nf4=True)
    weff = e4.state_dict()
    for k in list(sd):
        if "_proj" in k:
            sd[k] = weff[k]
    e16 = LlamaEngine(cfg, dev, max_batch=max_batch, max_seq_len=max_seq_len).load_state_dict(sd)
    return e4, e16


@pytest.mark.parametrize("cfg", [MIDSIZE, VICUNA_4L], ids=["midsize", "vicuna4l"])
def test_nf4_engine_against_bf16_weff(cuda, cfg):
    from vitron_b200 import ops
    S, NEW = 40, 10
    e4, e16 = _engines(cfg, cuda, 32, S + 2 * NEW)
    assert e4.nf4 and not e16.nf4
    assert e4.weight_bytes() < 0.45 * e16.weight_bytes()
    V = cfg["vocab_size"]
    for B in (8, 17, 32):
        ids = torch.randint(3, V, (B, S), generator=torch.Generator().manual_seed(B)).to(cuda)
        with torch.no_grad():
            l4, l16 = e4.prefill(e4.embed[ids]), e16.prefill(e16.embed[ids])
            scale = l16.abs().max().item()
            assert (l4 - l16).abs().max().item() <= 0.05 * scale, B
            # teacher-forced decode logits
            toks = ops.argmax_rows(l16)
            for _ in range(3):
                d4, d16 = e4.decode_one_logits(toks).clone(), e16.decode_one_logits(toks).clone()
                assert (d4 - d16).abs().max().item() <= 0.05 * d16.abs().max().item(), B
                toks = ops.argmax_rows(d16)
            # greedy graphed decode: tokens agree wherever the bf16 engine's top-2 margin is decisive
            runs = []
            for eng in (e4, e16, e4):
                logits = eng.prefill(eng.embed[ids])
                eng.start_decode(ops.argmax_rows(logits), NEW)
                eng.decode_steps(B, NEW - 1)
                runs.append(eng.token_log[:B, :NEW].clone())
            assert torch.equal(runs[0], runs[2]), B                       # reproducible across runs
            assert e4.launches_per_step <= e16.launches_per_step
            if B <= 16:
                assert e4.launches_per_step == e16.launches_per_step   # the same kernels, one NF4 GEMV per projection
            # first step: prefill logits decide token 0 for both engines
            top2 = l16.topk(2, -1).values
            decisive = (top2[:, 0] - top2[:, 1]) > 0.1 * scale
            assert torch.equal(runs[0][decisive, 0], runs[1][decisive, 0]), B


def test_nf4_sampled_decode(cuda):
    from vitron_b200 import ops
    e4, _ = _engines(MIDSIZE, cuda, 8, 64)
    ids = torch.randint(3, 2000, (8, 24), generator=torch.Generator().manual_seed(0)).to(cuda)
    out = []
    for _ in range(2):
        e4.set_sampling(0.8, 40, 0.9, seed=123)
        e4.start_decode(ops.sample_advance(e4.prefill(e4.embed[ids]), e4.d_sample), 12)
        e4.decode_steps(8, 11, sampled=True)
        out.append(e4.token_log[:8, :12].clone())
    assert torch.equal(out[0], out[1])
    assert bool((out[0] >= 0).all() and (out[0] < 2000).all())


def test_nf4_vitron_model_generate(cuda):
    """load_state_dict(nf4=True) on the full drop-in (projector and region extractor in NF4) runs generate."""
    import os
    from oracle.weights import seeded_state_dict
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fx = torch.load(os.path.join(root, "tests", "golden", "vitron_llm_tiny.pt"), weights_only=False)
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    vit = dict(fx["vit"], hidden_act="gelu")
    cfg = VitronConfig(llm=fx["llm"], vision=VisionConfig(**vit),
                       video=VisionConfig(**vit, add_time_attn=True, num_frames=fx["num_frames"]),
                       tokenizer_model_max_length=4096)
    model = VitronLlamaForCausalLM(cfg, cuda, max_batch=2, max_seq_len=256)
    model.load_state_dict(sd, nf4=True)
    assert isinstance(model.get_model().mm_projector.linears[0][0], nf4.NF4Weight)
    g = fx["gen_img"]
    with torch.no_grad():
        out = model.generate(g["input_ids"].to(cuda), images=[i.to(cuda) for i in g["images"]], regions=g["regions"],
                             do_sample=False, max_new_tokens=6, eos_token_id=-1)
    assert out.shape[1] == g["input_ids"].shape[1] + 6
