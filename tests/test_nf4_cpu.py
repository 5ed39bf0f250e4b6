"""CPU: the NF4 statement (vitron_b200/nf4.py) against literal per-element computations, argument validation of the NF4
entry points without a device, and `load_pretrained_model(..., load_4bit=True)` host logic with the NF4 GEMM replaced by
its torch statement."""
import json
import os

import numpy as np
import pytest
import torch

from vitron_b200 import nf4


def test_tables():
    assert nf4.NF4.shape == (16,) and nf4.NF4[7] == 0 and nf4.NF4[0] == -1 and nf4.NF4[15] == 1
    assert bool((nf4.NF4[1:] > nf4.NF4[:-1]).all())
    d = nf4.dynamic_map()
    assert d.shape == (256,) and bool((d[1:] >= d[:-1]).all())
    assert (d == 0).sum() == 1 and (d == 1.0).sum() == 1
    assert int((d > 0).sum()) == 128 and int((d < 0).sum()) == 127     # 127 positive midpoints + 1.0, 127 negative
    pos = sorted(x for x in d.tolist() if 0 < x < 1)
    assert pos == sorted(-x for x in d.tolist() if x < 0)                 # the negative half mirrors the positive one
    # the decade of exponent i holds 2^i midpoints of linspace(0.1, 1, 2^i + 1) * 10^(i - 6)
    for i in range(7):
        lo, hi = 0.1 * 10 ** (i - 6), 10 ** (i - 6)
        assert sum(1 for x in pos if lo <= x < hi) == 2 ** i, i


def _literal_codes(w):
    table = nf4.NF4.numpy()
    w = w.numpy().astype(np.float32)
    n, k = w.shape
    out = np.zeros((n, k), np.uint8)
    for r in range(n):
        for b in range(k // 64):
            blk = w[r, b * 64:(b + 1) * 64]
            am = np.float32(np.abs(blk).max())
            for e in range(64):
                if am == 0:
                    out[r, b * 64 + e] = 7
                    continue
                v = np.float32(blk[e] * np.float32(np.float32(1.0) / am))
                dist = [abs(np.float32(v - np.float32(t))) for t in table]
                out[r, b * 64 + e] = int(np.argmin(dist))     # first minimum: ties go to the lower index
    return out


def test_codes_match_literal_argmin_with_ties_and_zero_blocks():
    g = torch.Generator().manual_seed(0)
    w = torch.randn((6, 192), generator=g)
    w[1, 64:128] = 0                                          # an all-zero block
    mids = ((nf4.NF4[1:] + nf4.NF4[:-1]) / 2)                 # planted midpoint ties in a block whose absmax is 1
    w[2, :64] = 0
    w[2, 0] = 1.0
    w[2, 1:16] = mids
    w[2, 16:31] = -mids
    codes, absmax = nf4.quantize_codes(w)
    assert codes.dtype == torch.uint8
    assert np.array_equal(codes.numpy(), _literal_codes(w))
    assert bool((codes[1, 64:128] == 7).all())
    assert torch.equal(absmax, w.abs().reshape(6, 3, 64).amax(-1))


def test_scales_match_literal_double_quant():
    g = torch.Generator().manual_seed(1)
    absmax = torch.rand((7, 100), generator=g) * 0.3           # 700 values: two full 256-blocks and a partial one
    got = nf4.double_quant_scales(absmax).reshape(-1)
    flat = absmax.reshape(-1)
    offset = np.float32(flat.mean().item())
    dmap = nf4.dynamic_map().numpy()
    x = (flat - torch.tensor(offset)).numpy().astype(np.float32)
    for b0 in range(0, x.size, 256):
        blk = x[b0:b0 + 256]
        a2 = np.float32(np.abs(blk).max())
        for e, v in enumerate(blk):
            q = int(np.argmin(np.abs(np.float32(v * np.float32(np.float32(1) / a2)) - dmap)))
            want = np.float32(np.float32(dmap[q] * a2) + offset)
            assert got[b0 + e].item() == pytest.approx(float(want), rel=0, abs=1e-7), (b0 + e)


def test_pack_roundtrip_dequantize_and_k_check():
    g = torch.Generator().manual_seed(2)
    for k in (64, 128, 192, 4096 + 64):
        w = torch.randn((5, k), generator=g, dtype=torch.float32).to(torch.bfloat16)
        q = nf4.quantize(w)
        assert q.codes.shape == (5, (k + 127) // 128 * 64) and q.scales.shape == (5, k // 64)
        assert q.scales.dtype == torch.float16 and q.shape == (5, k)
        codes, absmax = nf4.quantize_codes(w)
        assert torch.equal(nf4.unpack_codes(q.codes, k), codes)
        scale = nf4.double_quant_scales(absmax).to(torch.float16).float()
        want = nf4.NF4[codes.long()] * scale.repeat_interleave(64, 1)
        assert torch.equal(nf4.dequantize(q), want)
        # half the widest NF4 gap (-1 .. -0.696) of the block's absmax, plus the fp16 / double-quant scale error
        assert ((nf4.dequantize(q) - w.float()).abs().reshape(5, -1, 64) <= 0.16 * w.float().abs().reshape(5, -1, 64).amax(-1, keepdim=True)).all()
    # lane t of superchunk s holds the codes of k = 128 s + 64 u + 32 h + 8 t + e in byte t*16 + u*8 + h*4 + e/2
    codes = torch.arange(128, dtype=torch.int64).remainder(16).to(torch.uint8)[None]
    packed = nf4.pack_codes(codes)
    t, u, h, e = 2, 1, 0, 6
    byte = packed[0, t * 16 + u * 8 + h * 4 + e // 2].item()
    k = 64 * u + 32 * h + 8 * t + e
    assert byte == (k % 16) | ((k + 1) % 16) << 4
    with pytest.raises(ValueError):
        nf4.quantize(torch.zeros((4, 96)))


def test_argument_validation_without_device():
    import ctypes as C
    from vitron_b200 import _lib, build
    from vitron_b200._lib import Epilogue
    build.build()
    lib = _lib.load()
    epi = Epilogue()
    buf = C.create_string_buffer(256)
    p = C.addressof(buf) + (-C.addressof(buf)) % 16
    assert lib.vb200_gemm_nf4(None, 64, p, p, None, p, 64, 1, 64, 64, C.byref(epi), None) == -1
    assert lib.vb200_gemm_nf4(p, 96, p, p, None, p, 64, 1, 64, 96, C.byref(epi), None) == -1       # K % 64
    assert lib.vb200_gemm_nf4(p, 64, p, p, None, p, 64, 33, 64, 64, C.byref(epi), None) == -4      # M > 32
    assert lib.vb200_gemm_nf4(p, 64, p + 1, p, None, p, 64, 1, 64, 64, C.byref(epi), None) == -1   # misaligned codes
    ks = C.cast(p + 4, C.POINTER(C.c_float))
    assert lib.vb200_gemm_nf4(p, 64, p, p, ks, p, 64, 1, 64, 64, C.byref(epi), None) == -1         # misaligned kscale
    assert lib.vb200_gemm_nf4(p, 68, p, p, None, p, 64, 1, 64, 64, C.byref(epi), None) == -1       # lda % 8 != 0
    assert lib.vb200_gemm_nf4(p, 64, p, p, None, p, 63, 1, 64, 64, C.byref(epi), None) == -1       # ldo < N
    epi.glu = 1
    assert lib.vb200_gemm_nf4(p, 64, p, p, None, p, 64, 1, 48, 64, C.byref(epi), None) == -1      # GLU needs N % 32
    assert lib.vb200_gemm_nf4(p, 64, p, p, None, p, 31, 1, 64, 64, C.byref(epi), None) == -1      # ldo < N / 2
    assert lib.vb200_nf4_dequant(None, p, None, p, 4, 64, None) == -1
    assert lib.vb200_nf4_dequant(p, p, None, p, 4, 100, None) == -1
    assert lib.vb200_nf4_dequant(p, p, None, p + 8, 4, 64, None) == -1


def nf4_gemm_statement(monkeypatch):
    """ops.gemm over the torch statements of tests/cpu_ops_emulator.py, with NF4 weights taken to
    bf16_rn(W_eff * kscale) (the nf4_dequant contract) before the product."""
    from tests import cpu_ops_emulator
    from vitron_b200 import ops
    cpu_ops_emulator.install(monkeypatch)
    dense = cpu_ops_emulator.gemm
    calls = []

    def gemm(a, w, kscale=None, **kw):
        if isinstance(w, nf4.NF4Weight):
            calls.append(w.shape)
            wd = nf4.dequantize(w)
            w = (wd * kscale[None, :] if kscale is not None else wd).to(torch.bfloat16)
        return dense(a, w, **kw)
    monkeypatch.setattr(ops, "gemm", gemm)
    return calls


def test_load_4bit_checkpoint_and_generate(tmp_path, monkeypatch):
    from oracle.weights import seeded_state_dict
    from tests.test_builder_cpu import GOLD, DummyTokenizer
    calls = nf4_gemm_statement(monkeypatch)
    from vitron_b200 import builder
    fx = torch.load(os.path.join(GOLD, "vitron_llm_tiny.pt"), weights_only=False)
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    llm, vit = fx["llm"], fx["vit"]
    ck, cache = tmp_path / "Vitron-merged", tmp_path / "cache"
    for d in (ck, cache / "LanguageBind_Image"):
        d.mkdir(parents=True)
    cfg = dict(llm, model_type="llava", mm_image_tower="LanguageBind_Image", mm_projector_type="mlp2x_gelu",
               mm_use_im_start_end=False, mm_use_im_patch_token=True, rms_norm_eps=1e-5, rope_theta=10000.0)
    json.dump(cfg, open(ck / "config.json", "w"))
    json.dump(dict(vision_config=dict(vit, hidden_act="gelu")), open(cache / "LanguageBind_Image" / "config.json", "w"))
    torch.save({k: v.to(torch.bfloat16) for k, v in sd.items()}, ck / "pytorch_model.bin")
    V = llm["vocab_size"]
    with pytest.raises(ValueError):
        builder.load_pretrained_model(str(ck), None, "vitron-llava-7b", True, False, device="cpu", tokenizer=DummyTokenizer(V))
    tok, model, proc, ctx = builder.load_pretrained_model(str(ck), None, "vitron-llava-7b", False, True, device="cpu",
                                                          cache_dir=str(cache), tokenizer=DummyTokenizer(V), max_batch=2,
                                                          max_seq_len=128)
    eng = model.engine
    assert eng.nf4 and eng.embed.dtype == torch.bfloat16 and eng.lm_head.dtype == torch.bfloat16
    for L in eng.layers:
        assert all(isinstance(L[n], nf4.NF4Weight) for n in ("wqkv", "wo", "wgu", "wdown"))
        assert L["g1"].dtype == torch.float32
    m = model.get_model()
    assert all(isinstance(w, nf4.NF4Weight) for w, _ in m.mm_projector.linears)
    assert all(b.dtype == torch.bfloat16 for _, b in m.mm_projector.linears)
    assert all(isinstance(w, nf4.NF4Weight) for w, _ in m.region_extractor.mlp)
    assert isinstance(m.region_extractor.loc[1][0], nf4.NF4Weight) and m.region_extractor.loc[0][0].dtype == torch.bfloat16
    # state_dict hands back W_eff under the reference names
    got = model.state_dict()
    q = nf4.quantize(sd["model.layers.1.mlp.up_proj.weight"].to(torch.bfloat16))
    assert torch.equal(got["model.layers.1.mlp.up_proj.weight"], nf4.dequantize(q).to(torch.bfloat16))
    w = sd["model.layers.0.self_attn.k_proj.weight"].to(torch.bfloat16).float()
    assert (got["model.layers.0.self_attn.k_proj.weight"].float() - w).abs().max() <= 0.16 * w.abs().max()
    assert eng.weight_bytes() < 2 * sum(v.numel() for k, v in sd.items() if "_proj" in k or k == "lm_head.weight")
    # generate() host logic runs on the NF4 weights
    ids = torch.tensor([[1, 5, 9, 11, 4, 7]])
    out = model.generate(ids, do_sample=False, max_new_tokens=4, eos_token_id=-1)
    assert out.shape == (1, 10) and torch.equal(out[:, :6], ids)
    assert calls and all(len(s) == 2 for s in calls)
    # the same tokens as a bf16 engine holding W_eff, with the gains applied as the column scale
    ref = {k: v.to(torch.bfloat16) for k, v in sd.items()}
    for n, t in got.items():
        if ".layers." in n and "_proj" in n:
            ref[n] = t
    from vitron_b200.llama import LlamaEngine
    e2 = LlamaEngine(llm, "cpu", max_batch=2, max_seq_len=128).load_state_dict(ref)
    lg1 = eng.prefill(eng.embed[ids[0]].unsqueeze(0))
    emb2 = torch.zeros_like(eng.embed)
    emb2[:V] = e2.embed[:V]
    lg2 = e2.prefill(emb2[ids[0]].unsqueeze(0))
    assert (lg1[:, :V] - lg2).abs().max() <= 0.05 * lg2.abs().max()
