"""CPU (no GPU): the C-ABI library builds/loads and exports every symbol include/vitron_b200.h declares;
the ctypes signature table covers exactly those symbols; argument validation works without a device;
host-side splice layout equals the oracle's restatement of the reference loop."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from vitron_b200 import _lib, build
    build.build()
    return _lib.load()


def header_symbols():
    text = open(os.path.join(ROOT, "include", "vitron_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vb200_\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol(lib):
    from vitron_b200 import _lib
    syms = header_symbols()
    assert len(syms) >= 27
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/vitron_b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == syms, set(_lib.SIGNATURES) ^ set(syms)
    assert b"sm_90a" in lib.vb200_version()


def test_argument_validation_without_device(lib):
    import ctypes as C
    from vitron_b200._lib import Epilogue
    epi = Epilogue()
    # null pointers / bad sizes are rejected before anything touches a device
    assert lib.vb200_gemm_bf16(None, 8, None, 8, None, 8, 8, 8, 8, C.byref(epi), None, 0, None) == -1
    assert lib.vb200_rmsnorm(None, 8, None, None, 8, 1, 8, 1e-5, None) == -1
    assert lib.vb200_attention_short(None, None, None, None, 1, 1, 64, 64, *([0] * 17), 1.0, None) == -1
    assert lib.vb200_gemm_bf16_workspace_size(128, 128, 128) == 0
    assert lib.vb200_gemm_bf16_workspace_size(8, 4096, 4096) == 0  # streaming kernel
    assert lib.vb200_gemm_bf16_workspace_size(32, 4096, 4096) > 0


def test_missing_library_fails_loudly(monkeypatch):
    from vitron_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libvitron_b200.so")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.load()


def test_glu_weight_packing_layout():
    from vitron_b200 import ops
    a = torch.arange(32 * 2, dtype=torch.float32).reshape(32, 2)
    b = -a
    w = ops.pack_glu_weight(a, b)
    assert w.shape == (64, 2)
    assert torch.equal(w[:16], a[:16]) and torch.equal(w[16:32], b[:16]) and torch.equal(w[32:48], a[16:])


def test_conv_weight_packing_layout():
    from vitron_b200 import ops
    w = torch.randn(5, 3, 3, 3)
    p = ops.pack_conv_weight(w)
    assert p.shape == (5, 9, 64) and p[:, :, 3:].abs().sum() == 0
    assert torch.allclose(p[2, 4, :3].float(), w[2, :, 1, 1].to(torch.bfloat16).float())
    w3 = torch.randn(4, 6, 3, 1, 1)
    assert ops.pack_conv_weight(w3).shape == (4, 3, 64)


def test_host_splice_layout_matches_oracle():
    from oracle import restate_llm as R
    from vitron_b200.vitron_model import layout_multimodal
    g = torch.Generator().manual_seed(0)
    d, V = 8, 50
    E = torch.randn((V, d), generator=g)
    feats = [torch.randn((4, d), generator=g) for _ in range(5)]          # 2 images + 3 video frames
    rfeats = [torch.randn((1, d), generator=g), torch.randn((1, d), generator=g), None, None, None]
    ids = torch.tensor([[1, 7, -200, 9, -300, 4, 0, 0, 0],
                        [1, -200, 8, 8, 8, -300, 3, 2, 6],
                        [1, -200, -200, -200, 5, 6, 0, 0, 0]])
    am = torch.tensor([[1] * 6 + [0] * 3, [1] * 9, [1] * 6 + [0] * 3]).bool()
    for left in (False, True):
        src, lab, m, pid, lens = layout_multimodal(ids, am, torch.full_like(ids, -100), [4] * 5,
                                                   [1, 1, None, None, None], 16, left)
        buf = torch.cat(feats + [r for r in rfeats if r is not None], 0)
        got = torch.zeros((*src.shape, d))
        for b in range(src.shape[0]):
            for s in range(src.shape[1]):
                v = int(src[b, s])
                if v >= 0:
                    got[b, s] = E[v]
                elif v != -2147483648:
                    got[b, s] = buf[-v - 1]
        want, wlens = R.splice({"model.embed_tokens.weight": E}, ids, am, feats, rfeats, True, 16,
                               "left" if left else "right")
        assert lens == wlens == [9, 12, 15]
        assert torch.equal(got, want)
        assert m.sum(1).tolist() == lens and (pid.max(1).values + 1).tolist() == lens
    # truncation to tokenizer_model_max_length
    src, *_ , lens = layout_multimodal(ids, am, torch.full_like(ids, -100), [4] * 5, [1, 1, None, None, None], 10, False)
    assert lens == [9, 10, 10] and src.shape[1] == 10
    with pytest.raises(ValueError):
        layout_multimodal(torch.tensor([[1, -300, 2]]), torch.ones((1, 3), dtype=torch.bool), torch.zeros((1, 3), dtype=torch.long), [4], None, None, False)


def test_focalnet_shape_table_matches_reference_names():
    """vitron_b200.param_shapes.focalnet_shapes == state-dict names / shapes of the unmodified reference class
    (recorded in tests/golden/focal_tiny.pt by oracle/gen_golden.py)."""
    import os
    import torch
    from vitron_b200 import param_shapes
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "focal_tiny.pt"), weights_only=False)
    assert param_shapes.focalnet_shapes(fx["cfg"]) == fx["shapes"]


def _rel(got, ref):
    got, ref = got.float(), ref.float()
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-6)).item(), ((got - ref).norm() / (ref.norm() + 1e-6)).item()


def test_focalnet_host_logic_against_reference_golden(monkeypatch):
    """Host side of vitron_b200.focal.FocalNet (weight folding / padding, in-place column slices, call order) with
    the kernels replaced by their torch statements (tests/cpu_ops_emulator.py): must reproduce the unmodified
    reference's golden outputs to bf16 accuracy. The kernels proper are checked on the GPU (test_zfocal_gpu.py)."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.focal import FocalNet
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "focal_tiny.pt"), weights_only=False)
    c = fx["cfg"]
    net = FocalNet(patch_size=c["patch_size"], embed_dim=c["embed_dim"], depths=c["depths"], mlp_ratio=c["mlp_ratio"],
                   patch_norm=c["patch_norm"], out_indices=c["out_indices"], focal_levels=c["focal_levels"],
                   focal_windows=c["focal_windows"], use_conv_embed=True, use_postln=c["use_postln"],
                   use_postln_in_modulation=c["use_postln_in_modulation"], scaling_modulator=c["scaling_modulator"],
                   use_layerscale=c["use_layerscale"], device="cpu")
    net.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"]))
    outs = net(fx["x"])
    for k, ref in fx["outs"].items():
        assert tuple(outs[k].shape) == tuple(ref.shape)
        e_inf, e_l2 = _rel(outs[k], ref)
        assert e_inf < 0.04 and e_l2 < 0.03, (k, e_inf, e_l2)


def test_focalnet_host_logic_preln_and_ragged(monkeypatch):
    import torch
    from oracle import restate_focal as FR
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200 import param_shapes
    from vitron_b200.focal import FocalNet
    cpu_ops_emulator.install(monkeypatch)
    cfg = dict(FR.FOCAL_L, embed_dim=64, depths=(1, 1, 1, 1), use_postln=False, use_postln_in_modulation=True,
               scaling_modulator=False, focal_levels=(3, 2, 2, 1), focal_windows=(5, 3, 7, 3))
    sd = seeded_state_dict(param_shapes.focalnet_shapes(cfg), 7)
    x = torch.randn((2, 3, 62, 90), generator=torch.Generator().manual_seed(2))
    ref = FR.focalnet_forward(sd, x, cfg)
    net = FocalNet(embed_dim=64, depths=cfg["depths"], focal_levels=cfg["focal_levels"], focal_windows=cfg["focal_windows"],
                   use_conv_embed=True, use_postln=False, use_postln_in_modulation=True, scaling_modulator=False,
                   use_layerscale=True, device="cpu").load_state_dict(sd)
    outs = net(x)
    for k, r in ref.items():
        e_inf, e_l2 = _rel(outs[k], r)
        assert e_inf < 0.04 and e_l2 < 0.03, (k, e_inf, e_l2)


def test_autoencoder_host_logic_against_reference_golden(monkeypatch):
    """Host side of vitron_b200.autoencoder.AutoencoderKL (quant_conv folding, channel padding, transposed-V attention,
    asymmetric downsample padding) with the kernels replaced by torch statements: reproduces the unmodified
    reference's golden encode moments and decode output to bf16 accuracy."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.autoencoder import AutoencoderKL
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vae_tiny.pt"), weights_only=False)
    ae = AutoencoderKL(fx["ddconfig"], 4, device="cpu").load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"], 0.8))
    post = ae.encode(fx["x"])
    for got, ref, what in ((post.mean, fx["mean"], "mean"), (post.std, fx["std"], "std"), (ae.decode(fx["z"]), fx["dec"], "dec")):
        assert got.shape == ref.shape
        e_inf, e_l2 = _rel(got, ref)
        assert e_inf < 0.05 and e_l2 < 0.04, (what, e_inf, e_l2)
    z = ae.encode_firsr_stage(fx["x"], 0.18215, generator=torch.Generator().manual_seed(0))
    assert z.shape == fx["mean"].shape


def test_vae_shape_table_matches_reference_names():
    import os
    import torch
    from vitron_b200 import param_shapes
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vae_tiny.pt"), weights_only=False)
    assert param_shapes.vae_shapes(fx["ddconfig"]) == fx["shapes"]


def test_gligen_unet_shape_table_and_host_logic(monkeypatch):
    """vitron_b200.gligen_unet.UNetModel: reference state-dict names (shape table == unmodified class) and host logic
    (block plan, batched time-embedding projection as conv row bias, channel padding, NHWC skip concat, position net)
    against the reference's golden output with the kernels replaced by torch statements."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200 import param_shapes
    from vitron_b200.gligen_unet import UNetModel
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "gligen_unet_tiny.pt"), weights_only=False)
    assert param_shapes.gligen_unet_shapes(fx["cfg"]) == fx["shapes"]
    cpu_ops_emulator.install(monkeypatch)
    net = UNetModel(**fx["cfg"], device="cpu").load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"], fx["gain"]))
    out = net(dict(fx["inputs"]))
    e_inf, e_l2 = _rel(out, fx["out"])
    assert out.shape == fx["out"].shape and e_inf < 0.05 and e_l2 < 0.04, (e_inf, e_l2)


def test_clip_embedder_host_logic_against_oracle(monkeypatch):
    """vitron_b200.clip_embedder (open_clip state-dict names, penultimate-layer rule, EOS pooling, image tower through the
    LanguageBind ViT path) against the restated / transformers-cross-checked oracle, kernels replaced by torch statements."""
    import torch
    from oracle import restate_openclip as OC
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from tests.test_oracle_cpu import OPENCLIP_TINY as cfg
    from vitron_b200.clip_embedder import FrozenOpenCLIPEmbedder, FrozenOpenCLIPTtxtVisualEmbedder
    cpu_ops_emulator.install(monkeypatch)
    sd = seeded_state_dict(OC.openclip_shapes(cfg), 3)
    g = torch.Generator().manual_seed(2)
    tokens = torch.randint(1, 298, (2, 16), generator=g)
    tokens[0, 9], tokens[1, 15] = 299, 299
    tokens[0, 10:] = 0
    img = torch.randn((2, 3, 56, 56), generator=g)
    both = FrozenOpenCLIPTtxtVisualEmbedder(None, device="cpu", layer="penultimate", arch_cfg=cfg).load_state_dict(sd)
    xi, xt, x = both(image=img, text=tokens)
    rt, rx = OC.encode_text(sd, tokens, cfg, layer_idx=1)
    for got, ref, what in ((x, rx, "tokens"), (xt, rt, "pooled text"), (xi, OC.encode_image(sd, img, cfg), "image")):
        e_inf, e_l2 = _rel(got, ref)
        assert got.shape == ref.shape and e_inf < 0.04 and e_l2 < 0.03, (what, e_inf, e_l2)
    emb = FrozenOpenCLIPEmbedder(None, device="cpu", layer="last", arch_cfg=cfg).load_state_dict(sd)
    e_inf, e_l2 = _rel(emb(tokens), OC.encode_text(sd, tokens, cfg, layer_idx=0)[1])
    assert e_inf < 0.04 and e_l2 < 0.03
    import pytest
    with pytest.raises(ValueError):
        emb("a caption")


def test_seem_host_logic_against_reference_golden(monkeypatch):
    """Host side of vitron_b200.seem (grouped K/V projections per feature level, FPN order, mask-head GEMM layout, mask
    reset rule, output dict) with the kernels replaced by torch statements, against the golden outputs of the UNMODIFIED
    reference pixel decoder + mask decoder (tests/golden/seem_tiny.pt)."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.seem import MultiScaleMaskedTransformerDecoder, TransformerEncoderPixelDecoder, XDecoderHead
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "seem_tiny.pt"), weights_only=False)
    t = fx["cfg"]
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    pd = TransformerEncoderPixelDecoder(t["in_channels"], t["C"], t["C"], t["heads"], t["ffn"], t["enc_layers"], device="cpu")
    pr = MultiScaleMaskedTransformerDecoder(t["C"], t["dim_proj"], t["Q"], t["heads"], t["ffn"], t["dec_layers"], t["C"], device="cpu")
    head = XDecoderHead(pd, pr).load_state_dict(sd)
    head.predictor.set_text_embeddings(fx["t_emb"], t["logit_scale"])
    mf, enc, multi = head.pixel_decoder.forward_features(fx["features"])
    pairs = [(mf, fx["mask_features"], "mask_features"), (enc, fx["enc_features"], "encoder features")]
    pairs += [(a, b, "multi-scale") for a, b in zip(multi, fx["multi_scale"])]
    for got, ref, what in pairs:
        e_inf, e_l2 = _rel(got, ref)
        assert tuple(got.shape) == tuple(ref.shape) and e_inf < 0.05 and e_l2 < 0.04, (what, e_inf, e_l2)
    out = head.predictor(fx["multi_scale"], fx["mask_features"])
    assert sorted(k for k in out if k.startswith("pred_") or k == "aux_outputs") == ["aux_outputs", "pred_logits", "pred_maskembs", "pred_masks"]
    a0, r0 = out["aux_outputs"][0], fx["out"]["aux_outputs"][0]
    for k in ("pred_masks", "pred_logits"):
        e_inf, e_l2 = _rel(a0[k], r0[k])
        assert e_inf < 0.03 and e_l2 < 0.03, (k, e_inf, e_l2)
    e_inf, e_l2 = _rel(out["pred_masks"], fx["out"]["pred_masks"])
    assert e_l2 < 0.08, (e_inf, e_l2)
    # inference mode (aux_outputs off): intermediate layers derive the attention masks from mask_features resized once per
    # level (bilinear is linear); the final outputs must still match the reference, the intermediate masks the aux-on run
    full_masks = out["attn_masks"]
    head.predictor.aux_outputs = False
    out2 = head.predictor(fx["multi_scale"], fx["mask_features"])
    assert out2["aux_outputs"] == []
    e_inf, e_l2 = _rel(out2["pred_masks"], fx["out"]["pred_masks"])
    assert e_l2 < 0.08, (e_inf, e_l2)
    e_inf, e_l2 = _rel(out2["pred_logits"], fx["out"]["pred_logits"])
    assert e_l2 < 0.08, (e_inf, e_l2)
    agree = [float((a == b).float().mean()) for a, b in zip(out2["attn_masks"], full_masks)]
    assert min(agree) > 0.97, agree


def test_unet_i2vgen_host_logic_against_reference_golden(monkeypatch):
    """Host side of vitron_b200.unet_i2vgen.UNetSD_I2VGen (block plan, batched time-embedding projection, NHWC skip concats,
    strided temporal attention views, context assembly, cached local-image adapter) with the kernels replaced by torch
    statements, against the golden output of the UNMODIFIED reference class (tests/golden/unet_tiny.pt)."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.unet_i2vgen import UNetSD_I2VGen
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "unet_tiny.pt"), weights_only=False)
    m = UNetSD_I2VGen(**fx["cfg"], device="cpu")
    m.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"], fx["gain"]))
    out = m(**fx["inputs"])
    e_inf, e_l2 = _rel(out, fx["out"])
    assert out.shape == fx["out"].shape and e_inf < 0.05 and e_l2 < 0.04, (e_inf, e_l2)


def test_cfg_denoiser_batched_equals_two_calls_and_rebind(monkeypatch):
    """Host logic of GraphedCFGDenoiser without a GPU (its _eval, i.e. what the CUDA graph captures, on the CPU emulator): the
    ONE batch-2 forward [cond | uncond] gives the same guidance result as the reference's two UNet calls
    (diffusion_ddim.py:153-158), mismatching conditioning dicts fall back to the two-call form, and rebind() refreshes the
    batched static tensors of both branches."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.unet_i2vgen import GraphedCFGDenoiser, UNetSD_I2VGen
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "unet_tiny.pt"), weights_only=False)
    m = UNetSD_I2VGen(**fx["cfg"], device="cpu")
    m.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"], fx["gain"]))
    i = fx["inputs"]
    pick = lambda j: dict(y=i["y"][j:j + 1].clone(), image=i["image"][j:j + 1].clone(), local_image=i["local_image"][:1].clone(),
                          fps=i["fps"][:1].clone())
    cond, unc = pick(0), pick(1)
    xt, t = i["x"][:1].float(), i["t"][:1]
    two = GraphedCFGDenoiser(m, cond, unc, 7.5, xt, t, batched=False)
    one = GraphedCFGDenoiser(m, cond, unc, 7.5, xt, t)
    assert one.batched and not two.batched
    ref, got = two._eval().float(), one._eval().float()
    assert got.shape == ref.shape == xt.shape
    # guidance amplifies the bf16-level differences between a batch-1 and a batch-2 evaluation of the same sample by (1 + 2 s)
    y_sep, u_sep = m(xt, t, **cond).float(), m(xt, t, **unc).float()
    yu = m(one.xt2, one.t2, **one.both).float()
    branch_scale = float(torch.maximum(y_sep.abs().max(), u_sep.abs().max()))
    assert (yu[:1] - y_sep).abs().max() <= 1e-2 * branch_scale and (yu[1:] - u_sep).abs().max() <= 1e-2 * branch_scale
    tol = 1e-2 * branch_scale * (1 + 2 * 7.5)
    assert (got - ref).abs().max() <= tol, (float((got - ref).abs().max()), tol)
    assert (got - (yu[1:] + 7.5 * (yu[:1] - yu[1:]))).abs().max() <= 2e-2 * got.abs().max() + 1e-3
    # a branch without the image embedding cannot be batched with one that has it
    unc_none = dict(unc, image=None)
    assert not GraphedCFGDenoiser(m, cond, unc_none, 7.5, xt, t).batched
    # rebind: new conditioning values reach the batched static tensors (cond rows first, uncond rows second)
    new_c = {k: (v + 0.25 if v.is_floating_point() else v) for k, v in cond.items()}
    new_u = {k: (v - 0.25 if v.is_floating_point() else v) for k, v in unc.items()}
    one.rebind(new_c, new_u)
    assert torch.equal(one.both["y"][:1], new_c["y"]) and torch.equal(one.both["y"][1:], new_u["y"])
    fresh = GraphedCFGDenoiser(m, new_c, new_u, 7.5, xt, t, batched=False)._eval().float()
    again = one._eval().float()
    assert (again - fresh).abs().max() <= tol, float((again - fresh).abs().max())


def test_gligen_block_host_logic_against_reference_golden(monkeypatch):
    """Host side of vitron_b200.gligen (concat-free gated self-attention over [visual ; grounding] rows, packed GEGLU
    weights, tanh-gated residual epilogues) with the kernels replaced by torch statements, against the golden outputs of
    the UNMODIFIED reference attention.py (tests/golden/gligen_tiny.pt)."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.gligen import BasicTransformerBlock
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "gligen_tiny.pt"), weights_only=False)
    for case in fx["cases"]:
        C, heads = case["C"], case["heads"]
        blk = BasicTransformerBlock(C, 768, 768, heads, C // heads, "gatedSA", device="cpu").load_state_dict(
            seeded_state_dict(case["shapes"], fx["seed"]))
        for got, ref, what in ((blk.fuser(case["x"], fx["objs"]), case["fuser_out"], "fuser"),
                               (blk(case["x"], fx["context"], fx["objs"]), case["block_out"], "block")):
            e_inf, e_l2 = _rel(got, ref)
            assert got.shape == ref.shape and e_inf < 0.04 and e_l2 < 0.03, (C, what, e_inf, e_l2)


def test_vitron_forward_host_logic_against_reference_golden(monkeypatch):
    """Host side of the vision-LLM path (rows a1-a7): LanguageBind tower, projector, region extractor, multimodal splice
    map, folded RMSNorm gains, packed SwiGLU weights, prefill bookkeeping — `VitronLlamaForCausalLM.forward` with the kernels
    replaced by torch statements must reproduce the UNMODIFIED reference's golden logits (tests/golden/vitron_llm_tiny.pt)."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vitron_llm_tiny.pt"), weights_only=False)
    vit = dict(fx["vit"], hidden_act="gelu")
    cfg = VitronConfig(llm=fx["llm"], vision=VisionConfig(**vit),
                       video=VisionConfig(**vit, add_time_attn=True, num_frames=fx["num_frames"]), tokenizer_model_max_length=4096)
    model = VitronLlamaForCausalLM(cfg, "cpu", max_batch=2, max_seq_len=256)
    model.load_state_dict(seeded_state_dict(fx["shapes"], fx["seed"]))
    g = fx["img"]
    out = model.forward(input_ids=g["input_ids"], attention_mask=g["attention_mask"], images=g["images"], regions=g["regions"])
    ref = g["logits"]
    for b, n in enumerate(model._last_lens):
        e_inf, e_l2 = _rel(out.logits[b, :n], ref[b, :n])
        assert e_inf < 0.05 and e_l2 < 0.04, (b, e_inf, e_l2)
    v = fx["vid"]                                   # video tower (temporal attention over the frames) + 8-sentinel splice
    out = model.forward(input_ids=v["input_ids"], images=[v["images"][0]])
    e_inf, e_l2 = _rel(out.logits, v["logits"])
    assert e_inf < 0.05 and e_l2 < 0.04, ("video", e_inf, e_l2)


def test_gligen_grounded_sample_host_logic(monkeypatch):
    """vitron_b200.gligen_sampler.grounded_sample (PLMS + scheduled gate + VAE decode) over the CUDA UNetModel / AutoencoderKL
    with the kernels replaced by torch statements, against the same chain built from the pinned oracles; also checks that
    set_alpha_scale reaches every gated fuser."""
    import os
    from functools import partial
    import torch
    from oracle import restate_gligen_unet as G, restate_vae as V
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200 import gligen_sampler as GS
    from vitron_b200.autoencoder import AutoencoderKL
    from vitron_b200.gligen_unet import UNetModel
    cpu_ops_emulator.install(monkeypatch)
    ufx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "gligen_unet_tiny.pt"), weights_only=False)
    vfx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vae_tiny.pt"), weights_only=False)
    usd = seeded_state_dict(ufx["shapes"], ufx["seed"], ufx["gain"])
    vsd = seeded_state_dict(vfx["shapes"], vfx["seed"], 0.8)
    cfg = dict(ufx["cfg"], image_size=8)
    unet = UNetModel(**cfg, device="cpu").load_state_dict(usd)
    vae = AutoencoderKL(vfx["ddconfig"], 4, device="cpu").load_state_dict(vsd)
    GS.set_alpha_scale(unet, 0.25)
    fusers = [b.fuser for e in unet.w.values() if isinstance(e, dict) and "blocks" in e for b in e["blocks"]]
    assert len(fusers) >= 3 and all(f.scale == 0.25 for f in fusers)
    inp = {k: v for k, v in ufx["inputs"].items() if k not in ("x", "timesteps")}
    g = torch.Generator().manual_seed(1)
    start = torch.randn((2, 4, 8, 8), generator=g)
    uc = torch.randn(inp["context"].shape, generator=g)
    steps, guide, atype = 5, 2.0, (0.4, 0.2, 0.4)
    img = GS.grounded_sample(unet, vae, GS.DDPM(), dict(inp, x=start.clone(), timesteps=None), uc, guidance_scale=guide, steps=steps,
                             alpha_type=atype)

    class OracleModel:          # the oracle UNet with the gate the sampler schedules
        scale = 1.0

        def __call__(self, d):
            return G.unet_forward(usd, cfg, d, alpha_scale=self.scale)
    om = OracleModel()
    sampler = GS.PLMSSampler(GS.DDPM(), om, alpha_generator_func=partial(GS.alpha_generator, type=list(atype)),
                             set_alpha_scale=lambda m, a: setattr(m, "scale", float(a)))
    lat = sampler.sample(S=steps, shape=(2, 4, 8, 8), input=dict(inp, x=start.clone(), timesteps=None), uc=uc, guidance_scale=guide)
    ref = V.decode(vsd, lat / 0.18215, vfx["ddconfig"])  # GLIGEN decode(z) = decoder(z / scale_factor) (autoencoder.py:40-45)
    e_inf, e_l2 = _rel(img, ref)
    assert img.shape == ref.shape and e_inf < 0.08 and e_l2 < 0.06, (e_inf, e_l2)


def test_seem_interactive_prompts_host_logic_against_reference_golden(monkeypatch):
    """SEEM interactive prompts (VERDICT r1 item 3): grounding / audio token prompts, spatial positive / negative point prompts
    and the refimg -> visual-prompt route of vitron_b200.seem against golden outputs of the UNMODIFIED reference decoder +
    AttentionDataStruct (tests/golden/seem_prompts_tiny.pt, oracle/gen_golden.py::gen_seem_prompts); kernels replaced by the
    torch statements of cpu_ops_emulator."""
    import os
    import torch
    from oracle.weights import seeded_state_dict
    from tests import cpu_ops_emulator
    from vitron_b200.seem import MultiScaleMaskedTransformerDecoder
    cpu_ops_emulator.install(monkeypatch)
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "seem_prompts_tiny.pt"), weights_only=False)
    t = fx["cfg"]
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    pr = MultiScaleMaskedTransformerDecoder(t["C"], t["dim_proj"], t["Q"], t["heads"], t["ffn"], t["dec_layers"], t["C"], device="cpu")
    pr.load_state_dict(sd, "predictor.")
    pr.set_text_embeddings(fx["t_emb"], t["logit_scale"])
    assert pr.mask_sptial_embed is not None and pr.pn_indicator is not None

    def check(out, ref, what):
        for k, v in ref.items():
            if k == "aux0":
                continue
            assert k in out, (what, k, sorted(out))
            e_inf, e_l2 = _rel(out[k], v)
            lim = (0.05, 0.04) if k in ("pred_pspatials", "pred_nspatials", "pred_pvisuals", "pred_nvisuals") else (0.3, 0.09)
            assert tuple(out[k].shape) == tuple(v.shape) and e_inf < lim[0] and e_l2 < lim[1], (what, k, e_inf, e_l2)
        for k, v in ref.get("aux0", {}).items():      # first decoder layer: no accumulated mask thresholding
            e_inf, e_l2 = _rel(out["aux_outputs"][0][k], v)
            assert e_inf < 0.04 and e_l2 < 0.03, (what, "aux0", k, e_inf, e_l2)
    for name, extra in fx["cases"].items():
        out = pr(fx["multi_scale"], fx["mask_features"], task="seg", extra=dict(extra))
        check(out, fx["out"][name], name)
    # refimg route (evaluate_referring_image): spatial prompts on a reference image become visual prompts of the target
    ref = pr(fx["multi_scale"], fx["mask_features"], task="refimg", extra=dict(fx["cases"]["spatial"]))
    assert sorted(ref) == ["src_visual_maskings", "src_visual_queries", "visual_query_neg", "visual_query_pos"]
    for k in ("visual_query_pos", "visual_query_neg"):
        e_inf, e_l2 = _rel(ref[k], fx["refimg"][k])
        assert e_inf < 0.04 and e_l2 < 0.03, (k, e_inf, e_l2)
    for a, b in zip(ref["src_visual_queries"], fx["refimg"]["src_visual_queries"]):
        e_inf, e_l2 = _rel(a, b)
        assert e_inf < 0.04 and e_l2 < 0.03, ("src_visual_queries", e_inf, e_l2)
    out = pr(fx["multi_scale"], fx["mask_features"], task="seg",
             extra={k: fx["refimg"][k] for k in ("visual_query_pos", "visual_query_neg", "src_visual_queries", "src_visual_maskings")})
    check(out, fx["out"]["visual"], "visual")


def test_argument_validation_of_the_widened_entry_points(lib):
    """Error behaviour of the §8(f) entry points without a device: null pointers, misaligned strides, unsupported kernel
    sizes and short workspaces are rejected with VB_ERR_* before any launch."""
    import ctypes as C
    ERR_ARG, ERR_WS, ERR_UNSUP = -1, -3, -4
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf)                                   # 16-byte aligned host memory stands in for device pointers:
    p += (-p) % 16                                         # every check below fails before the pointer is dereferenced
    assert lib.vb200_dwconv_nhwc(None, 64, None, None, 1, 8, 8, 64, 3, 1, None) == ERR_ARG
    assert lib.vb200_dwconv_nhwc(p, 60, p, p, 1, 8, 8, 64, 3, 1, None) == ERR_ARG          # ld_in < c / not a multiple of 8
    assert lib.vb200_dwconv_nhwc(p, 64, p, p, 1, 8, 8, 64, 3, 2, None) == ERR_ARG          # act: only NONE / GELU
    assert lib.vb200_dwconv_nhwc(p, 64, p, p, 1, 8, 8, 64, 4, 1, None) == ERR_UNSUP        # even kernel size
    assert lib.vb200_set_dwconv_impl(7) in (0, 1, 2, 3) and lib.vb200_set_dwconv_impl(0) in (0, 1, 2, 3)
    assert lib.vb200_colmean_workspace_size(2, 1000, 192) > 0
    assert lib.vb200_colmean(p, p, 1, 1000, 192, 1, p, 16, None) == ERR_WS                 # workspace too small
    assert lib.vb200_colmean(p, p, 1, 1000, 4096, 1, p, 1 << 30, None) == ERR_ARG          # c > 2048
    ptrs = (C.c_void_p * 7)(*([p] * 7))
    assert lib.vb200_focal_modulate(ptrs, 7, p, 400, p, p, 1, 64, 64, 1.0, None) == ERR_ARG  # > VB_FOCAL_MAX_LEVELS
    assert lib.vb200_mul_rows(p, 60, p, 64, p, 4, 64, None) == ERR_ARG
    assert lib.vb200_layernorm_add(p, 64, p, None, None, 0, p, 64, 4, 4096, 1e-5, None) == ERR_ARG  # d > 2048
    assert lib.vb200_im2col_nchw(p, 1, p, 1, 3, 32, 32, 7, 4, 2, 8, 8, 100, None) == ERR_ARG        # kpad < c*k*k / not % 8
    assert lib.vb200_softmax_rows(None, 8, p, 8, 1, 8, None) == ERR_ARG
    # 16-byte vector loads and stores: a pointer 2 bytes off (e.g. the row view x[:, 1:]) is refused, whichever it is
    q = p + 2
    for args in ((q, p, p, p), (p, q, p, p), (p, p, q, p), (p, p, p, q)):
        x, w, b, o = args
        assert lib.vb200_layernorm(x, 64, w, b, o, 64, 4, 64, 1e-5, None) == ERR_ARG, args
        if b == p:
            assert lib.vb200_rmsnorm(x, 64, w, o, 64, 4, 64, 1e-5, None) == ERR_ARG, args
    assert lib.vb200_layernorm(p, 64, p, None, q, 64, 4, 64, 1e-5, None) == ERR_ARG
    assert lib.vb200_row_rstd(q, 64, p, 4, 64, 1e-5, None) == ERR_ARG
    for x, o in ((q, p), (p, q)):
        assert lib.vb200_upsample2x_nhwc(x, o, 1, 4, 4, 64, None) == ERR_ARG
        assert lib.vb200_resize_bilinear_nhwc(x, o, 1, 4, 4, 64, 8, 8, None) == ERR_ARG
    for a, b, o in ((q, p, p), (p, q, p), (p, p, q)):
        assert lib.vb200_add_bf16(a, b, o, 64, 0, None) == ERR_ARG
        assert lib.vb200_add_rowgroup(a, b, o, 4, 64, 2, 2, None) == ERR_ARG
    m3 = (C.c_float * 3)(0.5, 0.5, 0.5)
    assert lib.vb200_preprocess_frames(p, p, 1, 32, 32, 224, 224, 10, 0, 224, 224, 1, 1, m3, m3, 1, 0, 0, None) == ERR_ARG  # crop outside
    assert lib.vb200_preprocess_frames(p, p, 1, 32, 32, 224, 224, 0, 0, 224, 224, 1, 1, m3, m3, 5, 0, 0, None) == ERR_ARG   # unknown mode


def test_outputs_that_are_not_row_views_are_refused(lib):
    """An out= (or in-place) tensor whose rows do not share one stride cannot be handed to a kernel as [rows, d]: a
    reshape would copy it, the kernel would write the copy and the caller's tensor would never change. The ops raise
    ValueError before any library call (CPU tensors: nothing here reaches a device)."""
    import torch
    from vitron_b200 import ops
    BF = torch.bfloat16
    x = torch.zeros((2, 5, 64), dtype=BF)
    w, b = torch.ones((64,), dtype=BF), torch.zeros((64,), dtype=BF)
    buf = torch.zeros((2, 8, 64), dtype=BF)
    bad = buf[:, :5]                                      # [B, S, d] slice of a longer sequence buffer
    with pytest.raises(ValueError):
        ops.rmsnorm(x, w, 1e-6, out=bad)
    with pytest.raises(ValueError):
        ops.layernorm(x, w, b, 1e-5, out=bad)
    with pytest.raises(ValueError):
        ops.layernorm_add(x, w, b, None, 1e-5, out=bad)
    with pytest.raises(ValueError):
        ops.gemm(x, torch.zeros((64, 64), dtype=BF), out=bad)
    with pytest.raises(ValueError):
        ops.rope_kv_append(bad, torch.zeros((10,), dtype=torch.int32), 1, 64, 1e4)
    with pytest.raises(ValueError):
        ops.add_rowgroup(x.reshape(10, 64), torch.zeros((2, 64), dtype=BF), 5, 2, out=bad.reshape(2, 5, 64)[0])
    with pytest.raises(ValueError):
        ops.add_rowgroup(x.reshape(10, 64), torch.zeros((2, 64), dtype=BF), 5, 2, out=torch.zeros((10, 64)))
    # a 3-D view whose rows do share one stride is fine: the reshape check is on views, not on dimensions
    assert ops._out_rows2d(buf[:1, :5])[1] == 64 and ops._out_rows2d(buf[:, :5][:, :, :32].contiguous())[1] == 32
    with pytest.raises(ValueError):
        ops._out_rows2d(buf[:, :5, :32])
