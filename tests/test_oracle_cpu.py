"""CPU: pins the oracle restatements (oracle/restate_*.py) against golden vectors produced by the
unmodified reference (oracle/gen_golden.py) and, when /root/reference is present, against the
reference itself on a fresh random configuration."""
import os

import pytest
import torch

from oracle import restate_llm as R
from oracle.weights import seeded_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def load(name):
    return torch.load(os.path.join(GOLD, name), weights_only=False)


def cfgs_of(fx):
    vit = dict(fx["vit"], hidden_act="gelu", layer_norm_eps=1e-5)
    return {"llm": dict(fx["llm"], rms_norm_eps=1e-5, rope_theta=10000.0), "vision": dict(vit, add_time_attn=False),
            "video": dict(vit, add_time_attn=True, num_frames=fx["num_frames"]), "max_len": 4096}


@pytest.fixture(scope="module")
def fx():
    return load("vitron_llm_tiny.pt")


@pytest.fixture(scope="module")
def sd(fx):
    return seeded_state_dict(fx["shapes"], fx["seed"])


def test_towers_and_adapters_match_reference_golden(fx, sd):
    c = cfgs_of(fx)
    t = fx["tower"]
    imgs = torch.stack(fx["img"]["images"])
    feats = R.clip_vit_hidden(sd, "model.image_tower.image_tower.", c["vision"], imgs)[:, 1:]
    assert torch.allclose(feats, t["image_feats"], atol=2e-4, rtol=1e-4)
    vf = R.clip_vit_hidden(sd, "model.video_tower.video_tower.", c["video"], fx["vid"]["images"][0][None])[:, :, 1:]
    assert torch.allclose(vf, t["video_feats"], atol=2e-4, rtol=1e-4)
    assert torch.allclose(R.projector(sd, "model.mm_projector.", feats), t["proj"], atol=2e-4, rtol=1e-4)
    rg = R.region_extractor(sd, "model.region_extractor.", feats, fx["img"]["regions"], fx["vit"]["image_size"])
    assert torch.allclose(rg, t["region"], atol=2e-4, rtol=1e-4)


def test_multimodal_logits_match_reference_golden(fx, sd):
    c = cfgs_of(fx)
    g = fx["img"]
    logits, lens = R.vitron_logits(sd, c, g["input_ids"], g["images"], g["regions"], g["attention_mask"])
    assert logits.shape == g["logits"].shape
    for b, n in enumerate(lens):  # padded positions are don't-care
        assert torch.allclose(logits[b, :n], g["logits"][b, :n], atol=2e-3, rtol=1e-3), b
    v = fx["vid"]
    lv, _ = R.vitron_logits(sd, c, v["input_ids"], v["images"])
    assert torch.allclose(lv, v["logits"], atol=2e-3, rtol=1e-3)


def test_greedy_tokens_match_reference_golden(fx, sd):
    c = cfgs_of(fx)
    g = fx["gen_img"]
    toks, gaps = R.greedy_generate(sd, c, g["input_ids"], g["images"], g["regions"], g["tokens"].shape[1])
    assert torch.equal(toks, g["tokens"]), (toks, g["tokens"], gaps)
    v = fx["vid"]
    toks, _ = R.greedy_generate(sd, c, v["input_ids"], v["images"], None, v["tokens"].shape[1])
    assert torch.equal(toks, v["tokens"])


@pytest.mark.skipif(not os.path.isdir("/root/reference/vitron"), reason="reference tree not present")
def test_oracle_against_live_reference():
    from oracle import refshim
    from oracle.weights import shapes_of
    llm = dict(hidden_size=64, intermediate_size=96, num_hidden_layers=3, num_attention_heads=4, vocab_size=97)
    vit = dict(hidden_size=48, intermediate_size=80, num_hidden_layers=4, num_attention_heads=3, image_size=42, patch_size=14)
    model = refshim.build_reference_vitron(llm, vit, with_video=False, hidden_act="quick_gelu")
    sd = seeded_state_dict(shapes_of(model), 5)
    model.load_state_dict(sd, strict=False)
    g = torch.Generator().manual_seed(1)
    img = torch.randn((3, 42, 42), generator=g)
    ids = torch.tensor([[1, 4, 9, -200, 17, 33, -300, 8]])
    with torch.no_grad():
        ref = model(input_ids=ids, images=[img], regions=[[3.0, 5.0, 30.0, 40.0]], use_cache=False).logits
    c = {"llm": dict(llm, rms_norm_eps=1e-5, rope_theta=10000.0),
         "vision": dict(vit, hidden_act="quick_gelu", layer_norm_eps=1e-5, add_time_attn=False), "max_len": 4096}
    got, _ = R.vitron_logits(sd, c, ids, [img], [[3.0, 5.0, 30.0, 40.0]])
    assert torch.allclose(got, ref.float(), atol=2e-3, rtol=1e-3)


def test_cached_decoder_equals_full_recompute(fx, sd):
    c = cfgs_of(fx)
    sdf = {k: v.float() for k, v in sd.items()}
    g = torch.Generator().manual_seed(0)
    emb = torch.randn((2, 9, fx["llm"]["hidden_size"]), generator=g)
    m = R.LlamaCPU(sdf, c["llm"])
    lg = m.prefill(emb)
    full = R.llama_forward(sdf, c["llm"], emb)
    assert torch.allclose(lg, full[:, -1], atol=1e-4, rtol=1e-4)
    tok = lg.argmax(-1)
    lg2 = m.step(tok)
    emb2 = torch.cat([emb, sdf["model.embed_tokens.weight"][tok][:, None]], 1)
    assert torch.allclose(lg2, R.llama_forward(sdf, c["llm"], emb2)[:, -1], atol=1e-4, rtol=1e-4)


# ------------------------------------------------------------------ i2vgen-xl UNet3D + DDIM
@pytest.fixture(scope="module")
def ufx():
    return load("unet_tiny.pt")


def test_unet_restatement_matches_reference_golden(ufx):
    from oracle import restate_unet as U
    sd = seeded_state_dict(ufx["shapes"], ufx["seed"], ufx["gain"])
    i = ufx["inputs"]
    out = U.unet_forward(sd, ufx["cfg"], i["x"], i["t"], y=i["y"], image=i["image"], local_image=i["local_image"], fps=i["fps"])
    ref = ufx["out"]
    assert out.shape == ref.shape
    assert torch.allclose(out, ref, atol=1e-3 * ref.abs().max().item(), rtol=1e-3), (out - ref).abs().max()


def test_ddim_restatement_matches_reference_golden(ufx):
    from oracle import restate_unet as U
    sd = seeded_state_dict(ufx["shapes"], ufx["seed"], ufx["gain"])
    d = ufx["ddim"]
    model = lambda xt, t, **kw: U.unet_forward(sd, ufx["cfg"], xt, t, **kw)
    out = U.ddim_sample_loop(d["noise"], model, [d["cond"], d["uncond"]], d["guide_scale"], d["ddim_timesteps"])
    assert torch.allclose(out, d["out"], atol=2e-3, rtol=2e-3), (out - d["out"]).abs().max()


# ------------------------------------------------------------------ GLIGEN gated self-attention
def test_gligen_restatement_matches_reference_golden():
    from oracle import restate_gligen as G
    fx = load("gligen_tiny.pt")
    for c in fx["cases"]:
        sd = seeded_state_dict(c["shapes"], fx["seed"])
        fo = G.gated_self_attention_dense(sd, "fuser.", c["x"], fx["objs"], c["heads"])
        assert torch.allclose(fo, c["fuser_out"], atol=1e-4, rtol=1e-4)
        bo = G.basic_transformer_block(sd, "", c["x"], fx["context"], fx["objs"], c["heads"])
        assert torch.allclose(bo, c["block_out"], atol=1e-4, rtol=1e-4)


# ------------------------------------------------------------------ SEEM (piecewise pin; detectron2 absent)
REF_SEEM = "/root/reference/modules/SEEM/demo_code/xdecoder"
needs_ref = pytest.mark.skipif(not os.path.isdir(REF_SEEM), reason="reference tree not present")


@needs_ref
def test_seem_position_embedding_matches_reference():
    from oracle import refshim, restate_seem as S
    pe = refshim.load_file("ref_seem_pe", "modules/SEEM/demo_code/xdecoder/modules/position_encoding.py")
    x = torch.zeros((2, 8, 5, 7))
    ref = pe.PositionEmbeddingSine(32, normalize=True)(x)
    assert torch.allclose(S.position_embedding_sine(x, 32), ref, atol=1e-6)
    # the product's own closed form (device-side cache) must agree too
    from vitron_b200.seem import position_embedding_sine as prod_pe
    got = prod_pe(5, 7, 32, torch.device("cpu")).view(5, 7, 64).permute(2, 0, 1)
    assert torch.allclose(got, ref[0], atol=1e-6)


@needs_ref
def test_seem_attention_matches_reference_mha():
    from oracle import refshim, restate_seem as S
    att = refshim.load_file("ref_seem_attn", "modules/SEEM/demo_code/xdecoder/body/decoder/utils/attn.py")
    torch.manual_seed(0)
    C, H, L, S_, B = 64, 4, 5, 9, 2
    m = att.MultiheadAttention(C, H, dropout=0.0).eval()
    sd = {"x." + k: v for k, v in m.state_dict().items()}
    q, k, v = torch.randn(L, B, C), torch.randn(S_, B, C), torch.randn(S_, B, C)
    mask = torch.rand(B * H, L, S_) < 0.5
    mask[3] = True  # fully masked head-rows -> nan_to_num() -> zeros
    with torch.no_grad():
        ref = m(q, k, v, attn_mask=mask)[0]
    assert torch.allclose(S.mha(q, k, v, sd, "x.", H, mask), ref, atol=1e-5)


@needs_ref
def test_seem_mask_rule_and_prepare_features_match_reference():
    from oracle import refshim, restate_seem as S
    ads = refshim.load_file("ref_seem_ads", "modules/SEEM/demo_code/xdecoder/body/decoder/utils/attention_data_struct.py")
    utl = refshim.load_file("ref_seem_utils", "modules/SEEM/demo_code/xdecoder/body/decoder/utils/utils.py")
    pe = refshim.load_file("ref_seem_pe2", "modules/SEEM/demo_code/xdecoder/modules/position_encoding.py")
    arch = {"VARIABLE": {"queries": ["object"]}, "SELF_ATTENTION": {"queries": {"object": ["queries_object"]}},
            "CROSS_ATTENTION": {"queries": {"object": True}}, "MASKING": [], "DUPLICATION": {}, "NUM_LAYERS": 1}
    d = ads.AttentionDataStruct(arch, {"mask": True, "bbox": False, "spatial": False, "grounding": False, "audio": False, "visual": False})
    d.reset({}, "seg", {})
    Q, N = 6, 12
    d.set("queries_object", "queries", torch.zeros(Q, 1, 4), torch.zeros(Q, 1, 4))
    d.cross_attn_variables()
    am = torch.rand(2, Q, N) < 0.6
    am[1, 2] = True
    d.set_results({"attn_mask": am.clone(), "predictions_class": None, "predictions_mask": None, "predictions_maskemb": None})
    ref = d.cross_attn_mask((3, 4), 2)
    mine = am.clone()
    mine[torch.where(mine.sum(-1) == mine.shape[-1])] = False
    assert torch.equal(ref, mine) and not ref[1, 2].any()
    # prepare_features
    import torch.nn as nn
    xs = [torch.randn(1, 8, 3, 4), torch.randn(1, 8, 6, 8), torch.randn(1, 8, 12, 16)]
    lvl = nn.Embedding(3, 8)
    src, pos, sizes = utl.prepare_features(xs, 3, pe.PositionEmbeddingSine(4, normalize=True), [nn.Sequential()] * 3, lvl)
    for i in range(3):
        assert torch.allclose(pos[i], S.position_embedding_sine(xs[i], 4).flatten(2).permute(2, 0, 1), atol=1e-6)
        assert torch.allclose(src[i], (xs[i].flatten(2) + lvl.weight[i][None, :, None]).permute(2, 0, 1))


def test_seem_restatement_runs_and_is_self_consistent():
    """Shapes / key names of the seg-path output dict (attention_data_struct.py:12-28,250-264)."""
    from oracle import restate_seem as S
    shapes = S.seem_shapes(in_channels=(16, 24, 32, 40), C=64, ffn=96, Q=7, enc_layers=1, dec_layers=3, dim_proj=32)
    sd = seeded_state_dict(shapes, 1)
    g = torch.Generator().manual_seed(0)
    feats = {f"res{i + 2}": torch.randn((1, c, 32 >> i, 48 >> i), generator=g) for i, c in enumerate((16, 24, 32, 40))}
    mf, enc, multi = S.pixel_decoder_forward(sd, feats, "pixel_decoder.", nheads=2, enc_layers=1)
    assert mf.shape == (1, 64, 32, 48) and [tuple(m.shape[-2:]) for m in multi] == [(4, 6), (8, 12), (16, 24)]
    out = S.mask_decoder_forward(sd, multi, mf, "predictor.", heads=2, num_layers=3, t_emb=torch.randn(5, 32), logit_scale=1.0)
    assert out["pred_logits"].shape == (1, 7, 5) and out["pred_masks"].shape == (1, 7, 32, 48)
    assert len(out["aux_outputs"]) == 3 and out["pred_maskembs"].shape == (1, 7, 64)


def _seem_restated(fx, sd, feats, t_emb):
    from oracle import restate_seem as S
    t = fx["cfg"]
    mf, enc, multi = S.pixel_decoder_forward(sd, feats, "pixel_decoder.", nheads=t["heads"], enc_layers=t["enc_layers"])
    out = S.mask_decoder_forward(sd, multi, mf, "predictor.", heads=t["heads"], num_layers=t["dec_layers"], t_emb=t_emb,
                                 logit_scale=t["logit_scale"])
    return mf, enc, multi, out


def _seem_compare(mf, enc, multi, out, ref_mf, ref_enc, ref_multi, ref_out, atol=3e-4):
    assert torch.allclose(mf, ref_mf, atol=atol, rtol=1e-4)
    assert torch.allclose(enc, ref_enc, atol=atol, rtol=1e-4)
    for a, b in zip(multi, ref_multi):
        assert torch.allclose(a, b, atol=atol, rtol=1e-4)
    for k in ("pred_logits", "pred_masks", "pred_maskembs"):
        assert torch.allclose(out[k], ref_out[k], atol=atol, rtol=1e-4), k
        for a, b in zip(out["aux_outputs"], ref_out["aux_outputs"]):
            assert torch.allclose(a[k], b[k], atol=atol, rtol=1e-4), ("aux", k)


def test_seem_restatement_matches_reference_golden():
    """Module-level pin of rows a10 + a11: the restatement reproduces what the UNMODIFIED reference classes
    TransformerEncoderPixelDecoder.forward_features + MultiScaleMaskedTransformerDecoder.forward(task='seg')
    computed (oracle/gen_golden.py::gen_seem, detectron2-layer stubs stated in refshim.setup_seem)."""
    fx = load("seem_tiny.pt")
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    mf, enc, multi, out = _seem_restated(fx, sd, fx["features"], fx["t_emb"])
    assert fx["out_keys"] == ["aux_outputs", "pred_logits", "pred_maskembs", "pred_masks"]
    assert len(out["aux_outputs"]) == len(fx["out"]["aux_outputs"]) == fx["cfg"]["dec_layers"]
    _seem_compare(mf, enc, multi, out, fx["mask_features"], fx["enc_features"], fx["multi_scale"], fx["out"])


def test_seem_restatement_matches_live_reference():
    from oracle import refshim
    if not refshim.available():
        pytest.skip("reference tree not present")
    from oracle import gen_golden as G
    t = dict(G.SEEM_TINY, C=96, ffn=160, Q=11, enc_layers=1, dec_layers=4, heads=3, in_channels=(16, 24, 40, 56))
    pd, md, sd, shapes = G.build_reference_seem(t, seed=77)
    g = torch.Generator().manual_seed(3)
    sizes = [(36, 28), (18, 14), (9, 7), (5, 4)]  # odd FPN chain: nearest-upsample to the lateral's size
    feats = {f"res{i + 2}": torch.randn((2, c, *sizes[i]), generator=g) for i, c in enumerate(t["in_channels"])}
    t_emb = torch.randn((t["n_text"], t["dim_proj"]), generator=g)
    md.lang_encoder.default_text_embeddings.copy_(t_emb)
    with torch.no_grad():
        r_mf, r_enc, r_multi = pd.forward_features(feats)
        r_out = md(r_multi, r_mf, task="seg", extra={})
    fx = {"cfg": t}
    mf, enc, multi, out = _seem_restated(fx, sd, feats, t_emb)
    _seem_compare(mf, enc, multi, out, r_mf, r_enc, r_multi, r_out)


def test_focal_restatement_matches_reference_golden():
    """§8(f1) FocalNet backbone: restatement == outputs of the unmodified reference class (golden)."""
    from oracle import restate_focal as FR
    fx = load("focal_tiny.pt")
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    outs = FR.focalnet_forward(sd, fx["x"], fx["cfg"])
    assert sorted(outs) == sorted(fx["outs"]) == ["res2", "res3", "res4", "res5"]
    for k, v in fx["outs"].items():
        assert outs[k].shape == v.shape
        assert torch.allclose(outs[k], v, atol=2e-4, rtol=1e-4), k


def test_focal_restatement_matches_live_reference():
    from oracle import refshim
    if not refshim.available():
        pytest.skip("reference tree not present")
    from oracle import gen_golden as G, restate_focal as FR
    cfg = dict(G.FOCAL_TINY, embed_dim=48, depths=(1, 2, 1, 1), focal_levels=(3, 2, 4, 1), focal_windows=(5, 3, 3, 7),
               scaling_modulator=False, use_postln=False, use_postln_in_modulation=True)
    net, sd, _ = G.build_reference_focalnet(cfg, seed=88)
    x = torch.randn((2, 3, 62, 90), generator=torch.Generator().manual_seed(4))  # exercises the pad-to-patch path
    with torch.no_grad():
        ref = net(x)
    outs = FR.focalnet_forward(sd, x, cfg)
    for k, v in ref.items():
        assert torch.allclose(outs[k], v, atol=2e-4, rtol=1e-4), k


def test_vae_restatement_matches_reference_golden():
    """§8(f2) i2vgen first-stage AutoencoderKL: restatement == unmodified reference class (golden)."""
    from oracle import restate_vae as V
    fx = load("vae_tiny.pt")
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    mean, logvar, std = V.encode_moments(sd, fx["x"], fx["ddconfig"])
    assert torch.allclose(mean, fx["mean"], atol=2e-4, rtol=1e-4)
    assert torch.allclose(logvar, fx["logvar"], atol=2e-4, rtol=1e-4)
    assert torch.allclose(std, fx["std"], atol=2e-4, rtol=1e-4)
    assert torch.allclose(V.decode(sd, fx["z"], fx["ddconfig"]), fx["dec"], atol=2e-4, rtol=1e-4)


def test_vae_restatement_matches_live_reference():
    from oracle import refshim
    if not refshim.available():
        pytest.skip("reference tree not present")
    from oracle import gen_golden as G, restate_vae as V
    dd = dict(G.VAE_TINY, ch=32, ch_mult=(1, 2, 4, 4), num_res_blocks=2)
    ae, sd, _ = G.build_reference_vae(dd, seed=99)
    g = torch.Generator().manual_seed(8)
    x, z = torch.randn((1, 3, 40, 24), generator=g), torch.randn((1, 4, 5, 3), generator=g)
    with torch.no_grad():
        post, dec = ae.encode(x), ae.decode(z)
        zz = ae.encode_firsr_stage(x, 0.18215)
    mean, logvar, std = V.encode_moments(sd, x, dd)
    assert torch.allclose(mean, post.mean, atol=2e-4, rtol=1e-4) and torch.allclose(std, post.std, atol=2e-4, rtol=1e-4)
    assert torch.allclose(V.decode(sd, z, dd), dec, atol=2e-4, rtol=1e-4)
    assert zz.shape == mean.shape  # encode_firsr_stage = scale_factor * posterior.sample(): stochastic, shape only


def test_gligen_autoencoder_scale_factor_matches_live_reference():
    """ADVICE r1 (high): GLIGEN's AutoencoderKL folds scale_factor into encode / decode (ldm/models/autoencoder.py:34-45).
    The product wrapper `gligen_sampler.GligenAutoencoder` over an unscaled VAE must reproduce the UNMODIFIED GLIGEN class
    with scale_factor = 0.18215 (decode exactly; encode with the posterior noise supplied)."""
    from oracle import refshim
    if not refshim.available():
        pytest.skip("reference tree not present")
    from oracle import gen_golden as G, restate_vae as V
    from vitron_b200.autoencoder import DiagonalGaussianDistribution
    from vitron_b200.gligen_sampler import GligenAutoencoder
    dd = dict(G.VAE_TINY, ch=32, ch_mult=(1, 2), num_res_blocks=1)
    _, sd, _ = G.build_reference_vae(dd, seed=5)
    ref = refshim.gligen_autoencoder_class()(dict(dd, dropout=0.0), 4, scale_factor=0.18215).eval()
    missing = ref.load_state_dict(sd, strict=False)
    assert not missing.missing_keys, missing.missing_keys

    class OracleVAE:  # the unscaled i2vgen-style interface the wrapper sits on (CPU stand-in for the CUDA AutoencoderKL)
        def encode(self, x):
            mean, logvar, _ = V.encode_moments(sd, x, dd)
            return DiagonalGaussianDistribution(torch.cat([mean, logvar], 1))

        def decode(self, z):
            return V.decode(sd, z, dd)

    wrap = GligenAutoencoder(OracleVAE(), 0.18215)
    g = torch.Generator().manual_seed(3)
    x, z = torch.randn((1, 3, 16, 16), generator=g), torch.randn((1, 4, 8, 8), generator=g)
    with torch.no_grad():
        want_dec = ref.decode(z)
        torch.manual_seed(11)
        want_enc = ref.encode(x)
        torch.manual_seed(11)
        noise = torch.randn(want_enc.shape)
    assert torch.allclose(wrap.decode(z), want_dec, atol=2e-4, rtol=1e-4)
    assert not torch.allclose(V.decode(sd, z, dd), want_dec, atol=1e-2)  # the unscaled decode is NOT the GLIGEN decode
    assert torch.allclose(wrap.encode(x, noise=noise), want_enc, atol=2e-4, rtol=1e-4)


def _rand_u8(shape, seed):
    return torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def test_image_transform_restatement_matches_reference_transform():
    """§8(f3): the restated image transform (antialiased variant) == the reference's own get_image_transform run with
    this image's torchvision (processing_image.py:15-25)."""
    from oracle import refshim, restate_preprocess as P
    if not refshim.available():
        pytest.skip("reference tree not present")
    import types
    from PIL import Image
    mod = refshim.load_file("ref_lb_processing_image", "vitron/model/multimodal_encoder/languagebind/image/processing_image.py")
    tf = mod.get_image_transform(types.SimpleNamespace(vision_config=None))
    for (h, w), seed in (((336, 336), 1), ((300, 451), 2), ((500, 333), 3), ((224, 224), 4), ((100, 150), 5)):
        u8 = _rand_u8((h, w, 3), seed)
        ref = tf(Image.fromarray(u8.numpy()))
        got = P.image_transform(u8, antialias=True)
        assert got.shape == ref.shape == (3, 224, 224)
        assert torch.allclose(got, ref, atol=1e-5), (h, w, (got - ref).abs().max())


def test_preprocess_kernel_formulas_match_oracle(monkeypatch):
    """The arithmetic coded in preprocess.cu (transcribed in tests/cpu_ops_emulator.py) reproduces ATen's bicubic /
    antialiased bicubic / bilinear resize through the host-side processors (geometry, crop, flip, layout)."""
    from oracle import restate_preprocess as P
    from tests import cpu_ops_emulator
    from vitron_b200 import processing
    cpu_ops_emulator.install(monkeypatch)
    for (h, w), seed in (((336, 336), 1), ((120, 181), 2), ((260, 230), 3), ((90, 64), 4)):
        u8 = _rand_u8((h, w, 3), seed)
        for aa in (False, True):
            got = processing.LanguageBindImageProcessor(device="cpu", antialias=aa).preprocess(u8.numpy())["pixel_values"][0]
            ref = P.image_transform(u8, antialias=aa)
            assert torch.allclose(got, ref, atol=2e-4), (h, w, aa, (got - ref).abs().max())
    for (h, w), seed, flip in (((240, 320), 5, False), ((300, 225), 6, True), ((224, 224), 7, True)):
        u8 = _rand_u8((4, h, w, 3), seed)
        got = processing.LanguageBindVideoProcessor(device="cpu").preprocess(u8, flip=flip)["pixel_values"][0]
        ref = P.video_transform(u8, flip)
        assert got.shape == ref.shape == (3, 4, 224, 224)
        assert torch.allclose(got, ref, atol=2e-4), (h, w, flip, (got - ref).abs().max())


def test_gligen_unet_restatement_matches_reference_golden():
    """§8(f2) GLIGEN grounded SD UNet: restatement == unmodified UNetModel (golden)."""
    from oracle import restate_gligen_unet as G
    fx = load("gligen_unet_tiny.pt")
    sd = seeded_state_dict(fx["shapes"], fx["seed"], fx["gain"])
    out = G.unet_forward(sd, fx["cfg"], fx["inputs"])
    assert out.shape == fx["out"].shape
    assert torch.allclose(out, fx["out"], atol=2e-5, rtol=2e-4), (out - fx["out"]).abs().max()


def test_gligen_unet_restatement_matches_live_reference():
    from oracle import refshim
    if not refshim.available():
        pytest.skip("reference tree not present")
    import contextlib
    import io
    from oracle import gen_golden as GG, restate_gligen_unet as G
    cfg = dict(GG.GLIGEN_UNET_TINY, model_channels=32, channel_mult=[1, 2, 4], num_res_blocks=2, attention_resolutions=[4, 1],
               num_heads=4, is_inpaint=True)
    net, sd, _ = GG.build_reference_gligen_unet(cfg, seed=72)
    inp = GG.gligen_unet_inputs(cfg, torch.Generator().manual_seed(5), b=1, n_obj=3, hw=(8, 12), inpaint=True)
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        ref = net(dict(inp))
        inp2 = {k: v for k, v in inp.items() if k not in ("boxes", "masks", "text_embeddings")}
        net.max_box = 30
        ref2 = net(dict(inp2))           # no grounding input: zero boxes -> learned null tokens (forward_position_net :393-399)
    out = G.unet_forward(sd, cfg, inp)
    assert torch.allclose(out, ref, atol=2e-5, rtol=2e-4), (out - ref).abs().max()
    assert torch.allclose(G.unet_forward(sd, cfg, inp2), ref2, atol=2e-5, rtol=2e-4)
    for mod in net.modules():                      # evaluator.py::set_alpha_scale (:35-39): the sampler's gate schedule
        if type(mod).__name__ == "GatedSelfAttentionDense":
            mod.scale = 0.3
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        ref3 = net(dict(inp))
    assert torch.allclose(G.unet_forward(sd, cfg, inp, alpha_scale=0.3), ref3, atol=2e-5, rtol=2e-4)
    assert not torch.allclose(ref3, ref, atol=1e-4)


OPENCLIP_TINY = dict(embed_dim=96, text=dict(width=128, layers=3, heads=2, context_length=16, vocab_size=300),
                     vision=dict(width=128, layers=2, heads=2, patch_size=14, image_size=56, mlp=256))


def test_openclip_restatement_matches_transformers_clip():
    """open_clip is absent (third-party): the restated published algorithm is cross-checked against the independent
    CLIP implementation in `transformers` with the same weights mapped (text: causal, EOS = argmax pooling; vision: CLS)."""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection, CLIPVisionConfig, CLIPVisionModelWithProjection
    from oracle import restate_openclip as OC
    cfg = OPENCLIP_TINY
    sd = seeded_state_dict(OC.openclip_shapes(cfg), 3)
    t, v = cfg["text"], cfg["vision"]

    def map_blocks(src, dst, n, d):
        out = {}
        for i in range(n):
            p, q = src + f"resblocks.{i}.", dst + f"encoder.layers.{i}."
            w, b = sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"]
            for j, nm in enumerate("qkv"):
                out[q + f"self_attn.{nm}_proj.weight"], out[q + f"self_attn.{nm}_proj.bias"] = w[j * d:(j + 1) * d], b[j * d:(j + 1) * d]
            out[q + "self_attn.out_proj.weight"], out[q + "self_attn.out_proj.bias"] = sd[p + "attn.out_proj.weight"], sd[p + "attn.out_proj.bias"]
            for a, bname in (("ln_1", "layer_norm1"), ("ln_2", "layer_norm2")):
                out[q + bname + ".weight"], out[q + bname + ".bias"] = sd[p + a + ".weight"], sd[p + a + ".bias"]
            out[q + "mlp.fc1.weight"], out[q + "mlp.fc1.bias"] = sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"]
            out[q + "mlp.fc2.weight"], out[q + "mlp.fc2.bias"] = sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"]
        return out

    tm = CLIPTextModelWithProjection(CLIPTextConfig(vocab_size=t["vocab_size"], hidden_size=t["width"], intermediate_size=4 * t["width"],
                                                    num_hidden_layers=t["layers"], num_attention_heads=t["heads"],
                                                    max_position_embeddings=t["context_length"], hidden_act="gelu",
                                                    projection_dim=cfg["embed_dim"], eos_token_id=t["vocab_size"] - 1,
                                                    attn_implementation="eager")).eval()
    hf = map_blocks("model.transformer.", "text_model.", t["layers"], t["width"])
    hf.update({"text_model.embeddings.token_embedding.weight": sd["model.token_embedding.weight"],
               "text_model.embeddings.position_embedding.weight": sd["model.positional_embedding"],
               "text_model.final_layer_norm.weight": sd["model.ln_final.weight"], "text_model.final_layer_norm.bias": sd["model.ln_final.bias"],
               "text_projection.weight": sd["model.text_projection"].t().contiguous()})
    missing, unexpected = tm.load_state_dict(hf, strict=False)
    assert not unexpected and all("position_ids" in m for m in missing), (missing, unexpected)
    g = torch.Generator().manual_seed(2)
    tokens = torch.randint(1, t["vocab_size"] - 1, (2, t["context_length"]), generator=g)
    tokens[0, 9], tokens[1, 15] = t["vocab_size"] - 1, t["vocab_size"] - 1       # EOS = highest id (argmax pooling)
    tokens[0, 10:] = 0
    with torch.no_grad():
        ref = tm(input_ids=tokens, output_hidden_states=True)
    xt, x = OC.encode_text(sd, tokens, cfg, layer_idx=0)
    assert torch.allclose(x, ref.last_hidden_state, atol=2e-4, rtol=1e-4)
    assert torch.allclose(xt, ref.text_embeds, atol=2e-4, rtol=1e-4)
    _, xp = OC.encode_text(sd, tokens, cfg, layer_idx=1)                            # "penultimate": ln_final(hidden_states[-2])
    with torch.no_grad():
        pen = tm.text_model.final_layer_norm(ref.hidden_states[-2])
    assert torch.allclose(xp, pen, atol=2e-4, rtol=1e-4)

    vm = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=v["width"], intermediate_size=v["mlp"], num_hidden_layers=v["layers"],
                                                        num_attention_heads=v["heads"], image_size=v["image_size"],
                                                        patch_size=v["patch_size"], hidden_act="gelu", projection_dim=cfg["embed_dim"],
                                                        attn_implementation="eager")).eval()
    hf = map_blocks("model.visual.transformer.", "vision_model.", v["layers"], v["width"])
    hf.update({"vision_model.embeddings.patch_embedding.weight": sd["model.visual.conv1.weight"],
               "vision_model.embeddings.class_embedding": sd["model.visual.class_embedding"],
               "vision_model.embeddings.position_embedding.weight": sd["model.visual.positional_embedding"],
               "vision_model.pre_layrnorm.weight": sd["model.visual.ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["model.visual.ln_pre.bias"],
               "vision_model.post_layernorm.weight": sd["model.visual.ln_post.weight"], "vision_model.post_layernorm.bias": sd["model.visual.ln_post.bias"],
               "visual_projection.weight": sd["model.visual.proj"].t().contiguous()})
    missing, unexpected = vm.load_state_dict(hf, strict=False)
    assert not unexpected and all("position_ids" in m for m in missing), (missing, unexpected)
    img = torch.randn((2, 3, 56, 56), generator=g)
    with torch.no_grad():
        iref = vm(pixel_values=img).image_embeds
    assert torch.allclose(OC.encode_image(sd, img, cfg), iref, atol=2e-4, rtol=1e-4)


def test_gligen_plms_sampler_matches_reference_sampler():
    """§8(f2) GLIGEN sampling loop: vitron_b200.gligen_sampler.{DDPM, PLMSSampler, alpha_generator} against the UNMODIFIED
    reference PLMSSampler / DDPM driven by the same analytic eps-model (CFG, gate schedule callback, inpainting blend).
    Pure fp32 host arithmetic: tight tolerance, no GPU involved."""
    from oracle import refshim
    if not refshim.available():
        pytest.skip("reference tree not present")
    from functools import partial
    from vitron_b200 import gligen_sampler as GS
    RefPLMS, RefDDPM = refshim.gligen_plms_classes()
    rd, md = RefDDPM(), GS.DDPM()
    assert torch.allclose(rd.alphas_cumprod, md.alphas_cumprod, atol=0, rtol=1e-6)
    # the vendored DDPM (ddpm.py) carries the schedule only; plms.py:98 calls `diffusion.q_sample`, which upstream GLIGEN
    # defines on its LatentDiffusion subclass (standard sqrt(ac) x0 + sqrt(1 - ac) eps): supply that to the reference object
    rd.q_sample = lambda x_start, t: (rd.sqrt_alphas_cumprod[t].view(-1, 1, 1, 1) * x_start
                                      + rd.sqrt_one_minus_alphas_cumprod[t].view(-1, 1, 1, 1) * torch.randn_like(x_start))
    g = torch.Generator().manual_seed(5)
    ctx, uc = torch.randn((2, 3, 4), generator=g), torch.randn((2, 3, 4), generator=g)
    bias = torch.randn((2, 4, 8, 8), generator=g) * 0.2

    class Model:
        scale = 1.0

        def __call__(self, inp):
            t = inp["timesteps"].view(-1, 1, 1, 1).float() / 1000.0
            return torch.tanh(inp["x"]) * 0.4 + bias * t * self.scale + inp["context"].mean(dim=(1, 2)).view(-1, 1, 1, 1) * 0.1

    calls_r, calls_m = [], []
    setter = lambda log: (lambda model, a: (log.append(float(a)), setattr(model, "scale", float(a)))[0])
    x_start = torch.randn((2, 4, 8, 8), generator=g)
    for kind in ("plain", "inpaint"):
        mask = (torch.rand((2, 1, 8, 8), generator=g) > 0.5).float() if kind == "inpaint" else None
        x0 = torch.randn((2, 4, 8, 8), generator=g) if kind == "inpaint" else None
        mr, mm = Model(), Model()
        ref_s = RefPLMS(rd, mr, alpha_generator_func=partial(GS.alpha_generator, type=[0.3, 0.2, 0.5]), set_alpha_scale=setter(calls_r))
        my_s = GS.PLMSSampler(md, mm, alpha_generator_func=partial(GS.alpha_generator, type=[0.3, 0.2, 0.5]), set_alpha_scale=setter(calls_m))
        torch.manual_seed(0)   # q_sample noise of the inpainting blend: both sides draw the same stream
        ref = ref_s.sample(S=10, shape=(2, 4, 8, 8), input=dict(x=x_start.clone(), timesteps=None, context=ctx), uc=uc,
                           guidance_scale=5.0, mask=mask, x0=x0)
        torch.manual_seed(0)
        got = my_s.sample(S=10, shape=(2, 4, 8, 8), input=dict(x=x_start.clone(), timesteps=None, context=ctx), uc=uc,
                          guidance_scale=5.0, mask=mask, x0=x0)
        assert torch.allclose(got, ref, atol=2e-5, rtol=1e-4), (kind, (got - ref).abs().max())
    assert calls_r == calls_m and len(calls_m) == 20
    ra = importlib_alpha = GS.alpha_generator(50, [0.3, 0.0, 0.7])
    assert ra[:15] == [1] * 15 and ra[15:] == [0] * 35
