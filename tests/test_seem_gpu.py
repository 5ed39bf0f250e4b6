"""GPU parity for SURVEY.md §8 rows a10 (SEEM pixel decoder) and a11 (SEEM mask decoder), task 'seg':
CUDA path vs the CPU oracle restatement (pinned at module level against the unmodified reference classes,
tests/test_oracle_cpu.py::test_seem_restatement_matches_*) and vs the reference's own golden outputs
(tests/golden/seem_tiny.pt). Float outputs: <= 5% inf / 4% L2;
bool attention masks: identical except where the oracle's mask logit is within the float tolerance
of the 0 threshold (mask-pixel decisions are bit-exact away from that band)."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def assert_close(got, ref, what, rel_inf=0.05, rel_l2=0.04):
    got, ref = got.float().cpu(), ref.float().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    scale = ref.abs().max().item() + 1e-6
    e_inf = (got - ref).abs().max().item() / scale
    e_l2 = ((got - ref).norm() / (ref.norm() + 1e-6)).item()
    assert e_inf < rel_inf and e_l2 < rel_l2, f"{what}: inf {e_inf:.4f} l2 {e_l2:.4f}"


def build(cuda, in_ch, C, ffn, Q, enc_layers, dec_layers, heads, dim_proj, seed):
    from oracle import restate_seem as S
    from oracle.weights import seeded_state_dict
    from vitron_b200.seem import MultiScaleMaskedTransformerDecoder, TransformerEncoderPixelDecoder, XDecoderHead
    shapes = S.seem_shapes(in_ch, C, ffn, Q, enc_layers, dec_layers, dim_proj)
    sd = seeded_state_dict(shapes, seed, 0.6)
    pd = TransformerEncoderPixelDecoder(in_ch, C, C, heads, ffn, enc_layers, device=cuda)
    pr = MultiScaleMaskedTransformerDecoder(C, dim_proj, Q, heads, ffn, dec_layers, C, device=cuda)
    head = XDecoderHead(pd, pr).load_state_dict(sd)
    return sd, head


@pytest.mark.parametrize("size", [(64, 96), (128, 128)])
def test_seem_pixel_and_mask_decoder_vs_oracle(cuda, size):
    from oracle import restate_seem as S
    in_ch, C, ffn, Q, heads, dim_proj = (64, 128, 192, 256), 512, 1024, 101, 8, 512
    enc_layers, dec_layers = 2, 9
    sd, head = build(cuda, in_ch, C, ffn, Q, enc_layers, dec_layers, heads, dim_proj, 4)
    g = torch.Generator().manual_seed(1)
    H, W = size
    feats = {f"res{i + 2}": torch.randn((1, c, H >> i, W >> i), generator=g) for i, c in enumerate(in_ch)}
    t_emb = torch.randn((20, dim_proj), generator=g)
    t_emb = t_emb / t_emb.norm(dim=-1, keepdim=True)
    head.predictor.set_text_embeddings(t_emb, 2.0)

    mf_r, enc_r, multi_r = S.pixel_decoder_forward(sd, feats, "pixel_decoder.", nheads=heads, enc_layers=enc_layers)
    mf, enc, multi = head.pixel_decoder.forward_features({k: v.to(cuda) for k, v in feats.items()})
    assert_close(enc, enc_r, "transformer encoder features")
    for a, b in zip(multi, multi_r):
        assert_close(a, b, "multi-scale feature")
    assert_close(mf, mf_r, "mask_features")

    # mask decoder on the ORACLE's pixel-decoder outputs (isolates a11 from a10's rounding)
    ref = S.mask_decoder_forward(sd, multi_r, mf_r, "predictor.", heads=heads, num_layers=dec_layers, t_emb=t_emb, logit_scale=2.0)
    out = head.predictor([m.to(cuda) for m in multi_r], mf_r.to(cuda))
    assert set(["pred_logits", "pred_masks", "pred_maskembs", "aux_outputs"]) <= set(out)
    assert len(out["aux_outputs"]) == dec_layers
    # first-layer quantities see no error accumulation: tight check incl. the bool masks
    a0, r0 = out["aux_outputs"][0], ref["aux_outputs"][0]
    assert_close(a0["pred_masks"], r0["pred_masks"], "layer-0 mask logits", 0.02, 0.02)
    check_masks(out["attn_masks"][0], ref["attn_masks"][0], r0["pred_masks"], heads, 0.03, (H >> 3, W >> 3))
    # after 9 layers of thresholded masks a borderline pixel may flip for one query: L2 stays tight, the
    # inf-norm bound is loose on purpose (the map is discontinuous at the threshold)
    assert_close(out["pred_maskembs"], ref["pred_maskembs"], "pred_maskembs", 0.3, 0.06)
    assert_close(out["pred_masks"], ref["pred_masks"], "pred_masks", 0.3, 0.06)
    assert_close(out["pred_logits"], ref["pred_logits"], "pred_logits", 0.3, 0.06)


def check_masks(got, ref_raw, ref_logits, heads, tol_frac, size):
    """got [B,1,Q,N] uint8 (reset applied); ref_raw [B*heads,Q,N] bool (raw); ref_logits [B,Q,H,W].
    Mask-pixel decisions must be IDENTICAL wherever the oracle's resized logit is further from the 0
    threshold than the float tolerance; inside that band either decision is admissible."""
    import torch.nn.functional as F
    B, _, Q, N = got.shape
    ref = ref_raw.view(B, heads, Q, N)[:, 0].clone()
    full = ref.sum(-1) == N
    ref[torch.where(full)] = False  # AttentionDataStruct.cross_attn_mask reset rule
    got = got[:, 0].bool().cpu()
    resized = F.interpolate(ref_logits.float(), size=size, mode="bilinear", align_corners=False).flatten(2)
    band = resized.abs() <= tol_frac * ref_logits.abs().max()
    # the fully-masked-row reset can be triggered on one side only by a pixel inside the band:
    #  - oracle row fully masked (reset to all-False): our raw row may keep True everywhere except band pixels
    #  - our row reset to all-False: every oracle-unmasked pixel of that row must lie inside the band
    ours_reset = (got.sum(-1) == 0) & (ref.sum(-1) > 0)
    normal = ~full & ~ours_reset
    bad = ((got != ref) & ~band & normal[:, :, None]).sum().item()
    bad += ((~ref) & ~band & ours_reset[:, :, None]).sum().item()
    bad += ((~got) & ~band & full[:, :, None] & (got.sum(-1) > 0)[:, :, None]).sum().item()
    assert bad == 0, f"{bad} mask pixels differ outside the tolerance band"
    assert band.float().mean().item() < 0.2


def test_seem_end_to_end_head(cuda):
    """XDecoderHead.layers(features) with tiny dims and an odd (non 2x) FPN size chain."""
    from oracle import restate_seem as S
    in_ch, C, ffn, Q, heads, dim_proj = (32, 64, 64, 96), 128, 256, 16, 2, 64
    sd, head = build(cuda, in_ch, C, ffn, Q, 1, 3, heads, dim_proj, 9)
    g = torch.Generator().manual_seed(5)
    sizes = [(36, 52), (18, 26), (9, 13), (5, 7)]
    feats = {f"res{i + 2}": torch.randn((2, c, *sizes[i]), generator=g) for i, c in enumerate(in_ch)}
    mf_r, enc_r, multi_r = S.pixel_decoder_forward(sd, feats, "pixel_decoder.", nheads=heads, enc_layers=1)
    ref = S.mask_decoder_forward(sd, multi_r, mf_r, "predictor.", heads=heads, num_layers=3)
    out = head({k: v.to(cuda) for k, v in feats.items()})
    assert out["pred_logits"] is None
    assert_close(out["aux_outputs"][0]["pred_masks"], ref["aux_outputs"][0]["pred_masks"], "e2e layer-0 masks", 0.06, 0.05)
    assert_close(out["pred_masks"], ref["pred_masks"], "e2e pred_masks", 0.12, 0.1)
    # interactive prompts (`extra` keys) are covered by test_seem_prompts_vs_reference_golden


def test_seem_vs_reference_golden(cuda):
    """Product path against outputs of the UNMODIFIED reference classes (tests/golden/seem_tiny.pt)."""
    import os
    from oracle.weights import seeded_state_dict
    from vitron_b200.seem import MultiScaleMaskedTransformerDecoder, TransformerEncoderPixelDecoder, XDecoderHead
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "seem_tiny.pt"), weights_only=False)
    t = fx["cfg"]
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    pd = TransformerEncoderPixelDecoder(t["in_channels"], t["C"], t["C"], t["heads"], t["ffn"], t["enc_layers"], device=cuda)
    pr = MultiScaleMaskedTransformerDecoder(t["C"], t["dim_proj"], t["Q"], t["heads"], t["ffn"], t["dec_layers"], t["C"], device=cuda)
    head = XDecoderHead(pd, pr).load_state_dict(sd)
    head.predictor.set_text_embeddings(fx["t_emb"], t["logit_scale"])
    mf, enc, multi = head.pixel_decoder.forward_features({k: v.to(cuda) for k, v in fx["features"].items()})
    assert_close(enc, fx["enc_features"], "golden transformer encoder features")
    for a, b in zip(multi, fx["multi_scale"]):
        assert_close(a, b, "golden multi-scale feature")
    assert_close(mf, fx["mask_features"], "golden mask_features")
    out = head.predictor([m.to(cuda) for m in fx["multi_scale"]], fx["mask_features"].to(cuda))
    ref = fx["out"]
    assert_close(out["aux_outputs"][0]["pred_masks"], ref["aux_outputs"][0]["pred_masks"], "golden layer-0 mask logits", 0.03, 0.03)
    assert_close(out["aux_outputs"][0]["pred_logits"], ref["aux_outputs"][0]["pred_logits"], "golden layer-0 class logits", 0.03, 0.03)
    assert_close(out["pred_masks"], ref["pred_masks"], "golden pred_masks", 0.3, 0.08)
    assert_close(out["pred_maskembs"], ref["pred_maskembs"], "golden pred_maskembs", 0.3, 0.08)


def test_seem_head_graph_replay_equals_eager(cuda):
    """XDecoderHead.enable_graph(): the CUDA-graph replay of the whole head returns exactly what the eager launch sequence
    returns (same kernels, same order), on two consecutive inputs (static buffers are refreshed)."""
    in_ch, C, ffn, Q, heads, dim_proj = (32, 64, 64, 96), 128, 256, 16, 2, 64
    sd, head = build(cuda, in_ch, C, ffn, Q, 1, 3, heads, dim_proj, 9)
    g = torch.Generator().manual_seed(5)
    sizes = [(32, 48), (16, 24), (8, 12), (4, 6)]
    outs = []
    for rep in range(2):
        feats = {f"res{i + 2}": torch.randn((1, c, *sizes[i]), generator=g).to(cuda) for i, c in enumerate(in_ch)}
        head.enable_graph(False)
        eager = head(feats)
        e_masks, e_emb = eager["pred_masks"].clone(), eager["pred_maskembs"].clone()
        head.enable_graph(True)
        got = head(feats)
        # same kernels in the same order; the GroupNorm group sums are fp32 atomics (order-dependent in the last bits), so the
        # comparison is to rounding level, not bit-wise
        for a, b_ in ((got["pred_masks"], e_masks), (got["pred_maskembs"], e_emb)):
            assert (a.float() - b_.float()).abs().max().item() <= 2e-2 * b_.float().abs().max().item(), rep
        outs.append(e_masks)
    assert not torch.equal(outs[0], outs[1])


def test_seem_inference_mode_without_aux_outputs(cuda):
    """predictor.aux_outputs = False (what the reference's evaluate() needs): intermediate layers derive only the next
    layer's attention mask, from mask_features resized once per level; final masks / logits / embeddings stay within
    rounding of the aux-on run, the intermediate attention masks agree except for logits next to the threshold."""
    in_ch, C, ffn, Q, heads, dim_proj = (32, 64, 64, 96), 128, 256, 16, 2, 64
    sd, head = build(cuda, in_ch, C, ffn, Q, 1, 3, heads, dim_proj, 9)
    g = torch.Generator().manual_seed(6)
    sizes = [(64, 96), (32, 48), (16, 24), (8, 12)]
    feats = {f"res{i + 2}": torch.randn((2, c, *sizes[i]), generator=g).to(cuda) for i, c in enumerate(in_ch)}
    full = head(feats)
    f_masks, f_emb, f_att = full["pred_masks"].clone(), full["pred_maskembs"].clone(), [m.clone() for m in full["attn_masks"]]
    assert len(full["aux_outputs"]) == 3   # dec_layers of this test head
    head.predictor.aux_outputs = False
    fast = head(feats)
    assert fast["aux_outputs"] == []
    assert_close(fast["pred_masks"], f_masks, "pred_masks aux off vs on", 0.08, 0.06)
    assert_close(fast["pred_maskembs"], f_emb, "pred_maskembs aux off vs on", 0.08, 0.06)
    agree = [float((a == b).float().mean()) for a, b in zip(fast["attn_masks"], f_att)]
    assert min(agree) > 0.97, agree
    head.enable_graph(True)       # and under graph replay (folded position terms are cached tensors)
    g1 = head(feats)
    assert_close(g1["pred_masks"], f_masks, "graph, aux off", 0.08, 0.06)


def test_seem_interactive_prompts_vs_reference_golden(cuda):
    """Grounding / audio token prompts, spatial point prompts and the refimg -> visual route on the CUDA kernels against the
    golden outputs of the UNMODIFIED reference decoder (tests/golden/seem_prompts_tiny.pt): the self-attention over
    [object queries | prompt tokens] runs as masked attention on the wgmma kernel."""
    import os
    from oracle.weights import seeded_state_dict
    from vitron_b200.seem import MultiScaleMaskedTransformerDecoder
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "seem_prompts_tiny.pt"), weights_only=False)
    t = fx["cfg"]
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    pr = MultiScaleMaskedTransformerDecoder(t["C"], t["dim_proj"], t["Q"], t["heads"], t["ffn"], t["dec_layers"], t["C"], device=cuda)
    pr.load_state_dict(sd, "predictor.")
    pr.set_text_embeddings(fx["t_emb"], t["logit_scale"])
    multi, mf = [m.to(cuda) for m in fx["multi_scale"]], fx["mask_features"].to(cuda)
    dev = lambda e: {k: ([m.to(cuda) for m in v] if isinstance(v, list) else v.to(cuda)) for k, v in e.items()}

    def check(out, ref, what):
        for k, v in ref.items():
            if k == "aux0":
                continue
            lim = (0.05, 0.04) if "spatial" in k or "visual" in k else (0.3, 0.09)
            assert_close(out[k], v, f"{what} {k}", *lim)
        for k, v in ref.get("aux0", {}).items():
            assert_close(out["aux_outputs"][0][k], v, f"{what} layer-0 {k}", 0.04, 0.03)
    for name, extra in fx["cases"].items():
        check(pr(multi, mf, task="seg", extra=dev(extra)), fx["out"][name], name)
    ref = pr(multi, mf, task="refimg", extra=dev(fx["cases"]["spatial"]))
    for k in ("visual_query_pos", "visual_query_neg"):
        assert_close(ref[k], fx["refimg"][k], k, 0.04, 0.03)
    vis = {k: ref[k] for k in ("visual_query_pos", "visual_query_neg", "src_visual_queries", "src_visual_maskings")}
    check(pr(multi, mf, task="seg", extra=vis), fx["out"]["visual"], "visual")
