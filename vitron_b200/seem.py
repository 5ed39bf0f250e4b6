"""SEEM pixel decoder + mask decoder on the vitron_b200 kernels (panoptic / 'seg' path).

Drop-ins for modules/SEEM/demo_code/xdecoder:
  * `TransformerEncoderPixelDecoder.forward_features(features)` — body/encoder/
    transformer_encoder_fpn.py:194-303 (FPN: 1x1 lateral + nearest-upsample add + 3x3 conv+GN+ReLU;
    6 post-norm encoder layers on res5 — body/transformer_blocks.py:154-232; 3x3 mask_features conv)
  * `MultiScaleMaskedTransformerDecoder.forward(x, mask_features, mask=None, target_queries=None,
    target_vlp=None, task='seg', extra={})` — body/decoder/seem.py:395-586 with
    CrossAttentionLayer/SelfAttentionLayer/FFNLayer :29-189 (post-norm), `prepare_features`
    (utils/utils.py:18-32), PositionEmbeddingSine (modules/position_encoding.py:18-52), the
    bool-mask rule of AttentionDataStruct.cross_attn_mask (attention_data_struct.py:173-187) and
    LanguageEncoder.compute_similarity (language/vlpencoder.py:293-299)
  * `XDecoderHead.layers` = pixel_decoder + predictor (body/xdecoder_head.py:103-118)
State-dict names are the reference's. Interactive prompts (spatial / grounding / visual / audio
`extra` keys) are not on the BASELINE path and raise NotImplementedError (DESIGN.md "next").

Design: NHWC bf16 throughout; the K/V projections of the memory for the 3 layers that share a
feature level are ONE grouped GEMM per level (N = 3 x 512); the mask head `einsum('bqc,bchw->bqhw')`
is a GEMM against the NHWC mask_features viewed as [HW, C]; the next layer's bool attention mask
(bilinear resize, sigmoid < 0.5, fully-masked-row reset) is one fused kernel with the threshold
decision in fp32; masked cross-attention never materialises Q x HW scores.
"""
import math

import torch
import torch.nn.functional as F

from . import ops

BF16 = torch.bfloat16


def position_embedding_sine(h, w, num_pos_feats, device, temperature=10000, scale=2 * math.pi):
    """PositionEmbeddingSine(normalize=True) for an unmasked h x w map -> [h*w, 2*num_pos_feats] fp32."""
    y_embed = torch.arange(1, h + 1, dtype=torch.float32, device=device)[:, None].expand(h, w)
    x_embed = torch.arange(1, w + 1, dtype=torch.float32, device=device)[None, :].expand(h, w)
    eps = 1e-6
    y_embed = y_embed / (y_embed[-1:, :] + eps) * scale
    x_embed = x_embed / (x_embed[:, -1:] + eps) * scale
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=device)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    pos_x = x_embed[:, :, None] / dim_t
    pos_y = y_embed[:, :, None] / dim_t
    pos_x = torch.stack((pos_x[:, :, 0::2].sin(), pos_x[:, :, 1::2].cos()), dim=3).flatten(2)
    pos_y = torch.stack((pos_y[:, :, 0::2].sin(), pos_y[:, :, 1::2].cos()), dim=3).flatten(2)
    return torch.cat((pos_y, pos_x), dim=2).reshape(h * w, 2 * num_pos_feats)


def _nhwc(x):
    """NCHW (any float dtype) -> contiguous NHWC bf16."""
    return x.permute(0, 2, 3, 1).to(BF16).contiguous()


def _nearest_to(y, h, w):
    n, hy, wy, c = y.shape
    if h == 2 * hy and w == 2 * wy:
        return ops.upsample2x_nhwc(y)
    iy = torch.div(torch.arange(h, device=y.device) * hy, h, rounding_mode="floor")
    ix = torch.div(torch.arange(w, device=y.device) * wy, w, rounding_mode="floor")
    return y[:, iy][:, :, ix].contiguous()


class _MHA:
    """nn.MultiheadAttention weights split for fused use: q/k share their input in every SEEM layer."""

    def __init__(self, sd, p, dev):
        g = lambda n: sd[p + n].detach().to(device=dev, dtype=BF16).contiguous()
        w, b = g("in_proj_weight"), g("in_proj_bias")
        d = w.shape[1]
        self.d = d
        self.wq, self.wk, self.wv = w[:d].contiguous(), w[d:2 * d].contiguous(), w[2 * d:].contiguous()
        self.bq, self.bk, self.bv = b[:d].contiguous(), b[d:2 * d].contiguous(), b[2 * d:].contiguous()
        self.wqk, self.bqk = w[:2 * d].contiguous(), b[:2 * d].contiguous()
        self.wo, self.bo = g("out_proj.weight"), g("out_proj.bias")


class TransformerEncoderPixelDecoder:
    def __init__(self, in_channels=(192, 384, 768, 1536), conv_dim=512, mask_dim=512, nheads=8, dim_feedforward=2048,
                 enc_layers=6, in_features=("res2", "res3", "res4", "res5"), device="cuda"):
        self.in_features = list(in_features)
        self.in_channels = list(in_channels)
        self.conv_dim, self.mask_dim, self.nheads, self.enc_layers = conv_dim, mask_dim, nheads, enc_layers
        self.device = torch.device(device)
        self.maskformer_num_feature_levels = 3
        self._pos = {}
        self._folded = {}   # per (layer, h, w): pos @ Wqk^T + b, the constant half of (src + pos) Wqk + b

    def load_state_dict(self, sd, prefix=""):
        self._folded = {}
        dev = self.device
        g = lambda n: sd[prefix + n].detach().to(device=dev, dtype=BF16).contiguous()
        L = len(self.in_features)
        w = {"input_proj": (g("input_proj.weight").reshape(self.conv_dim, -1).contiguous(), g("input_proj.bias"))}
        w["enc"] = []
        for i in range(self.enc_layers):
            p = f"transformer.encoder.layers.{i}."
            w["enc"].append(dict(att=_MHA(sd, prefix + p + "self_attn.", dev), l1=(g(p + "linear1.weight"), g(p + "linear1.bias")),
                                 l2=(g(p + "linear2.weight"), g(p + "linear2.bias")), n1=(g(p + "norm1.weight"), g(p + "norm1.bias")),
                                 n2=(g(p + "norm2.weight"), g(p + "norm2.bias"))))
        for idx in range(L):
            k = idx + 1
            w[f"layer_{k}"] = (ops.pack_conv_weight(g(f"layer_{k}.weight")), g(f"layer_{k}.norm.weight"), g(f"layer_{k}.norm.bias"))
            if idx != L - 1:
                aw = g(f"adapter_{k}.weight")
                w[f"adapter_{k}"] = (aw.reshape(aw.shape[0], -1).contiguous(), g(f"adapter_{k}.norm.weight"), g(f"adapter_{k}.norm.bias"))
        w["mask_features"] = (ops.pack_conv_weight(g("mask_features.weight")), g("mask_features.bias"))
        self.w = w
        return self

    def _pe(self, h, w):
        key = (h, w)
        if key not in self._pos:
            self._pos[key] = position_embedding_sine(h, w, self.conv_dim // 2, self.device).to(BF16).contiguous()
        return self._pos[key]

    def _out_conv(self, y, name):
        cw, gw, gb = self.w[name]
        return ops.groupnorm_nhwc(ops.conv_nhwc(y, cw, 3, 3), gw, gb, 32, 1e-5, act=ops.ACT_RELU)

    @torch.no_grad()
    def forward_features(self, features):
        """features: {'res2'..'res5': [B, C, H, W]} -> (mask_features, transformer_encoder_features,
        multi_scale_features[3]) as NCHW-shaped views of NHWC bf16 storage."""
        C, H = self.conv_dim, self.nheads
        hd = C // H
        multi = []
        y = None
        enc_feat = None
        for idx, f in enumerate(self.in_features[::-1]):
            x = _nhwc(features[f].to(self.device))
            n, h, w, cin = x.shape
            k = len(self.in_features) - idx
            if idx == 0:
                src = ops.gemm(x.view(n * h * w, cin), self.w["input_proj"][0], bias=self.w["input_proj"][1])
                pos = self._pe(h, w)
                for li, lw in enumerate(self.w["enc"]):
                    a = lw["att"]
                    if n == 1:   # (src + pos) Wqk + b = src Wqk + [pos Wqk + b]: constant per feature-map size
                        key = ("enc", li, h, w)
                        if key not in self._folded:
                            self._folded[key] = ops.gemm(pos, a.wqk, bias=a.bqk).contiguous()
                        qk = ops.gemm(src, a.wqk, rowbias=self._folded[key], rowbias_rows=1).view(n, h * w, 2, H, hd)
                    else:
                        qk = ops.gemm(ops.add(src, pos), a.wqk, bias=a.bqk).view(n, h * w, 2, H, hd)
                    v = ops.gemm(src, a.wv, bias=a.bv).view(n, h * w, H, hd)
                    att = ops.attention(qk[:, :, 0], qk[:, :, 1], v, scale=hd ** -0.5)
                    ops.gemm(att.view(n * h * w, C), a.wo, bias=a.bo, residual=src, out=src)
                    ops.layernorm(src, *lw["n1"], 1e-5, out=src)
                    ff = ops.gemm(src, lw["l1"][0], bias=lw["l1"][1], act=ops.ACT_RELU)
                    ops.gemm(ff, lw["l2"][0], bias=lw["l2"][1], residual=src, out=src)
                    ops.layernorm(src, *lw["n2"], 1e-5, out=src)
                enc_feat = src.view(n, h, w, C)
                y = self._out_conv(enc_feat, f"layer_{k}")
            else:
                aw, gw, gb = self.w[f"adapter_{k}"]
                cur = ops.gemm(x.view(n * h * w, cin), aw).view(n, h, w, C)
                cur = ops.groupnorm_nhwc(cur, gw, gb, 32, 1e-5)
                y = ops.add(cur, _nearest_to(y, h, w))
                y = self._out_conv(y, f"layer_{k}")
            if len(multi) < self.maskformer_num_feature_levels:
                multi.append(y)
        mf = ops.conv_nhwc(y, self.w["mask_features"][0], 3, 3, bias=self.w["mask_features"][1])
        nchw = lambda t: t.permute(0, 3, 1, 2)
        return nchw(mf), nchw(enc_feat), [nchw(m) for m in multi]


class MultiScaleMaskedTransformerDecoder:
    def __init__(self, hidden_dim=512, dim_proj=512, num_queries=101, nheads=8, dim_feedforward=2048, dec_layers=9,
                 mask_dim=512, device="cuda", task_switch=None, max_spatial_len=(512, 512, 512, 512)):
        self.hidden_dim, self.dim_proj, self.num_queries = hidden_dim, dim_proj, num_queries
        self.num_heads, self.num_layers, self.mask_dim = nheads, dec_layers, mask_dim
        self.num_feature_levels = 3
        self.device = torch.device(device)
        self.text_embeddings = None
        self.logit_scale = 0.0
        self._pos = {}
        # aux_outputs=True (reference behaviour): every layer's full-resolution pred_masks / pred_logits are computed and
        # returned under 'aux_outputs'. False (inference: the reference's evaluate() never reads them): intermediate layers
        # only produce the NEXT layer's attention mask, from mask_features resized once per level (bilinear is linear, see
        # vb200_resize_bilinear_nhwc) — no [Q, H, W] fp32 map, no class / caption logits for them; 'aux_outputs' is [].
        self.aux_outputs = True
        self._folded = {}
        # seem_focall_lang.yaml:60-86 enables MASK / SPATIAL / GROUNDING / VISUAL / AUDIO for the demo model
        self.task_switch = dict(mask=True, spatial=True, grounding=True, visual=True, audio=True)
        self.task_switch.update(task_switch or {})
        self.max_spatial_len = list(max_spatial_len)
        self.mask_sptial_embed = None   # (sic) seem.py:342
        self.pn_indicator = None

    def set_text_embeddings(self, t_emb, logit_scale):
        """Stand-in for lang_encoder.default_text_embeddings / logit_scale (vlpencoder.py:293-299)."""
        self.text_embeddings = t_emb.detach().to(device=self.device, dtype=BF16).contiguous()
        self.logit_scale = float(logit_scale)

    def load_state_dict(self, sd, prefix=""):
        self._folded = {}
        dev = self.device
        g = lambda n: sd[prefix + n].detach().to(device=dev, dtype=BF16).contiguous()
        L = self.num_layers
        self.cross = [dict(att=_MHA(sd, prefix + f"transformer_cross_attention_layers.{i}.multihead_attn.", dev),
                           n=(g(f"transformer_cross_attention_layers.{i}.norm.weight"), g(f"transformer_cross_attention_layers.{i}.norm.bias")))
                      for i in range(L)]
        self.selfa = [dict(att=_MHA(sd, prefix + f"transformer_self_attention_layers.{i}.self_attn.", dev),
                           n=(g(f"transformer_self_attention_layers.{i}.norm.weight"), g(f"transformer_self_attention_layers.{i}.norm.bias")))
                      for i in range(L)]
        self.ffn = [dict(l1=(g(f"transformer_ffn_layers.{i}.linear1.weight"), g(f"transformer_ffn_layers.{i}.linear1.bias")),
                         l2=(g(f"transformer_ffn_layers.{i}.linear2.weight"), g(f"transformer_ffn_layers.{i}.linear2.bias")),
                         n=(g(f"transformer_ffn_layers.{i}.norm.weight"), g(f"transformer_ffn_layers.{i}.norm.bias"))) for i in range(L)]
        self.decoder_norm = (g("decoder_norm.weight"), g("decoder_norm.bias"))
        self.query_feat, self.query_embed, self.level_embed = g("query_feat.weight"), g("query_embed.weight"), g("level_embed.weight")
        self.mask_embed = [(g(f"mask_embed.layers.{i}.weight"), g(f"mask_embed.layers.{i}.bias")) for i in range(3)]
        self.class_embed_t = g("class_embed").t().contiguous()  # [dim_proj, hidden] as a GEMM weight
        if prefix + "mask_sptial_embed.0" in sd:                  # spatial prompts (seem.py:342-347, 312)
            self.mask_sptial_embed = [g(f"mask_sptial_embed.{i}").t().contiguous() for i in range(3)]   # x @ E == gemm(x, E^T)
            self.pn_indicator = sd[prefix + "pn_indicator.weight"].detach().to(device=dev, dtype=torch.float32)
        # grouped K / V projection weights per feature level (level l feeds layers l, l+3, l+6)
        self.kgrp, self.vgrp = [], []
        for lvl in range(self.num_feature_levels):
            ids = [i for i in range(L) if i % self.num_feature_levels == lvl]
            self.kgrp.append((ids, torch.cat([self.cross[i]["att"].wk for i in ids], 0).contiguous(),
                              torch.cat([self.cross[i]["att"].bk for i in ids], 0).contiguous()))
            self.vgrp.append((ids, torch.cat([self.cross[i]["att"].wv for i in ids], 0).contiguous(),
                              torch.cat([self.cross[i]["att"].bv for i in ids], 0).contiguous()))
        return self

    def _pe(self, h, w):
        if (h, w) not in self._pos:
            self._pos[(h, w)] = position_embedding_sine(h, w, self.hidden_dim // 2, self.device).to(BF16).contiguous()
        return self._pos[(h, w)]

    def _heads(self, output, mask_rows, mask_hw, target_size, bs, small_rows=None):
        """forward_prediction_heads (seem.py:555-586). output [bs*Q, C] rows (batch-major). small_rows (aux_outputs off,
        intermediate layers): per-sample rows of mask_features already resized to target_size -> only the attention mask."""
        Q, C = self.num_queries, self.hidden_dim
        dec = ops.layernorm(output, *self.decoder_norm, 1e-5)
        if small_rows is not None:
            me = dec
            for i, (w, b) in enumerate(self.mask_embed):
                me = ops.gemm(me, w, bias=b, act=ops.ACT_RELU if i < 2 else ops.ACT_NONE)
            h2, w2 = int(target_size[0]), int(target_size[1])
            logits = torch.empty((bs, Q, h2 * w2), dtype=torch.float32, device=output.device)
            for b in range(bs):
                ops.gemm(me[b * Q:(b + 1) * Q], small_rows[b], out=logits[b], out_fp32=True)
            attn_mask = ops.seem_attn_mask(logits.view(bs * Q, h2, w2), h2, w2)     # same size: threshold + row reset only
            return dict(attn_mask=attn_mask.view(bs, 1, Q, -1))
        class_embed = ops.gemm(dec, self.class_embed_t)  # decoder_output @ class_embed
        outputs_class = None
        if self.text_embeddings is not None:
            ce = class_embed.float()
            v = (ce / (ce.norm(dim=-1, keepdim=True) + 1e-7)).to(BF16).contiguous()
            outputs_class = ops.gemm(v, self.text_embeddings, alpha=math.exp(self.logit_scale), out_fp32=True)
            outputs_class = outputs_class.view(bs, Q, -1)
        me = dec
        for i, (w, b) in enumerate(self.mask_embed):
            me = ops.gemm(me, w, bias=b, act=ops.ACT_RELU if i < 2 else ops.ACT_NONE)
        H, W = mask_hw
        outputs_mask = torch.empty((bs, Q, H * W), dtype=torch.float32, device=output.device)
        for b in range(bs):  # einsum('bqc,bchw->bqhw') == mask_embed[b] @ mask_features[b]^T over NHWC rows
            ops.gemm(me[b * Q:(b + 1) * Q], mask_rows[b], out=outputs_mask[b], out_fp32=True)
        outputs_mask = outputs_mask.view(bs, Q, H, W)
        attn_mask = ops.seem_attn_mask(outputs_mask.view(bs * Q, H, W), int(target_size[0]), int(target_size[1]))
        attn_mask = attn_mask.view(bs, 1, Q, -1)  # shared by the heads; rows that were fully masked are already reset
        return dict(attn_mask=attn_mask, predictions_class=outputs_class, predictions_mask=outputs_mask,
                    predictions_caption=class_embed.view(bs, Q, -1), predictions_maskemb=me.view(bs, Q, -1))

    # ------------------------------------------------------------------ interactive prompts (seem.py:398-500)
    @staticmethod
    def _rand_sample(x, max_len):
        """utils.py:11-16 (same RNG call, so a seeded torch generator reproduces the reference's subset)."""
        if x.shape[1] <= max_len:
            return x
        return x[:, torch.randperm(x.shape[1])[:max_len]]

    @staticmethod
    def _point_sample(inp, coords):
        """detectron2 point_rend.point_sample(input [N,C,H,W], coords [N,P,2] in [0,1], align_corners=True) -> [N,C,P]."""
        return F.grid_sample(inp, 2.0 * coords.unsqueeze(2) - 1.0, align_corners=True).squeeze(3)

    def _spatial_prompts(self, extra, mask_features_nchw, src_rows, size_list, bs, task):
        """Spatial-query pre-processing (seem.py:414-469): sampled positive / negative points -> mean-pooled mask-feature
        queries (reported as pred_pspatials / pred_nspatials) and, per feature level, point-sampled tokens of
        src @ mask_sptial_embed[level] + pn_indicator with their padding masks. Index / gather work in torch on the device."""
        if self.mask_sptial_embed is None:
            raise ValueError("spatial prompts need mask_sptial_embed / pn_indicator in the state dict")
        dev = self.device
        pos_masks, neg_masks = extra["spatial_query_pos_mask"], extra["spatial_query_neg_mask"]
        _, h, w = pos_masks[0].shape
        divisor = torch.tensor([h, w], device=dev)[None, ]
        pad = torch.nn.utils.rnn.pad_sequence
        mf = mask_features_nchw.float()

        def mean_query(masks):
            pts = [self._rand_sample((m.to(dev).nonzero()[:, 1:] / divisor).t(), self.max_spatial_len[-1]).t() for m in masks]
            pts = pad(pts, padding_value=-1).permute(1, 0, 2)
            dead = pts.sum(dim=-1) < 0
            q = self._point_sample(mf, pts.flip(dims=(2,)).type(mf.dtype))
            return torch.stack([xx[m].mean(dim=0, keepdim=True) for xx, m in zip(q.transpose(1, 2), ~dead)]).transpose(0, 1).nan_to_num()
        spatial_query_pos, spatial_query_neg = mean_query(pos_masks), mean_query(neg_masks)
        tokens, maskings = [], []
        for i in range(self.num_feature_levels):
            hi, wi = size_list[i]
            feat = ops.gemm(src_rows[i], self.mask_sptial_embed[i]).view(bs, hi, wi, -1).permute(0, 3, 1, 2).float()   # [bs,C,h,w]
            ppos = [self._rand_sample((m.to(dev).nonzero()[:, 1:] / divisor).t(), self.max_spatial_len[i]).t() for m in pos_masks]
            pneg = [self._rand_sample((m.to(dev).nonzero()[:, 1:] / divisor).t(), self.max_spatial_len[i]).t() for m in neg_masks]
            pts = [torch.cat([a, b_], dim=0) for a, b_ in zip(ppos, pneg)]
            ind = pad([torch.cat([torch.ones(a.shape[0], device=dev), -torch.ones(b_.shape[0], device=dev)]) for a, b_ in zip(ppos, pneg)],
                      padding_value=0)                                                   # [P, bs]
            pts = pad(pts, padding_value=-1).permute(1, 0, 2)
            dead = pts.sum(dim=-1) < 0
            pts[dead] = 0
            tok = self._point_sample(feat, pts.flip(dims=(2,)).type(feat.dtype)).permute(2, 0, 1)   # [P, bs, C]
            tok[ind == 1] += self.pn_indicator[0:1]
            tok[ind == -1] += self.pn_indicator[1:2]
            tokens.append(tok)
            maskings.append(dead)
        return spatial_query_pos, spatial_query_neg, tokens, maskings

    def _self_attn_mask(self, Q, groups, bs):
        """AttentionDataStruct.self_attn (attention_data_struct.py:173-225) for the shipped ATTENTION_ARCH
        (seem_focall_lang.yaml:114-139): queries_object sees itself and every token group; tokens_grounding / tokens_audio see
        queries_object and themselves; tokens_spatial / tokens_visual only themselves; padded tokens are masked both ways.
        groups: [(name, T, masking [bs, T] bool or None)]. Returns uint8 [bs, 1, L, L], 1 = masked."""
        L = Q + sum(t for _, t, _ in groups)
        m = torch.ones((bs, L, L), dtype=torch.bool, device=self.device)
        m[:, :Q, :Q] = False
        off = Q
        spans = {}
        for name, T, _ in groups:
            spans[name] = (off, off + T)
            off += T
        for name, T, masking in groups:
            a, b_ = spans[name]
            m[:, :Q, a:b_] = False                          # queries_object -> tokens_*
            m[:, a:b_, a:b_] = False                        # tokens_* -> itself
            if name in ("tokens_grounding", "tokens_audio"):
                m[:, a:b_, :Q] = False                      # -> queries_object
        for name, T, masking in groups:                      # MASKING: padded tokens (bi-directional inside the group,
            if masking is None:                              # uni-directional against the object queries)
                continue
            a, b_ = spans[name]
            mk = masking.to(self.device).bool()
            blk = m[:, a:b_, a:b_]
            blk[mk] = True
            blk.transpose(1, 2)[mk] = True
            m[:, :Q, a:b_].transpose(1, 2)[mk] = True        # pair [queries_object, tokens_*]: key2 in masking -> its columns
            if name in ("tokens_grounding", "tokens_audio"):
                m[:, a:b_, :Q][mk] = True                    # pair [tokens_*, queries_object]: key1 in masking -> its rows
        return m.unsqueeze(1).to(torch.uint8).contiguous()

    @torch.no_grad()
    def forward(self, x, mask_features, mask=None, target_queries=None, target_vlp=None, task="seg", extra={}):
        extra = extra or {}
        spatial_flag = ("spatial_query_pos_mask" in extra or task == "refimg") and self.task_switch.get("spatial", False)
        grounding_flag = "grounding_tokens" in extra and self.task_switch.get("grounding", False)
        visual_flag = "visual_query_pos" in extra and self.task_switch.get("visual", False)
        audio_flag = "audio_tokens" in extra and self.task_switch.get("audio", False)
        if "prev_mask" in extra:
            raise NotImplementedError("spatial memories (prev_mask) are not part of the shipped ATTENTION_ARCH's cross attention")
        assert len(x) == self.num_feature_levels
        Q, C, H = self.num_queries, self.hidden_dim, self.num_heads
        hd = C // H
        bs = x[0].shape[0]
        dev = self.device
        # prepare_features: src = feat + level_embed (V input), src + pos (K input); rows are (b, hw)
        size_list, kproj, vproj, src_rows = [], {}, {}, []
        for lvl in range(self.num_feature_levels):
            f = _nhwc(x[lvl].to(dev))
            n, h, w, c = f.shape
            size_list.append((h, w))
            ids, wk, bk = self.kgrp[lvl]
            _, wv, bv = self.vgrp[lvl]
            need_src = ("spatial_query_pos_mask" in extra or task == "refimg") and self.task_switch.get("spatial", False)
            if n == 1 and not need_src:
                # K = (f + level_embed + pos) Wk + bk = f Wk + [(level_embed + pos) Wk + bk]  (a per-row additive term that
                # depends on the feature-map size only), V = (f + level_embed) Wv + bv = f Wv + [level_embed Wv + bv]:
                # the two elementwise passes over the level's features disappear into the GEMM epilogues
                key = ("kv", lvl, h, w)
                if key not in self._folded:
                    le = self.level_embed[lvl].contiguous()
                    kb = ops.gemm(ops.add(self._pe(h, w), le), wk, bias=bk)                       # [h*w, len(ids)*C]
                    vb = ops.gemm(le.view(1, -1).contiguous(), wv, bias=bv)[0].contiguous()                  # [len(ids)*C]
                    self._folded[key] = (kb, vb)
                kb, vb = self._folded[key]
                frows = f.view(h * w, c)
                src_rows.append(None)
                kall = ops.gemm(frows, wk, rowbias=kb, rowbias_rows=1).view(n, h * w, len(ids), H, hd)
                vall = ops.gemm(frows, wv, bias=vb).view(n, h * w, len(ids), H, hd)
            else:
                src = ops.add(f.view(n * h * w, c), self.level_embed[lvl].contiguous())
                src_rows.append(src)
                kin = ops.add(src, self._pe(h, w))
                kall = ops.gemm(kin, wk, bias=bk).view(n, h * w, len(ids), H, hd)
                vall = ops.gemm(src, wv, bias=bv).view(n, h * w, len(ids), H, hd)
            for j, i in enumerate(ids):
                kproj[i], vproj[i] = kall[:, :, j], vall[:, :, j]
        mf = _nhwc(mask_features.to(dev))
        mask_hw = (mf.shape[1], mf.shape[2])
        mask_rows = [mf[b].view(-1, mf.shape[-1]) for b in range(bs)]

        output = self.query_feat.unsqueeze(0).repeat(bs, 1, 1).view(bs * Q, C).contiguous()
        qpos = self.query_embed.unsqueeze(0).repeat(bs, 1, 1).view(bs * Q, C).contiguous()

        # ---- prompts: token groups that join the self-attention (carried groups keep their updated value across layers)
        bt = lambda t: t.to(dev).permute(1, 0, 2).to(BF16).contiguous()          # [T, bs, C] -> [bs, T, C]
        carried = []                                                              # [name, value [bs,T,C], pos [bs,T,C], masking]
        if grounding_flag:
            carried.append(["tokens_grounding", bt(extra["grounding_tokens"]), bt(extra["grounding_tokens"]),
                            extra.get("grounding_nonzero_mask")])
        if audio_flag:
            carried.append(["tokens_audio", bt(extra["audio_tokens"]), bt(extra["audio_tokens"]), extra.get("audio_nonzero_mask")])
        spatial_query_pos = spatial_query_neg = None
        src_spatial_queries = src_spatial_maskings = None
        if spatial_flag:
            spatial_query_pos, spatial_query_neg, src_spatial_queries, src_spatial_maskings = self._spatial_prompts(
                extra, mask_features.to(dev), src_rows, size_list, bs, task)
            if "refimg" in task:                                                  # seem.py:459-465
                return dict(visual_query_pos=spatial_query_pos, visual_query_neg=spatial_query_neg,
                            src_visual_queries=src_spatial_queries, src_visual_maskings=src_spatial_maskings)
        visual_query_pos = visual_query_neg = None
        if visual_flag:
            visual_query_pos, visual_query_neg = extra["visual_query_pos"], extra["visual_query_neg"]
        has_prompts = bool(carried) or spatial_flag or visual_flag

        # aux_outputs off: mask_features resized once per level -> the intermediate heads need no full-resolution map
        small = None
        if not self.aux_outputs:
            small = {}
            for hw in set(size_list):
                r = ops.resize_bilinear_nhwc(mf, hw[0], hw[1])
                small[hw] = [r[b].view(-1, r.shape[-1]) for b in range(bs)]
        head = lambda out_rows, j, last=False: self._heads(out_rows, mask_rows, mask_hw, size_list[j % self.num_feature_levels], bs,
                                                           None if (small is None or last) else small[size_list[j % self.num_feature_levels]])
        # (output + query_pos) W + b = output W + [query_pos W + b]: the constant term becomes a per-row bias of the GEMM
        def qfold(name, i, w, b):
            key = (name, i, bs)
            if key not in self._folded:
                self._folded[key] = ops.gemm(qpos, w, bias=b).contiguous()
            return self._folded[key]
        results = [head(output, 0)]
        for i in range(self.num_layers):
            lvl = i % self.num_feature_levels
            # masked cross attention (post-norm)
            a = self.cross[i]["att"]
            q = ops.gemm(output, a.wq, rowbias=qfold("cq", i, a.wq, a.bq), rowbias_rows=1).view(bs, Q, H, hd)
            att = ops.attention(q, kproj[i], vproj[i], scale=hd ** -0.5, mask=results[-1]["attn_mask"])
            ops.gemm(att.view(bs * Q, C), a.wo, bias=a.bo, residual=output, out=output)
            ops.layernorm(output, *self.cross[i]["n"], 1e-5, out=output)
            a = self.selfa[i]["att"]
            if not has_prompts:
                # self attention among the object queries (mask all-False for task 'seg')
                qk = ops.gemm(output, a.wqk, rowbias=qfold("sqk", i, a.wqk, a.bqk), rowbias_rows=1).view(bs, Q, 2, H, hd)
                v = ops.gemm(output, a.wv, bias=a.bv).view(bs, Q, H, hd)
                att = ops.attention(qk[:, :, 0], qk[:, :, 1], v, scale=hd ** -0.5)
                ops.gemm(att.view(bs * Q, C), a.wo, bias=a.bo, residual=output, out=output)
                ops.layernorm(output, *self.selfa[i]["n"], 1e-5, out=output)
                # FFN
                f1 = ops.gemm(output, self.ffn[i]["l1"][0], bias=self.ffn[i]["l1"][1], act=ops.ACT_RELU)
                ops.gemm(f1, self.ffn[i]["l2"][0], bias=self.ffn[i]["l2"][1], residual=output, out=output)
                ops.layernorm(output, *self.ffn[i]["n"], 1e-5, out=output)
            else:
                # the token groups of this layer: carried ones + the level's spatial / visual tokens (re-set every layer,
                # seem.py:512-527), sequence = [queries_object | groups...] per sample
                groups = [(g_[0], g_[1], g_[2], g_[3]) for g_ in carried]
                if spatial_flag:
                    tk = bt(src_spatial_queries[lvl])
                    groups.append(("tokens_spatial", tk, tk, src_spatial_maskings[lvl]))
                if visual_flag:
                    tk = bt(extra["src_visual_queries"][lvl])
                    groups.append(("tokens_visual", tk, tk, extra["src_visual_maskings"][lvl]))
                order = {"tokens_grounding": 0, "tokens_spatial": 1, "tokens_visual": 2, "tokens_audio": 3}   # SELF_ATTENTION dict order
                groups.sort(key=lambda g_: order[g_[0]])
                X = torch.cat([output.view(bs, Q, C)] + [g_[1] for g_ in groups], 1)
                P = torch.cat([qpos.view(bs, Q, C)] + [g_[2] for g_ in groups], 1)
                Ltot = X.shape[1]
                X = X.reshape(bs * Ltot, C).contiguous()
                sm = self._self_attn_mask(Q, [(g_[0], g_[1].shape[1], g_[3]) for g_ in groups], bs)
                qk = ops.gemm(ops.add(X, P.reshape(bs * Ltot, C).contiguous()), a.wqk, bias=a.bqk).view(bs, Ltot, 2, H, hd)
                v = ops.gemm(X, a.wv, bias=a.bv).view(bs, Ltot, H, hd)
                att = ops.attention(qk[:, :, 0], qk[:, :, 1], v, scale=hd ** -0.5, mask=sm)
                ops.gemm(att.view(bs * Ltot, C), a.wo, bias=a.bo, residual=X, out=X)
                ops.layernorm(X, *self.selfa[i]["n"], 1e-5, out=X)
                f1 = ops.gemm(X, self.ffn[i]["l1"][0], bias=self.ffn[i]["l1"][1], act=ops.ACT_RELU)
                ops.gemm(f1, self.ffn[i]["l2"][0], bias=self.ffn[i]["l2"][1], residual=X, out=X)
                ops.layernorm(X, *self.ffn[i]["n"], 1e-5, out=X)
                X3 = X.view(bs, Ltot, C)
                output = X3[:, :Q].reshape(bs * Q, C).contiguous()
                off = Q
                for g_ in groups:                                  # update_variables(output, 'self_attn')
                    T = g_[1].shape[1]
                    for cg in carried:
                        if cg[0] == g_[0]:
                            cg[1] = X3[:, off:off + T].contiguous()
                    off += T
            results.append(head(output, i + 1, last=(i == self.num_layers - 1)))
        # organize_output (attention_data_struct.py:250-264) for the object queries
        names = {"predictions_class": "pred_logits", "predictions_mask": "pred_masks", "predictions_maskemb": "pred_maskembs"}
        if grounding_flag or audio_flag:
            names["predictions_caption"] = "pred_captions"        # attention_data_struct.py:12-28 (queries_object slice)
        out = {v: results[-1][k] for k, v in names.items()}
        out["aux_outputs"] = [{v: r[k] for k, v in names.items()} for r in results[:-1]] if self.aux_outputs else []
        extras_out = {}
        if spatial_flag:
            extras_out.update(pred_pspatials=spatial_query_pos.transpose(0, 1), pred_nspatials=spatial_query_neg.transpose(0, 1))
        if visual_flag:
            extras_out.update(pred_pvisuals=visual_query_pos.transpose(0, 1), pred_nvisuals=visual_query_neg.transpose(0, 1))
        out.update(extras_out)
        for a_ in out["aux_outputs"]:
            a_.update(extras_out)
        out["attn_masks"] = [r["attn_mask"] for r in results]  # extra (not in the reference dict): for parity tests
        return out

    __call__ = forward


class XDecoderHead:
    """sem_seg_head: layers(features) = predictor(*pixel_decoder.forward_features(features))
    (body/xdecoder_head.py:100-118)."""

    def __init__(self, pixel_decoder, predictor):
        self.pixel_decoder, self.predictor = pixel_decoder, predictor
        self._graphed = None

    def enable_graph(self, on=True):
        """Replay the whole head (pixel decoder + 9 decoder layers + 10 prediction heads, ~400 launches) from one CUDA graph
        per feature-shape signature. The returned tensors are then static buffers, overwritten by the next call."""
        self._graphed = ops.GraphedCall(lambda **f: self.layers(f)) if on else None
        return self

    def load_state_dict(self, sd, prefix=""):
        self.pixel_decoder.load_state_dict(sd, prefix + "pixel_decoder.")
        self.predictor.load_state_dict(sd, prefix + "predictor.")
        return self

    def forward(self, features, mask=None, target_queries=None, target_vlp=None, task="seg", extra={}):
        if (self._graphed is not None and not extra and mask is None and target_queries is None and target_vlp is None
                and task == "seg" and all(torch.is_tensor(v) and v.is_cuda for v in features.values())):
            return self._graphed(**features)
        return self.layers(features, mask, target_queries, target_vlp, task, extra)

    def layers(self, features, mask=None, target_queries=None, target_vlp=None, task="seg", extra={}):
        mask_features, enc_feats, multi = self.pixel_decoder.forward_features(features)
        return self.predictor(multi, mask_features, mask, target_queries, target_vlp, task, extra)

    __call__ = forward
