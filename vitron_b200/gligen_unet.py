"""GLIGEN's grounded Stable-Diffusion UNet on the vitron_b200 kernels (SURVEY.md §8 f2: "the rest of the GLIGEN UNet").

Drop-in for modules/GLIGEN/demo/gligen/ldm/modules/diffusionmodules/openaimodel.py::UNetModel (:234-502) with
ResBlock (:113-230), Downsample / Upsample (:51-110), TimestepEmbedSequential (:34-48), SpatialTransformer
(ldm/modules/attention.py:352-386), PositionNet (diffusionmodules/positionnet.py:9-50) and `timestep_embedding` /
FourierEmbedder (diffusionmodules/util.py:160-180, 12-26): same constructor keywords, state-dict names and
`forward(input)` with the reference's input dict (`x`, `timesteps`, `context`, `boxes`, `masks`, `text_embeddings`,
optional `inpainting_extra_input`). The transformer blocks are `vitron_b200.gligen.BasicTransformerBlock` (row a12).

Design: NHWC bf16 end to end (the reference flips 'b c h w' <-> 'b (h w) c' around every SpatialTransformer);
3x3 convs, stride-2 downsample and the conv after the nearest upsample are the TMA implicit-GEMM wgmma kernel; the
time-embedding projections of ALL ResBlocks are one GEMM per forward and enter conv1 as a per-sample row bias in its
epilogue; GroupNorm(32)+SiLU is one fused kernel; skip 1x1 convs, proj_in / proj_out are GEMMs on the pixel rows with
the residual in the epilogue.
"""
import math

import torch

from . import ops
from .gligen import BasicTransformerBlock

BF16 = torch.bfloat16


def timestep_embedding(timesteps, dim, max_period=10000):
    """diffusionmodules/util.py:160-180 (repeat_only=False)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / half)
    args = timesteps[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


def fourier_embed(x, num_freqs=8, temperature=100):
    """FourierEmbedder.__call__ (util.py:12-26): [.., 4] -> [.., num_freqs*2*4], (sin, cos) per frequency band."""
    bands = temperature ** (torch.arange(num_freqs, device=x.device) / num_freqs)
    out = []
    for f in bands:
        out.append(torch.sin(f * x))
        out.append(torch.cos(f * x))
    return torch.cat(out, -1)


class UNetModel:
    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, use_checkpoint=False, num_heads=8,
                 use_scale_shift_norm=False, transformer_depth=1, positive_len=768, context_dim=None, fuser_type=None,
                 is_inpaint=False, is_style=False, device="cuda"):
        if fuser_type != "gatedSA":
            raise NotImplementedError("only the gatedSA fuser is on the Vitron path (attention.py:329-334)")
        if use_scale_shift_norm or dims != 2 or not conv_resample or is_style:
            raise NotImplementedError("scale-shift norm / 3-D / pooled resampling / style position net are not used by GLIGEN's SD config")
        self.image_size, self.in_channels, self.model_channels, self.out_channels = image_size, in_channels, model_channels, out_channels
        self.num_res_blocks, self.attention_resolutions = num_res_blocks, list(attention_resolutions)
        self.channel_mult, self.num_heads, self.transformer_depth = tuple(channel_mult), num_heads, transformer_depth
        self.positive_len, self.context_dim, self.fuser_type = positive_len, context_dim, fuser_type
        self.is_inpaint = is_inpaint
        self.device = torch.device(device)
        self.max_box = 30
        # ---- block plan, mirrors UNetModel.__init__ :283-372 (entries: ("conv"|"res"|"st"|"down"|"up", prefix, cin, cout))
        mc = model_channels
        total_in = in_channels + in_channels + 1 if is_inpaint else in_channels
        self.total_in = total_in
        plan_in = [[("conv", "input_blocks.0.0.", total_in, mc)]]
        chans = [mc]
        ch, ds, idx = mc, 1, 1
        for level, mult in enumerate(self.channel_mult):
            for _ in range(num_res_blocks):
                layers = [("res", f"input_blocks.{idx}.0.", ch, mult * mc)]
                ch = mult * mc
                if ds in self.attention_resolutions:
                    layers.append(("st", f"input_blocks.{idx}.1.", ch, ch))
                plan_in.append(layers)
                chans.append(ch)
                idx += 1
            if level != len(self.channel_mult) - 1:
                plan_in.append([("down", f"input_blocks.{idx}.0.", ch, ch)])
                chans.append(ch)
                ds *= 2
                idx += 1
        self.plan_in = plan_in
        self.plan_mid = [("res", "middle_block.0.", ch, ch), ("st", "middle_block.1.", ch, ch), ("res", "middle_block.2.", ch, ch)]
        plan_out, idx = [], 0
        for level, mult in list(enumerate(self.channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                ich = chans.pop()
                layers = [("res", f"output_blocks.{idx}.0.", ch + ich, mc * mult)]
                ch = mc * mult
                j = 1
                if ds in self.attention_resolutions:
                    layers.append(("st", f"output_blocks.{idx}.{j}.", ch, ch))
                    j += 1
                if level and i == num_res_blocks:
                    layers.append(("up", f"output_blocks.{idx}.{j}.", ch, ch))
                    ds //= 2
                plan_out.append(layers)
                idx += 1
        self.plan_out = plan_out
        self.final_ch = ch
        self.w = None

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd, strict=True):
        dev = self.device
        f32 = lambda n: sd[n].detach().to(device=dev, dtype=torch.float32)
        bf = lambda t: t.to(BF16).contiguous()
        gn = lambda p: (bf(f32(p + "weight")), bf(f32(p + "bias")))

        def conv3(p, cin_pad=None):
            w = f32(p + "weight")
            if cin_pad is not None and cin_pad != w.shape[1]:
                wp = torch.zeros((w.shape[0], cin_pad, *w.shape[2:]), dtype=w.dtype, device=dev)
                wp[:, :w.shape[1]] = w
                w = wp
            return ops.pack_conv_weight(w), bf(f32(p + "bias"))

        lin = lambda p: (bf(f32(p + "weight").flatten(1)), bf(f32(p + "bias")))
        w = {"time": (lin("time_embed.0."), lin("time_embed.2."))}
        emb_w, emb_b, self.emb_slices, off = [], [], {}, 0
        heads = self.num_heads
        for layers in self.plan_in + [self.plan_mid] + self.plan_out:
            for kind, p, cin, cout in layers:
                if kind == "conv":
                    self.cin_pad = (cin + 7) // 8 * 8
                    w[p] = conv3(p, self.cin_pad)
                elif kind == "res":
                    r = dict(n1=gn(p + "in_layers.0."), c1=conv3(p + "in_layers.2."), n2=gn(p + "out_layers.0."),
                             c2=conv3(p + "out_layers.3."))
                    if cin != cout:
                        r["skip"] = lin(p + "skip_connection.")
                    emb_w.append(f32(p + "emb_layers.1.weight"))
                    emb_b.append(f32(p + "emb_layers.1.bias"))
                    self.emb_slices[p] = (off, off + cout)
                    off += cout
                    w[p] = r
                elif kind == "st":
                    blocks = [BasicTransformerBlock(cout, self.context_dim, self.context_dim, heads, cout // heads, self.fuser_type,
                                                    device=dev).load_state_dict(sd, p + f"transformer_blocks.{d}.")
                              for d in range(self.transformer_depth)]
                    w[p] = dict(n=gn(p + "norm."), pin=lin(p + "proj_in."), pout=lin(p + "proj_out."), blocks=blocks)
                elif kind == "down":
                    w[p] = conv3(p + "op.")
                elif kind == "up":
                    w[p] = conv3(p + "conv.")
        w["emb_all"] = (bf(torch.cat(emb_w, 0)), bf(torch.cat(emb_b, 0)))
        w["out_gn"] = gn("out.0.")
        w["out_conv"] = conv3("out.2.")
        pn = "position_net."
        w["pos"] = dict(l0=lin(pn + "linears.0."), l1=lin(pn + "linears.2."), l2=lin(pn + "linears.4."),
                        null_pos=f32(pn + "null_positive_feature"), null_xyxy=f32(pn + "null_position_feature"))
        self.w = w
        return self

    # ------------------------------------------------------------------ pieces
    def forward_position_net(self, input):
        """UNetModel.forward_position_net :388-405 + PositionNet.forward :30-50 -> objs [B, N, context_dim] bf16."""
        if "boxes" in input:
            boxes, masks, text = input["boxes"], input["masks"], input["text_embeddings"]
            self.max_box = text.shape[1]
        else:
            b = input["x"].shape[0]
            boxes = torch.zeros((b, self.max_box, 4), device=self.device)
            masks = torch.zeros((b, self.max_box), device=self.device)
            text = torch.zeros((b, self.max_box, self.positive_len), device=self.device)
        p = self.w["pos"]
        boxes, masks, text = boxes.to(self.device).float(), masks.to(self.device).float().unsqueeze(-1), text.to(self.device).float()
        B, N, _ = boxes.shape
        xyxy = fourier_embed(boxes)
        text = text * masks + (1 - masks) * p["null_pos"].view(1, 1, -1)
        xyxy = xyxy * masks + (1 - masks) * p["null_xyxy"].view(1, 1, -1)
        h = torch.cat([text, xyxy], dim=-1).reshape(B * N, -1).to(BF16).contiguous()
        h = ops.gemm(h, p["l0"][0], bias=p["l0"][1], act=ops.ACT_SILU)
        h = ops.gemm(h, p["l1"][0], bias=p["l1"][1], act=ops.ACT_SILU)
        return ops.gemm(h, p["l2"][0], bias=p["l2"][1]).view(B, N, -1)

    def _res(self, p, x, emb_all):
        r = self.w[p]
        n, h, w, cin = x.shape
        lo, hi = self.emb_slices[p]
        a = ops.groupnorm_nhwc(x, *r["n1"], 32, 1e-5, act=ops.ACT_SILU)
        rb = emb_all[:, lo:hi].contiguous()                                     # [B, cout]: + emb_out[..., None, None]
        hcur = ops.conv_nhwc(a, r["c1"][0], 3, 3, bias=r["c1"][1], rowbias=rb, rowbias_rows=h * w)
        a = ops.groupnorm_nhwc(hcur, *r["n2"], 32, 1e-5, act=ops.ACT_SILU)
        if "skip" in r:
            skip = ops.gemm(x.view(n * h * w, cin), r["skip"][0], bias=r["skip"][1]).view(n, h, w, -1)
        else:
            skip = x
        return ops.conv_nhwc(a, r["c2"][0], 3, 3, bias=r["c2"][1], residual=skip)

    def _st(self, p, x, context, objs):
        s = self.w[p]
        n, h, w, c = x.shape
        xn = ops.groupnorm_nhwc(x, *s["n"], 32, 1e-6)
        t = ops.gemm(xn.view(n * h * w, c), s["pin"][0], bias=s["pin"][1]).view(n, h * w, -1)
        for blk in s["blocks"]:
            t = blk(t, context, objs)
        return ops.gemm(t.reshape(n * h * w, -1), s["pout"][0], bias=s["pout"][1], residual=x.view(n * h * w, c)).view(n, h, w, c)

    def _run(self, layers, x, emb_all, context, objs):
        for kind, p, cin, cout in layers:
            if kind == "conv":
                x = ops.conv_nhwc(x, self.w[p][0], 3, 3, bias=self.w[p][1])
            elif kind == "res":
                x = self._res(p, x, emb_all)
            elif kind == "st":
                x = self._st(p, x, context, objs)
            elif kind == "down":
                x = ops.conv_nhwc(x, self.w[p][0], 3, 3, stride=2, bias=self.w[p][1])
            elif kind == "up":
                x = ops.conv_nhwc(ops.upsample2x_nhwc(x), self.w[p][0], 3, 3, bias=self.w[p][1])
        return x

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, input):
        if self.w is None:
            raise RuntimeError("UNetModel: load_state_dict() first")
        dev = self.device
        objs = self.forward_position_net(input)
        t_emb = timestep_embedding(input["timesteps"].to(dev), self.model_channels).to(BF16).contiguous()
        (w0, b0), (w1, b1) = self.w["time"]
        # emb is only ever consumed through the ResBlocks' emb_layers = Sequential(SiLU, Linear): the SiLU is the epilogue
        # of time_embed.2, and every ResBlock's Linear is one row block of a single GEMM
        emb_act = ops.gemm(ops.gemm(t_emb, w0, bias=b0, act=ops.ACT_SILU), w1, bias=b1, act=ops.ACT_SILU)
        emb_all = ops.gemm(emb_act, self.w["emb_all"][0], bias=self.w["emb_all"][1])
        h = input["x"].to(dev)
        if self.is_inpaint:
            extra = input["inpainting_extra_input"].to(dev)
            if extra.shape[2] != h.shape[2]:
                raise NotImplementedError("inpainting_extra_input at a different resolution than x (openaimodel.py:468-471)")
            h = torch.cat([h, extra], dim=1)
        B, cin, H, W = h.shape
        x = torch.zeros((B, H, W, self.cin_pad), dtype=BF16, device=dev)
        x[..., :cin] = h.permute(0, 2, 3, 1)
        context = input["context"].to(dev).to(BF16).contiguous()
        hs = []
        for layers in self.plan_in:
            x = self._run(layers, x, emb_all, context, objs)
            hs.append(x)
        x = self._run(self.plan_mid, x, emb_all, context, objs)
        for layers in self.plan_out:
            skip = hs.pop()
            if skip.shape[1] != x.shape[1]:
                raise NotImplementedError("skip connection at a different resolution (odd latent sizes, openaimodel.py:483-489)")
            x = self._run(layers, torch.cat([x, skip], dim=-1), emb_all, context, objs)
        a = ops.groupnorm_nhwc(x, *self.w["out_gn"], 32, 1e-5, act=ops.ACT_SILU)
        out = ops.conv_nhwc(a, self.w["out_conv"][0], 3, 3, bias=self.w["out_conv"][1])
        return out.permute(0, 3, 1, 2).float().contiguous()

    __call__ = forward


SD14_GLIGEN_UNET = dict(image_size=64, in_channels=4, model_channels=320, out_channels=4, num_res_blocks=2,
                        attention_resolutions=[4, 2, 1], channel_mult=[1, 2, 4, 4], num_heads=8, transformer_depth=1,
                        context_dim=768, fuser_type="gatedSA", use_checkpoint=False)
"""GLIGEN's generation_text config (gligen/configs: SD-1.4 UNet with gatedSA fusers)."""
