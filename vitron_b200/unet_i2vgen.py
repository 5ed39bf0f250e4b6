"""UNetSD_I2VGen (i2vgen-xl UNet3D) on the vitron_b200 kernels + the DDIM / CFG sampler.

Drop-in for modules/i2vgen-xl/tools/modules/unet/unet_i2vgen.py:20-418 (same constructor keywords,
same `forward(x, t, y, image, local_image, masked, fps, ...)`, same state-dict names) and for
`DiffusionDDIM.ddim_sample_loop` (tools/modules/diffusions/diffusion_ddim.py:143-250). Blocks follow
tools/modules/unet/util.py: ResBlock :610-730, TemporalConvBlock_v2 :1347-1392, SpatialTransformer
:311-373, BasicTransformerBlock :510-540, GEGLU/FeedForward :543-577, TemporalTransformer :992-1089,
Upsample/Downsample :579-607,732-756, TransformerV2 :1129-1148, sinusoidal_embedding :177-189.

Design: activations stay NHWC bf16 `[(b f), h, w, c]` end to end — the reference's ~40
`rearrange(...).contiguous()` layout flips per forward disappear because (i) Conv2d 3x3 / Conv3d
(3,1,1) are im2col-free implicit GEMMs reading the NHWC tensor through 4-D TMA maps, (ii) every
Linear is a row-wise wgmma GEMM with bias / GEGLU / residual fused, (iii) temporal attention reads
its length-f sequences with strides. All 22 ResBlock time-embedding projections are one GEMM.
The tiny x-independent local-image adapter (4..32 channels, <0.01 % of FLOPs) runs once per
conditioning through torch ops and is cached.
"""
import math

import torch
import torch.nn.functional as F

from . import ops

BF16 = torch.bfloat16


def sinusoidal_embedding(timesteps, dim):
    half = dim // 2
    timesteps = timesteps.float()
    sinusoid = torch.outer(timesteps, torch.pow(10000, -torch.arange(half, device=timesteps.device).to(timesteps).div(half)))
    x = torch.cat([torch.cos(sinusoid), torch.sin(sinusoid)], dim=1)
    if dim % 2 != 0:
        x = torch.cat([x, torch.zeros_like(x[:, :1])], dim=1)
    return x


class UNetSD_I2VGen:
    def __init__(self, config=None, in_dim=4, dim=320, y_dim=1024, context_dim=1024, hist_dim=156, concat_dim=4,
                 dim_condition=4, out_dim=4, num_tokens=4, dim_mult=(1, 2, 4, 4), num_heads=8, head_dim=64,
                 num_res_blocks=2, attn_scales=(1.0, 0.5, 0.25), use_scale_shift_norm=True, dropout=0.1,
                 temporal_attn_times=1, temporal_attention=True, use_checkpoint=False, use_image_dataset=False,
                 use_sim_mask=False, training=False, inpainting=True, p_all_zero=0.1, p_all_keep=0.1, zero_y=None,
                 adapter_transformer_layers=1, device="cuda", **kwargs):
        if not temporal_attention or use_image_dataset:
            raise NotImplementedError("only the shipped inference configuration (temporal transformers on) is supported")
        self.device = torch.device(device)
        self.in_dim, self.dim, self.y_dim, self.context_dim = in_dim, dim, y_dim, context_dim
        self.out_dim, self.num_tokens, self.head_dim = out_dim, num_tokens, head_dim
        self.embed_dim = dim * 4
        self.num_heads = num_heads if num_heads else dim // 32
        self.zero_y = zero_y
        self.concat_dim = in_dim
        self.adapter_layers = adapter_transformer_layers
        dim_mult, attn_scales = list(dim_mult), list(attn_scales)
        # ---- block plan, mirroring the reference constructor (unet_i2vgen.py:133-233)
        enc_dims = [dim * u for u in [1] + dim_mult]
        dec_dims = [dim * u for u in [dim_mult[-1]] + dim_mult[::-1]]
        shortcut, scale = [dim], 1.0
        self.input_plan = [[("conv_in", "input_blocks.0.0", in_dim + self.concat_dim, dim),
                            ("tt", "input_blocks.0.1", dim, self.num_heads)]]
        idx = 1
        for i, (cin, cout) in enumerate(zip(enc_dims[:-1], enc_dims[1:])):
            for j in range(num_res_blocks):
                blk = [("res", f"input_blocks.{idx}.0", cin, cout)]
                if scale in attn_scales:
                    blk.append(("st", f"input_blocks.{idx}.1", cout, cout // head_dim))
                    blk.append(("tt", f"input_blocks.{idx}.2", cout, cout // head_dim))
                cin = cout
                self.input_plan.append(blk)
                shortcut.append(cout)
                idx += 1
                if i != len(dim_mult) - 1 and j == num_res_blocks - 1:
                    self.input_plan.append([("down", f"input_blocks.{idx}", cout, cout)])
                    shortcut.append(cout)
                    scale /= 2.0
                    idx += 1
        c = enc_dims[-1]
        self.middle_plan = [("res", "middle_block.0", c, c), ("st", "middle_block.1", c, c // head_dim),
                            ("tt", "middle_block.2", c, c // head_dim), ("res", "middle_block.3", c, c)]
        self.output_plan = []
        idx = 0
        for i, (cin, cout) in enumerate(zip(dec_dims[:-1], dec_dims[1:])):
            for j in range(num_res_blocks + 1):
                blk = [("res", f"output_blocks.{idx}.0", cin + shortcut.pop(), cout)]
                k = 1
                if scale in attn_scales:
                    blk.append(("st", f"output_blocks.{idx}.1", cout, cout // head_dim))
                    blk.append(("tt", f"output_blocks.{idx}.2", cout, cout // head_dim))
                    k = 3
                cin = cout
                if i != len(dim_mult) - 1 and j == num_res_blocks:
                    blk.append(("up", f"output_blocks.{idx}.{k}", cout, cout))
                    scale *= 2.0
                self.output_plan.append(blk)
                idx += 1
        self.final_dim = dec_dims[-1]
        self.w = {}
        self._adapter_cache = None

    # ------------------------------------------------------------------ weights
    def _all_blocks(self):
        for blk in self.input_plan:
            yield from blk
        yield from self.middle_plan
        for blk in self.output_plan:
            yield from blk

    def load_state_dict(self, sd, strict=True):
        dev = self.device
        g = lambda n: sd[n].detach().to(device=dev, dtype=BF16).contiguous()
        g32 = lambda n: sd[n].detach().to(device=dev, dtype=torch.float32).contiguous()
        w = {}

        def lin(p):
            return g(p + ".weight"), (g(p + ".bias") if (p + ".bias") in sd else None)

        def transformer_block(p, ctx_self):
            t = {}
            for a in ("attn1", "attn2"):
                cross = (a == "attn2") and not ctx_self
                if cross:
                    t[a] = dict(wq=g(f"{p}.{a}.to_q.weight"),
                                wkv=torch.cat([g(f"{p}.{a}.to_k.weight"), g(f"{p}.{a}.to_v.weight")], 0).contiguous())
                else:
                    t[a] = dict(wqkv=torch.cat([g(f"{p}.{a}.to_q.weight"), g(f"{p}.{a}.to_k.weight"),
                                                g(f"{p}.{a}.to_v.weight")], 0).contiguous())
                t[a]["wo"], t[a]["bo"] = lin(f"{p}.{a}.to_out.0")
            for n in ("norm1", "norm2", "norm3"):
                t[n] = lin(f"{p}.{n}")
            pw, pb = g(f"{p}.ff.net.0.proj.weight"), g(f"{p}.ff.net.0.proj.bias")
            inner = pw.shape[0] // 2
            t["ff1"] = (ops.pack_glu_weight(pw[:inner], pw[inner:]), ops.pack_glu_weight(pb[:inner], pb[inner:]))
            t["ff2"] = lin(f"{p}.ff.net.2")
            return t

        emb_w, emb_b, off = [], [], 0
        for kind, p, cin, cout in self._all_blocks():
            if kind == "conv_in":
                w[p] = dict(w=ops.pack_conv_weight(g(p + ".weight")), b=g(p + ".bias"))
            elif kind == "res":
                r = dict(gn1=lin(p + ".in_layers.0"), conv1=ops.pack_conv_weight(g(p + ".in_layers.2.weight")),
                         b1=g(p + ".in_layers.2.bias"), gn2=lin(p + ".out_layers.0"),
                         conv2=ops.pack_conv_weight(g(p + ".out_layers.3.weight")), b2=g(p + ".out_layers.3.bias"))
                ew, eb = lin(p + ".emb_layers.1")
                emb_w.append(ew)
                emb_b.append(eb)
                r["emb"] = (off, off + cout)
                off += cout
                if cin != cout:
                    r["skip"] = (g(p + ".skip_connection.weight").reshape(cout, cin).contiguous(), g(p + ".skip_connection.bias"))
                tc = []
                for ci, li in ((1, 2), (2, 3), (3, 3), (4, 3)):
                    tc.append(dict(gn=lin(f"{p}.temopral_conv.conv{ci}.0"),
                                   w=ops.pack_conv_weight(g(f"{p}.temopral_conv.conv{ci}.{li}.weight")),
                                   b=g(f"{p}.temopral_conv.conv{ci}.{li}.bias")))
                r["tconv"] = tc
                w[p] = r
            elif kind == "st":
                w[p] = dict(gn=lin(p + ".norm"), pin=lin(p + ".proj_in"), pout=lin(p + ".proj_out"),
                            blk=transformer_block(p + ".transformer_blocks.0", ctx_self=False))
            elif kind == "tt":
                pin_w = g(p + ".proj_in.weight")
                pout_w = g(p + ".proj_out.weight")
                w[p] = dict(gn=lin(p + ".norm"), pin=(pin_w.reshape(pin_w.shape[0], -1).contiguous(), g(p + ".proj_in.bias")),
                            pout=(pout_w.reshape(pout_w.shape[0], -1).contiguous(), g(p + ".proj_out.bias")),
                            blk=transformer_block(p + ".transformer_blocks.0", ctx_self=True))
            elif kind == "down":
                w[p] = dict(w=ops.pack_conv_weight(g(p + ".op.weight")), b=g(p + ".op.bias"))
            elif kind == "up":
                w[p] = dict(w=ops.pack_conv_weight(g(p + ".conv.weight")), b=g(p + ".conv.bias"))
        w["emb_all"] = (torch.cat(emb_w, 0).contiguous(), torch.cat(emb_b, 0).contiguous())
        for name in ("time_embed", "fps_embedding", "context_embedding"):
            w[name] = (lin(name + ".0"), lin(name + ".2"))
        w["out_gn"] = lin("out.0")
        w["out_conv"] = (ops.pack_conv_weight(g("out.2.weight")), g("out.2.bias"))
        # tiny local-image adapter: fp32 torch weights (see module docstring)
        w["adapter"] = {k: g32(k) for k in sd if k.startswith(("local_image_concat.", "local_temporal_encoder.",
                                                               "local_image_embedding."))}
        self.w = w
        self._adapter_cache = None
        return self

    # ------------------------------------------------------------------ blocks
    def _res(self, p, x, emb_all, b, f):
        """x [(b f), h, w, cin] -> [(b f), h, w, cout] (ResBlock + TemporalConvBlock_v2)."""
        r = self.w[p]
        n, h, wd, cin = x.shape
        a = ops.groupnorm_nhwc(x, *r["gn1"], 32, 1e-5, act=ops.ACT_SILU)
        lo, hi = r["emb"]
        rb = emb_all[:, lo:hi].contiguous()
        hcur = ops.conv_nhwc(a, r["conv1"], 3, 3, bias=r["b1"], rowbias=rb, rowbias_rows=f * h * wd)
        a = ops.groupnorm_nhwc(hcur, *r["gn2"], 32, 1e-5, act=ops.ACT_SILU)
        if "skip" in r:
            skip = ops.gemm(x.view(-1, cin), r["skip"][0], bias=r["skip"][1]).view(n, h, wd, -1)
        else:
            skip = x
        hcur = ops.conv_nhwc(a, r["conv2"], 3, 3, bias=r["b2"], residual=skip)
        cout = hcur.shape[-1]
        ident = hcur
        t = hcur
        for i, tc in enumerate(r["tconv"]):
            a = ops.groupnorm_nhwc(t, *tc["gn"], 32, 1e-5, act=ops.ACT_SILU, n=b)
            res = ident.view(b, f, h * wd, cout) if i == 3 else None
            t = ops.conv_nhwc(a.view(b, f, h * wd, cout), tc["w"], 3, 1, pad_h=1, pad_w=0, bias=tc["b"], residual=res)
        return t.view(n, h, wd, cout)

    def _self_attn(self, a, z, t, heads, shape5=None):
        """z += to_out(attention(LN-ed rows a)). shape5 = (b, f, hw) selects temporal sequences."""
        rows, inner = a.shape
        hd = inner // heads
        qkv = ops.gemm(a, t["wqkv"])
        if shape5 is None:
            raise AssertionError
        b, f, hw = shape5
        q5 = qkv.view(b, f, hw, 3, heads, hd).permute(3, 0, 2, 1, 4, 5)  # [3, b, hw, f, H, hd]
        att = torch.empty((b, f, hw, heads, hd), dtype=BF16, device=a.device)
        ops.attention_short(q5[0], q5[1], q5[2], scale=hd ** -0.5, out=att.permute(0, 2, 1, 3, 4))
        return ops.gemm(att.view(rows, inner), t["wo"], bias=t["bo"], residual=z, out=z)

    def _ff(self, z, t):
        a = ops.layernorm(z, *t["norm3"], 1e-5)
        gl = ops.gemm(a, t["ff1"][0], bias=t["ff1"][1], glu=ops.GLU_GEGLU)
        return ops.gemm(gl, t["ff2"][0], bias=t["ff2"][1], residual=z, out=z)

    def _st(self, p, x, context, b, f, heads):
        """SpatialTransformer: x [(b f), h, w, c]; context [b, L, ctx]."""
        s = self.w[p]
        n, h, wd, c = x.shape
        hw = h * wd
        xn = ops.groupnorm_nhwc(x, *s["gn"], 32, 1e-6)
        z = ops.gemm(xn.view(n * hw, c), s["pin"][0], bias=s["pin"][1])
        inner = z.shape[1]
        hd = inner // heads
        t = s["blk"]
        a = ops.layernorm(z, *t["norm1"], 1e-5)
        qkv = ops.gemm(a, t["attn1"]["wqkv"]).view(n, hw, 3, heads, hd)
        att = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], scale=hd ** -0.5)
        ops.gemm(att.view(n * hw, inner), t["attn1"]["wo"], bias=t["attn1"]["bo"], residual=z, out=z)
        a = ops.layernorm(z, *t["norm2"], 1e-5)
        q = ops.gemm(a, t["attn2"]["wq"]).view(b, f, hw, heads, hd)
        L = context.shape[1]
        kv = ops.gemm(context.reshape(b * L, -1), t["attn2"]["wkv"]).view(b, L, 2, heads, hd)
        att = torch.empty((b, f, hw, heads, hd), dtype=BF16, device=x.device)
        for bi in range(b):  # context is shared by the f frames of a sample: K/V projected once, stride-0 over f
            ops.attention(q[bi], kv[bi:bi + 1, :, 0].expand(f, L, heads, hd), kv[bi:bi + 1, :, 1].expand(f, L, heads, hd),
                          scale=hd ** -0.5, out=att[bi])
        ops.gemm(att.view(n * hw, inner), t["attn2"]["wo"], bias=t["attn2"]["bo"], residual=z, out=z)
        self._ff(z, t)
        out = ops.gemm(z, s["pout"][0], bias=s["pout"][1], residual=x.view(n * hw, c))
        return out.view(n, h, wd, c)

    def _tt(self, p, x, b, f, heads):
        """TemporalTransformer (only_self_att): GroupNorm over (f,h,w), two self-attentions over f, GEGLU FF."""
        s = self.w[p]
        n, h, wd, c = x.shape
        hw = h * wd
        xn = ops.groupnorm_nhwc(x, *s["gn"], 32, 1e-6, n=b)
        z = ops.gemm(xn.view(n * hw, c), s["pin"][0], bias=s["pin"][1])
        t = s["blk"]
        a = ops.layernorm(z, *t["norm1"], 1e-5)
        self._self_attn(a, z, t["attn1"], heads, (b, f, hw))
        a = ops.layernorm(z, *t["norm2"], 1e-5)
        self._self_attn(a, z, t["attn2"], heads, (b, f, hw))
        self._ff(z, t)
        out = ops.gemm(z, s["pout"][0], bias=s["pout"][1], residual=x.view(n * hw, c))
        return out.view(n, h, wd, c)

    def _run(self, blk, x, emb_all, context, b, f):
        for kind, p, cin, cout in blk:
            if kind == "conv_in":
                x = ops.conv_nhwc(x, self.w[p]["w"], 3, 3, bias=self.w[p]["b"])
            elif kind == "res":
                x = self._res(p, x, emb_all, b, f)
            elif kind == "st":
                x = self._st(p, x, context, b, f, cout)
            elif kind == "tt":
                x = self._tt(p, x, b, f, cout)
            elif kind == "down":
                x = ops.conv_nhwc(x, self.w[p]["w"], 3, 3, stride=2, bias=self.w[p]["b"])
            elif kind == "up":
                x = ops.conv_nhwc(ops.upsample2x_nhwc(x), self.w[p]["w"], 3, 3, bias=self.w[p]["b"])
        return x

    # ------------------------------------------------------------------ local-image adapter (cached)
    def _adapter(self, local_image, batch, f, h, w):
        key = (local_image.data_ptr(), local_image._version, tuple(local_image.shape), f)
        if self._adapter_cache is not None and self._adapter_cache[0] == key:
            return self._adapter_cache[1]
        A = self.w["adapter"]
        li = local_image.float()
        if f > 1:
            mask_pos = torch.cat([torch.ones_like(li[:, :, :1]) * ((tpos + 1) / (f - 1)) for tpos in range(f - 1)], dim=2)
            ximg = torch.cat([li[:, :, :1], mask_pos], dim=2)
        else:
            ximg = li
        ximg = ximg.permute(0, 2, 1, 3, 4).reshape(batch * f, -1, h, w)
        ximg = F.conv2d(ximg, A["local_image_concat.0.weight"], A["local_image_concat.0.bias"], padding=1)
        ximg = F.conv2d(F.silu(ximg), A["local_image_concat.2.weight"], A["local_image_concat.2.bias"], padding=1)
        ximg = F.conv2d(F.silu(ximg), A["local_image_concat.4.weight"], A["local_image_concat.4.bias"], padding=1)
        cd = ximg.shape[1]
        s = ximg.view(batch, f, cd, h, w).permute(0, 3, 4, 1, 2).reshape(batch * h * w, f, cd)
        for li_ in range(self.adapter_layers):  # TransformerV2 (util.py:1129-1148): heads=2, dim_head=cd
            p = f"local_temporal_encoder.layers.{li_}."
            y = F.layer_norm(s, (cd,), A[p + "0.norm.weight"], A[p + "0.norm.bias"])
            qkv = F.linear(y, A[p + "0.fn.to_qkv.weight"]).view(s.shape[0], f, 3, 2, cd).permute(2, 0, 3, 1, 4)
            att = torch.softmax(qkv[0] @ qkv[1].transpose(-1, -2) * cd ** -0.5, -1) @ qkv[2]
            att = att.permute(0, 2, 1, 3).reshape(s.shape[0], f, 2 * cd)
            s = F.linear(att, A[p + "0.fn.to_out.0.weight"], A[p + "0.fn.to_out.0.bias"]) + s
            y = F.linear(F.gelu(F.linear(s, A[p + "1.net.0.0.weight"], A[p + "1.net.0.0.bias"])),
                         A[p + "1.net.2.weight"], A[p + "1.net.2.bias"])
            s = y + s
        concat = s.view(batch, h, w, f, cd).permute(0, 3, 1, 2, 4) * 2.0  # "concat += _ximg" twice (:294-295)
        lc = local_image[:, :, 0].float() if local_image.ndim == 5 else local_image.float()
        lc = F.silu(F.conv2d(lc, A["local_image_embedding.0.weight"], A["local_image_embedding.0.bias"], padding=1))
        lc = F.adaptive_avg_pool2d(lc, (32, 32))
        lc = F.silu(F.conv2d(lc, A["local_image_embedding.3.weight"], A["local_image_embedding.3.bias"], stride=2, padding=1))
        lc = F.conv2d(lc, A["local_image_embedding.5.weight"], A["local_image_embedding.5.bias"], stride=2, padding=1)
        local_context = lc.flatten(2).transpose(1, 2)  # [b, 64, 1024]
        out = (concat.reshape(batch * f, h, w, cd).contiguous(), local_context)
        self._adapter_cache = (key, out)
        return out

    @torch.no_grad()
    def refresh_adapter(self, local_image, batch, f, h, w):
        """Recompute the cached local-image adapter output for a local_image whose storage was updated in place and write
        it INTO the existing cache buffers: a captured CUDA graph that reads them (GraphedCFGDenoiser) stays valid."""
        old = self._adapter_cache
        self._adapter_cache = None
        if local_image.ndim == 5 and local_image.size(2) > 1:
            local_image = local_image[:, :, :1]
        elif local_image.ndim != 5:
            local_image = local_image.unsqueeze(2)
        new = self._adapter(local_image, batch, f, h, w)
        if old is not None and all(o.shape == n.shape for o, n in zip(old[1], new)):
            for o, n in zip(old[1], new):
                o.copy_(n)
            self._adapter_cache = (self._adapter_cache[0], old[1])

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x, t, y=None, image=None, local_image=None, masked=None, fps=None, video_mask=None,
                focus_present_mask=None, prob_focus_present=0., mask_last_frame_num=0, **kwargs):
        batch, c, f, h, w = x.shape
        dev = self.device
        if local_image.ndim == 5 and local_image.size(2) > 1:
            local_image = local_image[:, :, :1]
        elif local_image.ndim != 5:
            local_image = local_image.unsqueeze(2)
        concat, local_context = self._adapter(local_image, batch, f, h, w)

        def mlp(name, v):
            (w0, b0), (w1, b1) = self.w[name]
            return ops.gemm(ops.gemm(v.to(BF16).contiguous(), w0, bias=b0, act=ops.ACT_SILU), w1, bias=b1)

        emb = mlp("time_embed", sinusoidal_embedding(t, self.dim)).float() + \
            mlp("fps_embedding", sinusoidal_embedding(fps, self.dim)).float()
        emb_all = ops.gemm(F.silu(emb).to(BF16).contiguous(), self.w["emb_all"][0], bias=self.w["emb_all"][1])

        ctx = [y.to(device=dev, dtype=torch.float32)] if y is not None else [self.zero_y.repeat(batch, 1, 1)[:, :1].float()]
        ctx.append(local_context)
        if image is not None:
            ic = mlp("context_embedding", image.reshape(-1, image.shape[-1]))
            ctx.append(ic.float().view(-1, self.num_tokens, self.context_dim))
        context = torch.cat(ctx, dim=1).to(BF16).contiguous()  # [b, L, ctx]; shared by the f frames

        xin = torch.cat([x.float().permute(0, 2, 3, 4, 1).reshape(batch * f, h, w, c), concat], dim=-1).to(BF16).contiguous()
        xs = []
        cur = xin
        for blk in self.input_plan:
            cur = self._run(blk, cur, emb_all, context, batch, f)
            xs.append(cur)
        cur = self._run(self.middle_plan, cur, emb_all, context, batch, f)
        for blk in self.output_plan:
            cur = torch.cat([cur, xs.pop()], dim=-1)
            cur = self._run(blk, cur, emb_all, context, batch, f)
        a = ops.groupnorm_nhwc(cur, *self.w["out_gn"], 32, 1e-5, act=ops.ACT_SILU)
        out = ops.conv_nhwc(a, self.w["out_conv"][0], 3, 3, bias=self.w["out_conv"][1])
        return out.view(batch, f, h, w, self.out_dim).permute(0, 4, 1, 2, 3).float()

    __call__ = forward


class GraphedCFGDenoiser:
    """One classifier-free-guidance evaluation  u + s (y - u), captured in a CUDA graph (≈1500 kernel launches per DDIM step
    would otherwise be bound by the host launch rate). The conditioning (y / image / local_image / fps) is fixed per video;
    xt and t are static buffers.
    The reference evaluates the two branches as two UNet calls (diffusion_ddim.py:153-154). Nothing in the network mixes
    samples of a batch (GroupNorm statistics, attention sequences and the adapter are per sample), so the same two results
    come out of ONE batch-2 forward [cond | uncond] — which is what runs here when both conditionings carry the same tensors:
    the 1280-channel levels (20-80 tiles per GEMM / conv) and every latency-bound launch (GroupNorm, small GEMMs) do twice the
    work per launch. batched=False keeps the two-call form."""

    def __init__(self, unet, cond, uncond, guide_scale, xt_like, t_like, batched=True):
        self.unet, self.cond, self.uncond, self.scale = unet, cond, uncond, float(guide_scale)
        self.xt = xt_like.detach().clone().float().contiguous()
        self.t = t_like.detach().clone()
        self.graph = None
        self.out = None
        keys = set(cond) | set(uncond)
        self.batched = bool(batched) and all(
            (torch.is_tensor(cond.get(k)) and torch.is_tensor(uncond.get(k)) and cond[k].shape == uncond[k].shape
             and cond[k].dtype == uncond[k].dtype) or (cond.get(k) is None and uncond.get(k) is None) for k in keys)
        if self.batched:   # static [cond | uncond] tensors the captured graph reads
            self.both = {k: (torch.cat([cond[k], uncond[k]], 0).contiguous() if torch.is_tensor(cond.get(k)) else None) for k in keys}
            self.xt2 = torch.cat([self.xt, self.xt], 0)
            self.t2 = torch.cat([self.t, self.t], 0)

    @torch.no_grad()
    def rebind(self, cond, uncond):
        """New conditioning for the SAME captured graph (next video of a serving loop): the values are copied into the
        static tensors the graph reads and the UNet's cached adapter output is refreshed in place. Shapes must match."""
        seen = set()
        for dst, src in ((self.cond, cond), (self.uncond, uncond)):
            for k, v in dst.items():
                if torch.is_tensor(v) and id(v) not in seen:
                    seen.add(id(v))
                    v.copy_(src[k].to(v.device))
                elif v is None and src.get(k) is not None:
                    raise ValueError(f"conditioning '{k}' was None when the graph was captured")
        b, _, f, h, w = self.xt.shape
        if self.batched:
            for k, v in self.both.items():
                if v is not None:
                    v[:b].copy_(self.cond[k])
                    v[b:].copy_(self.uncond[k])
            self.unet.refresh_adapter(self.both["local_image"], 2 * b, f, h, w)
        else:
            self.unet.refresh_adapter(self.cond["local_image"], b, f, h, w)

    def _eval(self):
        if self.batched:
            b = self.xt.shape[0]
            self.xt2[:b].copy_(self.xt)
            self.xt2[b:].copy_(self.xt)
            self.t2[:b].copy_(self.t)
            self.t2[b:].copy_(self.t)
            yu = self.unet(self.xt2, self.t2, **self.both).float()
            return ops.cfg_combine(yu[:b].contiguous(), yu[b:].contiguous(), self.scale)
        y = self.unet(self.xt, self.t, **self.cond).float().contiguous()
        u = self.unet(self.xt, self.t, **self.uncond).float().contiguous()
        return ops.cfg_combine(y, u, self.scale)

    def __call__(self, xt, t):
        self.xt.copy_(xt)
        self.t.copy_(t)
        if self.graph is None:
            s = torch.cuda.Stream(device=self.xt.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):  # warm-up: workspaces, adapter cache, lazy attributes
                    self._eval()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            l0 = ops.launch_count()
            with torch.cuda.graph(g), ops.pdl(True):
                self.out = self._eval()
            self.launches = ops.launch_count() - l0
            self.graph = g
        self.graph.replay()
        ops.count_launches(self.launches)
        return self.out


class GraphedBranch:
    """ONE UNet forward with fixed conditioning, captured in a CUDA graph (xt / t are static buffers). Building block of the
    CFG-branch split: each GPU of a pair owns one of the two classifier-free-guidance branches."""

    def __init__(self, unet, cond, xt_like, t_like):
        self.unet, self.cond = unet, cond
        self.xt = xt_like.detach().clone().float().contiguous()
        self.t = t_like.detach().clone()
        self.graph, self.out, self.launches = None, None, 0

    def __call__(self, xt, t):
        self.xt.copy_(xt)
        self.t.copy_(t)
        if self.graph is None:
            s = torch.cuda.Stream(device=self.xt.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    self.unet(self.xt, self.t, **self.cond)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            l0 = ops.launch_count()
            with torch.cuda.graph(g), ops.pdl(True):
                self.out = self.unet(self.xt, self.t, **self.cond).float().contiguous()
            self.launches = ops.launch_count() - l0
            self.graph = g
        self.graph.replay()
        ops.count_launches(self.launches)
        return self.out


class CFGSplitDenoiser:
    """Classifier-free guidance with the two UNet evaluations of a DDIM step on TWO ranks (SURVEY.md §8e: the cond / uncond
    branches of diffusion_ddim.py:153-158 are independent given x_t). Rank `role` 0 of the pair evaluates the conditional
    branch, role 1 the unconditional one; ONE collective per step — an all_gather of the two [b, 4, f, h, w] fp32 branch outputs
    inside the pair's process group (655 KB at the 16 x 40 x 64 latent) — after which both ranks hold (y, u), compute the same
    u + s (y - u) and therefore the same x_{t-1}: no broadcast of the latent is needed, the pair stays in lock-step.

    `branch` is any callable (xt, t) -> branch output (GraphedBranch on the GPU); `combine(y, u, scale)` defaults to the
    cfg_combine kernel; `group` is the 2-rank torch.distributed group (None = the default group of a 2-rank job)."""

    def __init__(self, branch, role, guide_scale, group=None, combine=None):
        self.branch, self.role, self.scale, self.group = branch, int(role), float(guide_scale), group
        self.combine = combine or ops.cfg_combine
        self._buf = None

    def __call__(self, xt, t):
        import torch.distributed as dist
        mine = self.branch(xt, t).float().contiguous()
        b = mine.shape[0]
        if self._buf is None or self._buf.shape[0] != 2 * b or self._buf.shape[1:] != mine.shape[1:]:
            self._buf = torch.empty((2 * b, *mine.shape[1:]), dtype=mine.dtype, device=mine.device)
        dist.all_gather_into_tensor(self._buf, mine, group=self.group)   # rows [0, b) = role 0 (cond), [b, 2b) = role 1
        return self.combine(self._buf[:b], self._buf[b:], self.scale)


# ====================================================================================== DDIM sampler
def _cosine_betas(num_timesteps=1000, cosine_s=0.008, zero_terminal_snr=True):
    """schedules.py:50-57 (+ rescale_zero_terminal_snr :121-143), float64."""
    fn = lambda u: math.cos((u + cosine_s) / (1 + cosine_s) * math.pi / 2) ** 2
    betas = torch.tensor([min(1.0 - fn((s + 1) / num_timesteps) / fn(s / num_timesteps), 0.999)
                          for s in range(num_timesteps)], dtype=torch.float64)
    if zero_terminal_snr and betas.max() != 1.0:
        abs_ = (1 - betas).cumprod(0).sqrt()
        a0, aT = abs_[0].clone(), abs_[-1].clone()
        abs_ = (abs_ - aT) * a0 / (a0 - aT)
        ab = abs_ ** 2
        alphas = torch.cat([ab[0:1], ab[1:] / ab[:-1]])
        betas = 1 - alphas
    return betas


class DiffusionDDIM:
    """`ddim_sample_loop` with classifier-free guidance, mean_type 'v' | 'eps', var_type 'fixed_small'
    (tools/modules/config.py:55-68). Per step: 2 UNet forwards, u + s (y - u) (cfg_combine kernel),
    v -> x0 -> eps -> x_{t-1} in fp32."""

    def __init__(self, schedule="cosine", schedule_param=None, mean_type="v", var_type="fixed_small", **kwargs):
        sp = dict(num_timesteps=1000, cosine_s=0.008, zero_terminal_snr=True)
        sp.update(schedule_param or {})
        if schedule != "cosine":
            raise NotImplementedError(schedule)
        if mean_type not in ("v", "eps") or not var_type.startswith("fixed"):
            raise NotImplementedError((mean_type, var_type))
        self.mean_type = mean_type
        self.betas = _cosine_betas(**sp)
        self.num_timesteps = len(self.betas)
        ac = torch.cumprod(1 - self.betas, 0)
        self.alphas_cumprod = ac
        self.sqrt_alphas_cumprod = ac.sqrt()
        self.sqrt_one_minus_alphas_cumprod = (1 - ac).sqrt()
        self.sqrt_recip_alphas_cumprod = (1 / ac).sqrt()
        self.sqrt_recipm1_alphas_cumprod = (1 / ac - 1).sqrt()

    def _i(self, tensor, t, x):
        return tensor.to(x.device)[t].view(x.size(0), *((1,) * (x.ndim - 1))).to(x)

    @torch.no_grad()
    def ddim_sample(self, xt, t, model, model_kwargs, guide_scale=None, ddim_timesteps=20, eta=0.0, clamp=None):
        stride = self.num_timesteps // ddim_timesteps
        if isinstance(model, (GraphedCFGDenoiser, CFGSplitDenoiser)):
            out = model(xt, t)
        elif guide_scale is None:
            out = model(xt, t, **model_kwargs).float()
        else:
            y_out = model(xt, t, **model_kwargs[0]).float().contiguous()
            u_out = model(xt, t, **model_kwargs[1]).float().contiguous()
            out = ops.cfg_combine(y_out, u_out, guide_scale)
        if self.mean_type == "v":
            x0 = self._i(self.sqrt_alphas_cumprod, t, xt) * xt - self._i(self.sqrt_one_minus_alphas_cumprod, t, xt) * out
        else:
            x0 = self._i(self.sqrt_recip_alphas_cumprod, t, xt) * xt - self._i(self.sqrt_recipm1_alphas_cumprod, t, xt) * out
        if clamp is not None:
            x0 = x0.clamp(-clamp, clamp)
        eps = (self._i(self.sqrt_recip_alphas_cumprod, t, xt) * xt - x0) / self._i(self.sqrt_recipm1_alphas_cumprod, t, xt)
        alphas = self._i(self.alphas_cumprod, t, xt)
        alphas_prev = self._i(self.alphas_cumprod, (t - stride).clamp(0), xt)
        sigmas = eta * torch.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
        direction = torch.sqrt(1 - alphas_prev - sigmas ** 2) * eps
        # the reference draws the noise unconditionally (diffusion_ddim.py:233), also at eta = 0 where it is multiplied
        # by sigma = 0: the draw is kept so that a shared torch RNG stream stays aligned with the reference's
        noise = torch.randn_like(xt)
        mask = t.ne(0).float().view(-1, *((1,) * (xt.ndim - 1)))
        xt_1 = torch.sqrt(alphas_prev) * x0 + direction + mask * sigmas * noise
        return xt_1, x0

    @torch.no_grad()
    def ddim_sample_loop(self, noise, model, model_kwargs={}, clamp=None, percentile=None, condition_fn=None,
                         guide_scale=None, ddim_timesteps=20, eta=0.0, use_graph=False):
        """Reference signature (+ use_graph: capture the per-step CFG evaluation of a UNetSD_I2VGen in a
        CUDA graph)."""
        if percentile is not None or condition_fn is not None:
            raise NotImplementedError("percentile / condition_fn are not used by the i2vgen-xl inference entrance")
        b = noise.size(0)
        xt = noise.float()
        if use_graph and guide_scale is not None and isinstance(model, UNetSD_I2VGen):
            model = GraphedCFGDenoiser(model, model_kwargs[0], model_kwargs[1], guide_scale, xt,
                                       torch.zeros((b,), dtype=torch.long, device=xt.device))
        steps = (1 + torch.arange(0, self.num_timesteps, self.num_timesteps // ddim_timesteps)).clamp(
            0, self.num_timesteps - 1).flip(0)
        for step in steps:
            t = torch.full((b,), int(step), dtype=torch.long, device=xt.device)
            xt, _ = self.ddim_sample(xt, t, model, model_kwargs, guide_scale, ddim_timesteps, eta, clamp)
        return xt
