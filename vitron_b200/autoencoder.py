"""i2vgen-xl first-stage AutoencoderKL (Stable-Diffusion VAE) on the vitron_b200 kernels (SURVEY.md §8 f2).

Drop-in for modules/i2vgen-xl/tools/modules/autoencoder.py::AutoencoderKL (:31-112) with Encoder (:483-578),
Decoder (:581-686), ResnetBlock (:276-336), AttnBlock (:391-442), Upsample / Downsample (:444-481) and
DiagonalGaussianDistribution (:212-253): same constructor (`ddconfig`, `embed_dim`), state-dict names and
`encode / encode_firsr_stage / decode` entry points the i2vgen entrance calls
(tools/inferences/inference_i2vgen_entrance.py:172-173, 205-208).

Design: NHWC bf16 end to end; every 3x3 conv (incl. stride-2 downsample and the conv after the nearest
upsample) is the TMA implicit-GEMM wgmma kernel with bias / residual in the epilogue; GroupNorm(32, eps 1e-6) +
SiLU is one fused NHWC kernel; the 1x1 shortcut / q,k,v / proj_out convs are GEMMs on the pixel rows (q and k
share one GEMM); the single-head c-channel attention (head_dim = 512, outside the flash kernels' range) is
QK^T GEMM (fp32 scores, scale in the epilogue) -> row softmax kernel -> PV GEMM with V produced already
transposed ([c, hw] = Wv @ x^T) so no transpose is materialised, and V's bias added after the PV product
(softmax rows sum to one). `quant_conv` is folded into the encoder's conv_out at load time (two linear maps in a
row); 3- and 4-channel ends are zero-padded to 8 channels for 16-byte rows.
"""
import torch
import torch.nn.functional as F

from . import ops

BF16 = torch.bfloat16


class DiagonalGaussianDistribution:
    """autoencoder.py:212-253 on (mean, logvar) tensors [B, z, h, w] fp32."""

    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if self.deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator=None, noise=None):
        """mean + std * N(0, 1); `noise` (same shape) may be supplied for reproducible comparisons, `generator` may be
        a CPU or device generator."""
        if noise is None:
            gdev = generator.device if generator is not None else self.mean.device
            noise = torch.randn(self.mean.shape, device=gdev, dtype=self.mean.dtype, generator=generator)
        return self.mean + self.std * noise.to(self.mean.device)

    def mode(self):
        return self.mean


def _pad_cin(w, cin_to):
    """[cout, cin, kh, kw] -> zero-padded input channels."""
    cout, cin, kh, kw = w.shape
    out = torch.zeros((cout, cin_to, kh, kw), dtype=w.dtype, device=w.device)
    out[:, :cin] = w
    return out


def _pad_cout(w, b, cout_to):
    out = torch.zeros((cout_to, *w.shape[1:]), dtype=w.dtype, device=w.device)
    out[:w.shape[0]] = w
    bo = torch.zeros((cout_to,), dtype=b.dtype, device=b.device)
    bo[:b.shape[0]] = b
    return out, bo


class AutoencoderKL:
    def __init__(self, ddconfig, embed_dim, pretrained=None, ignore_keys=(), image_key="image", colorize_nlabels=None,
                 monitor=None, ema_decay=None, learn_logvar=False, use_vid_decoder=False, device="cuda", **kwargs):
        if not ddconfig["double_z"]:
            raise AssertionError("double_z")
        if tuple(ddconfig.get("attn_resolutions", ())) != ():
            raise NotImplementedError("attention at non-mid resolutions (attn_resolutions) is not used by i2vgen-xl")
        self.dd = dict(ddconfig)
        self.embed_dim = embed_dim
        self.ch = ddconfig["ch"]
        self.ch_mult = tuple(ddconfig["ch_mult"])
        self.num_res_blocks = ddconfig["num_res_blocks"]
        self.z_channels = ddconfig["z_channels"]
        self.out_ch = ddconfig["out_ch"]
        self.in_channels = ddconfig["in_channels"]
        self.device = torch.device(device)
        self.w = None

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd, strict=True):
        dev = self.device
        f32 = lambda n: sd[n].detach().to(device=dev, dtype=torch.float32)
        bf = lambda t: t.to(BF16).contiguous()
        conv3 = lambda p: (ops.pack_conv_weight(f32(p + "weight")), bf(f32(p + "bias")))
        lin = lambda p: (bf(f32(p + "weight").flatten(1)), bf(f32(p + "bias")))
        gn = lambda p: (bf(f32(p + "weight")), bf(f32(p + "bias")))

        def res(p):
            r = dict(n1=gn(p + "norm1."), c1=conv3(p + "conv1."), n2=gn(p + "norm2."), c2=conv3(p + "conv2."))
            if p + "nin_shortcut.weight" in sd:
                r["nin"] = lin(p + "nin_shortcut.")
            elif p + "conv_shortcut.weight" in sd:
                r["csc"] = conv3(p + "conv_shortcut.")
            return r

        def attn(p):
            wq, bq = f32(p + "q.weight").flatten(1), f32(p + "q.bias")
            wk, bk = f32(p + "k.weight").flatten(1), f32(p + "k.bias")
            return dict(n=gn(p + "norm."), qk=(bf(torch.cat([wq, wk], 0)), bf(torch.cat([bq, bk], 0))),
                        v=lin(p + "v."), o=lin(p + "proj_out."))

        nres = len(self.ch_mult)
        w = {"enc": {}, "dec": {}}
        e = w["enc"]
        wi = f32("encoder.conv_in.weight")
        e["conv_in"] = (ops.pack_conv_weight(_pad_cin(wi, 8)), bf(f32("encoder.conv_in.bias")))
        e["down"] = []
        for i in range(nres):
            lvl = {"blocks": [res(f"encoder.down.{i}.block.{j}.") for j in range(self.num_res_blocks)]}
            if i != nres - 1:
                lvl["down"] = conv3(f"encoder.down.{i}.downsample.conv.")
            e["down"].append(lvl)
        e["mid1"], e["attn"], e["mid2"] = res("encoder.mid.block_1."), attn("encoder.mid.attn_1."), res("encoder.mid.block_2.")
        e["norm_out"] = gn("encoder.norm_out.")
        # quant_conv (1x1, linear) folded into conv_out: W' = Wq @ Wout, b' = Wq @ bout + bq
        wo, bo = f32("encoder.conv_out.weight"), f32("encoder.conv_out.bias")
        wq, bq = f32("quant_conv.weight").flatten(1), f32("quant_conv.bias")
        wf = torch.einsum("om,mikl->oikl", wq, wo)
        wf, bfold = _pad_cout(wf, wq @ bo + bq, 8 * ((wf.shape[0] + 7) // 8))
        e["conv_out"] = (ops.pack_conv_weight(wf), bf(bfold))
        self.moment_ch = wq.shape[0]

        d = w["dec"]
        wp, bp = f32("post_quant_conv.weight"), f32("post_quant_conv.bias")       # [z, embed, 1, 1]
        wp8, bp8 = _pad_cout(wp, bp, 8)
        d["pqc"] = (bf(wp8.permute(0, 2, 3, 1).reshape(8, 1, wp.shape[1])), bf(bp8))  # conv_direct layout [cout, kh*kw, cin]
        d["conv_in"] = (ops.pack_conv_weight(_pad_cin(f32("decoder.conv_in.weight"), 8)), bf(f32("decoder.conv_in.bias")))
        d["mid1"], d["attn"], d["mid2"] = res("decoder.mid.block_1."), attn("decoder.mid.attn_1."), res("decoder.mid.block_2.")
        d["up"] = []
        for i in range(nres):
            lvl = {"blocks": [res(f"decoder.up.{i}.block.{j}.") for j in range(self.num_res_blocks + 1)]}
            if i != 0:
                lvl["up"] = conv3(f"decoder.up.{i}.upsample.conv.")
            d["up"].append(lvl)
        d["norm_out"] = gn("decoder.norm_out.")
        wo, bo = _pad_cout(f32("decoder.conv_out.weight"), f32("decoder.conv_out.bias"), 8)
        d["conv_out"] = (ops.pack_conv_weight(wo), bf(bo))
        self.w = w
        return self

    # ------------------------------------------------------------------ blocks (x: [n, h, w, c] bf16 NHWC)
    @staticmethod
    def _res(x, r):
        n, h, w, cin = x.shape
        a = ops.groupnorm_nhwc(x, *r["n1"], 32, 1e-6, act=ops.ACT_SILU)
        hcur = ops.conv_nhwc(a, r["c1"][0], 3, 3, bias=r["c1"][1])
        a = ops.groupnorm_nhwc(hcur, *r["n2"], 32, 1e-6, act=ops.ACT_SILU)
        if "nin" in r:
            skip = ops.gemm(x.view(n * h * w, cin), r["nin"][0], bias=r["nin"][1]).view(n, h, w, -1)
        elif "csc" in r:
            skip = ops.conv_nhwc(x, r["csc"][0], 3, 3, bias=r["csc"][1])
        else:
            skip = x
        return ops.conv_nhwc(a, r["c2"][0], 3, 3, bias=r["c2"][1], residual=skip)

    @staticmethod
    def _attn(x, a):
        """AttnBlock.forward (autoencoder.py:418-442): one head of c channels over the h*w pixels of each image."""
        n, h, w, c = x.shape
        T = h * w
        hn = ops.groupnorm_nhwc(x, *a["n"], 32, 1e-6).view(n * T, c)
        qk = ops.gemm(hn, a["qk"][0], bias=a["qk"][1])                      # [n*T, 2c]
        att = torch.empty((n * T, c), dtype=BF16, device=x.device)
        scores = torch.empty((T, T), dtype=torch.float32, device=x.device)
        for b in range(n):
            rows = slice(b * T, (b + 1) * T)
            ops.gemm(qk[rows, :c], qk[rows, c:], alpha=float(c) ** -0.5, out=scores, out_fp32=True)   # q k^T / sqrt(c)
            p = ops.softmax_rows(scores)
            vt = ops.gemm(a["v"][0], hn[rows])                              # [c, T] = Wv @ x^T (bias added below)
            ops.gemm(p, vt, bias=a["v"][1], out=att[rows])                  # P V^T' + bv
        return ops.gemm(att, a["o"][0], bias=a["o"][1], residual=x.view(n * T, c)).view(n, h, w, c)

    # ------------------------------------------------------------------ encoder / decoder
    @torch.no_grad()
    def _encode_moments(self, x):
        """x [B, 3, H, W] float -> moments [B, 2*embed, H/8, W/8] fp32 (Encoder.forward + quant_conv)."""
        if self.w is None:
            raise RuntimeError("AutoencoderKL: load_state_dict() first")
        e = self.w["enc"]
        x = x.to(self.device)
        B, cin, H, W = x.shape
        x8 = torch.zeros((B, H, W, 8), dtype=BF16, device=self.device)
        x8[..., :cin] = x.permute(0, 2, 3, 1)
        h = ops.conv_nhwc(x8, e["conv_in"][0], 3, 3, bias=e["conv_in"][1])
        for lvl in e["down"]:
            for r in lvl["blocks"]:
                h = self._res(h, r)
            if "down" in lvl:   # Downsample: zero pad right/bottom by one, conv k3 s2 p0 (autoencoder.py:474-479)
                h = ops.conv_nhwc(F.pad(h, (0, 0, 0, 1, 0, 1)).contiguous(), lvl["down"][0], 3, 3, stride=2, pad_h=0, pad_w=0,
                                  bias=lvl["down"][1])
        h = self._res(h, e["mid1"])
        h = self._attn(h, e["attn"])
        h = self._res(h, e["mid2"])
        h = ops.groupnorm_nhwc(h, *e["norm_out"], 32, 1e-6, act=ops.ACT_SILU)
        m = ops.conv_nhwc(h, e["conv_out"][0], 3, 3, bias=e["conv_out"][1])
        return m[..., :self.moment_ch].permute(0, 3, 1, 2).float().contiguous()

    def encode(self, x):
        return DiagonalGaussianDistribution(self._encode_moments(x))

    def encode_firsr_stage(self, x, scale_factor=1.0, generator=None, noise=None):
        """(sic) autoencoder.py:85-90: scale_factor * posterior.sample()."""
        return scale_factor * self.encode(x).sample(generator, noise)

    @torch.no_grad()
    def decode(self, z, **kwargs):
        """z [B, z_channels, h, w] -> [B, out_ch, 8h, 8w] fp32 (post_quant_conv + Decoder.forward)."""
        if self.w is None:
            raise RuntimeError("AutoencoderKL: load_state_dict() first")
        d = self.w["dec"]
        z = z.to(self.device)
        zn = z.permute(0, 2, 3, 1).to(BF16).contiguous()
        h = ops.conv_nhwc_direct(zn, d["pqc"][0], d["pqc"][1], 1, 1)             # [B, h, w, 8], channels >= z are zero
        h = ops.conv_nhwc(h, d["conv_in"][0], 3, 3, bias=d["conv_in"][1])
        h = self._res(h, d["mid1"])
        h = self._attn(h, d["attn"])
        h = self._res(h, d["mid2"])
        for i in reversed(range(len(d["up"]))):
            lvl = d["up"][i]
            for r in lvl["blocks"]:
                h = self._res(h, r)
            if "up" in lvl:
                h = ops.conv_nhwc(ops.upsample2x_nhwc(h), lvl["up"][0], 3, 3, bias=lvl["up"][1])
        h = ops.groupnorm_nhwc(h, *d["norm_out"], 32, 1e-6, act=ops.ACT_SILU)
        out = ops.conv_nhwc(h, d["conv_out"][0], 3, 3, bias=d["conv_out"][1])
        return out[..., :self.out_ch].permute(0, 3, 1, 2).float().contiguous()

    def forward(self, input, sample_posterior=True):
        posterior = self.encode(input)
        z = posterior.sample() if sample_posterior else posterior.mode()
        return self.decode(z), posterior

    __call__ = forward


SD_VAE_DDCONFIG = dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                       num_res_blocks=2, attn_resolutions=[], dropout=0.0, video_kernel_size=[3, 1, 1])
"""tools/modules/config.py:110-127."""
