"""FocalNet backbone of SEEM on the vitron_b200 kernels (SURVEY.md §8 f1).

Drop-in for modules/SEEM/demo_code/xdecoder/backbone/focal.py: `FocalNet` (:340-590) keeps the reference's
constructor keywords, state-dict names and `forward(x) -> {"res2".."res5": [B, C_i, H_i, W_i]}`; `D2FocalNet`
(:598-672) builds it from the `cfg['BACKBONE']['FOCAL']` block of configs/seem/seem_focall_lang.yaml:29-47.

Design (NHWC bf16 end to end, no NCHW round trips — the reference permutes to NCHW and back inside every
FocalModulation, :101,114):
  * every Linear / 1x1 conv is the wgmma GEMM (`f` is padded to N = 2C+8 so q | ctx | gates are column
    slices of ONE output buffer: no torch.split copy); fc1 carries the exact-erf GELU in its epilogue;
  * the focal levels are a register-sliding-window depthwise conv kernel with the GELU fused (FFMA2),
    reading its first input in place from the `f` output (strided view);
  * ctx_global is a deterministic two-stage column mean; gating + scaling_modulator is one pass over the levels;
  * post-LN + layerscale + residual is one kernel: gamma is folded into the LayerNorm affine at load time
    (pre-LN variant: gamma is folded into the proj / fc2 weights and the residual rides the GEMM epilogue);
  * downsample (Conv k3 s2) is the im2col-free TMA implicit-GEMM conv, the stem (cin = 3, k7 s4) is an
    im2col kernel + GEMM.
Outputs are NCHW-shaped views of NHWC storage, which the pixel decoder consumes without a copy.
"""
import torch

from . import ops

BF16 = torch.bfloat16


def _ceil(a, b):
    return (a + b - 1) // b * b


class FocalNet:
    def __init__(self, pretrain_img_size=1600, patch_size=4, in_chans=3, embed_dim=96, depths=(2, 2, 6, 2),
                 mlp_ratio=4., drop_rate=0., drop_path_rate=0.2, norm_layer=None, patch_norm=True,
                 out_indices=(0, 1, 2, 3), frozen_stages=-1, focal_levels=(2, 2, 2, 2), focal_windows=(9, 9, 9, 9),
                 use_conv_embed=False, use_postln=False, use_postln_in_modulation=False, scaling_modulator=False,
                 use_layerscale=False, use_checkpoint=False, device="cuda"):
        if not use_conv_embed:
            raise NotImplementedError("only the overlapped conv embedding (USE_CONV_EMBED: True, seem_focall_lang.yaml:40) is built")
        self.patch_size = int(patch_size)
        self.in_chans = in_chans
        self.embed_dim = embed_dim
        self.depths = list(depths)
        self.num_layers = len(self.depths)
        self.mlp_ratio = mlp_ratio
        self.patch_norm = patch_norm
        self.out_indices = list(out_indices)
        self.focal_levels = list(focal_levels)
        self.focal_windows = list(focal_windows)
        self.focal_factor = 2
        self.use_postln = use_postln
        self.use_postln_in_modulation = use_postln_in_modulation
        self.scaling_modulator = scaling_modulator
        self.use_layerscale = use_layerscale
        self.num_features = [int(embed_dim * 2 ** i) for i in range(self.num_layers)]
        self.device = torch.device(device)
        self.w = None

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd, prefix=""):
        dev = self.device
        f32 = lambda n: sd[prefix + n].detach().to(device=dev, dtype=torch.float32)
        bf = lambda t: t.to(BF16).contiguous()
        w = {}
        pw = f32("patch_embed.proj.weight")  # [C, 3, 7, 7]
        C0 = pw.shape[0]
        self.stem_k = pw.shape[2]
        kreal = pw.shape[1] * pw.shape[2] * pw.shape[3]
        self.stem_kpad = _ceil(kreal, 64)
        wp = torch.zeros((C0, self.stem_kpad), dtype=torch.float32, device=dev)
        wp[:, :kreal] = pw.reshape(C0, kreal)
        w["stem"] = (bf(wp), bf(f32("patch_embed.proj.bias")))
        if self.patch_norm:
            w["stem_norm"] = (bf(f32("patch_embed.norm.weight")), bf(f32("patch_embed.norm.bias")))
        w["layers"] = []
        for i in range(self.num_layers):
            C = self.num_features[i]
            L = self.focal_levels[i]
            blocks = []
            for j in range(self.depths[i]):
                p = f"layers.{i}.blocks.{j}."
                b = {}
                g1 = f32(p + "gamma_1") if self.use_layerscale else torch.ones(C, device=dev)
                g2 = f32(p + "gamma_2") if self.use_layerscale else torch.ones(C, device=dev)
                # f: rows [0, C) = q, [C, 2C) = ctx, [2C, 2C+L+1) = gates; padded to 2C+8 rows (zero rows)
                fw, fb = f32(p + "modulation.f.weight"), f32(p + "modulation.f.bias")
                npad = 2 * C + _ceil(L + 1, 8)
                fwp = torch.zeros((npad, C), dtype=torch.float32, device=dev)
                fbp = torch.zeros((npad,), dtype=torch.float32, device=dev)
                fwp[:fw.shape[0]], fbp[:fb.shape[0]] = fw, fb
                b["f"] = (bf(fwp), bf(fbp))
                b["focal"] = []
                for l in range(L):
                    k = self.focal_factor * l + self.focal_windows[i]
                    b["focal"].append((ops.pack_dwconv_weight(f32(p + f"modulation.focal_layers.{l}.0.weight")), k))
                b["h"] = (bf(f32(p + "modulation.h.weight").reshape(C, C)), bf(f32(p + "modulation.h.bias")))
                if self.use_postln_in_modulation:
                    b["ln"] = (bf(f32(p + "modulation.ln.weight")), bf(f32(p + "modulation.ln.bias")))
                pjw, pjb = f32(p + "modulation.proj.weight"), f32(p + "modulation.proj.bias")
                f1w, f1b = f32(p + "mlp.fc1.weight"), f32(p + "mlp.fc1.bias")
                f2w, f2b = f32(p + "mlp.fc2.weight"), f32(p + "mlp.fc2.bias")
                n1w, n1b = f32(p + "norm1.weight"), f32(p + "norm1.bias")
                n2w, n2b = f32(p + "norm2.weight"), f32(p + "norm2.bias")
                if self.use_postln:  # x = shortcut + gamma * LN(branch): gamma folded into the LN affine
                    b["proj"], b["fc2"] = (bf(pjw), bf(pjb)), (bf(f2w), bf(f2b))
                    b["n1"], b["n2"] = (bf(g1 * n1w), bf(g1 * n1b)), (bf(g2 * n2w), bf(g2 * n2b))
                else:                # x = shortcut + gamma * branch(LN(x)): gamma folded into the last Linear
                    b["proj"] = (bf(g1[:, None] * pjw), bf(g1 * pjb))
                    b["fc2"] = (bf(g2[:, None] * f2w), bf(g2 * f2b))
                    b["n1"], b["n2"] = (bf(n1w), bf(n1b)), (bf(n2w), bf(n2b))
                b["fc1"] = (bf(f1w), bf(f1b))
                blocks.append(b)
            layer = {"blocks": blocks}
            if i < self.num_layers - 1:
                p = f"layers.{i}.downsample."
                layer["down"] = (ops.pack_conv_weight(f32(p + "proj.weight")), bf(f32(p + "proj.bias")),
                                 bf(f32(p + "norm.weight")), bf(f32(p + "norm.bias")))
            if i in self.out_indices:
                layer["norm"] = (bf(f32(f"norm{i}.weight")), bf(f32(f"norm{i}.bias")))
            w["layers"].append(layer)
        self.w = w
        return self

    # ------------------------------------------------------------------ forward
    def _modulation(self, xin, b, nb, H, W, C, L):
        """FocalModulation.forward (focal.py:91-118) on rows [nb*H*W, C]."""
        fo = ops.gemm(xin, b["f"][0], bias=b["f"][1])                      # [T, 2C + 8]
        ld = fo.shape[1]
        q, gates = fo[:, :C], fo[:, 2 * C:]
        cur = fo.view(nb, H, W, ld)[..., C:2 * C]                           # ctx, read in place
        levels = []
        for wt, k in b["focal"]:
            cur = ops.dwconv_nhwc(cur, wt, k, act=ops.ACT_GELU)
            levels.append(cur.view(nb * H * W, C))
        glob = ops.colmean(levels[-1], nb, act=ops.ACT_GELU)                # GELU(mean_hw(ctx_L))
        scale = 1.0 / (L + 1) if self.scaling_modulator else 1.0
        ctx_all = ops.focal_modulate(levels, gates, glob, nb, scale)
        hq = ops.gemm(ctx_all, b["h"][0], bias=b["h"][1])
        x_out = ops.mul_rows(q, hq)
        if self.use_postln_in_modulation:
            x_out = ops.layernorm(x_out, *b["ln"], 1e-5)
        return x_out

    def _block(self, x, b, nb, H, W, C, L):
        """FocalModulationBlock.forward (focal.py:172-203); x [nb*H*W, C] is updated and returned."""
        if self.use_postln:
            m = ops.gemm(self._modulation(x, b, nb, H, W, C, L), b["proj"][0], bias=b["proj"][1])
            x = ops.layernorm_add(m, b["n1"][0], b["n1"][1], x, 1e-5)
            h1 = ops.gemm(x, b["fc1"][0], bias=b["fc1"][1], act=ops.ACT_GELU)
            h2 = ops.gemm(h1, b["fc2"][0], bias=b["fc2"][1])
            return ops.layernorm_add(h2, b["n2"][0], b["n2"][1], x, 1e-5)
        xin = ops.layernorm(x, *b["n1"], 1e-5)
        x = ops.gemm(self._modulation(xin, b, nb, H, W, C, L), b["proj"][0], bias=b["proj"][1], residual=x)
        h1 = ops.gemm(ops.layernorm(x, *b["n2"], 1e-5), b["fc1"][0], bias=b["fc1"][1], act=ops.ACT_GELU)
        return ops.gemm(h1, b["fc2"][0], bias=b["fc2"][1], residual=x)

    @torch.no_grad()
    def forward_nhwc(self, x):
        """x [B, 3, H, W] (fp32 or bf16, NCHW) -> {"res2"..: [B, H_i, W_i, C_i] bf16 NHWC}."""
        if self.w is None:
            raise RuntimeError("FocalNet: load_state_dict() first")
        x = x.to(self.device)
        if x.dtype not in (torch.float32, BF16):
            x = x.float()
        x = x.contiguous()
        nb, _, Hin, Win = x.shape
        ps = self.patch_size
        Hp, Wp = _ceil(Hin, ps), _ceil(Win, ps)                              # PatchEmbed pads to the patch size
        k, stride, pad = self.stem_k, 4, 2                                   # conv embed stem (focal.py:314)
        H, W = (Hp + 2 * pad - k) // stride + 1, (Wp + 2 * pad - k) // stride + 1
        rows = ops.im2col_nchw(x, k, stride, pad, H, W, self.stem_kpad)
        t = ops.gemm(rows, self.w["stem"][0], bias=self.w["stem"][1])
        if self.patch_norm:
            t = ops.layernorm(t, *self.w["stem_norm"], 1e-5)
        outs = {}
        for i, layer in enumerate(self.w["layers"]):
            C, L = self.num_features[i], self.focal_levels[i]
            for b in layer["blocks"]:
                t = self._block(t, b, nb, H, W, C, L)
            if "norm" in layer:
                outs[f"res{i + 2}"] = ops.layernorm(t, *layer["norm"], 1e-5).view(nb, H, W, C)
            if "down" in layer:
                cw, cb, nw, nbias = layer["down"]
                d = ops.conv_nhwc(t.view(nb, H, W, C), cw, 3, 3, stride=2, bias=cb)
                H, W = d.shape[1], d.shape[2]
                t = ops.layernorm(d.view(nb * H * W, 2 * C), nw, nbias, 1e-5)
        return outs

    def forward(self, x):
        """Reference face: NCHW-shaped outputs (views of NHWC storage)."""
        return {k: v.permute(0, 3, 1, 2) for k, v in self.forward_nhwc(x).items()}

    __call__ = forward


class D2FocalNet(FocalNet):
    """focal.py:598-672: built from cfg = cfg['MODEL'] (keys BACKBONE.FOCAL.*)."""

    def __init__(self, cfg, input_shape=None, device="cuda"):
        fc = cfg["BACKBONE"]["FOCAL"]
        super().__init__(fc["PRETRAIN_IMG_SIZE"], fc["PATCH_SIZE"], 3, fc["EMBED_DIM"], fc["DEPTHS"], fc["MLP_RATIO"],
                         fc["DROP_RATE"], fc["DROP_PATH_RATE"], None, fc["PATCH_NORM"], fc["OUT_INDICES"],
                         focal_levels=fc["FOCAL_LEVELS"], focal_windows=fc["FOCAL_WINDOWS"],
                         use_conv_embed=fc["USE_CONV_EMBED"], use_postln=fc["USE_POSTLN"],
                         use_postln_in_modulation=fc["USE_POSTLN_IN_MODULATION"],
                         scaling_modulator=fc.get("SCALING_MODULATOR", False), use_layerscale=fc["USE_LAYERSCALE"],
                         use_checkpoint=fc.get("USE_CHECKPOINT", False), device=device)
        self._out_features = fc["OUT_FEATURES"]
        self._out_feature_strides = {"res2": 4, "res3": 8, "res4": 16, "res5": 32}
        self._out_feature_channels = {f"res{i + 2}": c for i, c in enumerate(self.num_features)}

    def forward(self, x):
        if x.dim() != 4:
            raise AssertionError(f"SwinTransformer takes an input of shape (N, C, H, W). Got {tuple(x.shape)} instead!")
        return {k: v for k, v in super().forward(x).items() if k in self._out_features}

    __call__ = forward

    def output_shape(self):
        return {n: dict(channels=self._out_feature_channels[n], stride=self._out_feature_strides[n]) for n in self._out_features}

    @property
    def size_divisibility(self):
        return 32


FOCAL_L_CFG = {"BACKBONE": {"FOCAL": dict(
    PRETRAIN_IMG_SIZE=224, PATCH_SIZE=4, EMBED_DIM=192, DEPTHS=[2, 2, 18, 2], FOCAL_LEVELS=[4, 4, 4, 4],
    FOCAL_WINDOWS=[3, 3, 3, 3], DROP_PATH_RATE=0.3, MLP_RATIO=4.0, DROP_RATE=0.0, PATCH_NORM=True, USE_CONV_EMBED=True,
    SCALING_MODULATOR=True, USE_CHECKPOINT=False, USE_POSTLN=True, USE_POSTLN_IN_MODULATION=False, USE_LAYERSCALE=True,
    OUT_FEATURES=["res2", "res3", "res4", "res5"], OUT_INDICES=[0, 1, 2, 3])}}
"""configs/seem/seem_focall_lang.yaml:29-47."""
