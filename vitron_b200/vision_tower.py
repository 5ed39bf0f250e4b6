"""LanguageBind ViT-L/14 image / video towers on the vitron_b200 kernels.

Drop-in for the reference's `LanguageBindImageTower` / `LanguageBindVideoTower`
(vitron/model/multimodal_encoder/languagebind/__init__.py:69-233) wrapping `CLIPVisionTransformer`
(languagebind/image/modeling_image.py:596-672, video/modeling_video.py:596-676) with
`CLIPEncoderLayer` (modeling_image.py:65-158; video variant has temporal attention and no temporal
MLP, modeling_video.py:83-134).  Same forward signatures and attributes; parameters are read from
a state dict with the reference's names (SURVEY.md Appendix B).

Mechanism differences: patch-embed is patchify + wgmma GEMM, q/k/v is one fused GEMM, attention
never materialises S x S scores, bias/activation/residual live in GEMM epilogues, only the layers
that influence `hidden_states[select_layer]` are executed (the reference computes and discards the
rest), and the video tower's two `rearrange` transposes per layer are replaced by strided attention.
"""
from types import SimpleNamespace

import torch

from . import ops

BF16 = torch.bfloat16
_ACTS = {"gelu": ops.ACT_GELU, "quick_gelu": ops.ACT_QUICK_GELU, "relu": ops.ACT_RELU, "silu": ops.ACT_SILU}


class VisionConfig(SimpleNamespace):
    """Subset of CLIPVisionConfig the path reads (configuration_image.py:183-205)."""

    def __init__(self, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                 image_size=224, patch_size=14, hidden_act="gelu", layer_norm_eps=1e-5, num_channels=3,
                 add_time_attn=False, num_frames=1, **kw):
        super().__init__(hidden_size=hidden_size, intermediate_size=intermediate_size,
                         num_hidden_layers=num_hidden_layers, num_attention_heads=num_attention_heads,
                         image_size=image_size, patch_size=patch_size, hidden_act=hidden_act,
                         layer_norm_eps=layer_norm_eps, num_channels=num_channels, add_time_attn=add_time_attn,
                         num_frames=num_frames, **kw)


class VisionTransformerB200:
    """CLIPVisionTransformer.forward restricted to what the towers consume: the hidden state
    selected by `select_layer` (all tokens)."""

    def __init__(self, config, device):
        self.config = config
        self.device = torch.device(device)
        self.act = _ACTS[config.hidden_act]
        self.kpad = (config.num_channels * config.patch_size ** 2 + 63) // 64 * 64
        self.layers = []
        self.w = {}

    # parameter names relative to the vision transformer root (e.g. 'encoder.layers.0.mlp.fc1.weight')
    def load_state_dict(self, sd, prefix=""):
        dev, c = self.device, self.config

        def get(name):
            return sd[prefix + name].detach().to(device=dev, dtype=BF16).contiguous()

        d = c.hidden_size
        pw = get("embeddings.patch_embedding.weight").reshape(d, -1)
        wpatch = torch.zeros((d, self.kpad), dtype=BF16, device=dev)
        wpatch[:, :pw.shape[1]] = pw
        self.w = dict(cls=get("embeddings.class_embedding").reshape(-1),
                      pos=get("embeddings.position_embedding.weight"), wpatch=wpatch,
                      pre_w=get("pre_layrnorm.weight"), pre_b=get("pre_layrnorm.bias"))
        for n in ("post_layernorm.weight", "post_layernorm.bias"):   # not on the path (hidden_states[-2]); kept for state_dict()
            if prefix + n in sd:
                self.w[n] = get(n)
        self.layers = []
        for i in range(c.num_hidden_layers):
            p = f"encoder.layers.{i}."
            L = dict(
                wqkv=torch.cat([get(p + f"self_attn.{n}_proj.weight") for n in "qkv"], 0).contiguous(),
                bqkv=torch.cat([get(p + f"self_attn.{n}_proj.bias") for n in "qkv"], 0).contiguous(),
                wo=get(p + "self_attn.out_proj.weight"), bo=get(p + "self_attn.out_proj.bias"),
                ln1w=get(p + "layer_norm1.weight"), ln1b=get(p + "layer_norm1.bias"),
                ln2w=get(p + "layer_norm2.weight"), ln2b=get(p + "layer_norm2.bias"),
                w1=get(p + "mlp.fc1.weight"), b1=get(p + "mlp.fc1.bias"),
                w2=get(p + "mlp.fc2.weight"), b2=get(p + "mlp.fc2.bias"))
            if c.add_time_attn:
                L.update(
                    temb=get(p + "temporal_embedding").reshape(-1, d).contiguous(),
                    twqkv=torch.cat([get(p + f"temporal_attn.{n}_proj.weight") for n in "qkv"], 0).contiguous(),
                    tbqkv=torch.cat([get(p + f"temporal_attn.{n}_proj.bias") for n in "qkv"], 0).contiguous(),
                    two=get(p + "temporal_attn.out_proj.weight"), tbo=get(p + "temporal_attn.out_proj.bias"),
                    tlnw=get(p + "temporal_layer_norm1.weight"), tlnb=get(p + "temporal_layer_norm1.bias"))
                if (prefix + p + "temporal_mlp.fc1.weight") in sd:  # image-variant layer with time attention
                    L.update(tw1=get(p + "temporal_mlp.fc1.weight"), tb1=get(p + "temporal_mlp.fc1.bias"),
                             tw2=get(p + "temporal_mlp.fc2.weight"), tb2=get(p + "temporal_mlp.fc2.bias"),
                             tln2w=get(p + "temporal_layer_norm2.weight"), tln2b=get(p + "temporal_layer_norm2.bias"))
            self.layers.append(L)
        return self

    def state_dict(self, prefix=""):
        """The reference's parameter names (SURVEY.md Appendix B) rebuilt from the packed device tensors."""
        c, out, d = self.config, {}, self.config.hidden_size
        w = self.w
        out[prefix + "embeddings.class_embedding"] = w["cls"]
        out[prefix + "embeddings.position_embedding.weight"] = w["pos"]
        k = c.num_channels * c.patch_size ** 2
        out[prefix + "embeddings.patch_embedding.weight"] = w["wpatch"][:, :k].reshape(d, c.num_channels, c.patch_size, c.patch_size)
        out[prefix + "pre_layrnorm.weight"], out[prefix + "pre_layrnorm.bias"] = w["pre_w"], w["pre_b"]
        for n in ("post_layernorm.weight", "post_layernorm.bias"):
            if n in w:
                out[prefix + n] = w[n]
        for i, L in enumerate(self.layers):
            p = f"{prefix}encoder.layers.{i}."
            for n, wq, bq in zip("qkv", L["wqkv"].split(d, 0), L["bqkv"].split(d, 0)):
                out[p + f"self_attn.{n}_proj.weight"], out[p + f"self_attn.{n}_proj.bias"] = wq, bq
            out[p + "self_attn.out_proj.weight"], out[p + "self_attn.out_proj.bias"] = L["wo"], L["bo"]
            out[p + "layer_norm1.weight"], out[p + "layer_norm1.bias"] = L["ln1w"], L["ln1b"]
            out[p + "layer_norm2.weight"], out[p + "layer_norm2.bias"] = L["ln2w"], L["ln2b"]
            out[p + "mlp.fc1.weight"], out[p + "mlp.fc1.bias"] = L["w1"], L["b1"]
            out[p + "mlp.fc2.weight"], out[p + "mlp.fc2.bias"] = L["w2"], L["b2"]
            if "temb" in L:
                out[p + "temporal_embedding"] = L["temb"].reshape(1, -1, d)
                for n, wq, bq in zip("qkv", L["twqkv"].split(d, 0), L["tbqkv"].split(d, 0)):
                    out[p + f"temporal_attn.{n}_proj.weight"], out[p + f"temporal_attn.{n}_proj.bias"] = wq, bq
                out[p + "temporal_attn.out_proj.weight"], out[p + "temporal_attn.out_proj.bias"] = L["two"], L["tbo"]
                out[p + "temporal_layer_norm1.weight"], out[p + "temporal_layer_norm1.bias"] = L["tlnw"], L["tlnb"]
            if "tw1" in L:
                out[p + "temporal_mlp.fc1.weight"], out[p + "temporal_mlp.fc1.bias"] = L["tw1"], L["tb1"]
                out[p + "temporal_mlp.fc2.weight"], out[p + "temporal_mlp.fc2.bias"] = L["tw2"], L["tb2"]
                out[p + "temporal_layer_norm2.weight"], out[p + "temporal_layer_norm2.bias"] = L["tln2w"], L["tln2b"]
        return out

    def parameters(self):
        yield from self.w.values()
        for L in self.layers:
            yield from L.values()

    def num_layers_for(self, select_layer):
        L = self.config.num_hidden_layers
        idx = select_layer if select_layer >= 0 else L + 1 + select_layer
        if not 0 <= idx <= L:
            raise ValueError(f"select_layer {select_layer} out of range for {L} layers")
        return idx

    def forward_hidden(self, pixel_values, select_layer=-2):
        """pixel_values [B,3,H,W] or [B,3,T,H,W] -> hidden_states[select_layer] as
        [B, 1+np, d] (image) or [B, T, 1+np, d] (video), bf16."""
        c = self.config
        if pixel_values.dim() == 5:
            B, _, T = pixel_values.shape[:3]
            px = pixel_values.permute(0, 2, 1, 3, 4).reshape(B * T, *pixel_values.shape[1:2], *pixel_values.shape[3:])
        else:
            B, T = pixel_values.shape[0], 1
            px = pixel_values
        px = px.contiguous()
        if px.dtype not in (torch.float32, BF16):
            px = px.float()
        nb = px.shape[0]
        d, H = c.hidden_size, c.num_attention_heads
        hd = d // H
        npatch = (c.image_size // c.patch_size) ** 2
        N = npatch + 1
        A = ops.patchify(px, c.patch_size, self.kpad)
        po = ops.gemm(A, self.w["wpatch"])
        h = ops.vit_embed_ln(po, self.w["cls"], self.w["pos"], self.w["pre_w"], self.w["pre_b"], nb, npatch,
                             c.layer_norm_eps).view(nb * N, d)
        for L in self.layers[:self.num_layers_for(select_layer)]:
            if c.add_time_attn:
                if T != 1:
                    ops.add_rowgroup(h, L["temb"], N, T, out=h)
                x = ops.layernorm(h, L["tlnw"], L["tlnb"], c.layer_norm_eps)
                qkv = ops.gemm(x, L["twqkv"], bias=L["tbqkv"])
                # rows are (b, t, n); sequences run over t for fixed (b, n)
                q5 = qkv.view(B, T, N, 3, H, hd).permute(3, 0, 2, 1, 4, 5)  # [3, B, N, T, H, hd]
                att = torch.empty((B, T, N, H, hd), dtype=BF16, device=h.device)
                ops.attention_short(q5[0], q5[1], q5[2], scale=hd ** -0.5, out=att.permute(0, 2, 1, 3, 4))
                ops.gemm(att.view(nb * N, d), L["two"], bias=L["tbo"], residual=h, out=h)
                if "tw1" in L:
                    x = ops.layernorm(h, L["tln2w"], L["tln2b"], c.layer_norm_eps)
                    f = ops.gemm(x, L["tw1"], bias=L["tb1"], act=self.act)
                    ops.gemm(f, L["tw2"], bias=L["tb2"], residual=h, out=h)
            x = ops.layernorm(h, L["ln1w"], L["ln1b"], c.layer_norm_eps)
            qkv = ops.gemm(x, L["wqkv"], bias=L["bqkv"]).view(nb, N, 3, H, hd)
            att = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], scale=hd ** -0.5)
            ops.gemm(att.view(nb * N, d), L["wo"], bias=L["bo"], residual=h, out=h)
            x = ops.layernorm(h, L["ln2w"], L["ln2b"], c.layer_norm_eps)
            f = ops.gemm(x, L["w1"], bias=L["b1"], act=self.act)
            ops.gemm(f, L["w2"], bias=L["b2"], residual=h, out=h)
        h = h.view(nb, N, d)
        return h.view(B, T, N, d) if pixel_values.dim() == 5 else h


class _TowerBase:
    is_loaded = True

    def __init__(self, config, device, select_layer=-2, select_feature="patch"):
        self.vit = VisionTransformerB200(config, device)
        self.select_layer = select_layer
        self.select_feature = select_feature

    def load_model(self):  # reference API; weights come from load_state_dict here
        self.is_loaded = True

    # nn.Module face used by the reference's builder (builder.py:152-163: `tower.to(device=..., dtype=...)`)
    def to(self, *args, **kwargs):
        from .module_face import check_to
        check_to(self.device, args, kwargs)
        return self

    def eval(self):
        return self

    def parameters(self):
        return self.vit.parameters()

    def state_dict(self, prefix=""):
        attr = "video_tower." if isinstance(self, LanguageBindVideoTower) else "image_tower."
        return self.vit.state_dict(prefix + attr)

    @property
    def config(self):
        return self.vit.config

    @property
    def hidden_size(self):
        return self.vit.config.hidden_size

    @property
    def num_patches(self):
        return (self.vit.config.image_size // self.vit.config.patch_size) ** 2

    @property
    def dtype(self):
        return BF16

    @property
    def device(self):
        return self.vit.device

    @property
    def dummy_feature(self):
        return torch.zeros(1, self.hidden_size, device=self.device, dtype=self.dtype)

    def __call__(self, x):
        return self.forward(x)


class LanguageBindImageTower(_TowerBase):
    """forward(images [B,3,H,W] | list of [3,H,W]) -> [B, 256, 1024] (languagebind/__init__.py:106-121)."""

    def feature_select(self, hidden):
        if self.select_feature == "patch":
            return hidden[:, 1:]
        if self.select_feature == "cls_patch":
            return hidden
        raise ValueError(f"Unexpected select feature: {self.select_feature}")

    @torch.no_grad()
    def forward(self, images):
        if isinstance(images, list):
            return [self.feature_select(self.vit.forward_hidden(im.unsqueeze(0).to(self.device), self.select_layer))
                    .to(im.dtype if im.dtype.is_floating_point else BF16) for im in images]
        h = self.vit.forward_hidden(images.to(self.device), self.select_layer)
        return self.feature_select(h)


class LanguageBindVideoTower(_TowerBase):
    """forward(videos [B,3,T,H,W]) -> [B, T, 256, 1024] (languagebind/__init__.py:192-204)."""

    def feature_select(self, hidden):
        if self.select_feature == "patch":
            return hidden[:, :, 1:]
        raise ValueError(f"Unexpected select feature: {self.select_feature}")

    @torch.no_grad()
    def forward(self, videos):
        if isinstance(videos, list):
            return [self.feature_select(self.vit.forward_hidden(v.unsqueeze(0).to(self.device), self.select_layer))
                    for v in videos]
        return self.feature_select(self.vit.forward_hidden(videos.to(self.device), self.select_layer))


def build_image_tower(config, device, state_dict=None, prefix="", **kw):
    """cf. multimodal_encoder/builder.py:7-15 — here the tower is built from an explicit VisionConfig."""
    t = LanguageBindImageTower(config, device, kw.get("select_layer", -2), kw.get("select_feature", "patch"))
    if state_dict is not None:
        t.vit.load_state_dict(state_dict, prefix)
    return t


def build_video_tower(config, device, state_dict=None, prefix="", **kw):
    t = LanguageBindVideoTower(config, device, kw.get("select_layer", -2), kw.get("select_feature", "patch"))
    if state_dict is not None:
        t.vit.load_state_dict(state_dict, prefix)
    return t
