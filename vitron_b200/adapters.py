"""mm_projector and region_extractor on the vitron_b200 kernels.

`build_vision_projector` mirrors vitron/model/multimodal_projector/builder.py:33-51 (linear /
mlpNx_gelu / identity); `RegionExtractor` mirrors vitron/model/region_extractor/layer.py:59-130
(bbox -> binary canvas mask -> bilinear 16x16 -> >0 -> normalised mask pooling -> 3-layer ReLU MLP,
plus the 4 -> 2048 -> 4096 location encoder, summed), including its quirk that x indexes rows.
"""
import re

import torch

from . import nf4 as _nf4
from . import ops

BF16 = torch.bfloat16


def _linear_weight(w, nf4):
    """bf16 weight, or with nf4 (the reference's load_4bit, whose replace_with_bnb_linear converts every Linear these
    modules hold) an NF4Weight; a Linear whose input width is not a multiple of 64 (the 4-input location encoder) stays
    bf16, the one place where the NF4 format of vitron_b200.nf4 does not reach."""
    return _nf4.quantize(w) if nf4 and w.shape[1] % _nf4.BLOCK == 0 else w


def _dense(w):
    return _nf4.dequantize(w).to(BF16) if isinstance(w, _nf4.NF4Weight) else w


def _tensors(w):
    return (w.codes, w.scales) if isinstance(w, _nf4.NF4Weight) else (w,)


class VisionProjector:
    def __init__(self, projector_type, mm_hidden_size, hidden_size, device):
        self.device = torch.device(device)
        self.projector_type = projector_type
        self.linears = []  # [(w, b)]
        if projector_type == "linear":
            self.depth = 1
        elif projector_type == "identity":
            self.depth = 0
        else:
            m = re.match(r"^mlp(\d+)x_gelu$", projector_type)
            if not m:
                raise ValueError(f"Unknown projector type: {projector_type}")
            self.depth = int(m.group(1))
        self.mm_hidden_size, self.hidden_size = mm_hidden_size, hidden_size

    def load_state_dict(self, sd, prefix="", nf4=False):
        """names: '<prefix>weight/bias' (linear) or '<prefix>{0,2,4..}.weight/bias' (mlpNx_gelu). nf4: weights in NF4,
        biases bf16."""
        get = lambda n: sd[prefix + n].detach().to(device=self.device, dtype=BF16).contiguous()
        w = lambda n: _linear_weight(get(n), nf4)
        if self.projector_type == "linear":
            self.linears = [(w("weight"), get("bias"))]
        else:
            self.linears = [(w(f"{2 * i}.weight"), get(f"{2 * i}.bias")) for i in range(self.depth)]
        return self

    def state_dict(self, prefix=""):
        if self.projector_type == "linear":
            return {prefix + "weight": _dense(self.linears[0][0]), prefix + "bias": self.linears[0][1]}
        out = {}
        for i, (w, b) in enumerate(self.linears):
            out[f"{prefix}{2 * i}.weight"], out[f"{prefix}{2 * i}.bias"] = _dense(w), b
        return out

    def parameters(self):
        for w, b in self.linears:
            yield from _tensors(w)
            yield b

    def __call__(self, x):
        if self.depth == 0:
            return x
        shp = x.shape
        h = x.reshape(-1, shp[-1])
        if h.dtype != BF16:
            h = h.to(BF16)
        if not h.is_contiguous():
            h = h.contiguous()
        for i, (w, b) in enumerate(self.linears):
            last = i == len(self.linears) - 1
            h = ops.gemm(h, w, bias=b, act=ops.ACT_NONE if last else ops.ACT_GELU)
        return h.view(*shp[:-1], h.shape[-1])


def build_vision_projector(config, device, state_dict=None, prefix="", **kwargs):
    p = VisionProjector(getattr(config, "mm_projector_type", "linear"), config.mm_hidden_size, config.hidden_size,
                        device)
    if state_dict is not None:
        p.load_state_dict(state_dict, prefix)
    return p


class RegionExtractor:
    def __init__(self, in_dim=1024, out_dim=4096, patch_size=14, image_size=224, device="cuda"):
        self.in_dim, self.out_dim = in_dim, out_dim
        self.patch_size, self.image_size = patch_size, image_size
        self.device = torch.device(device)
        self.mlp = []
        self.loc = []

    def load_state_dict(self, sd, prefix="", nf4=False):
        """names: region_linear.layers.{0,1,2}.{weight,bias}, loc_encoder.loc_encoder.{0,2}.{weight,bias}. nf4: weights
        in NF4 (except the 4-input location layer), biases bf16."""
        get = lambda n: sd[prefix + n].detach().to(device=self.device, dtype=BF16).contiguous()
        self.mlp = [(_linear_weight(get(f"region_linear.layers.{i}.weight"), nf4), get(f"region_linear.layers.{i}.bias"))
                    for i in range(3)]
        w0 = get("loc_encoder.loc_encoder.0.weight")  # [hidden/2, 4] -> pad K to 8 for 16-byte rows
        w0p = torch.zeros((w0.shape[0], 8), dtype=BF16, device=self.device)
        w0p[:, :4] = w0
        self.loc = [(w0p, get("loc_encoder.loc_encoder.0.bias")),
                    (_linear_weight(get("loc_encoder.loc_encoder.2.weight"), nf4), get("loc_encoder.loc_encoder.2.bias"))]
        return self

    def state_dict(self, prefix=""):
        out = {}
        for i, (w, b) in enumerate(self.mlp):
            out[f"{prefix}region_linear.layers.{i}.weight"], out[f"{prefix}region_linear.layers.{i}.bias"] = _dense(w), b
        out[prefix + "loc_encoder.loc_encoder.0.weight"] = self.loc[0][0][:, :4].contiguous()
        out[prefix + "loc_encoder.loc_encoder.0.bias"] = self.loc[0][1]
        out[prefix + "loc_encoder.loc_encoder.2.weight"] = _dense(self.loc[1][0])
        out[prefix + "loc_encoder.loc_encoder.2.bias"] = self.loc[1][1]
        return out

    def parameters(self):
        for w, b in self.mlp + self.loc:
            yield from _tensors(w)
            yield b

    def forward(self, feats, regions):
        """feats [B, S, C] patch features, regions: list of B [x1, y1, x2, y2] -> [B, 1, out_dim]."""
        b, s, c = feats.shape
        if len(regions) != b:
            raise ValueError(f"{b} feature maps but {len(regions)} regions")
        boxes = torch.tensor([[float(v) for v in r] for r in regions], dtype=torch.float32).to(self.device)
        f = feats.to(BF16).contiguous()
        pooled = ops.region_mask_pool(f, boxes, self.image_size)
        h = pooled
        for i, (w, bias) in enumerate(self.mlp):
            h = ops.gemm(h, w, bias=bias, act=ops.ACT_RELU if i < 2 else ops.ACT_NONE)
        bx = torch.zeros((b, 8), dtype=BF16, device=self.device)
        bx[:, :4] = boxes.to(BF16)
        l = ops.gemm(bx, self.loc[0][0], bias=self.loc[0][1], act=ops.ACT_RELU)
        out = ops.gemm(l, self.loc[1][0], bias=self.loc[1][1], residual=h)
        return out.unsqueeze(1)

    __call__ = forward


def build_region_extractor(config, device, state_dict=None, prefix="", **kwargs):
    r = RegionExtractor(in_dim=getattr(config, "mm_hidden_size", 1024), out_dim=config.hidden_size,
                        patch_size=getattr(config, "mm_patch_size", 14),
                        image_size=getattr(config, "mm_image_size", 224), device=device)
    if state_dict is not None:
        r.load_state_dict(state_dict, prefix)
    return r
