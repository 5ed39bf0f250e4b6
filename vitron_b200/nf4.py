"""NF4 weight format: the statement the kernels of csrc/gemv_nf4.cu are tested against.

The reference's `load_pretrained_model(..., load_4bit=True)` (vitron/model/builder.py:36-46) loads the language model
through bitsandbytes with `load_in_4bit`, `bnb_4bit_quant_type='nf4'` and `bnb_4bit_use_double_quant=True`. This module
restates that quantisation with torch:

  * each weight [N, K] (checkpoint dtype, taken to fp32; K % 64 == 0) is cut into blocks of 64 consecutive elements
    of a row; `absmax` per block; code = the nearest NF4 value to `w * (1 / absmax)` in fp32, ties to the lower index,
    an all-zero block gets code 7 (the value 0)  -- `quantize_4bit(blocksize=64)`;
  * the absmax values are double-quantised as `compress_statistics` does: offset = mean(absmax) over the tensor, then
    `absmax - offset` is quantised in blocks of 256 against the signed 8-bit dynamic map with a per-block fp32 absmax2;
    the scale a block uses is `dmap[q] * absmax2 + offset` in fp32.

Device format (`NF4Weight`): packed 4-bit codes and one fp16 scale per (row, 64-column block), the double-dequantised
scale rounded to fp16. A per-row scale leaves the row order free, so q/k/v concatenation and the 16-row gate/up
interleave of `ops.pack_glu_weight` apply to quantised rows as they do to bf16 ones. `dequantize` defines W_eff, the
matrix the format stands for. The dequantiser kernel rounds W_eff * kscale to bf16 bit for bit. The M <= 32
weight-streaming kernel multiplies bf16_rn(NF4[code]) * scale instead, which is at most 3.1e-3 relative from W_eff;
tests/test_nf4_kernels_gpu.py pins it against those operands and bounds its distance to W_eff. Parity of this quantiser
with bitsandbytes itself is not pinned (the library is not a dependency)."""
import torch

NF4 = torch.tensor([-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
                    -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
                    0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941,
                    0.7229568362236023, 1.0], dtype=torch.float32)
BLOCK = 64          # quantisation block (elements of one row)
BLOCK2 = 256        # double-quantisation block (absmax values)
_ROWS_PER_PASS = 512


def dynamic_map():
    """bitsandbytes `create_dynamic_map(signed=True, max_exponent_bits=7, total_bits=8)`: for i in 0..6 the 2^i midpoints
    of linspace(0.1, 1, 2^i + 1) scaled by +-10^(i-6), plus 0 and 1.0, sorted (256 fp32 entries)."""
    data = []
    for i in range(7):
        b = torch.linspace(0.1, 1, 2 ** i + 1)
        means = ((b[:-1] + b[1:]) / 2.0).tolist()
        data += [10 ** (i - 6) * m for m in means]
        data += [-(10 ** (i - 6)) * m for m in means]
    data += [0.0, 1.0]
    data.sort()
    return torch.tensor(data, dtype=torch.float32)


def _nearest(v, table):
    """Index of the nearest table entry to each element of fp32 v (ties: the lower index)."""
    return (v.unsqueeze(-1) - table).abs().argmin(-1)


def quantize_codes(w):
    """w [N, K] -> (codes uint8 [N, K] in 0..15, absmax fp32 [N, K / 64])."""
    if w.dim() != 2 or w.shape[1] % BLOCK != 0:
        raise ValueError(f"NF4 needs a [N, K] weight with K % {BLOCK} == 0, got {tuple(w.shape)}")
    n, k = w.shape
    table = NF4.to(w.device)
    codes = torch.empty((n, k), dtype=torch.uint8, device=w.device)
    absmax = torch.empty((n, k // BLOCK), dtype=torch.float32, device=w.device)
    for r in range(0, n, _ROWS_PER_PASS):   # bounded fp32 temporaries on the load device
        blk = w[r:r + _ROWS_PER_PASS].to(torch.float32).reshape(-1, k // BLOCK, BLOCK)
        am = blk.abs().amax(-1)
        c = _nearest(blk * (1.0 / am).unsqueeze(-1), table)
        c = torch.where((am == 0).unsqueeze(-1), torch.full_like(c, 7), c)
        codes[r:r + _ROWS_PER_PASS] = c.reshape(-1, k).to(torch.uint8)
        absmax[r:r + _ROWS_PER_PASS] = am
    return codes, absmax


def double_quant_scales(absmax):
    """The fp32 scale each 64-block uses after double quantisation: dmap[q] * absmax2 + offset."""
    flat = absmax.reshape(-1).to(torch.float32)
    offset = flat.mean()
    x = flat - offset
    pad = (-x.numel()) % BLOCK2
    xb = torch.cat([x, x.new_zeros(pad)]).reshape(-1, BLOCK2)
    a2 = xb.abs().amax(-1, keepdim=True)
    dmap = dynamic_map().to(absmax.device)
    q = _nearest(xb * torch.where(a2 > 0, 1.0 / a2, torch.zeros_like(a2)), dmap)
    scale = dmap[q] * a2 + offset
    return scale.reshape(-1)[:flat.numel()].reshape(absmax.shape)


def pack_codes(codes):
    """codes uint8 [N, K] (natural order) -> [N, ceil(K/128) * 64] in the kernel's byte order: per 128 k and per lane
    t = 0..3, 16 bytes hold the codes of k in {64u + 32h + 8t + e : u, h in 0..1, e in 0..7} (the k positions a lane of
    gemv.cu owns in two consecutive 64-blocks), byte u*8 + h*4 + e/2 = code(e even) | code(e odd) << 4."""
    n, k = codes.shape
    kp = (k + 127) // 128 * 128
    c = torch.zeros((n, kp), dtype=torch.uint8, device=codes.device)
    c[:, :k] = codes
    c = c.view(n, kp // 128, 2, 2, 4, 4, 2).permute(0, 1, 4, 2, 3, 5, 6)   # [n, s, u, h, t, pair, lo/hi] -> [n, s, t, u, h, pair, lo/hi]
    return (c[..., 0] | (c[..., 1] << 4)).reshape(n, kp // 2).contiguous()


def unpack_codes(packed, k):
    """Inverse of pack_codes: [N, ceil(K/128) * 64] -> codes uint8 [N, K]."""
    n = packed.shape[0]
    kp = (k + 127) // 128 * 128
    b = packed.view(n, kp // 128, 4, 2, 2, 4)                                # [n, s, t, u, h, pair]
    c = torch.stack([b & 15, b >> 4], -1).permute(0, 1, 3, 4, 2, 5, 6)       # [n, s, u, h, t, pair, lo/hi]
    return c.reshape(n, kp)[:, :k].contiguous()


class NF4Weight:
    """One NF4-quantised weight [N, K]: packed codes (uint8 [N, ceil(K/128) * 64]) and fp16 scales [N, K / 64]."""

    def __init__(self, codes, scales, k):
        self.codes, self.scales, self.k = codes, scales, int(k)

    @property
    def shape(self):
        return (self.codes.shape[0], self.k)

    @property
    def device(self):
        return self.codes.device

    @property
    def nbytes(self):
        return self.codes.numel() + 2 * self.scales.numel()

    def rows(self, i, j):
        return NF4Weight(self.codes[i:j], self.scales[i:j], self.k)

    @staticmethod
    def cat(ws):
        """Row concatenation (q | k | v)."""
        return NF4Weight(torch.cat([w.codes for w in ws]).contiguous(), torch.cat([w.scales for w in ws]).contiguous(), ws[0].k)


def quantize(w):
    """w [N, K] (any float dtype, any device) -> NF4Weight on w's device."""
    codes, absmax = quantize_codes(w)
    scales = double_quant_scales(absmax).to(torch.float16)
    return NF4Weight(pack_codes(codes), scales.contiguous(), w.shape[1])


def dequantize(w):
    """W_eff fp32 [N, K] = NF4[code] * float(scale)."""
    codes = unpack_codes(w.codes, w.k).long()
    vals = NF4.to(w.device)[codes].view(w.shape[0], -1, BLOCK)
    return (vals * w.scales.float().unsqueeze(-1)).reshape(w.shape)
