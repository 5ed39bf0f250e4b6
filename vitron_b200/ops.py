"""Torch-tensor wrappers over the C ABI (include/vitron_b200.h).

torch is used only for device memory, streams and shapes: every function here enqueues one or two
hand-written CUDA kernels from libvitron_b200.so on the current torch stream. No fallbacks.
"""
import ctypes as C
import math
import struct

import torch

from . import _lib, beam
from .nf4 import NF4Weight
from ._lib import (ACT_GELU, ACT_NONE, ACT_QUICK_GELU, ACT_RELU, ACT_SILU, GLU_GEGLU, GLU_NONE,
                   GLU_SWIGLU, Epilogue, check)

BF16 = torch.bfloat16
_ws = {}
_launches = [0]


def launch_count():
    """Number of vitron_b200 kernels enqueued so far through this module (bench.py: gpu_launches)."""
    return _launches[0]


def count_launches(n):
    _launches[0] += int(n)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


_ws_retired = []


def workspace(nbytes, device, tag="main"):
    """Grow-only per-(device, tag) scratch buffer, zero-filled at allocation (the split-K / split-KV
    arrival counters at its head must start at zero; the kernels leave them zeroed). A buffer that is outgrown is
    RETIRED, never freed: captured CUDA graphs keep the address they were captured with, and every buffer is
    self-consistent (its own counters), so an old graph replaying against its old buffer stays correct."""
    key = (device.index if device.index is not None else torch.cuda.current_device(), tag)
    buf = _ws.get(key)
    if buf is None or buf.numel() < nbytes:
        if buf is not None:
            _ws_retired.append(buf)
        buf = torch.zeros(max(int(nbytes), 1 << 20), dtype=torch.uint8, device=device)
        _ws[key] = buf
    return buf


def reserve_decode_workspace(max_batch, n_heads, head_dim, device):
    """Pre-size the split-KV decode workspace for the largest batch an engine will ever run."""
    need = _lib.load().vb200_attn_decode_workspace_size(max_batch, n_heads, head_dim, 32)
    return workspace(need, torch.device(device), "dec")


class pdl:
    """Context manager: launch the vitron_b200 kernels issued inside with programmatic dependent launch (every kernel
    launched through vb_launch starts with griddepcontrol.launch_dependents / .wait): consecutive kernels of a stream or of
    a captured CUDA graph overlap launch latency and prologue (barrier init, tensor-map prefetch) with the predecessor's tail."""

    def __init__(self, enabled=True):
        self.enabled, self.prev = enabled, None

    def __enter__(self):
        self.prev = _lib.load().vb200_set_pdl(1 if self.enabled else 0)
        return self

    def __exit__(self, *exc):
        _lib.load().vb200_set_pdl(self.prev)
        return False


class GraphedCall:
    """Capture `fn(**tensors)` (any composition of the ops below + allocation-only torch calls, no host syncs) in one CUDA graph
    per input signature and replay it: launch-bound chains (the ~290 kernels of the SEEM mask decoder, ~10 us of host time
    each) run at device speed. Inputs are copied into static buffers; the RETURNED tensors are static too and are overwritten
    by the next call with the same signature — consume or clone them first."""

    def __init__(self, fn, warmup=2):
        self.fn, self.warmup, self.graphs = fn, warmup, {}

    def __call__(self, **tensors):
        key = tuple((k, tuple(v.shape), v.dtype, v.device.index) for k, v in sorted(tensors.items()))
        ent = self.graphs.get(key)
        if ent is None:
            static = {k: v.detach().clone() for k, v in tensors.items()}
            dev = next(iter(static.values())).device
            s = torch.cuda.Stream(device=dev)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(self.warmup):  # workspaces, cached tables, cudaFuncSetAttribute calls
                    self.fn(**static)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            l0 = launch_count()
            with torch.cuda.graph(g), pdl(True):
                out = self.fn(**static)
            ent = (g, static, out, launch_count() - l0)
            self.graphs[key] = ent
        g, static, out, n = ent
        for k, v in tensors.items():
            static[k].copy_(v, non_blocking=True)
        g.replay()
        count_launches(n)
        return out


def _req(cond, msg):
    if not cond:
        raise ValueError(msg)


def _rows2d(x):
    """View x as [rows, d] with unit inner stride; returns (tensor2d, ld)."""
    _req(x.stride(-1) == 1, "inner dimension must be contiguous")
    if x.dim() == 2:
        return x, x.stride(0)
    x2 = x.reshape(-1, x.shape[-1])
    return x2, x2.stride(0)


def pack_glu_weight(w_a, w_b):
    """Interleave two [F, K] weights (or [F] biases) in 16-row blocks: rows [32i,32i+16) = a,
    [32i+16,32i+32) = b — the layout the fused GLU epilogue expects."""
    f = w_a.shape[0]
    _req(f % 16 == 0 and w_a.shape == w_b.shape, "GLU halves must match and be multiples of 16 rows")
    rest = w_a.shape[1:]
    a = w_a.reshape(f // 16, 16, *rest)
    b = w_b.reshape(f // 16, 16, *rest)
    return torch.stack([a, b], dim=1).reshape(2 * f, *rest).contiguous()


def gemm(a, w, bias=None, act=ACT_NONE, glu=GLU_NONE, residual=None, alpha=1.0, rowbias=None,
         rowbias_rows=0, out=None, out_fp32=False, rowscale=None, rms_eps=0.0, kscale=None):
    """out[M, N'] = epilogue(a[M, K] @ w[N, K]^T) on wgmma tensor cores. w is bf16, or an NF4Weight (nf4.py): then
    out = epilogue(a @ diag(kscale) @ W_eff^T) with the optional fp32 column scale kscale [K], on the NF4 weight-streaming
    kernel for M <= 32 and as an NF4 -> bf16 dequantisation into a workspace followed by the bf16 GEMM above that."""
    lib = _lib.load()
    a2, lda = _rows2d(a)
    q4 = isinstance(w, NF4Weight)
    _req(a2.dtype == BF16 and (q4 or w.dtype == BF16), "gemm operands must be bf16 (or an NF4Weight)")
    _req(len(w.shape) == 2 and w.shape[1] == a2.shape[1] and (q4 or w.stride(1) == 1), "weight must be [N, K] row-major")
    _req(kscale is None or (q4 and kscale.dtype == torch.float32 and kscale.is_contiguous()
                            and kscale.numel() == a2.shape[1]), "kscale: fp32 [K], NF4 weights only")
    M, K = a2.shape
    N = w.shape[0]
    small = M <= (NF4_MAX_M if q4 else 16)      # the weight-streaming kernels compute the RMS row scale themselves
    n_out = N // 2 if glu != GLU_NONE else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.float32 if out_fp32 else BF16, device=a.device)
    else:
        _req(out.shape[-1] == n_out and out.stride(-1) == 1, "bad out shape")
        _req(out.dtype == (torch.float32 if out_fp32 else BF16), "bad out dtype")
    out2, ldo = _rows2d(out)
    epi = Epilogue()
    epi.bias = _ptr(bias)
    epi.rowbias = _ptr(rowbias)
    epi.rowbias_rows = int(rowbias_rows)
    epi.alpha = float(alpha)
    epi.act = int(act)
    epi.glu = int(glu)
    epi.out_fp32 = 1 if out_fp32 else 0
    if rowscale is not None:
        _req(rowscale.dtype == torch.float32 and rowscale.numel() == M and rowscale.is_contiguous(), "bad rowscale")
        epi.rowscale = rowscale.data_ptr()
    elif rms_eps > 0:
        if small:
            epi.rms_eps = float(rms_eps)  # computed inside the weight-streaming kernel
        else:
            rs = row_rstd(a2, rms_eps)
            epi.rowscale = rs.data_ptr()
    if residual is not None:
        r2, ldr = _rows2d(residual)
        _req(r2.dtype == BF16 and r2.shape == (M, n_out), "bad residual")
        epi.residual = r2.data_ptr()
        epi.ldr = ldr
    if bias is not None:
        _req(bias.dtype == BF16 and bias.numel() == N and bias.is_contiguous(), "bad bias")
    if M == 0:
        return out.reshape(*a.shape[:-1], n_out) if a.dim() != 2 else out
    if q4 and small:
        check(lib.vb200_gemm_nf4(a2.data_ptr(), lda, w.codes.data_ptr(), w.scales.data_ptr(), _ptr(kscale),
                                 out2.data_ptr(), ldo, M, N, K, C.byref(epi), _stream()), "vb200_gemm_nf4")
        _launches[0] += 1
        return out.reshape(*a.shape[:-1], n_out) if a.dim() != 2 else out
    if q4:
        w = nf4_dequant(w, kscale, workspace(2 * N * K, a.device, "nf4"))
    need = lib.vb200_gemm_bf16_workspace_size(M, N, K)
    ws = workspace(need, a.device) if need else None
    check(lib.vb200_gemm_bf16(a2.data_ptr(), lda, w.data_ptr(), w.stride(0), out2.data_ptr(), ldo, M, N, K,
                              C.byref(epi), _ptr(ws), need, _stream()), "vb200_gemm_bf16")
    _launches[0] += 1
    return out.reshape(*a.shape[:-1], n_out) if a.dim() != 2 else out


NF4_MAX_M = 32   # rows of A that vb200_gemm_nf4 takes; larger M dequantises into a workspace and runs the bf16 GEMM


def nf4_dequant(w, kscale=None, out=None):
    """bf16 [N, K] = bf16_rn((NF4[code] * scale) * kscale[k]) of an NF4Weight (bit-identical to nf4.dequantize).
    out: a bf16 [N, K] tensor or a uint8 workspace of at least 2 N K bytes."""
    N, K = w.shape
    if out is None:
        out = torch.empty((N, K), dtype=BF16, device=w.device)
    else:
        _req(out.is_contiguous() and out.numel() * out.element_size() >= 2 * N * K, "nf4_dequant: out too small")
        out = out.view(torch.uint8)[:2 * N * K].view(BF16).view(N, K) if out.dtype != BF16 else out.view(N, K)
    _req(kscale is None or (kscale.dtype == torch.float32 and kscale.is_contiguous() and kscale.numel() == K), "bad kscale")
    check(_lib.load().vb200_nf4_dequant(w.codes.data_ptr(), w.scales.data_ptr(), _ptr(kscale), out.data_ptr(), N, K,
                                        _stream()), "vb200_nf4_dequant")
    _launches[0] += 1
    return out


def reserve_nf4_workspace(weights, device):
    """Pre-size the dequantisation workspace for the largest of `weights` (NF4Weight), so that a CUDA graph captured at
    M > NF4_MAX_M never sees the workspace move."""
    need = max((2 * w.shape[0] * w.shape[1] for w in weights), default=0)
    return workspace(need, torch.device(device), "nf4") if need else None


def set_gemm_impl(impl):
    """0 = specialised v2 kernel whenever eligible (default), 1 = generic kernel only; returns the previous setting."""
    return _lib.load().vb200_set_gemm_impl(int(impl))


def set_gemm_debug(resident_b=-1, dbg=-1):
    """Measurement aids (see include/vitron_b200.h); returns the previous packed setting."""
    return _lib.load().vb200_set_gemm_debug(int(resident_b), int(dbg))


def pack_conv_weight(w):
    """[cout, cin, kh, kw] (torch Conv2d) or [cout, cin, kt, 1, 1] (Conv3d (k,1,1)) ->
    [cout, kh*kw, ceil64(cin)] bf16, zero padded: the K-major layout of the implicit GEMM."""
    if w.dim() == 5:
        w = w[:, :, :, 0, 0].unsqueeze(-1)  # [cout, cin, kt, 1]
    cout, cin, kh, kw = w.shape
    cpad = (cin + 63) // 64 * 64
    out = torch.zeros((cout, kh * kw, cpad), dtype=BF16, device=w.device)
    out[:, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, kh * kw, cin).to(BF16)
    return out.contiguous()


def conv_nhwc(x, wt, kh, kw, stride=1, pad_h=None, pad_w=None, bias=None, act=ACT_NONE, glu=GLU_NONE,
              residual=None, alpha=1.0, rowbias=None, rowbias_rows=0, out=None):
    """x [nb, h, w, cin] bf16 NHWC, wt from pack_conv_weight -> [nb, ho, wo, cout]."""
    lib = _lib.load()
    _req(x.dtype == BF16 and x.is_contiguous() and x.dim() == 4, "x must be contiguous NHWC bf16")
    nb, h, w, cin = x.shape
    cout = wt.shape[0]
    pad_h = kh // 2 if pad_h is None else pad_h
    pad_w = kw // 2 if pad_w is None else pad_w
    ho = (h + 2 * pad_h - kh) // stride + 1
    wo = (w + 2 * pad_w - kw) // stride + 1
    n_out = cout // 2 if glu != GLU_NONE else cout
    if out is None:
        out = torch.empty((nb, ho, wo, n_out), dtype=BF16, device=x.device)
    _req(wt.shape[1] == kh * kw and wt.shape[2] == (cin + 63) // 64 * 64, "weight not packed for this conv")
    epi = Epilogue()
    epi.bias = _ptr(bias)
    epi.rowbias = _ptr(rowbias)
    epi.rowbias_rows = int(rowbias_rows)
    epi.alpha = float(alpha)
    epi.act = int(act)
    epi.glu = int(glu)
    if residual is not None:
        _req(residual.is_contiguous() and residual.shape == out.shape, "bad residual")
        epi.residual = residual.data_ptr()
        epi.ldr = n_out
    need = lib.vb200_conv_nhwc_workspace_size(nb, h, w, cin, cout, kh, kw, stride, pad_h, pad_w)
    ws = workspace(need, x.device) if need else None
    check(lib.vb200_conv_nhwc_bf16(x.data_ptr(), wt.data_ptr(), out.data_ptr(), nb, h, w, cin, cout, kh, kw,
                                   stride, pad_h, pad_w, C.byref(epi), _ptr(ws), need, _stream()), "vb200_conv_nhwc_bf16")
    _launches[0] += 1
    return out


def conv_nhwc_direct(x, w_khwc, bias, kh, kw, stride=1, pad_h=None, pad_w=None):
    """Tiny layers only. w_khwc: [cout, kh*kw, cin] bf16 (unpadded)."""
    lib = _lib.load()
    nb, h, w, cin = x.shape
    cout = w_khwc.shape[0]
    pad_h = kh // 2 if pad_h is None else pad_h
    pad_w = kw // 2 if pad_w is None else pad_w
    ho = (h + 2 * pad_h - kh) // stride + 1
    wo = (w + 2 * pad_w - kw) // stride + 1
    out = torch.empty((nb, ho, wo, cout), dtype=BF16, device=x.device)
    check(lib.vb200_conv_nhwc_direct(x.data_ptr(), w_khwc.data_ptr(), _ptr(bias), out.data_ptr(), nb, h, w, cin,
                                     cout, kh, kw, stride, pad_h, pad_w, _stream()), "vb200_conv_nhwc_direct")
    _launches[0] += 1
    return out


def rmsnorm(x, weight, eps, out=None):
    lib = _lib.load()
    x2, ldx = _rows2d(x)
    out = torch.empty_like(x) if out is None else out
    o2, ldo = _rows2d(out)
    check(lib.vb200_rmsnorm(x2.data_ptr(), ldx, weight.data_ptr(), o2.data_ptr(), ldo, x2.shape[0], x2.shape[1],
                            float(eps), _stream()), "vb200_rmsnorm")
    _launches[0] += 1
    return out


def layernorm(x, weight, bias, eps, out=None):
    lib = _lib.load()
    x2, ldx = _rows2d(x)
    if out is None:
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
    o2, ldo = _rows2d(out)
    check(lib.vb200_layernorm(x2.data_ptr(), ldx, weight.data_ptr(), _ptr(bias), o2.data_ptr(), ldo, x2.shape[0],
                              x2.shape[1], float(eps), _stream()), "vb200_layernorm")
    _launches[0] += 1
    return out


def groupnorm_nhwc(x, weight, bias, groups, eps, act=ACT_NONE, n=None, out=None):
    """x [..., c] viewed as [n, spatial, c]; statistics over (spatial, c/groups) per n."""
    lib = _lib.load()
    _req(x.is_contiguous() and x.dtype == BF16, "x must be contiguous bf16")
    c = x.shape[-1]
    n = x.shape[0] if n is None else n
    spatial = x.numel() // (n * c)
    out = torch.empty_like(x) if out is None else out
    need = lib.vb200_groupnorm_workspace_size(n, groups, c)
    ws = workspace(need, x.device, "gn")
    check(lib.vb200_groupnorm_nhwc(x.data_ptr(), weight.data_ptr(), bias.data_ptr(), out.data_ptr(), n, spatial, c,
                                   groups, float(eps), int(act), ws.data_ptr(), need, _stream()),
          "vb200_groupnorm_nhwc")
    _launches[0] += 1
    return out


def _bsh(t):
    """(batch, seq, head) element strides of a [B, S, H, D] view."""
    _req(t.dim() == 4 and t.stride(3) == 1, "expect [B, S, H, D] with contiguous D")
    return t.stride(0), t.stride(1), t.stride(2)


def attention(q, k, v, scale=None, causal=False, kv_len=None, mask=None, out=None):
    """q [B, Sq, H, D], k/v [B, Skv, H, D] (any strides with contiguous D) -> [B, Sq, H, D].
    mask: bool/uint8 [B or 1, H or 1, Sq, Skv], True = masked out."""
    lib = _lib.load()
    B, Sq, H, D = q.shape
    Skv = k.shape[1]
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    if out is None:
        out = torch.empty((B, Sq, H, D), dtype=BF16, device=q.device)
    m_ptr, m_sb, m_sh, m_sq = 0, 0, 0, 0
    if mask is not None:
        if mask.dtype == torch.bool:
            mask = mask.view(torch.uint8)
        _req(mask.dim() == 4 and mask.stride(3) == 1 and mask.shape[2] == Sq and mask.shape[3] == Skv, "bad mask")
        m_ptr = mask.data_ptr()
        m_sb = mask.stride(0) if mask.shape[0] > 1 else 0
        m_sh = mask.stride(1) if mask.shape[1] > 1 else 0
        m_sq = mask.stride(2)
    need = lib.vb200_attention_workspace_size(B, H, Sq, Skv, D, 1 if causal else 0) if kv_len is None else 0
    ws = workspace(need, q.device, "attn") if need else None
    check(lib.vb200_attention_ws(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, Sq, Skv, D,
                                 *_bsh(q), *_bsh(k), *_bsh(v), *_bsh(out), float(scale), 1 if causal else 0,
                                 _ptr(kv_len), m_ptr, m_sb, m_sh, m_sq, _ptr(ws), need, _stream()), "vb200_attention_ws")
    _launches[0] += 2 if need else 1
    return out


def attention_paged(q, k_pages, v_pages, block_table, q_start, q_len, max_kv_len, scale=None, out=None):
    """A chunk of queries over the paged KV cache (vb200_attention_paged): q [B, Sq, H, 128] strided view with RoPE
    applied, k_pages / v_pages [num_pages, H, 64, 128], block_table int32 [B, max_pages] (contiguous), q_start /
    q_len int32 [B] on the device (keys cached before the chunk, valid queries), max_kv_len >= q_start + q_len on the host.
    -> [B, Sq, H, 128]; query i of row b sees keys j <= q_start[b] + i, rows i >= q_len[b] are zeros."""
    lib = _lib.load()
    B, Sq, H, D = q.shape
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    _req(block_table.dim() == 2 and block_table.shape[0] >= B and block_table.is_contiguous(),
         "block_table: contiguous int32 [>= B, max_pages]")
    _req(k_pages.is_contiguous() and v_pages.is_contiguous() and k_pages.shape == v_pages.shape, "contiguous pages")
    if out is None:
        out = torch.empty((B, Sq, H, D), dtype=BF16, device=q.device)
    need = lib.vb200_attention_paged_workspace_size(B, H, Sq, D, int(max_kv_len))
    ws = workspace(need, q.device, "attn") if need else None
    check(lib.vb200_attention_paged(q.data_ptr(), *_bsh(q), k_pages.data_ptr(), v_pages.data_ptr(), k_pages.shape[0],
                                    block_table.data_ptr(), block_table.shape[1], q_start.data_ptr(), q_len.data_ptr(),
                                    out.data_ptr(), *_bsh(out), B, H, Sq, D, k_pages.shape[2], int(max_kv_len),
                                    float(scale), _ptr(ws), need, _stream()), "vb200_attention_paged")
    _launches[0] += 2 if need else 1
    return out


def set_attention_impl(impl):
    """0 = automatic, 1 = mma.sync kernel only, 2 = wgmma kernel whenever the shape is supported."""
    check(_lib.load().vb200_set_attention_impl(int(impl)), "vb200_set_attention_impl")


def attention_watchdog():
    """(site, block, thread) of the first expired wait in the wgmma attention kernel since the last call;
    site 0 = none. Synchronises."""
    import ctypes
    buf = (ctypes.c_uint32 * 3)()
    torch.cuda.synchronize()
    check(_lib.load().vb200_attention_watchdog(ctypes.addressof(buf)), "vb200_attention_watchdog")
    return tuple(buf)


def attention_short(q, k, v, scale=None, out=None):
    """q/k/v [nseq, S, H, 64] or [outer, inner, S, H, 64] strided views (sequence = leading dims),
    S <= 32. out defaults to a fresh tensor of q's shape."""
    lib = _lib.load()
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    if out is None:
        out = torch.empty(q.shape, dtype=BF16, device=q.device)
    if q.dim() == 4:
        nseq, S, H, D = q.shape
        inner, so = 0, (0, 0, 0, 0)
        b3 = [_bsh(t) for t in (q, k, v, out)]
    else:
        _req(q.dim() == 5, "expect 4-D or 5-D q")
        outer, inner, S, H, D = q.shape
        nseq = outer * inner
        so = tuple(t.stride(0) for t in (q, k, v, out))
        for t in (q, k, v, out):
            _req(t.stride(4) == 1, "contiguous head dim")
        b3 = [(t.stride(1), t.stride(2), t.stride(3)) for t in (q, k, v, out)]
    check(lib.vb200_attention_short(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), nseq, H, S, D,
                                    *b3[0], *b3[1], *b3[2], *b3[3], inner, *so, float(scale), _stream()),
          "vb200_attention_short")
    _launches[0] += 1
    return out


def add_rowgroup(x, table, group_rows, period, out=None):
    """x [rows, d] + table[(row // group_rows) % period]."""
    lib = _lib.load()
    x2, _ = _rows2d(x)
    _req(x.is_contiguous() and table.is_contiguous(), "contiguous")
    out = torch.empty_like(x) if out is None else out
    check(lib.vb200_add_rowgroup(x2.data_ptr(), table.data_ptr(), out.data_ptr(), x2.shape[0], x2.shape[1],
                                 group_rows, period, _stream()), "vb200_add_rowgroup")
    _launches[0] += 1
    return out


def rope_kv_append(qkv, positions, n_heads, head_dim, theta, k_pages=None, v_pages=None, block_table=None,
                   batch_of_token=None, slot_of_token=None, page_size=0):
    lib = _lib.load()
    q2, ld = _rows2d(qkv)
    max_pages = block_table.shape[1] if block_table is not None else 0
    check(lib.vb200_rope_kv_append(q2.data_ptr(), ld, positions.data_ptr(), _ptr(batch_of_token),
                                   _ptr(slot_of_token), _ptr(k_pages), _ptr(v_pages), _ptr(block_table),
                                   max_pages, q2.shape[0], n_heads, head_dim, page_size, float(theta), _stream()),
          "vb200_rope_kv_append")
    _launches[0] += 1
    return qkv


def attn_decode_paged(q, k_pages, v_pages, block_table, kv_len, n_heads, head_dim, page_size, max_kv_len,
                      scale=None, out=None):
    """q [B, >= n_heads*head_dim] rows (e.g. the fused qkv buffer) -> out [B, n_heads*head_dim]."""
    lib = _lib.load()
    B = q.shape[0]
    scale = 1.0 / math.sqrt(head_dim) if scale is None else scale
    if out is None:
        out = torch.empty((B, n_heads * head_dim), dtype=BF16, device=q.device)
    need = lib.vb200_attn_decode_workspace_size(B, n_heads, head_dim, 32)
    ws = workspace(need, q.device, "dec")
    check(lib.vb200_attn_decode_paged(q.data_ptr(), q.stride(0), k_pages.data_ptr(), v_pages.data_ptr(),
                                      block_table.data_ptr(), block_table.shape[1], kv_len.data_ptr(),
                                      out.data_ptr(), out.stride(0), B, n_heads, head_dim, page_size, max_kv_len,
                                      float(scale), ws.data_ptr(), need, _stream()), "vb200_attn_decode_paged")
    _launches[0] += 1
    return out


def rope_table(positions, head_dim, theta, out=None):
    """fp32 [B, head_dim]: cos | sin of every sequence's current position (once per decode step)."""
    lib = _lib.load()
    B = positions.shape[0]
    if out is None:
        out = torch.empty((B, head_dim), dtype=torch.float32, device=positions.device)
    check(lib.vb200_rope_table(positions.data_ptr(), out.data_ptr(), B, head_dim, float(theta), _stream()),
          "vb200_rope_table")
    _launches[0] += 1
    return out


def attn_decode_rope(qkv, table, k_pages, v_pages, block_table, kv_len, n_heads, head_dim, page_size, max_kv_len,
                     scale=None, out=None):
    """Decode attention with RoPE + KV append fused in (qkv rows hold the un-rotated q|k|v of the new token;
    table = rope_table(positions))."""
    lib = _lib.load()
    B = qkv.shape[0]
    scale = 1.0 / math.sqrt(head_dim) if scale is None else scale
    if out is None:
        out = torch.empty((B, n_heads * head_dim), dtype=BF16, device=qkv.device)
    need = lib.vb200_attn_decode_workspace_size(B, n_heads, head_dim, 32)
    ws = workspace(need, qkv.device, "dec")
    check(lib.vb200_attn_decode_rope(qkv.data_ptr(), qkv.stride(0), table.data_ptr(), k_pages.data_ptr(),
                                     v_pages.data_ptr(), block_table.data_ptr(), block_table.shape[1],
                                     kv_len.data_ptr(), out.data_ptr(), out.stride(0), B, n_heads, head_dim, page_size,
                                     max_kv_len, float(scale), ws.data_ptr(), need, _stream()),
          "vb200_attn_decode_rope")
    _launches[0] += 1
    return out


def attn_decode_rope_beam(qkv, table, k_pages, v_pages, block_table, kv_len, beam_src, gen_start, n_heads, head_dim,
                          page_size, max_kv_len, scale=None, out=None):
    """attn_decode_rope for beam rows: key j >= gen_start[b] of row b is read from the pages of row beam_src[b, j]
    (int32 [B, >= max_kv_len], rows index block_table); the new token's K / V still go to row b's own pages."""
    lib = _lib.load()
    B = qkv.shape[0]
    _req(beam_src.dtype == torch.int32 and beam_src.dim() == 2 and beam_src.stride(1) == 1 and beam_src.shape[0] >= B
         and gen_start.dtype == torch.int32 and gen_start.numel() >= B, "beam_src int32 [B, S], gen_start int32 [B]")
    _req(beam_src.shape[1] >= max_kv_len, "beam_src must cover max_kv_len positions")
    scale = 1.0 / math.sqrt(head_dim) if scale is None else scale
    if out is None:
        out = torch.empty((B, n_heads * head_dim), dtype=BF16, device=qkv.device)
    need = lib.vb200_attn_decode_workspace_size(B, n_heads, head_dim, 32)
    ws = workspace(need, qkv.device, "dec")
    check(lib.vb200_attn_decode_rope_beam(qkv.data_ptr(), qkv.stride(0), table.data_ptr(), k_pages.data_ptr(),
                                          v_pages.data_ptr(), block_table.data_ptr(), block_table.shape[1],
                                          kv_len.data_ptr(), beam_src.data_ptr(), beam_src.stride(0),
                                          gen_start.data_ptr(), out.data_ptr(), out.stride(0), B, n_heads, head_dim,
                                          page_size, max_kv_len, float(scale), ws.data_ptr(), need, _stream()),
          "vb200_attn_decode_rope_beam")
    _launches[0] += 1
    return out


def row_rstd(x, eps):
    """fp32 [rows] = rsqrt(mean(x_row^2) + eps)."""
    lib = _lib.load()
    x2, ldx = _rows2d(x)
    out = torch.empty((x2.shape[0],), dtype=torch.float32, device=x.device)
    check(lib.vb200_row_rstd(x2.data_ptr(), ldx, out.data_ptr(), x2.shape[0], x2.shape[1], float(eps), _stream()),
          "vb200_row_rstd")
    _launches[0] += 1
    return out


def splice_multimodal(embed, feats, srcmap, out=None):
    lib = _lib.load()
    rows = srcmap.numel()
    d = embed.shape[1]
    if out is None:
        out = torch.empty((*srcmap.shape, d), dtype=BF16, device=embed.device)
    nfeat = 0 if feats is None else feats.shape[0]
    check(lib.vb200_splice_multimodal(embed.data_ptr(), embed.shape[0], _ptr(feats), nfeat, srcmap.data_ptr(),
                                      out.data_ptr(), rows, d, _stream()), "vb200_splice_multimodal")
    _launches[0] += 1
    return out


def argmax_rows(logits, out=None):
    lib = _lib.load()
    l2, ld = _rows2d(logits)
    if out is None:
        out = torch.empty((l2.shape[0],), dtype=torch.int64, device=logits.device)
    check(lib.vb200_argmax_rows(l2.data_ptr(), 1 if l2.dtype == torch.float32 else 0, ld, l2.shape[0], l2.shape[1],
                                out.data_ptr(), _stream()), "vb200_argmax_rows")
    _launches[0] += 1
    return out


def argmax_advance(logits, out_idx, next_src=None, positions=None, kv_len=None, token_log=None, prompt_len=None):
    lib = _lib.load()
    _req(logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1, "fp32 logits [B, V]")
    check(lib.vb200_argmax_advance(logits.data_ptr(), logits.stride(0), logits.shape[0], logits.shape[1],
                                   out_idx.data_ptr(), _ptr(next_src), _ptr(positions), _ptr(kv_len),
                                   _ptr(token_log), token_log.shape[1] if token_log is not None else 0,
                                   _ptr(prompt_len), _stream()), "vb200_argmax_advance")
    _launches[0] += 1
    return out_idx


SAMPLE_PARAMS = struct.Struct("<fifIQ")   # vb_sample_params: temperature, top_k, top_p, reserved, seed


def sample_params(temperature, top_k, top_p, seed):
    """vb_sample_params packed into a CPU uint8 tensor (copy it into the device buffer vb200_sample_advance reads).
    top_k 0 = off, top_p >= 1 = off; the temperature is used as given."""
    raw = SAMPLE_PARAMS.pack(float(temperature), int(top_k), float(top_p), 0, int(seed) & (2 ** 64 - 1))
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8)


def sample_advance(logits, params, out_idx=None, next_src=None, positions=None, kv_len=None, token_log=None,
                   prompt_len=None):
    """Sampled sibling of argmax_advance: temperature, top-k, top-p and a Philox draw per row (contract in
    include/vitron_b200.h), parameters read from the device buffer `params` (sample_params). Without kv_len /
    prompt_len the draw is step 0 and no state advances (the token of the prefill logits)."""
    lib = _lib.load()
    _req(logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1, "fp32 logits [B, V]")
    _req(params.dtype == torch.uint8 and params.numel() == SAMPLE_PARAMS.size and params.is_contiguous()
         and params.device == logits.device, "params: uint8 [24] sampling buffer on the logits' device")
    if out_idx is None:
        out_idx = torch.empty((logits.shape[0],), dtype=torch.int64, device=logits.device)
    check(lib.vb200_sample_advance(logits.data_ptr(), logits.stride(0), logits.shape[0], logits.shape[1],
                                   params.data_ptr(), out_idx.data_ptr(), _ptr(next_src), _ptr(positions), _ptr(kv_len),
                                   _ptr(token_log), token_log.shape[1] if token_log is not None else 0,
                                   _ptr(prompt_len), _stream()), "vb200_sample_advance")
    _launches[0] += 1
    return out_idx


def reserve_beam_workspace(rows, device):
    """Pre-size the beam-step workspace for the most rows an engine will run (its address is baked into decode graphs)."""
    return workspace(_lib.load().vb200_beam_workspace_size(rows), torch.device(device), "beam")


def _beam_args(logits, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count, hyp_ids,
               next_src, positions, kv_len, token_log, prompt_len):
    """Checks of the beam-step buffers; returns the leading C arguments and the workspace of vb200_beam_(sample_)advance."""
    lib = _lib.load()
    _req(logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1, "fp32 logits [B * k, V]")
    R = logits.shape[0]
    _req(k > 0 and R % k == 0, f"{R} rows are not a multiple of k = {k}")
    _req(params.dtype == torch.uint8 and params.is_contiguous() and params.device == logits.device,
         "params: uint8 beam parameter buffer on the logits' device")
    _req(params.numel() == beam.PARAMS.size, f"params: {beam.PARAMS.size}-byte vb_beam_params buffer")
    dev = logits.device
    for name, t, dt in (("beam_src", beam_src, torch.int32), ("hyp_ids", hyp_ids, torch.int64),
                        ("token_log", token_log, torch.int64)):
        _req(t.dtype == dt and t.dim() == 2 and t.stride(1) == 1 and t.shape[0] >= R and t.device == dev,
             f"{name}: {dt} [>= {R}, S] with unit inner stride on the logits' device")
    for name, t, dt in (("beam_score", beam_score, torch.float32), ("hyp_score", hyp_score, torch.float64),
                        ("parent", parent, torch.int32), ("done", done, torch.int32), ("hyp_len", hyp_len, torch.int32),
                        ("hyp_seq", hyp_seq, torch.int32), ("hyp_count", hyp_count, torch.int32),
                        ("next_src", next_src, torch.int32), ("positions", positions, torch.int32),
                        ("kv_len", kv_len, torch.int32), ("prompt_len", prompt_len, torch.int32)):
        _req(t.dtype == dt and t.dim() == 1 and t.is_contiguous() and t.numel() >= R and t.device == dev,
             f"{name}: contiguous {dt} [>= {R}] on the logits' device")
    need = lib.vb200_beam_workspace_size(R)
    ws = workspace(need, logits.device, "beam")
    return (logits.data_ptr(), logits.stride(0), R // k, k, logits.shape[1], params.data_ptr(), beam_score.data_ptr(),
            parent.data_ptr(), done.data_ptr(), beam_src.data_ptr(), beam_src.stride(0), hyp_score.data_ptr(),
            hyp_len.data_ptr(), hyp_seq.data_ptr(), hyp_count.data_ptr(), hyp_ids.data_ptr(), hyp_ids.stride(0),
            next_src.data_ptr(), positions.data_ptr(), kv_len.data_ptr(), token_log.data_ptr(), token_log.stride(0),
            prompt_len.data_ptr(), ws.data_ptr(), need)


def beam_advance(logits, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count, hyp_ids,
                 next_src, positions, kv_len, token_log, prompt_len):
    """One beam-search step for B = rows / k requests (contract in include/vitron_b200.h, statement in
    vitron_b200.beam): parameters from the device buffer `params` (beam.pack_params), state updated in place."""
    args = _beam_args(logits, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count,
                      hyp_ids, next_src, positions, kv_len, token_log, prompt_len)
    check(_lib.load().vb200_beam_advance(*args, _stream()), "vb200_beam_advance")
    _launches[0] += 1


def beam_sample_advance(logits, k, params, sample_params, beam_score, parent, done, beam_src, hyp_score, hyp_len,
                        hyp_seq, hyp_count, hyp_ids, next_src, positions, kv_len, token_log, prompt_len):
    """One beam-sampling step (HF 4.31 beam_sample) for B = rows / k searches: beam_advance's arguments plus the device
    buffer `sample_params` (sample_params: temperature, top_k, top_p, seed). Contract in include/vitron_b200.h,
    statement in vitron_b200.beam.beam_sample_advance."""
    _req(sample_params.dtype == torch.uint8 and sample_params.numel() == SAMPLE_PARAMS.size
         and sample_params.is_contiguous() and sample_params.device == logits.device,
         f"sample_params: uint8 [{SAMPLE_PARAMS.size}] sampling buffer on the logits' device")
    args = _beam_args(logits, k, params, beam_score, parent, done, beam_src, hyp_score, hyp_len, hyp_seq, hyp_count,
                      hyp_ids, next_src, positions, kv_len, token_log, prompt_len)
    check(_lib.load().vb200_beam_sample_advance(*args, sample_params.data_ptr(), _stream()), "vb200_beam_sample_advance")
    _launches[0] += 1


def patchify(pixels, patch, kpad):
    lib = _lib.load()
    _req(pixels.is_contiguous() and pixels.dim() == 4, "pixels must be contiguous NCHW")
    _req(pixels.dtype in (torch.float32, BF16), "pixels must be fp32 or bf16")
    nb, c, h, w = pixels.shape
    out = torch.empty((nb * (h // patch) * (w // patch), kpad), dtype=BF16, device=pixels.device)
    check(lib.vb200_patchify(pixels.data_ptr(), 1 if pixels.dtype == torch.float32 else 0, out.data_ptr(), nb, c, h,
                             w, patch, kpad, _stream()), "vb200_patchify")
    _launches[0] += 1
    return out


def vit_embed_ln(patch_out, cls, pos, ln_w, ln_b, nb, npatch, eps):
    lib = _lib.load()
    d = patch_out.shape[-1]
    out = torch.empty((nb, npatch + 1, d), dtype=BF16, device=patch_out.device)
    check(lib.vb200_vit_embed_ln(patch_out.data_ptr(), cls.data_ptr(), pos.data_ptr(), ln_w.data_ptr(),
                                 ln_b.data_ptr(), out.data_ptr(), nb, npatch, d, float(eps), _stream()),
          "vb200_vit_embed_ln")
    _launches[0] += 1
    return out


def upsample2x_nhwc(x):
    lib = _lib.load()
    nb, h, w, c = x.shape
    out = torch.empty((nb, 2 * h, 2 * w, c), dtype=BF16, device=x.device)
    check(lib.vb200_upsample2x_nhwc(x.data_ptr(), out.data_ptr(), nb, h, w, c, _stream()), "vb200_upsample2x_nhwc")
    _launches[0] += 1
    return out


def add(a, b, out=None):
    """a + b (bf16); b may be a broadcast operand whose numel divides a's (period)."""
    lib = _lib.load()
    _req(a.is_contiguous() and b.is_contiguous(), "add operands must be contiguous")
    out = torch.empty_like(a) if out is None else out
    period = 0 if b.numel() == a.numel() else b.numel()
    check(lib.vb200_add_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), period, _stream()),
          "vb200_add_bf16")
    _launches[0] += 1
    return out


def cfg_combine(y, u, scale):
    lib = _lib.load()
    _req(y.dtype == torch.float32 and u.dtype == torch.float32 and y.is_contiguous() and u.is_contiguous(), "fp32")
    out = torch.empty_like(y)
    check(lib.vb200_cfg_combine(y.data_ptr(), u.data_ptr(), out.data_ptr(), float(scale), y.numel(), _stream()),
          "vb200_cfg_combine")
    _launches[0] += 1
    return out


def region_mask_pool(feats, boxes, image_size):
    """feats [B, g*g, C] bf16, boxes fp32 [B, 4] -> [B, C]."""
    lib = _lib.load()
    B, n, c = feats.shape
    g = int(math.isqrt(n))
    out = torch.empty((B, c), dtype=BF16, device=feats.device)
    check(lib.vb200_region_mask_pool(feats.data_ptr(), boxes.data_ptr(), out.data_ptr(), B, g, c, image_size,
                                     _stream()), "vb200_region_mask_pool")
    _launches[0] += 1
    return out


def seem_attn_mask(mask_logits, h2, w2):
    """mask_logits fp32 [Q, H, W] -> uint8 [Q, h2*w2], 1 = masked out."""
    lib = _lib.load()
    Q, H, W = mask_logits.shape
    out = torch.empty((Q, h2 * w2), dtype=torch.uint8, device=mask_logits.device)
    check(lib.vb200_seem_attn_mask(mask_logits.data_ptr(), out.data_ptr(), Q, H, W, h2, w2, _stream()),
          "vb200_seem_attn_mask")
    _launches[0] += 1
    return out


def resize_bilinear_nhwc(x, h2, w2):
    """bf16 NHWC [nb, H, W, C] -> [nb, h2, w2, C], F.interpolate(bilinear, align_corners=False) semantics."""
    lib = _lib.load()
    _req(x.dim() == 4 and x.is_contiguous() and x.dtype == BF16 and x.shape[-1] % 8 == 0, "x: contiguous NHWC bf16, C % 8 == 0")
    nb, H, W, C = x.shape
    out = torch.empty((nb, h2, w2, C), dtype=BF16, device=x.device)
    check(lib.vb200_resize_bilinear_nhwc(x.data_ptr(), out.data_ptr(), nb, H, W, C, int(h2), int(w2), _stream()),
          "vb200_resize_bilinear_nhwc")
    _launches[0] += 1
    return out


# ---- FocalNet backbone glue (focal.cu) ---------------------------------------------------------

def im2col_nchw(pixels, k, stride, pad, ho, wo, kpad):
    """NCHW fp32/bf16 pixels -> [nb*ho*wo, kpad] bf16 rows ordered (c, ky, kx); zero outside the image."""
    lib = _lib.load()
    _req(pixels.is_contiguous() and pixels.dim() == 4 and pixels.dtype in (torch.float32, BF16), "pixels: contiguous NCHW fp32/bf16")
    nb, c, h, w = pixels.shape
    out = torch.empty((nb * ho * wo, kpad), dtype=BF16, device=pixels.device)
    check(lib.vb200_im2col_nchw(pixels.data_ptr(), 1 if pixels.dtype == torch.float32 else 0, out.data_ptr(), nb, c, h, w,
                                k, stride, pad, ho, wo, kpad, _stream()), "vb200_im2col_nchw")
    _launches[0] += 1
    return out


def pack_dwconv_weight(w):
    """[c, 1, k, k] (torch depthwise Conv2d) -> [k*k, c] bf16 tap-major."""
    c, one, kh, kw = w.shape
    _req(one == 1 and kh == kw, "depthwise square kernel expected")
    return w.reshape(c, kh * kw).t().to(BF16).contiguous()


def set_dwconv_impl(impl):
    """0 = automatic (default), 1 = 8-channel kernel, 2 / 3 = channel-pair kernel with 16 / 32-pixel strips."""
    return _lib.load().vb200_set_dwconv_impl(int(impl))


def dwconv_nhwc(x, wt, k, act=ACT_NONE):
    """x: [nb, h, w, c] bf16, either contiguous or a channel slice of a contiguous [nb, h, w, ld] tensor."""
    lib = _lib.load()
    nb, h, w, c = x.shape
    ld = x.stride(2)
    _req(x.dtype == BF16 and x.stride(3) == 1 and x.stride(1) == w * ld and x.stride(0) == h * w * ld, "x must be a channel slice of an NHWC tensor")
    _req(wt.shape == (k * k, c) and wt.is_contiguous() and wt.dtype == BF16, "weight must be [k*k, c] bf16")
    out = torch.empty((nb, h, w, c), dtype=BF16, device=x.device)
    check(lib.vb200_dwconv_nhwc(x.data_ptr(), ld, wt.data_ptr(), out.data_ptr(), nb, h, w, c, k, int(act), _stream()),
          "vb200_dwconv_nhwc")
    _launches[0] += 1
    return out


def colmean(x, nb, act=ACT_NONE):
    """x [nb*t, c] (or [nb, ..., c]) contiguous bf16 -> fp32 [nb, c] = act(mean over the t rows of each batch)."""
    lib = _lib.load()
    _req(x.is_contiguous() and x.dtype == BF16, "x must be contiguous bf16")
    c = x.shape[-1]
    t = x.numel() // (nb * c)
    out = torch.empty((nb, c), dtype=torch.float32, device=x.device)
    need = lib.vb200_colmean_workspace_size(nb, t, c)
    ws = workspace(need, x.device, "colmean")
    check(lib.vb200_colmean(x.data_ptr(), out.data_ptr(), nb, t, c, int(act), ws.data_ptr(), need, _stream()), "vb200_colmean")
    _launches[0] += 2
    return out


def focal_modulate(levels, gates, glob, nb, scale):
    """levels: list of contiguous [nb*t, c] bf16; gates: bf16 column slice [nb*t, >= len(levels)+1]; glob fp32 [nb, c]."""
    lib = _lib.load()
    c = levels[0].shape[-1]
    t = levels[0].numel() // (nb * c)
    for l in levels:
        _req(l.is_contiguous() and l.dtype == BF16 and l.numel() == nb * t * c, "bad ctx level")
    _req(gates.dtype == BF16 and gates.stride(-1) == 1 and gates.shape[-1] >= len(levels) + 1, "bad gates")
    _req(glob.dtype == torch.float32 and glob.is_contiguous() and glob.shape == (nb, c), "bad glob")
    g2 = gates.reshape(-1, gates.shape[-1]) if gates.dim() != 2 else gates
    ptrs = (C.c_void_p * len(levels))(*[l.data_ptr() for l in levels])
    out = torch.empty((nb * t, c), dtype=BF16, device=glob.device)
    check(lib.vb200_focal_modulate(ptrs, len(levels), g2.data_ptr(), g2.stride(0), glob.data_ptr(), out.data_ptr(), nb, t, c,
                                   float(scale), _stream()), "vb200_focal_modulate")
    _launches[0] += 1
    return out


def mul_rows(a, b):
    """a [rows, c] (row-strided view), b [rows, c] -> a * b, contiguous bf16."""
    lib = _lib.load()
    _req(a.dim() == 2 and b.dim() == 2 and a.shape == b.shape and a.stride(1) == 1 and b.stride(1) == 1, "2-D operands")
    out = torch.empty(a.shape, dtype=BF16, device=a.device)
    check(lib.vb200_mul_rows(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), a.shape[0], a.shape[1],
                             _stream()), "vb200_mul_rows")
    _launches[0] += 1
    return out


def layernorm_add(x, weight, bias, residual, eps, out=None):
    """residual + LayerNorm(x) * weight + bias (residual / bias may be None); out may alias residual."""
    lib = _lib.load()
    x2, ldx = _rows2d(x)
    if out is None:
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
    o2, ldo = _rows2d(out)
    r_ptr, ldr = 0, 0
    if residual is not None:
        r2, ldr = _rows2d(residual)
        _req(r2.shape == x2.shape and r2.dtype == BF16, "bad residual")
        r_ptr = r2.data_ptr()
    check(lib.vb200_layernorm_add(x2.data_ptr(), ldx, weight.data_ptr(), _ptr(bias), r_ptr, ldr, o2.data_ptr(), ldo,
                                  x2.shape[0], x2.shape[1], float(eps), _stream()), "vb200_layernorm_add")
    _launches[0] += 1
    return out


def softmax_rows(x, out=None):
    """fp32 [rows, n] -> bf16 softmax over the last dim."""
    lib = _lib.load()
    _req(x.dim() == 2 and x.dtype == torch.float32 and x.stride(1) == 1, "x must be fp32 [rows, n]")
    if out is None:
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
    check(lib.vb200_softmax_rows(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), x.shape[0], x.shape[1], _stream()),
          "vb200_softmax_rows")
    _launches[0] += 1
    return out


def preprocess_frames(frames, rh, rw, top, left, oh, ow, mean, std, mode, flip=False, layout="image", dtype=torch.float32):
    """frames uint8 [n, h, w, 3] (device) -> normalised [n, 3, oh, ow] (layout "image") or [3, n, oh, ow] ("video")."""
    lib = _lib.load()
    _req(frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3 and frames.is_contiguous(), "uint8 [n,h,w,3]")
    _req(dtype in (torch.float32, BF16), "fp32 or bf16 output")
    n, h, w, _ = frames.shape
    if layout == "image":
        out = torch.empty((n, 3, oh, ow), dtype=dtype, device=frames.device)
        dn, dc = 3 * oh * ow, oh * ow
    else:
        out = torch.empty((3, n, oh, ow), dtype=dtype, device=frames.device)
        dn, dc = oh * ow, n * oh * ow
    m3 = (C.c_float * 3)(*[float(v) for v in mean])
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    check(lib.vb200_preprocess_frames(frames.data_ptr(), out.data_ptr(), n, h, w, rh, rw, top, left, oh, ow, dn, dc, m3, s3,
                                      int(mode), 1 if flip else 0, 1 if dtype == BF16 else 0, _stream()), "vb200_preprocess_frames")
    _launches[0] += 1
    return out
