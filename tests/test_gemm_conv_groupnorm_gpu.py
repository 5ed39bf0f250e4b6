"""GPU: the wgmma GEMM above 64 rows, the implicit-GEMM convolution and the NHWC GroupNorm against float64 references, on
the branches the prefill, ViT, UNet, GLIGEN, SEEM and VAE paths take:
- `ops.gemm` (`gemm_v2_kernel<BN, STAGES, F, RESB>`): every tile width with every specialised epilogue and the run-time
  (F_ALL / F_ALL_GLU) variants, resident B, split-K with `splitk_reduce_kernel`, the no-workspace fallback, at ragged
  shapes and at the model calls, writing into strided views of NaN-filled buffers;
- `ops.conv_nhwc` (the same kernel with a 4-D TMA A operand) at the model convolutions and at the tiling edges, plus
  `ops.conv_nhwc_direct`;
- `ops.groupnorm_nhwc` (`gn_onepass_kernel<ACT, CACHED>`) on every launch plan, with group means far from zero;
- Python statements of the host planners (plan_tiles, resb_tile, use_swap, swap_splits, conv_pixel_tile, gn_plan),
  checked against the library's workspace sizes and, in a profiler trace, against the kernel instantiations launched.

References. GEMM and convolution: float64 over the exact bf16 operands, S = sum_k |a_k w_k| (for a convolution over the
in-bounds taps), and the epilogue in float64 in the kernel's order (gemm_v2.cuh epilogue, epi_store2, reduce_item):
rowscale, then bias and rowbias, then the activation or the GLU, then residual + alpha * v; GELU is exact erf.
GroupNorm: float64 statistics over the bf16 input (biased variance), then the affine and the activation.

GEMM / convolution bound. The products of bf16 operands are exact in fp32. wgmma adds the products of each k16 step to the
fp32 accumulator; we assume (NVIDIA documents no more) that each such step, group sum and addition together, is off by at
most one fp32 ulp of the running partial sum, and the partial is at most S in magnitude. Truncation instead of rounding is
allowed for, so the ulp is 2^-23 relative rather than 2^-24. Over K_eff / 16 steps this gives
    |acc - sum| <= tau * S,   tau = (ceil(K_eff / 16) + 8) * 2^-23,
where K_eff counts the k-blocks the kernel runs (a convolution's kh * kw * ceil64(cin)), and the 8 spare ulps cover the
split-K reduce (<= 8 fp32 additions of partials in split order) and the rowscale product. Propagated through the epilogue:
    |out - ref| <= 2 * 2^-9 * |ref| + |alpha| * E + 2^-20 * |alpha| * P + 1e-6,
    E = L * tau * S * |rs| after an activation (L = 1.13 bounds |act'| for GELU, quick-GELU, SiLU and ReLU), tau S |rs>
        without one; SwiGLU: |b| L tau S_a |rs| + |silu(a)| tau S_b |rs|; GEGLU (a * gelu(b)): |gelu(b)| tau S_a |rs| +
        |a| L tau S_b |rs|;
    P = (1 + |v|) for an activation, (1 + |a|)(1 + |b|) for a GLU: the fp32 bias additions, the __expf / erf
        approximations (gelu_erf_fast is within 1.5e-7 in erf) and the fp32 residual update;
    2 * 2^-9 |ref| is the bf16 rounding of the output (one half-ulp is 2^-9 relative; the factor 2 leaves room for ref
        landing on a rounding boundary); an fp32 output drops it.
Dropping one k-element, one tap or one row breaks this bound: at K = 4096 with 0.02-scaled weights tau S is ~1.6e-3
against |a_k w_k| ~ 1e-2.

GroupNorm bound. The kernel sums x and x^2, and x - K and (x - K)^2 around a pivot K per (sample, group), in fp32, in
chains of at most ~2^8 additions per thread before the fixed-order tree, so the relative error of each mean of these is at
most ~2^-16, and that of var is at most 2^-16 (1 + (mu - K)^2 / var). It takes the plain sums (K = 0) when |mu| <= 2 std,
a factor of at most 5, and the pivot sums otherwise, with the pivot within a few standard deviations of the group mean.
With C_STAT = 2^-12 (> 2^-16 * 13, the pivot up to sqrt(12) standard deviations off):
    |y - y_ref| <= 2 * 2^-9 * |y_ref| + L * (C_STAT * (|x - mu| rstd + 1) |gamma| + 2^-22 (|x| rstd |gamma| + |beta|))
                   + 2^-12 |y_pre| (SiLU only: tanh.approx.f32 is within ~2^-11, and silu = 0.5 y (1 + tanh(y / 2))) + 1e-6,
where the 2^-22 term is the fp32 affine y = x * (rstd gamma) + (beta - mean rstd gamma). Without the pivot (K = 0), an
fp32 one-pass variance loses (mu / sigma)^2 * 2^-24 relative: at a group mean 64 standard deviations from zero that
is past C_STAT, and a count off by one sample row moves the mean by mu / spatial, which the offset cases catch."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U9, U23 = 2.0 ** -9, 2.0 ** -23
L_ACT = 1.13
C_STAT = 2.0 ** -12
F_RS, F_RB, F_RES, F_ACT, F_GLU, F_F32, F_WS = 1, 2, 4, 8, 16, 32, 64
F_ALL = F_RS | F_RB | F_RES | F_ACT | F_F32
F_ALL_GLU = F_GLU | F_RS | F_RB | F_RES | F_F32
STAGES = {256: 4, 160: 5, 128: 6, 64: 8, 32: 8}
RESB_STAGES = {256: 3, 160: 6, 128: 3}
SMEM_LIMIT = 227 * 1024
GN_DYN_SMEM_MAX, GN_MAX_N = 220 * 1024, 1024
RATIOS = {}                       # test group -> largest err / tol seen


# ---------------------------------------------------------------------------------------------------- helpers
def gen(cuda, seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, device=g.device, generator=g, dtype=torch.float32) * scale + shift


def close(out, ref, tol, group, what):
    """|out - ref| <= tol element by element (NaN fails); records the largest err / tol of the group."""
    ratio = ((out.to(F64) - ref).abs() / tol).nan_to_num(float("inf"))
    r = float(ratio.max()) if ratio.numel() else 0.0
    RATIOS[group] = max(RATIOS.get(group, 0.0), r)
    if r > 1:
        idx = [int(i) for i in torch.nonzero(ratio > 1)[0]]
        n = int((ratio > 1).sum())
        raise AssertionError(f"{what}: {n}/{ratio.numel()} elements over the bound, max err/tol {r:.3g}; first at {idx}: "
                             f"got {float(out[tuple(idx)]):.6g}, want {float(ref[tuple(idx)]):.6g}")


def kernels_of(fn):
    """Names (spaces removed) of the CUDA kernels `fn` launches, from a torch.profiler trace kept in memory. A trace
    that came back without any of this library's kernels (the profiler occasionally drops a session's GPU activity
    records) is taken again."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name.replace(" ", "") for e in prof.events()}
        if any("vb::" in n for n in names):
            break
    return names


def launched(names, pattern):
    return any(pattern.replace(" ", "") in n for n in names)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class gemm_mode:
    """set_gemm_impl / resident-B switch / VB200_FORCE_BN for the duration of a block, restored afterwards."""

    def __init__(self, impl=0, resb=None, force_bn=None):
        self.impl, self.resb, self.force = impl, resb, force_bn

    def __enter__(self):
        from vitron_b200 import ops
        self.prev_impl = ops.set_gemm_impl(self.impl)
        self.prev_dbg = ops.set_gemm_debug(-1, -1)
        if self.resb is not None:
            ops.set_gemm_debug(self.resb, -1)
        self.prev_env = os.environ.get("VB200_FORCE_BN")
        if self.force is not None:
            os.environ["VB200_FORCE_BN"] = str(self.force)
        return self

    def __exit__(self, *exc):
        from vitron_b200 import ops
        ops.set_gemm_impl(self.prev_impl)
        ops.set_gemm_debug(self.prev_dbg & 0xff, self.prev_dbg >> 8)
        if self.prev_env is None:
            os.environ.pop("VB200_FORCE_BN", None)
        else:
            os.environ["VB200_FORCE_BN"] = self.prev_env
        return False


# ---------------------------------------------------------------------------------------------------- planner statement
def _f(x):
    return np.float32(x)


def plan_tiles(mb, N, kblocks, allow_split, out_rows, force_bn=None):
    """Statement of plan_tiles() (gemm.cu) on this device, in fp32 like the C code: (bn, splits)."""
    if force_bn in (256, 160, 128, 64, 32):
        return force_bn, 1
    s = sms()
    tk = {256: 1.0, 160: 0.78, 128: 0.76, 64: 0.625, 32: 0.57}
    best, best_t = (256, 1), _f(1e30)
    for bn in (256, 160, 128, 64, 32):
        tiles = mb * -(-N // bn)
        for sp in range(1, 9):
            if sp > 1:
                if not allow_split or tiles * 10 >= s * 7 or kblocks // sp < 4 or sp * out_rows * N * 4 > (64 << 20):
                    break
            waves = -(-(tiles * sp) // s)
            kpu = -(-kblocks // sp)
            t = _f(waves) * (_f(kpu) * _f(tk[bn]) + _f(1.5 if sp > 1 else 0.0))
            t = _f(t + _f(2.0) * _f(bn) / _f(256.0))
            if sp > 1:
                t = _f(t + _f(sp) * _f(out_rows) * _f(N) * _f(8.0) / _f(5.0e6) / _f(0.27) + _f(9.0))
            if t < best_t - _f(1e-4):
                best_t, best = t, (bn, sp)
    return best


def resb_smem(bn, nkb):
    return nkb * bn * 128 + RESB_STAGES[bn] * 128 * 128 + 1280


def resb_tile(M, N, nkb, need, impl=0, resb=1):
    """Statement of resb_tile() (gemm.cu): the resident-B tile width, or 0."""
    if impl == 1 or not (resb & 3) or need not in (0, F_RES, F_GLU, F_ACT):
        return 0
    if nkb > 5 and not (resb & 2):
        return 0
    if M < 4096:
        return 0
    best, best_cost = 0, _f(1e30)
    for bn in (160, 256, 128):
        nb = -(-N // bn)
        if resb_smem(bn, nkb) > SMEM_LIMIT or nb > sms():
            continue
        groups = sms() // nb
        per_cta = -(-(-(-M // 128)) // groups)
        mma, astream = _f(bn) / _f(256.0), _f(0.55 if bn == 160 else 0.9)
        cost = _f(per_cta) * _f(nkb) * max(mma, astream)
        if cost < best_cost:
            best, best_cost = bn, cost
    return best


def use_swap(M, N, K):
    return M <= 64 and N * K > (4 << 20)


def swap_splits(M, N, K):
    """Statement of swap_splits() (gemm.cu)."""
    s = sms()
    m_blocks, kblocks = -(-N // 128), -(-K // 64)
    best, best_score = 1, _f(-1.0)
    for sp in range(1, min(32, kblocks) + 1):
        if sp * M * N * 4 > (96 << 20):
            break
        units = m_blocks * sp
        waves = -(-units // s)
        util = _f(units) / _f(waves * s)
        bal = _f(kblocks) / _f(sp * -(-kblocks // sp))
        score = _f(util * bal - _f(0.01) * _f(sp))
        if score > best_score + _f(1e-6):
            best_score, best = score, sp
    return best


def v2_need(splits, rowscale=False, rowbias=False, residual=False, alpha=1.0, act=0, glu=0, out_fp32=False):
    if splits > 1:
        return F_WS
    return ((F_RS if rowscale else 0) | (F_RB if rowbias else 0) | (F_RES if residual or alpha != 1.0 else 0) |
            (F_ACT if act else 0) | (F_GLU if glu else 0) | (F_F32 if out_fp32 else 0))


def v2_variant(need, impl):
    """The F template argument dispatch_v2 picks for `need`."""
    if need & F_WS:
        return F_WS
    if impl == 0 and need in (0, F_ACT, F_RES, F_GLU, F_GLU | F_RS, F_RS, F_RB):
        return need
    return F_ALL_GLU if need & F_GLU else F_ALL


def conv_pixel_tile(wo, ho, nb):
    """Statement of conv_pixel_tile() (gemm.cu): (tw, th, tn)."""
    best, tile = -1, (1, 1, 1)
    for cw in range(min(wo, 128), 0, -1):
        for ch in range(min(128 // cw, ho), 0, -1):
            cn = min(128 // (cw * ch), nb)
            blocks = -(-wo // cw) * -(-ho // ch) * -(-nb // cn)
            if best < 0 or blocks < best:
                best, tile = blocks, (cw, ch, cn)
    return tile


def gemm_plan(M, N, K, impl=0, resb=1, force_bn=None, workspace=True, **epi):
    """What vb200_gemm_bf16 launches for M > 64: dict(bn, splits, F, resb, kernel) with the kernel-name pattern."""
    assert M > 64
    nkb = -(-K // 64)
    need1 = v2_need(1, **epi)
    rbn = resb_tile(M, N, nkb, need1, impl, resb)
    if rbn:
        return dict(bn=rbn, splits=1, F=need1, resb=True, fallback=None,
                    kernel=f"gemm_v2_kernel<{rbn},{RESB_STAGES[rbn]},{need1},true>")
    mb = -(-M // 128)
    bn, sp = plan_tiles(mb, N, nkb, True, M, force_bn)
    fallback = None
    if sp > 1 and not workspace:
        bn, sp = plan_tiles(mb, N, nkb, False, M, force_bn)
        fallback = "no-workspace"
    Fv = v2_variant(v2_need(sp, **epi), impl)
    return dict(bn=bn, splits=sp, F=Fv, resb=False, fallback=fallback,
                kernel=f"gemm_v2_kernel<{bn},{STAGES[bn]},{Fv},false>")


def conv_plan(nb, h, w, cin, cout, kh, kw, stride, ph, pw, impl=0, force_bn=None, **epi):
    ho, wo = (h + 2 * ph - kh) // stride + 1, (w + 2 * pw - kw) // stride + 1
    tw, th, tn = conv_pixel_tile(wo, ho, nb)
    mb = -(-wo // tw) * -(-ho // th) * -(-nb // tn)
    kb = kh * kw * -(-cin // 64)
    bn, sp = plan_tiles(mb, cout, kb, True, nb * ho * wo, force_bn)
    Fv = v2_variant(v2_need(sp, **epi), impl)
    return dict(bn=bn, splits=sp, F=Fv, tile=(tw, th, tn), ho=ho, wo=wo, kernel=f"gemm_v2_kernel<{bn},{STAGES[bn]},{Fv},false>")


def gn_plan(n, spatial, c):
    """Statement of gn_plan() (norm.cu)."""
    vec = c // 8
    rpp = min(max(512 // vec, 1), spatial)
    threads = (vec * rpp + 31) // 32 * 32
    s = sms()
    per = 1 if n >= s else s // n
    per = min(per, (spatial + 4 * rpp - 1) // (4 * rpp))
    if n >= 8 and spatial * c * 2 + rpp * c * 8 <= 128 * 1024:
        per = 1
    per = max(per, 1)
    rpc = -(-spatial // per)
    per = -(-spatial // rpc)
    part = rpp * c * 8
    cached = part + rpc * c * 2 <= GN_DYN_SMEM_MAX
    return dict(rpp=rpp, threads=threads, per=per, rpc=rpc, cached=cached)


def gn_launches(n, spatial, c):
    """The launches of vb200_groupnorm_nhwc: a list of (samples, plan), following its chunking over GN_MAX_N and its
    halving of uncached batches into cached chunks."""
    if n > GN_MAX_N:
        out = []
        for s0 in range(0, n, GN_MAX_N):
            out += gn_launches(min(GN_MAX_N, n - s0), spatial, c)
        return out
    pl = gn_plan(n, spatial, c)
    if not pl["cached"] and n > 1:
        nc = n
        while nc > 1:
            nc = (nc + 1) // 2
            if gn_plan(nc, spatial, c)["cached"]:
                break
        if gn_plan(nc, spatial, c)["cached"]:
            out = []
            for s0 in range(0, n, nc):
                out += gn_launches(min(nc, n - s0), spatial, c)
            return out
    return [(n, pl)]


# ---------------------------------------------------------------------------------------------------- references
def act64(v, act):
    from vitron_b200 import ops
    if act == ops.ACT_GELU:
        return F.gelu(v)
    if act == ops.ACT_QUICK_GELU:
        return v * torch.sigmoid(1.702 * v)
    if act == ops.ACT_RELU:
        return F.relu(v)
    if act == ops.ACT_SILU:
        return F.silu(v)
    return v


def tau(k_eff):
    return (math.ceil(k_eff / 16) + 8) * U23


def epi_ref(acc, S, k_eff, bias=None, act=0, glu=0, residual=None, alpha=1.0, rowbias=None, rowbias_rows=0,
            rowscale=None, out_fp32=False):
    """float64 epilogue over acc [rows, N] and S = sum |a w| in the kernel's order; returns (ref, tol) of the bound in the
    module docstring."""
    rs = rowscale.to(F64)[:, None] if rowscale is not None else torch.ones((acc.shape[0], 1), dtype=F64, device=acc.device)
    v = acc * rs
    e = tau(k_eff) * S * rs.abs()
    if bias is not None:
        v = v + bias.to(F64)
    if rowbias is not None:
        grp = torch.arange(acc.shape[0], device=acc.device) // max(int(rowbias_rows), 1)
        v = v + rowbias.to(F64)[grp]
    if glu:
        col = torch.arange(acc.shape[1], device=acc.device)
        ia, ib = col[(col % 32) < 16], col[(col % 32) >= 16]
        va, vb, ea, eb = v[:, ia], v[:, ib], e[:, ia], e[:, ib]
        if glu == 1:
            r = F.silu(va) * vb
            err = vb.abs() * L_ACT * ea + F.silu(va).abs() * eb
        else:
            r = va * F.gelu(vb)
            err = F.gelu(vb).abs() * ea + va.abs() * L_ACT * eb
        P = (1 + va.abs()) * (1 + vb.abs())
    else:
        r = act64(v, act)
        err = L_ACT * e if act else e
        P = 1 + v.abs()
    r = (residual.to(F64) + alpha * r) if residual is not None else alpha * r
    tol = abs(alpha) * err + 2.0 ** -20 * abs(alpha) * P + 1e-6
    if not out_fp32:
        tol = tol + 2 * U9 * r.abs()
    return r, tol


def gemm_ref(a, w, k_eff=None, **epi):
    a64, w64 = a.to(F64), w.to(F64)
    return epi_ref(a64 @ w64.t(), a64.abs() @ w64.abs().t(), k_eff or -(-a.shape[1] // 64) * 64, **epi)


def conv_ref(x, wt, kh, kw, stride, ph, pw, k_eff=None, **epi):
    """x [nb, h, w, cin] bf16, wt [cout, cin, kh, kw] bf16 -> (ref, tol) flattened to [nb*ho*wo, cout']; taps that fall
    outside the image read zeros."""
    nb, h, w, cin = x.shape
    cout = wt.shape[0]
    ho, wo = (h + 2 * ph - kh) // stride + 1, (w + 2 * pw - kw) // stride + 1
    xp = F.pad(x.to(F64), (0, 0, pw, pw, ph, ph))
    cols = [xp[:, dy:dy + stride * (ho - 1) + 1:stride, dx:dx + stride * (wo - 1) + 1:stride, :]
            for dy in range(kh) for dx in range(kw)]
    A = torch.stack(cols, 3).reshape(nb * ho * wo, kh * kw * cin)
    W = wt.to(F64).permute(0, 2, 3, 1).reshape(cout, kh * kw * cin)
    return epi_ref(A @ W.t(), A.abs() @ W.abs().t(), k_eff or kh * kw * -(-cin // 64) * 64, **epi)


def guarded(rows, cols, dtype, device, grow=(2, 13), off=(1, 3)):
    """A NaN-filled buffer with guard rows and columns around an out= view [rows, cols] at row / column offset `off`
    (the view's base is not 16-byte aligned and its row stride exceeds its width)."""
    buf = torch.full((rows + grow[0], cols + grow[1]), float("nan"), dtype=dtype, device=device)
    return buf, buf[off[0]:off[0] + rows, off[1]:off[1] + cols]


def check_guards(buf, view, what):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    r0 = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    keep.view(-1)[torch.as_strided(torch.arange(buf.numel(), device=buf.device), view.shape, view.stride(), r0).reshape(-1)] = False
    n = int((~buf[keep].isnan()).sum())
    assert n == 0, f"{what}: {n} elements written outside the out= view"


def strided_a(a, g):
    """a [M, K] as a view with a 16-byte base offset and lda = K + 72 into a buffer holding 1000 elsewhere."""
    M, K = a.shape
    big = torch.full((M, K + 72), 1000.0, dtype=BF, device=a.device)
    big[:, 8:8 + K] = a
    return big[:, 8:8 + K]


def run_gemm(cuda, g, a, w, group, what, out_fp32=False, **epi):
    """ops.gemm into a guarded strided out= view; checks the guards, the bound and the bit-identical repeat."""
    from vitron_b200 import ops
    M = a.shape[0]
    n_out = w.shape[0] // 2 if epi.get("glu") else w.shape[0]
    buf, out = guarded(M, n_out, F32 if out_fp32 else BF, cuda)
    res = ops.gemm(a, w, out=out, out_fp32=out_fp32, **epi)
    assert res.data_ptr() == out.data_ptr()
    check_guards(buf, out, what)
    ref, tol = gemm_ref(a, w, out_fp32=out_fp32, **epi)
    close(out, ref, tol, group, what)
    again = ops.gemm(a, w, out_fp32=out_fp32, **epi)
    assert torch.equal(again, out), f"{what}: repeat differs"
    return out


FEATURES = {   # name -> epilogue builder(g, M, N)
    "plain": lambda g, M, N: {},
    "gelu": lambda g, M, N: dict(bias=randn((N,), g).to(BF), act=1),
    "quick_gelu": lambda g, M, N: dict(bias=randn((N,), g).to(BF), act=2),
    "relu": lambda g, M, N: dict(bias=randn((N,), g).to(BF), act=3),
    "silu": lambda g, M, N: dict(bias=randn((N,), g).to(BF), act=4),
    "residual": lambda g, M, N: dict(bias=randn((N,), g).to(BF), residual=randn((M, N), g).to(BF), alpha=-0.75),
    "alpha": lambda g, M, N: dict(alpha=0.5),
    "swiglu": lambda g, M, N: dict(bias=randn((N,), g).to(BF), glu=1),
    "geglu": lambda g, M, N: dict(bias=randn((N,), g).to(BF), glu=2),
    "swiglu+rowscale": lambda g, M, N: dict(glu=1, rowscale=(torch.rand((M,), device=g.device, generator=g) * 2 + 0.25)),
    "rowscale": lambda g, M, N: dict(rowscale=(torch.rand((M,), device=g.device, generator=g) * 2 + 0.25)),
    "rowbias": lambda g, M, N: dict(rowbias=randn((-(-M // 40), N), g).to(BF), rowbias_rows=40),
    # combinations without a specialised variant: F_ALL / F_ALL_GLU
    "rowbias+act+residual": lambda g, M, N: dict(rowbias=randn((-(-M // 7), N), g).to(BF), rowbias_rows=7, act=4,
                                                 residual=randn((M, N), g).to(BF), bias=randn((N,), g).to(BF)),
    "rowscale+fp32": lambda g, M, N: dict(rowscale=(torch.rand((M,), device=g.device, generator=g) + 0.5), out_fp32=True),
    "geglu+residual": lambda g, M, N: dict(glu=2, residual=randn((M, N // 2), g).to(BF), alpha=2.0),
    "fp32": lambda g, M, N: dict(bias=randn((N,), g).to(BF), out_fp32=True),
}


def epi_flags(epi):
    keys = ("rowscale", "rowbias", "residual", "alpha", "act", "glu", "out_fp32")
    return {k: (epi[k] is not None if k in ("rowscale", "rowbias", "residual") else epi[k]) for k in keys if k in epi}


# ---------------------------------------------------------------------------------------------------- A: GEMM, M > 64
VARIANT_SHAPES = {bn: [(257, 3 * bn + (32 if bn != 32 else 64), 200), (383, 2 * bn + 41, 136)] for bn in (256, 160, 128, 64, 32)}


@pytest.mark.parametrize("impl", [0, 1], ids=["specialised", "generic"])
@pytest.mark.parametrize("bn", [256, 160, 128, 64, 32])
def test_gemm_variant_matrix(cuda, bn, impl):
    """Every tile width forced, every feature set, at M = 128k +- 1, N not a multiple of the tile (odd where GLU is
    off), K = 64k + 8; A is a strided view with a 16-byte offset; out is a guarded strided view."""
    g = gen(cuda, 100 * bn + impl)
    for M, N, K in VARIANT_SHAPES[bn]:
        a = strided_a(randn((M, K), g).to(BF), g)
        for name, mk in FEATURES.items():
            glu = name.startswith(("swiglu", "geglu"))
            n = N - N % 32 if glu else N
            if glu and n % 32:
                continue
            w = (randn((n, K), g, 0.05)).to(BF)
            epi = mk(g, M, n)
            out_fp32 = epi.pop("out_fp32", False)
            plan = gemm_plan(M, n, K, impl=impl, resb=0, force_bn=bn, out_fp32=out_fp32, **epi_flags(epi))
            assert plan["bn"] == bn and plan["splits"] == 1
            with gemm_mode(impl, resb=0, force_bn=bn):
                run_gemm(cuda, g, a, w, "gemm variants", f"BN {bn} impl {impl} {name} {M}x{n}x{K}", out_fp32=out_fp32, **epi)


RESB_CASES = [(4224, 320, 320), (8192, 640, 320), (5000, 2560, 320), (4097, 336, 128)]


def resb_wide():
    """(M, N, K, resident-B mode, width): N one 160-wide n-block past the SM count takes BN = 256; K = 640 with mode 3
    takes BN = 128."""
    return [(4096, 160 * sms() + 32, 320, 1, 256), (4096, 128 * sms(), 640, 3, 128)]


@pytest.mark.parametrize("need", ["plain", "residual", "geglu", "silu"])
def test_gemm_resident_b(cuda, need):
    """The resident-B variants with each feature set they exist for, at shapes the planner sends to them, against the
    same calls with resident B off."""
    from vitron_b200 import ops
    g = gen(cuda, 300 + len(need))
    for M, N, K, mode in [c + (1,) for c in RESB_CASES] + [c[:4] for c in resb_wide()]:
        a = randn((M, K), g).to(BF)
        w = randn((N, K), g, 0.05).to(BF)
        epi = FEATURES[need](g, M, N)
        if need == "geglu" and N % 32:
            continue
        plan = gemm_plan(M, N, K, resb=mode, **epi_flags(epi))
        assert plan["resb"], (M, N, K, plan)
        with gemm_mode(0, resb=mode):
            out = run_gemm(cuda, g, a, w, "gemm resident B", f"resb {need} {M}x{N}x{K}", **epi)
        with gemm_mode(0, resb=0):
            off = ops.gemm(a, w, **epi)
        ref, tol = gemm_ref(a, w, **epi)
        close(off, ref, tol, "gemm resident B", f"resb off {need} {M}x{N}x{K}")
        assert out.shape == off.shape


# LLaMA-7B prefill (Vicuna widths), ViT-L/14, UNet, GLIGEN / SEEM query rows; rows scaled x1 .. x30
LLAMA_ROWS = [65, 127, 128, 129, 768]
LLAMA_CALLS = ["qkv", "gate_up", "o_proj", "down", "lm_head-32000", "lm_head-32001", "lm_head-32002"]


@pytest.fixture(scope="module")
def vicuna(cuda):
    from vitron_b200 import ops
    g = gen(cuda, 31)
    w = {n: randn(s, g, 0.02).to(BF) for n, s in (("qkv", (12288, 4096)), ("o_proj", (4096, 4096)),
                                                   ("gate", (11008, 4096)), ("up", (11008, 4096)),
                                                   ("down", (4096, 11008)), ("lm_head", (32002, 4096)))}
    w["gate_up"] = ops.pack_glu_weight(w["gate"], w["up"])
    return w


@pytest.mark.parametrize("M", LLAMA_ROWS)
def test_gemm_llama_prefill(cuda, vicuna, M):
    """The LlamaEngine prefill calls: qkv / gate_up with the RMS row scale (row_rstd -> rowscale), o / down with the
    in-place residual, lm_head in fp32 at three vocabulary sizes; rows scaled x1 to x30."""
    from vitron_b200 import ops
    w = vicuna
    g = gen(cuda, 7000 + M)
    eps = 1e-5
    for call in LLAMA_CALLS:
        K = 11008 if call == "down" else 4096
        scale = (1 + 29 * torch.rand((M, 1), device=cuda, generator=g))
        x = (randn((M, K), g) * scale).to(BF)
        what = f"{call} M={M}"
        if call in ("o_proj", "down"):
            h0 = randn((M, 4096), g).to(BF)
            h = h0.clone()
            got = ops.gemm(x, w[call], residual=h, out=h)
            assert got.data_ptr() == h.data_ptr()
            ref, tol = gemm_ref(x, w[call], residual=h0)
            close(h, ref, tol, "gemm llama", what)
            assert torch.equal(ops.gemm(x, w[call], residual=h0), h), f"{what}: in-place residual differs"
            continue
        rs = ops.row_rstd(x, eps)
        rs64 = torch.rsqrt(x.to(F64).pow(2).mean(-1) + eps)
        assert bool(((rs.to(F64) - rs64).abs() <= 2.0 ** -16 * rs64).all()), f"{what}: row_rstd"
        if call.startswith("lm_head"):
            V = int(call.split("-")[1])
            wv = w["lm_head"][:V]
            buf, out = guarded(M, V, F32, cuda)
            ops.gemm(x, wv, rms_eps=eps, out=out, out_fp32=True)
            check_guards(buf, out, what)
            ref, tol = gemm_ref(x, wv, rowscale=rs, out_fp32=True)
        else:
            glu = 1 if call == "gate_up" else 0
            buf, out = guarded(M, w[call].shape[0] // (2 if glu else 1), BF, cuda)
            ops.gemm(x, w[call], glu=glu, rms_eps=eps, out=out)
            check_guards(buf, out, what)
            ref, tol = gemm_ref(x, w[call], rowscale=rs, glu=glu)
        close(out, ref, tol, "gemm llama", what)


MODEL_GEMMS = {   # name: (M, N, K, epilogue)
    "vit-fc1": (257 * 2, 4096, 1024, dict(bias=True, act=2)),
    "vit-fc2": (257 * 2, 1024, 4096, dict(bias=True, residual=True)),
    "vit-qkv": (257, 3072, 1024, dict(bias=True)),
    "unet-proj": (40960, 320, 320, dict(bias=True, residual=True)),
    "unet-geglu": (40960, 2560, 320, dict(bias=True, glu=2)),
    "unet-ff-out": (40960, 320, 1280, dict(bias=True, residual=True)),
    "unet-l2-geglu": (2560, 10240, 1280, dict(bias=True, glu=2)),
    "gligen-101": (101, 768, 768, dict(bias=True, act=1)),
    "seem-101-mlp": (101, 512, 512, dict(bias=True, act=3)),
    "seem-101-logits": (101, 4096, 512, dict(out_fp32=True)),
    "split-640x1280x3840": (640, 1280, 3840, dict(bias=True)),
    "split-200x1280x5120": (200, 1280, 5120, dict(bias=True, residual=True)),
    "split-2560x1280x11520": (2560, 1280, 11520, dict(bias=True)),
    "split-128x256x4096": (128, 256, 4096, dict()),
    "split-640x336x2048": (640, 336, 2048, dict(act=4)),
    "split-300x1280x4096": (300, 1280, 4096, dict(bias=True, act=1)),
}


@pytest.mark.parametrize("impl", [0, 1], ids=["specialised", "generic"])
@pytest.mark.parametrize("name", list(MODEL_GEMMS))
def test_gemm_model_shapes(cuda, name, impl):
    M, N, K, spec = MODEL_GEMMS[name]
    g = gen(cuda, 500 + list(MODEL_GEMMS).index(name))
    a = (randn((M, K), g) * (1 + 29 * torch.rand((M, 1), device=cuda, generator=g)) / 8).to(BF)
    w = randn((N, K), g, 0.02).to(BF)
    n_out = N // 2 if spec.get("glu") else N
    epi = {}
    if spec.get("bias"):
        epi["bias"] = randn((N,), g).to(BF)
    if spec.get("residual"):
        epi["residual"] = randn((M, n_out), g).to(BF)
    for k in ("act", "glu"):
        if k in spec:
            epi[k] = spec[k]
    with gemm_mode(impl):
        run_gemm(cuda, g, a, w, "gemm model", f"{name} impl {impl}", out_fp32=spec.get("out_fp32", False), **epi)


SPLIT_SHAPES = [(200, 1280, 5120), (200, 1282, 5120), (200, 1284, 5120), (200, 1286, 5120), (300, 1280, 4096),
                (256, 512, 4096), (128, 256, 4096)]


@pytest.mark.parametrize("M,N,K", SPLIT_SHAPES)
def test_gemm_splitk_reduce(cuda, M, N, K):
    """splitk_reduce_kernel with every epilogue feature (GLU where N % 32 == 0), N % 8 in {0, 2, 4, 6}, rowbias and
    rowscale together, into guarded views at an unaligned column; repeats and the in-place residual are bit-identical."""
    from vitron_b200 import ops
    plan = gemm_plan(M, N, K)
    assert plan["splits"] > 1, plan
    g = gen(cuda, M + N + K)
    a = strided_a(randn((M, K), g).to(BF), g)
    w = randn((N, K), g, 0.02).to(BF)
    names = [n for n in FEATURES if not n.startswith(("swiglu", "geglu"))] + ["rowbias+rowscale"]
    if N % 32 == 0:
        names += ["swiglu", "geglu", "swiglu+rowscale", "geglu+residual"]
    for name in names:
        if name == "rowbias+rowscale":
            epi = dict(rowbias=randn((-(-M // 40), N), g).to(BF), rowbias_rows=40,
                       rowscale=torch.rand((M,), device=cuda, generator=g) + 0.5, bias=randn((N,), g).to(BF))
        else:
            epi = FEATURES[name](g, M, N)
        out_fp32 = epi.pop("out_fp32", False)
        run_gemm(cuda, g, a, w, "gemm split-K", f"split {name} {M}x{N}x{K}", out_fp32=out_fp32, **epi)
    h0 = randn((M, N), g).to(BF)
    h = h0.clone()
    ops.gemm(a, w, residual=h, out=h, alpha=0.5)
    assert torch.equal(ops.gemm(a, w, residual=h0, alpha=0.5), h), "split in-place residual differs"


def test_gemm_no_workspace_fallback(cuda):
    """A split-K shape called through the C ABI without a workspace runs the unsplit plan (same numbers, within the
    bound; no partials anywhere)."""
    import ctypes as C
    from vitron_b200 import _lib
    lib = _lib.load()
    M, N, K = 200, 1280, 5120
    plan, fb = gemm_plan(M, N, K), gemm_plan(M, N, K, workspace=False)
    assert plan["splits"] > 1 and fb["splits"] == 1 and fb["fallback"] == "no-workspace"
    g = gen(cuda, 77)
    a, w, bias = randn((M, K), g).to(BF), randn((N, K), g, 0.02).to(BF), randn((N,), g).to(BF)
    buf, out = guarded(M, N, BF, cuda)
    epi = _lib.Epilogue()
    epi.bias, epi.alpha = bias.data_ptr(), 1.0
    _lib.check(lib.vb200_gemm_bf16(a.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), out.stride(0), M, N, K, C.byref(epi),
                                   None, 0, torch.cuda.current_stream().cuda_stream), "vb200_gemm_bf16")
    torch.cuda.synchronize()
    check_guards(buf, out, "no workspace")
    ref, tol = gemm_ref(a, w, bias=bias)
    close(out, ref, tol, "gemm split-K", "no-workspace fallback")


# ---------------------------------------------------------------------------------------------------- B: convolution
def run_conv(cuda, g, nb, h, w, cin, cout, kh, kw, stride=1, ph=None, pw=None, group="conv", what="", amp=1.0,
             wscale=None, **epi):
    """ops.conv_nhwc into out= at an offset inside a NaN-filled flat buffer; border pixels asserted on their own."""
    from vitron_b200 import ops
    ph = kh // 2 if ph is None else ph
    pw = kw // 2 if pw is None else pw
    x = randn((nb, h, w, cin), g, amp).to(BF)
    wt = randn((cout, cin, kh, kw), g, wscale or 1.0 / math.sqrt(cin * kh * kw)).to(BF)
    ho, wo = (h + 2 * ph - kh) // stride + 1, (w + 2 * pw - kw) // stride + 1
    n_out = cout // 2 if epi.get("glu") else cout
    for k, v in list(epi.items()):
        if v == "rand":
            epi[k] = {"bias": lambda: randn((cout,), g).to(BF), "residual": lambda: randn((nb, ho, wo, n_out), g).to(BF)}[k]()
    guard = 40
    flat = torch.full((nb * ho * wo * n_out + 2 * guard,), float("nan"), dtype=BF, device=cuda)
    out = flat[guard:guard + nb * ho * wo * n_out].view(nb, ho, wo, n_out)
    ops.conv_nhwc(x, ops.pack_conv_weight(wt), kh, kw, stride=stride, pad_h=ph, pad_w=pw, out=out, **epi)
    assert bool(flat[:guard].isnan().all() and flat[-guard:].isnan().all()), f"{what}: wrote outside out="
    ref_epi = {k: v for k, v in epi.items()}
    if "residual" in ref_epi:
        ref_epi["residual"] = ref_epi["residual"].reshape(-1, n_out)
    ref, tol = conv_ref(x, wt, kh, kw, stride, ph, pw, **ref_epi)
    ref, tol = ref.view(nb, ho, wo, n_out), tol.view(nb, ho, wo, n_out)
    for name, sl in (("top row", (slice(None), 0)), ("bottom row", (slice(None), ho - 1)),
                     ("left column", (slice(None), slice(None), 0)), ("right column", (slice(None), slice(None), wo - 1))):
        close(out[sl], ref[sl], tol[sl], group, f"{what}: {name}")
    close(out, ref, tol, group, what)
    return x, wt, out


UNET_LEVELS = [(40, 64, 320), (20, 32, 640), (10, 16, 1280), (5, 8, 1280)]


@pytest.mark.parametrize("impl", [0, 1], ids=["specialised", "generic"])
@pytest.mark.parametrize("level", range(4))
def test_conv_unet_levels(cuda, level, impl):
    """UNetSD_I2VGen ResBlock convolutions at f = 16 frames: bias + time-embedding rowbias, bias + residual; the stride-2
    downsample, the upsample-then-conv, the temporal Conv3d (3, 1, 1) with pad_w = 0 and a residual."""
    h, w, c = UNET_LEVELS[level]
    g = gen(cuda, 600 + level)
    f = 16
    with gemm_mode(impl):
        rb = randn((1, c), g).to(BF)
        run_conv(cuda, g, f, h, w, c, c, 3, 3, group="conv unet", what=f"L{level} conv1 rowbias",
                 bias="rand", rowbias=rb, rowbias_rows=f * h * w)
        run_conv(cuda, g, f, h, w, c, c, 3, 3, group="conv unet", what=f"L{level} conv2 residual", bias="rand",
                 residual="rand")
        if level < 3:
            run_conv(cuda, g, f, h, w, c, c, 3, 3, stride=2, group="conv unet", what=f"L{level} downsample", bias="rand")
        if level > 0:
            from vitron_b200 import ops
            x = randn((f, h, w, c), g).to(BF)
            up = ops.upsample2x_nhwc(x)
            assert torch.equal(up, x.repeat_interleave(2, 1).repeat_interleave(2, 2)), "upsample2x"
        run_conv(cuda, g, 1, f, h * w, c, c, 3, 1, ph=1, pw=0, group="conv unet", what=f"L{level} temporal", bias="rand",
                 residual="rand")


VAE_CONVS = {   # name: (nb, h, w, cin, cout, kh, kw, stride, ph, pw, epi)
    "conv_in-cin8": (1, 128, 128, 8, 128, 3, 3, 1, 1, 1, dict(bias="rand")),
    "res-128": (1, 128, 128, 128, 128, 3, 3, 1, 1, 1, dict(bias="rand", residual="rand")),
    "down-128-pad0": (1, 129, 129, 128, 128, 3, 3, 2, 0, 0, dict(bias="rand")),
    "res-256": (1, 64, 64, 256, 256, 3, 3, 1, 1, 1, dict(bias="rand")),
    "csc-128-256": (1, 64, 64, 128, 256, 3, 3, 1, 1, 1, dict(bias="rand")),
    "down-256-pad0": (1, 65, 65, 256, 256, 3, 3, 2, 0, 0, dict(bias="rand")),
    "res-512": (1, 32, 32, 512, 512, 3, 3, 1, 1, 1, dict(bias="rand", residual="rand")),
    "conv_out-512-8": (1, 32, 32, 512, 8, 3, 3, 1, 1, 1, dict(bias="rand")),
    "seem-fpn-256": (1, 64, 64, 256, 256, 3, 3, 1, 1, 1, dict()),
    "seem-fpn-512": (1, 32, 32, 512, 512, 3, 3, 1, 1, 1, dict()),
    "focal-down-96": (1, 56, 56, 96, 192, 3, 3, 2, 1, 1, dict(bias="rand")),
    "focal-down-192": (1, 28, 28, 192, 384, 3, 3, 2, 1, 1, dict(bias="rand")),
}


@pytest.mark.parametrize("name", list(VAE_CONVS))
def test_conv_vae_seem_focal(cuda, name):
    """VAE convolutions (conv_in at cin = 8, pad = 0 downsample after F.pad), SEEM FPN 3x3 (+ GroupNorm + ReLU as the
    model runs it), FocalNet stride-2 downsample at cin = 96 / 192."""
    from vitron_b200 import ops
    nb, h, w, cin, cout, kh, kw, stride, ph, pw, epi = VAE_CONVS[name]
    g = gen(cuda, 700 + list(VAE_CONVS).index(name))
    x, wt, out = run_conv(cuda, g, nb, h, w, cin, cout, kh, kw, stride, ph, pw, group="conv vae/seem/focal", what=name,
                          **dict(epi))
    if name.startswith("seem"):
        gw, gb = (1 + 0.2 * randn((cout,), g)).to(BF), (0.2 * randn((cout,), g)).to(BF)
        y = ops.groupnorm_nhwc(out, gw, gb, 32, 1e-5, act=ops.ACT_RELU)
        ref, tol = gn_ref(out.view(1, -1, cout), gw, gb, 32, 1e-5, ops.ACT_RELU)
        close(y.view(1, -1, cout), ref, tol, "groupnorm model", f"{name} + GN ReLU")


CONV_EDGES = [  # nb, h, w, cin, cout, kh, kw, stride
    (2, 12, 12, 8, 320, 3, 3, 1), (2, 9, 11, 72, 64, 3, 3, 1), (2, 10, 10, 96, 128, 3, 3, 1), (1, 17, 19, 160, 96, 3, 3, 1),
    (2, 9, 13, 128, 96, 3, 3, 2), (1, 33, 65, 64, 128, 3, 3, 2), (3, 7, 7, 32, 64, 3, 3, 2),
    (1, 8, 300, 64, 64, 3, 3, 1), (2, 7, 130, 64, 64, 3, 3, 1), (5, 5, 8, 64, 64, 3, 3, 1), (7, 3, 5, 64, 160, 3, 3, 1),
    (3, 10, 16, 320, 640, 1, 1, 1), (1, 33, 200, 192, 512, 1, 1, 1),
    (16, 10, 16, 1280, 1280, 3, 3, 1), (1, 16, 40, 1280, 1280, 3, 1, 1), (16, 5, 8, 2560, 1280, 3, 3, 1),
    (2, 5, 8, 640, 48, 3, 3, 1),
]


@pytest.mark.parametrize("impl", [0, 1], ids=["specialised", "generic"])
@pytest.mark.parametrize("nb,h,w,cin,cout,kh,kw,stride", CONV_EDGES)
def test_conv_edges(cuda, nb, h, w, cin, cout, kh, kw, stride, impl):
    """cin % 64 in {8, 32} (weight padding against the OOB zero-fill), stride 2 on odd sizes, wo below and above 128, nb
    not a multiple of tn, ragged pixel tiles, split-K convolutions, 1x1 and (3, 1) kernels."""
    g = gen(cuda, nb * 1000 + h * 10 + w + cin + impl)
    with gemm_mode(impl):
        run_conv(cuda, g, nb, h, w, cin, cout, kh, kw, stride, group="conv edges", what=f"{(nb, h, w, cin, cout, kh, kw, stride)}",
                 bias="rand")


@pytest.mark.parametrize("bn", [256, 160, 128, 64, 32])
def test_conv_forced_bn(cuda, bn):
    """One convolution per forced tile width with the ResBlock epilogue (bias + rowbias + residual: F_ALL)."""
    g = gen(cuda, 800 + bn)
    with gemm_mode(0, force_bn=bn):
        rb = randn((2, 200), g).to(BF)
        run_conv(cuda, g, 2, 11, 13, 96, 200, 3, 3, group="conv edges", what=f"forced BN {bn}", bias="rand",
                 residual="rand", rowbias=rb, rowbias_rows=11 * 13)
        run_conv(cuda, g, 3, 9, 10, 128, 2 * bn + 64, 3, 3, stride=2, group="conv edges", what=f"forced BN {bn} s2")


def test_conv_direct(cuda):
    """conv_nhwc_direct (tiny layers) against the same float64 reference; its tau counts one step per FMA of its fp32
    chains (kh * kw * cin of them) instead of one per k16 MMA."""
    from vitron_b200 import ops
    g = gen(cuda, 900)
    for nb, h, w, cin, cout in [(2, 9, 7, 8, 16), (1, 16, 16, 64, 32), (3, 5, 6, 24, 8)]:
        x = randn((nb, h, w, cin), g).to(BF)
        wt = randn((cout, cin, 3, 3), g, 0.2).to(BF)
        bias = randn((cout,), g).to(BF)
        out = ops.conv_nhwc_direct(x, wt.permute(0, 2, 3, 1).reshape(cout, 9, cin).contiguous(), bias, 3, 3)
        ref, tol = conv_ref(x, wt, 3, 3, 1, 1, 1, k_eff=16 * 9 * cin, bias=bias)
        close(out.reshape(-1, cout), ref, tol, "conv direct", f"direct {(nb, h, w, cin, cout)}")


# ---------------------------------------------------------------------------------------------------- C: GroupNorm
def gn_ref(x, w, b, groups, eps, act):
    """float64 GroupNorm over x [n, spatial, c] bf16 (biased variance), then the activation; returns (ref, tol)."""
    from vitron_b200 import ops
    n, sp, c = x.shape
    cpg = c // groups
    x64 = x.to(F64).view(n, sp, groups, cpg)
    mu = x64.mean((1, 3), keepdim=True)
    var = (x64 - mu).pow(2).mean((1, 3), keepdim=True)
    rstd = torch.rsqrt(var + eps)
    gam, bet = w.to(F64).view(groups, cpg), b.to(F64).view(groups, cpg)
    ypre = ((x64 - mu) * rstd * gam + bet).view(n, sp, c)
    y = ypre.clamp_min(0) if act == ops.ACT_RELU else F.silu(ypre) if act == ops.ACT_SILU else ypre
    stat = C_STAT * ((x64 - mu).abs() * rstd + 1) * gam.abs() + 2.0 ** -22 * (x64.abs() * rstd * gam.abs() + bet.abs())
    tol = 2 * U9 * y.abs() + (L_ACT if act else 1.0) * stat.view(n, sp, c) + 1e-6
    if act == ops.ACT_SILU:
        tol = tol + 2.0 ** -12 * ypre.abs()
    return y, tol


def gn_operands(g, n, sp, c, groups=32, r=0.0, channel_spread=0.0, const_group=False):
    """x = mean + N(0, 1): the per-(sample, group) mean is r * (+-1) (r spreads of the group), channels of a group get
    extra means in [-channel_spread, channel_spread]; const_group makes group 1 of every sample one constant."""
    cpg = c // groups
    sign = torch.randint(0, 2, (n, 1, groups, 1), device=g.device, generator=g).to(F32) * 2 - 1
    chan = (torch.rand((1, 1, groups, cpg), device=g.device, generator=g) * 2 - 1) * channel_spread
    x = randn((n, sp, groups, cpg), g) + r * sign + chan
    if const_group:
        x[:, :, 1, :] = 3.25
    w = (1 + 0.3 * randn((c,), g)).to(BF)
    b = (0.5 * randn((c,), g)).to(BF)
    return x.reshape(n, sp, c).to(BF), w, b


def run_gn(cuda, x, w, b, groups, eps, act, group, what, n=None):
    from vitron_b200 import ops
    nn = x.shape[0] if n is None else n
    y = ops.groupnorm_nhwc(x, w, b, groups, eps, act=act, n=n)
    c = x.shape[-1]
    ref, tol = gn_ref(x.reshape(nn, -1, c), w, b, groups, eps, act)
    close(y.reshape(nn, -1, c), ref, tol, group, what)
    ws = ops.workspace(0, cuda, "gn")
    assert int(ws[:8 * GN_MAX_N].view(torch.int32).abs().sum()) == 0, f"{what}: counters left non-zero"
    return y


GN_MODEL = {   # name: (n, spatial, c, eps, act, n_view)
    "unet-l0-silu": (16, 2560, 320, 1e-5, 4, None), "unet-l1-silu": (16, 640, 640, 1e-5, 4, None),
    "unet-l2-silu": (16, 160, 1280, 1e-5, 4, None), "unet-l3-silu": (16, 40, 1280, 1e-5, 4, None),
    "unet-cat-640": (16, 2560, 640, 1e-5, 4, None), "unet-cat-960": (16, 2560, 960, 1e-5, 4, None),
    "unet-cat-1920": (16, 640, 1920, 1e-5, 4, None), "unet-cat-2560": (16, 160, 2560, 1e-5, 4, None),
    "unet-l3-cat-2560": (16, 40, 2560, 1e-5, 4, None),
    "unet-temporal-conv": (16, 2560, 320, 1e-5, 4, 1), "unet-spatial-tf": (16, 2560, 320, 1e-6, 0, None),
    "unet-temporal-tf": (16, 640, 640, 1e-6, 0, 1), "unet-l3-temporal": (16, 40, 1280, 1e-6, 0, 1),
    "gligen-l0": (2, 4096, 320, 1e-5, 4, None), "gligen-l2": (2, 256, 1280, 1e-5, 4, None),
    "gligen-tf": (2, 4096, 320, 1e-6, 0, None), "gligen-l3": (2, 64, 1280, 1e-5, 4, None),
    "vae-128": (1, 128 * 128, 128, 1e-6, 4, None), "vae-256": (1, 64 * 64, 256, 1e-6, 4, None),
    "vae-512": (1, 32 * 32, 512, 1e-6, 4, None), "vae-attn": (1, 32 * 32, 512, 1e-6, 0, None),
    "vae-dec-512px": (1, 512 * 512, 128, 1e-6, 4, None),
    "seem-fpn": (1, 64 * 64, 256, 1e-5, 3, None), "seem-mask": (1, 16 * 16, 256, 1e-5, 0, None),
}


@pytest.mark.parametrize("name", list(GN_MODEL))
def test_groupnorm_model_shapes(cuda, name):
    n, sp, c, eps, act, nv = GN_MODEL[name]
    g = gen(cuda, 1100 + list(GN_MODEL).index(name))
    x, w, b = gn_operands(g, n, sp, c, r=1.5)
    run_gn(cuda, x, w, b, 32, eps, act, "groupnorm model", name, n=nv)


GN_OFFSET_SHAPES = [(1, 40960, 320), (1, 2560, 320), (8, 128, 64), (16, 256, 160), (1, 512 * 512, 128), (2, 40960, 320),
                    (3, 3, 320), (2, 50, 2560)]


@pytest.mark.parametrize("r", [0, 8, 64, 256])
@pytest.mark.parametrize("n,sp,c", GN_OFFSET_SHAPES)
def test_groupnorm_offsets(cuda, n, sp, c, r):
    """Group means r spreads away from zero, channel means that differ inside a group, a constant group (its output is
    beta), on every launch plan (cached, one CTA per sample, uncached, halved into chunks, rpp > spatial)."""
    from vitron_b200 import ops
    g = gen(cuda, 1200 + r + n + c)
    x, w, b = gn_operands(g, n, sp, c, r=float(r), channel_spread=3.0, const_group=True)
    for act in (ops.ACT_NONE, ops.ACT_SILU):
        y = run_gn(cuda, x, w, b, 32, 1e-5, act, "groupnorm offsets", f"r {r} {(n, sp, c)} act {act}")
        if act == ops.ACT_NONE:
            cpg = c // 32
            beta, gam = b[cpg:2 * cpg].to(F64), w[cpg:2 * cpg].to(F64)
            tol = 2 * U9 * beta.abs() + 2.0 ** -22 * (3.25 * 1e-5 ** -0.5 * gam.abs() + beta.abs()) + 1e-6
            close(y.view(n, sp, c)[:, :, cpg:2 * cpg], beta.expand(n, sp, cpg), tol.expand(n, sp, cpg),
                  "groupnorm offsets", f"r {r} {(n, sp, c)}: constant group is beta")


GN_PLAN_CASES = [(1, 40960, 320), (8, 128, 64), (16, 256, 160), (1, 512 * 512, 128), (2, 40960, 320), (3, 40960, 320),
                 (1100, 16, 64), (4, 1, 64), (3, 3, 320), (2, 33, 960), (2, 50, 2560), (2, 5000, 1920), (2, 300, 128),
                 (1, 64 * 64, 512), (16, 640, 640), (16, 160, 1280)]


@pytest.mark.parametrize("n,sp,c", GN_PLAN_CASES)
def test_groupnorm_plans(cuda, n, sp, c):
    """The planner cases (see test_case_list_reaches_every_branch) at offset r = 8 with ReLU and groups 32, 16 and 8."""
    from vitron_b200 import ops
    g = gen(cuda, 1300 + n + sp + c)
    for groups in (32, 16, 8):
        if c % groups:
            continue
        x, w, b = gn_operands(g, n, sp, c, groups=groups, r=8.0)
        run_gn(cuda, x, w, b, groups, 1e-5, ops.ACT_RELU, "groupnorm plans", f"{(n, sp, c)} groups {groups}")


def test_groupnorm_workspace_interleaved(cuda):
    """Calls of different n / groups interleaved on the one workspace are bit-identical to the same calls made alone,
    the in-place form is bit-identical, and the counter prefix is zero after every call."""
    from vitron_b200 import ops
    g = gen(cuda, 1400)
    cases = [(1, 40960, 320, 32), (16, 640, 640, 16), (2, 40960, 320, 32), (8, 128, 64, 8), (1, 512 * 512, 128, 32),
             (1100, 16, 64, 32), (3, 3, 320, 32)]
    ops_in = [gn_operands(g, n, sp, c, groups=gr, r=4.0) + (gr,) for n, sp, c, gr in cases]
    alone = []
    for x, w, b, gr in ops_in:
        alone.append(ops.groupnorm_nhwc(x, w, b, gr, 1e-5, act=ops.ACT_SILU).clone())
        torch.cuda.synchronize()
    for rnd in range(2):
        for i in (list(range(len(cases))) if rnd == 0 else list(reversed(range(len(cases))))):
            x, w, b, gr = ops_in[i]
            y = ops.groupnorm_nhwc(x, w, b, gr, 1e-5, act=ops.ACT_SILU)
            assert torch.equal(y, alone[i]), f"interleaved call {cases[i]} differs"
            assert int(ops.workspace(0, cuda, "gn")[:8 * GN_MAX_N].view(torch.int32).abs().sum()) == 0
    for i, (x, w, b, gr) in enumerate(ops_in):
        xi = x.clone()
        ops.groupnorm_nhwc(xi, w, b, gr, 1e-5, act=ops.ACT_SILU, out=xi)
        assert torch.equal(xi, alone[i]), f"in-place {cases[i]} differs"


# ---------------------------------------------------------------------------------------------------- D: planner reach
def test_case_list_reaches_every_branch(cuda):
    """The cases of this file reach every branch of the planners on this device (statements above), and the statements
    agree with the library's own workspace sizes."""
    from vitron_b200 import _lib
    lib = _lib.load()
    # statement of the planners = the library's workspace sizes
    for M, N, K in [(M, N, K) for M, N, K in SPLIT_SHAPES] + [(m[0], m[1], m[2]) for m in MODEL_GEMMS.values()] + \
            [(17, 4096, 4096), (33, 12288, 4096), (64, 4096, 11008), (40, 2048, 512)]:
        if M <= 16:
            continue
        if use_swap(M, N, K):
            want = swap_splits(M, N, K) * M * N * 4
        else:
            bn, sp = plan_tiles(-(-M // 128), N, -(-K // 64), True, M)
            want = sp * M * N * 4 if sp > 1 else 0
        assert lib.vb200_gemm_bf16_workspace_size(M, N, K) == want, (M, N, K)
    convs = [c[:8] for c in CONV_EDGES] + [(16, h, w, c, c, 3, 3, 1) for h, w, c in UNET_LEVELS]
    for nb, h, w, cin, cout, kh, kw, stride in convs:
        p = conv_plan(nb, h, w, cin, cout, kh, kw, stride, kh // 2, kw // 2)
        want = p["splits"] * nb * p["ho"] * p["wo"] * cout * 4 if p["splits"] > 1 else 0
        assert lib.vb200_conv_nhwc_workspace_size(nb, h, w, cin, cout, kh, kw, stride, kh // 2, kw // 2) == want
    # GEMM: every BN unsplit, split-K 2..8, resident B per width and feature set, resident-B fallbacks
    unsplit = {gemm_plan(M, N, K, resb=0, force_bn=bn)["bn"] for bn, shapes in VARIANT_SHAPES.items() for M, N, K in shapes}
    assert unsplit == {256, 160, 128, 64, 32}
    splits = {gemm_plan(M, N, K)["splits"] for M, N, K in SPLIT_SHAPES} | \
             {gemm_plan(M, N, K)["splits"] for M, N, K, _ in MODEL_GEMMS.values() if M > 64}
    assert any(2 <= s <= 8 for s in splits) and max(splits) <= 8, splits
    conv_splits = {conv_plan(*c[:8], c[5] // 2, c[6] // 2)["splits"] for c in CONV_EDGES}
    assert max(conv_splits) > 1, conv_splits
    resb = {}
    for M, N, K in RESB_CASES:
        for need, epi in (("plain", {}), ("residual", dict(residual=True)), ("geglu", dict(glu=2)), ("silu", dict(act=4))):
            p = gemm_plan(M, N, K, **epi)
            if p["resb"]:
                resb.setdefault(p["bn"], set()).add(p["F"])
    assert resb.get(160) == {0, F_RES, F_GLU, F_ACT}, resb
    for M, N, K, mode, bn_want in resb_wide():
        for epi in ({}, dict(residual=True), dict(glu=2), dict(act=4)):
            p = gemm_plan(M, N, K, resb=mode, **epi)
            assert p["resb"] and p["bn"] == bn_want and p["F"] == v2_need(1, **epi), (M, N, K, p)
    big_n = 256 * (sms() + 1)
    assert not gemm_plan(4096, big_n, 320)["resb"]                       # nb > SMs at every width
    assert not gemm_plan(40960, 320, 320, rowscale=True)["resb"]         # no resident-B variant with F_RS
    assert gemm_plan(200, 1280, 5120, workspace=False)["splits"] == 1
    # conv pixel tiles: wo < 128, wo > 128, nb not a multiple of tn, ragged last tiles
    tiles = {c: conv_pixel_tile((c[2] + 2 - 3) // c[7] + 1, (c[1] + 2 - 3) // c[7] + 1, c[0]) for c in CONV_EDGES if c[5] == 3}
    assert any((c[2] - 1) // c[7] + 1 > 128 for c in tiles) and any((c[2] - 1) // c[7] + 1 < 128 for c in tiles)
    assert any(c[0] % t[2] for c, t in tiles.items())
    assert any(((c[2] + 2 - 3) // c[7] + 1) % t[0] for c, t in tiles.items())
    # GroupNorm: each launch plan
    kinds = set()
    for n, sp, c in GN_PLAN_CASES + [s for s in GN_OFFSET_SHAPES]:
        launches = gn_launches(n, sp, c)
        for ns, pl in launches:
            kinds.add("cached-multi" if pl["cached"] and pl["per"] > 1 else "one-cta" if pl["per"] == 1 and ns >= 8
                      else "uncached" if not pl["cached"] else "cached-single")
            if pl["rpp"] > sp or 512 // (c // 8) > sp:
                kinds.add("rpp>spatial")
        if n > GN_MAX_N:
            kinds.add("n>1024")
        elif n > 1 and len(launches) > 1:
            kinds.add("halved")
        if 512 % (c // 8):
            kinds.add("c/8 not dividing 512")
    assert {"cached-multi", "one-cta", "uncached", "halved", "n>1024", "rpp>spatial", "c/8 not dividing 512"} <= kinds, kinds
    cpgs = {c // 32 for _, _, c in GN_PLAN_CASES + GN_OFFSET_SHAPES}
    assert {4, 10, 20, 40} <= cpgs, cpgs


# ---------------------------------------------------------------------------------------------------- E: which variant ran
def check_trace_cases(cuda):
    """Each case family runs the instantiation the planner statement predicts."""
    from vitron_b200 import ops
    g = gen(cuda, 1900)
    want = []

    def gemm_case(M, N, K, impl=0, resb=None, force=None, **epi):
        a, w = randn((M, K), g).to(BF), randn((N, K), g, 0.05).to(BF)
        out_fp32 = epi.pop("out_fp32", False)
        e = {k: (randn((M, N // 2 if epi.get("glu") else N), g).to(BF) if k == "residual" else
                 torch.rand((M,), device=cuda) + 0.5 if k == "rowscale" else
                 randn((-(-M // 40), N), g).to(BF) if k == "rowbias" else v) for k, v in epi.items()}
        if "rowbias" in e:
            e["rowbias_rows"] = 40
        plan = gemm_plan(M, N, K, impl=impl, resb=1 if resb is None else resb, force_bn=force, out_fp32=out_fp32,
                         **epi_flags(e))

        def fn():
            with gemm_mode(impl, resb=resb, force_bn=force):
                ops.gemm(a, w, out_fp32=out_fp32, **e)
        names = kernels_of(fn)
        want.append((names, [plan["kernel"]] + (["splitk_reduce_kernel"] if plan["splits"] > 1 else []),
                     [] if plan["splits"] > 1 else ["splitk_reduce_kernel"], (M, N, K, impl, epi)))

    for bn in (256, 160, 128, 64, 32):
        M, N, K = VARIANT_SHAPES[bn][0]
        for impl in (0, 1):
            gemm_case(M, N, K, impl, resb=0, force=bn)
            gemm_case(M, N, K, impl, resb=0, force=bn, glu=1, rowscale=True)
            gemm_case(M, N, K, impl, resb=0, force=bn, rowbias=True, act=4, residual=True)
            gemm_case(M, N, K, impl, resb=0, force=bn, rowscale=True, out_fp32=True)
        gemm_case(M, N, K, 0, resb=0, force=bn, act=2)
        gemm_case(M, N, K, 0, resb=0, force=bn, rowbias=True)
    for M, N, K in RESB_CASES:
        gemm_case(M, N, K)
        gemm_case(M, N, K, residual=True)
        gemm_case(M, N, K, act=4)
        gemm_case(M, N, K, rowscale=True)
    gemm_case(40960, 2560, 320, glu=2)
    for M, N, K, mode, _ in resb_wide():
        gemm_case(M, N, K, resb=mode)
        gemm_case(M, N, K, resb=mode, glu=2)
    for M, N, K in SPLIT_SHAPES:
        gemm_case(M, N, K)
        gemm_case(M, N, K, rowbias=True, rowscale=True)
    for name in ("vit-fc1", "unet-l2-geglu", "gligen-101", "seem-101-logits"):
        M, N, K, spec = MODEL_GEMMS[name]
        gemm_case(M, N, K, **{k: v for k, v in spec.items() if k in ("act", "glu", "out_fp32")})
    # convolutions
    for c in CONV_EDGES[:6] + CONV_EDGES[-4:]:
        nb, h, w, cin, cout, kh, kw, stride = c
        x = randn((nb, h, w, cin), g).to(BF)
        wt = ops.pack_conv_weight(randn((cout, cin, kh, kw), g, 0.05).to(BF))
        bias = randn((cout,), g).to(BF)
        plan = conv_plan(nb, h, w, cin, cout, kh, kw, stride, kh // 2, kw // 2)
        names = kernels_of(lambda: ops.conv_nhwc(x, wt, kh, kw, stride=stride, bias=bias))
        want.append((names, [plan["kernel"]] + (["splitk_reduce_kernel"] if plan["splits"] > 1 else []),
                     [] if plan["splits"] > 1 else ["splitk_reduce_kernel"], c))
    # GroupNorm
    for n, sp, c in GN_PLAN_CASES:
        for act in (0, 3, 4):
            if act != 4 and (n, sp, c) not in ((1, 40960, 320), (1, 512 * 512, 128)):
                continue
            x = randn((n, sp, c), g).to(BF)
            wgt, b = torch.ones((c,), dtype=BF, device=cuda), torch.zeros((c,), dtype=BF, device=cuda)
            kinds = {pl["cached"] for _, pl in gn_launches(n, sp, c)}
            names = kernels_of(lambda: ops.groupnorm_nhwc(x, wgt, b, 32, 1e-5, act=act))
            want.append((names, [f"gn_onepass_kernel<{act},{'true' if k else 'false'}>" for k in kinds],
                         [f"gn_onepass_kernel<{act},{'false' if k else 'true'}>" for k in kinds if len(kinds) == 1], (n, sp, c, act)))
    for i, (names, present, absent, case) in enumerate(want):
        for p in present:
            assert launched(names, p), (i, case, p, sorted(n for n in names if "vb::" in n))
        for a in absent:
            assert not launched(names, a), (i, case, a, sorted(n for n in names if "vb::" in n))
    print(f"trace ok: {len(want)} calls")


def test_dispatch_branches_in_trace(cuda):
    """check_trace_cases in a fresh Python process: a profiler session in a process that has already captured a CUDA
    graph (other test files do) can come back without kernel records."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import sys; sys.path.insert(0, {root!r}); import torch; import tests.test_gemm_conv_groupnorm_gpu as t; "
            "t.check_trace_cases(torch.device('cuda:0'))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "trace ok" in r.stdout, (r.stdout[-4000:] + r.stderr[-4000:])


def test_report(cuda):
    """Prints the largest err / tol per group seen in this file."""
    for group, r in sorted(RATIOS.items()):
        print(f"max err/tol {group}: {r:.3f}")
