"""GPU: the NF4 kernels of csrc/gemv_nf4.cu against float64 references, on the branches a `load_4bit` model takes:
- `ops.gemm(x, NF4Weight)` at M <= 32 (`gemv_nf4_kernel<ROWS, NT>`): 16- and 32-row tiles, one, two and four token
  tiles, every epilogue, the engine's four Vicuna-7B projections, the region MLP / location encoder calls, K with an odd
  number of 64-blocks, k-slices without a superchunk, fewer tiles than the grid cap and three tiles per CTA, with probes
  where one (row, block), one token row, one byte value or one kscale block decides the output;
- `ops.gemm(x, NF4Weight)` above 32 rows (`nf4_dequant_kernel` into the "nf4" workspace, then `gemm_v2_kernel`) at the
  LLaMA prefill, mm_projector and region MLP calls, through workspace growth;
- both inside a CUDA graph captured under PDL, and the graphed NF4 decode of a `LlamaEngine` at batch > 32;
- a Python statement of the GEMV's host plan (tile height, token tiles, grid, per-warp k-slices), checked against a trace
  of the launched instantiations.

What the GEMV multiplies. Its shared-memory table holds T[c] = bf16_rn(NF4[c]) (13 of the 16 NF4 values are not bf16
numbers; the largest relative difference is 3.1e-3, code 2), the products T[c] * x~ run on mma.sync with fp32
accumulation, and the fp16 block scale s multiplies each 64-block's partial sum in fp32. With kscale the activations are
x~ = bf16_rn(fp32(x) * kscale[k]) (torch: `(x.float() * ks).to(bf16)`), otherwise x~ = x. The RMS row scale comes from the
raw x: rs = rsqrt(mean_k x^2 + eps). The reference is therefore float64 over exactly these operands,
    acc[m, n] = sum_k x~[m, k] T[code(n, k)] s[n, k / 64],        v = rs * acc,
followed by the epilogue in float64 in the kernel's order: rowscale, bias and rowbias, activation or GLU, then
residual + alpha * v.

GEMV bound. Let S[m, n] = sum_k |x~| |T| |s| and let the k-slice of a warp hold nb 64-blocks at most (nb = 2 *
max(s1 - s0) of the plan). A bf16 * bf16 product is exact in fp32. Every fp32 stage is taken to be off by at most one
unit of 2^-23 of the largest partial sum it can see (2^-23 rather than 2^-24 allows the tensor core to truncate):
    mma: four k16 steps per block, partial <= sum over the block of |x~ T|, then the exact scaling by s inside fmaf;
    fmaf(tmp, s, acc) over the slice's blocks: nb steps, partial <= S;
    the sum over the KS k-slices in the epilogue: KS steps; the product by rs: one more, and one spare.
So |acc_kernel - acc| <= tau S with tau = (4 + nb + KS + 2) 2^-23. The RMS scale: the kernel sums x^2 in fp32 per thread
over 16 nb terms, then two shuffles and KS slice sums, divides by K, adds eps and takes rsqrtf (2 ulp), so
    |rs_kernel / rs - 1| <= rho = ((16 nb + KS + 5) / 2 + 2) 2^-23
(the square root halves the sum's relative error). Before the epilogue |v_kernel - v| <= E = tau S |rs| + rho |v|.
Through the epilogue (L = 1.13 bounds |act'| for GELU, quick-GELU, SiLU and ReLU):
    activation: L E; SwiGLU: |b| L E_a + |silu(a)| E_b + L E_a E_b; GEGLU (a * gelu(b)): |gelu(b)| E_a + |a| L E_b + L E_a E_b;
    plus 2^-20 P with P = 1 + |v| (activation) or (1 + |a|)(1 + |b|) (GLU): fp32 bias additions, __expf / erff and the
    fp32 residual update, all relative errors of a few 2^-24 of values of that size; everything times |alpha|;
    output: bf16 rounding is at most 2^-8 of the rounded value, so tol' = (1 + 2^-8) tol + 2^-8 |ref|; an fp32 output
    adds 2^-23 (|ref| + |residual|).
The same value against W_eff = NF4[c] * s (the format's statement, nf4.dequantize) adds the exact table term
    E_tab = |rs| sum_k |x~| |s| |T[c] - NF4[c]|
to E. At K = 4096 with unit-scale rows tau S is ~1e-5 of S: dropping one 64-block of 4096 k, a wrong block scale, or
an RMS sum that misses one k-slice is an error of 1e-2 of S or more.

Prefill bound (M > 32). The dequantiser is bit-identical to bf16_rn(nf4.dequantize(w) * kscale) (tests/test_nf4_gpu.py),
so the reference is float64 over that bf16 matrix and the bf16 GEMM bound of tests/test_gemm_conv_groupnorm_gpu.py:
tau = (ceil(K / 16) + 8) 2^-23 over S = sum |a| |w|, with the kernel's row_rstd as the row scale. Each result must also be
bit-identical to `ops.gemm` over that bf16 matrix."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from vitron_b200 import nf4

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U8, U23 = 2.0 ** -8, 2.0 ** -23
L_ACT = 1.13
EPS = 1e-5
MS = [1, 2, 7, 8, 9, 15, 16, 17, 24, 25, 31, 32]
RATIOS = {}                       # test group -> largest err / tol seen


# ---------------------------------------------------------------------------------------------------- helpers
def gen(cuda, seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, device=g.device, generator=g, dtype=torch.float32) * scale + shift


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


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


def guarded(rows, cols, dtype, device):
    """A NaN-filled buffer with guard rows and columns around an out= view [rows, cols] at offset (1, 3)."""
    buf = torch.full((rows + 2, cols + 13), float("nan"), dtype=dtype, device=device)
    return buf, buf[1:1 + rows, 3:3 + cols]


def check_guards(buf, view, what):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    r0 = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    keep.view(-1)[torch.as_strided(torch.arange(buf.numel(), device=buf.device), view.shape, view.stride(), r0).reshape(-1)] = False
    n = int((~buf[keep].isnan()).sum())
    assert n == 0, f"{what}: {n} elements written outside the out= view"


def x_view(x):
    """x [M, K] as a view with a 16-byte base offset and lda = K + 24 into a NaN-filled buffer."""
    M, K = x.shape
    big = torch.full((M, K + 24), float("nan"), dtype=BF, device=x.device)
    big[:, 8:8 + K] = x
    return big[:, 8:8 + K]


def kernels_of(fn):
    """Names (spaces removed) of the CUDA kernels `fn` launches, from a torch.profiler trace kept in memory; a trace
    without any of this library's kernels (the profiler occasionally drops a session's GPU records) is taken again."""
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


# ---------------------------------------------------------------------------------------------------- host plan statement
def nf4_plan(M, N, K, glu=False):
    """Statement of vb200_gemm_nf4's launch and of the per-warp k-slices of gemv_nf4_kernel."""
    rows = 32 if glu or N // 16 > 6 * sms() else 16
    nt = 1 if M <= 8 else 2 if M <= 16 else 4
    tiles = -(-N // rows)
    grid = min(tiles, 2 * sms())
    ks = 8 // (rows // 16)
    g = 1 if nt == 4 else 2
    chunks = K // 64
    nsc = (chunks + 1) // 2
    base, rem = divmod(nsc, ks)
    slices = []
    for w in range(ks):
        s0 = w * base + min(w, rem)
        s1 = s0 + base + (1 if w < rem else 0)
        ngroups = -(-(s1 - s0) // g)
        slices.append(dict(s0=s0, s1=s1, ngroups=ngroups, npairs=(ngroups + 1) // 2))
    return dict(rows=rows, nt=nt, tiles=tiles, grid=grid, ks=ks, g=g, chunks=chunks, nsc=nsc, slices=slices,
                nb=2 * max(s["s1"] - s["s0"] for s in slices), kernel=f"gemv_nf4_kernel<{rows},{nt}>")


def tau_gemv(plan):
    return (4 + plan["nb"] + plan["ks"] + 2) * U23


def rho_gemv(plan):
    return ((16 * plan["nb"] + plan["ks"] + 5) / 2 + 2) * U23


# ---------------------------------------------------------------------------------------------------- weights
class W4:
    """An NF4 weight built from chosen codes uint8 [N, K] and fp16 scales [N, K / 64], with the packed code bytes past K
    (K % 128 == 64) holding nonzero codes, and its float64 operands."""

    def __init__(self, codes, scales, g=None):
        n, k = codes.shape
        kp = -(-k // 128) * 128
        full = torch.zeros((n, kp), dtype=torch.uint8, device=codes.device)
        full[:, :k] = codes
        if kp > k:
            full[:, k:] = torch.randint(1, 16, (n, kp - k), device=codes.device, generator=g, dtype=torch.int64).to(torch.uint8) \
                if g is not None else 11
        self.w = nf4.NF4Weight(nf4.pack_codes(full), scales.contiguous(), k)
        self.codes, self.scales, self.n, self.k = codes, scales, n, k
        self._m = None

    def with_scales(self, scales):
        """The same codes (and padding bytes) with other scales."""
        o = W4.__new__(W4)
        o.w = nf4.NF4Weight(self.w.codes, scales.contiguous(), self.k)
        o.codes, o.scales, o.n, o.k, o._m = self.codes, scales, self.n, self.k, None
        return o

    def mats(self, keep=True):
        """float64 [N, K]: T[c] s, |T[c] s|, NF4[c] s, |T[c] - NF4[c]| |s|."""
        if self._m is not None:
            return self._m
        dev = self.codes.device
        t64, e64 = nf4.NF4.to(BF).to(F64).to(dev), nf4.NF4.to(F64).to(dev)
        s = self.scales.to(F64).repeat_interleave(64, 1)
        c = self.codes.long()
        m = (t64[c] * s, t64.abs()[c] * s.abs(), e64[c] * s, (t64 - e64).abs()[c] * s.abs())
        if keep:
            self._m = m
        return m


def rand_codes(g, n, k):
    return torch.randint(0, 16, (n, k), device=g.device, generator=g, dtype=torch.int64).to(torch.uint8)


def rand_scales(g, n, k, spread=3.0, base=0.02):
    """fp16 scales base * 2^U(-spread, spread) per (row, block): blocks and rows differ by up to 2^(2 spread)."""
    e = (torch.rand((n, k // 64), device=g.device, generator=g) * 2 - 1) * spread
    return (base * torch.exp2(e)).to(torch.float16)


def rand_w4(g, n, k, spread=3.0, base=0.02):
    return W4(rand_codes(g, n, k), rand_scales(g, n, k, spread, base), g)


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


def epi64(v, e, bias=None, rowbias=None, rowbias_rows=0, act=0, glu=0, residual=None, alpha=1.0, out_fp32=False):
    """float64 epilogue of v [M, N] (row scale applied) with |v_kernel - v| <= e; returns (ref, tol)."""
    if bias is not None:
        v = v + bias.to(F64)
    if rowbias is not None:
        grp = torch.arange(v.shape[0], device=v.device) // max(int(rowbias_rows), 1)
        v = v + rowbias.to(F64)[grp]
    if glu:
        col = torch.arange(v.shape[1], device=v.device)
        ia, ib = col[(col % 32) < 16], col[(col % 32) >= 16]
        va, vb, ea, eb = v[:, ia], v[:, ib], e[:, ia], e[:, ib]
        if glu == 1:
            r = F.silu(va) * vb
            err = vb.abs() * L_ACT * ea + F.silu(va).abs() * eb + L_ACT * ea * eb
        else:
            r = va * F.gelu(vb)
            err = F.gelu(vb).abs() * ea + va.abs() * L_ACT * eb + L_ACT * ea * eb
        P = (1 + va.abs()) * (1 + vb.abs())
    else:
        r = act64(v, act)
        err = L_ACT * e if act else e
        P = 1 + v.abs()
    r = (residual.to(F64) + alpha * r) if residual is not None else alpha * r
    tol = abs(alpha) * err + 2.0 ** -20 * abs(alpha) * P + 1e-30
    if out_fp32:
        tol = tol + U23 * (r.abs() + (residual.to(F64).abs() if residual is not None else 0))
    else:
        tol = (1 + U8) * tol + U8 * r.abs()
    return r, tol


def gemv_ref(x, W, plan, kscale=None, rms_eps=0.0, rowscale=None, **epi):
    """((ref, tol) against the operands the GEMV multiplies, (ref, tol) against W_eff) of the module docstring."""
    Wt, Wa, We, Wd = W.mats()
    xt = ((x.float() * kscale).to(BF) if kscale is not None else x).to(F64)
    acc, S = xt @ Wt.t(), xt.abs() @ Wa.t()
    acc_e, D = xt @ We.t(), xt.abs() @ Wd.t()
    rho = 0.0
    if rowscale is not None:
        rs = rowscale.to(F64)[:, None]
    elif rms_eps > 0:
        rs = torch.rsqrt(x.to(F64).pow(2).mean(-1, keepdim=True) + rms_eps)
        rho = rho_gemv(plan)
    else:
        rs = torch.ones((x.shape[0], 1), dtype=F64, device=x.device)
    e = tau_gemv(plan) * S * rs.abs()
    v, v_e, d = acc * rs, acc_e * rs, D * rs.abs()
    return epi64(v, e + rho * v.abs(), **epi), epi64(v_e, e + d + rho * (v_e.abs() + d), **epi)


def run_gemv(cuda, x, W, group, what, out_fp32=False, guard=True, **kw):
    """ops.gemm(x, W) at M <= 32 into a guarded out= view (x as an offset view with NaN padding); checks the plan, the
    guards, both bounds and a bit-identical repeat. Returns the output."""
    from vitron_b200 import ops
    M = x.shape[0]
    glu = kw.get("glu", 0)
    plan = nf4_plan(M, W.n, W.k, glu=bool(glu))
    n_out = W.n // 2 if glu else W.n
    xv = x_view(x)
    buf, out = guarded(M, n_out, F32 if out_fp32 else BF, cuda)
    res = ops.gemm(xv, W.w, out=out, out_fp32=out_fp32, **kw)
    assert res.data_ptr() == out.data_ptr()
    check_guards(buf, out, what)
    (ref, tol), (ref_e, tol_e) = gemv_ref(x, W, plan, out_fp32=out_fp32, **kw)
    close(out, ref, tol, group, what)
    close(out, ref_e, tol_e, group + " vs W_eff", what + " vs W_eff")
    again = ops.gemm(x, W.w, out_fp32=out_fp32, **kw)
    assert torch.equal(again, out), f"{what}: repeat differs"
    return out


# ---------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def vicuna(cuda):
    """NF4 weights of one Vicuna-7B layer in the engine's layout (qkv concatenated, gate / up interleaved in 16-row blocks)
    with their float64 operands, the RMSNorm gains, and the region MLP / location encoder weights."""
    from vitron_b200 import ops
    g = gen(cuda, 41)
    w = {}
    for name, (n, k) in (("qkv", (12288, 4096)), ("o_proj", (4096, 4096)), ("down", (4096, 11008))):
        w[name] = W4(*nf4_codes_scales(g, n, k))
    gate, up = nf4_codes_scales(g, 11008, 4096), nf4_codes_scales(g, 11008, 4096)
    w["gate_up"] = W4(ops.pack_glu_weight(gate[0], up[0]), ops.pack_glu_weight(gate[1], up[1]))
    for name, (n, k) in (("region0", (4096, 1024)), ("region1", (4096, 4096)), ("loc1", (4096, 2048))):
        w[name] = W4(*nf4_codes_scales(g, n, k))
    for W in w.values():
        W.mats()
    w["g1"] = (1 + 0.5 * torch.rand((4096,), device=cuda, generator=g)).contiguous()
    w["g2"] = (1 + 0.5 * torch.rand((4096,), device=cuda, generator=g)).contiguous()
    w["bias"] = {n: randn((4096,), g, 0.1).to(BF) for n in ("region0", "region1", "loc1")}
    return w


def nf4_codes_scales(g, n, k):
    """(codes, scales) of nf4.quantize over a 0.02-scaled normal weight: the model's code and scale distribution."""
    q = nf4.quantize(randn((n, k), g, 0.02).to(BF))
    return nf4.unpack_codes(q.codes, k), q.scales


def engine_call(ops, w, call, x, h=None, out=None):
    """The LlamaEngine._layer calls (llama.py) on NF4 weights: qkv / gate_up with the RMS scale and the RMSNorm gain as
    kscale, o_proj / down with the residual in place."""
    if call == "qkv":
        return ops.gemm(x, w["qkv"].w, rms_eps=EPS, kscale=w["g1"], out=out)
    if call == "gate_up":
        return ops.gemm(x, w["gate_up"].w, glu=ops.GLU_SWIGLU, rms_eps=EPS, kscale=w["g2"], out=out)
    return ops.gemm(x, w[call].w, residual=h, out=h)


# ---------------------------------------------------------------------------------------------------- the case list
EDGE_N = ["37", "200", "rows32"]
EDGE_K = [64, 128, 192, 1088, 4160]


def edge_n(name):
    return 16 * (6 * sms() + 1) if name == "rows32" else int(name)


def test_case_list_reaches_every_branch(cuda):
    """The shapes of this file reach, on this device, every <ROWS, NT> instantiation, fewer tiles than the grid cap,
    three tiles on one CTA (the RMS scale reused), odd block counts, k-slices without a superchunk, an odd group count
    and slices of unequal length."""
    plans = []
    for M in MS:
        for N, K, glu in [(12288, 4096, False), (22016, 4096, True), (4096, 4096, False), (4096, 11008, False),
                          (4096, 1024, False), (4096, 2048, False)]:
            plans.append(nf4_plan(M, N, K, glu))
        for n in EDGE_N:
            for K in EDGE_K:
                plans.append(nf4_plan(M, edge_n(n), K))
    assert {(p["rows"], p["nt"]) for p in plans} == {(r, t) for r in (16, 32) for t in (1, 2, 4)}
    assert any(p["tiles"] < 2 * sms() for p in plans)
    assert any(p["tiles"] > 2 * p["grid"] for p in plans)
    assert any(p["chunks"] % 2 for p in plans)
    assert any(s["s1"] == s["s0"] for p in plans for s in p["slices"])
    assert any(s["ngroups"] % 2 for p in plans for s in p["slices"])
    assert any(len({s["s1"] - s["s0"] for s in p["slices"]}) > 1 for p in plans)
    assert nf4_plan(1, 12288, 4096)["rows"] == 16 and nf4_plan(1, edge_n("rows32"), 64)["rows"] == 32
    # the single-block probes below sit at the first and last superchunk of every k-slice at KS = 8 and KS = 4
    assert nf4_plan(1, 4096, 4160)["ks"] == 8 and nf4_plan(1, edge_n("rows32"), 4160)["ks"] == 4


# ---------------------------------------------------------------------------------------------------- A: decode shapes
@pytest.mark.parametrize("M", MS)
def test_vicuna_decode_projections(cuda, vicuna, M):
    """The engine's four projections at every row count: qkv and gate/up with rms_eps and kscale, o_proj and down with
    the in-place residual, compared with the out-of-place residual bit for bit; rows scaled x1 .. x30."""
    from vitron_b200 import ops
    w = vicuna
    g = gen(cuda, 100 + M)
    for call in ("qkv", "gate_up", "o_proj", "down"):
        W = w[call]
        scale = 1 + 29 * torch.rand((M, 1), device=cuda, generator=g)
        x = (randn((M, W.k), g) * scale).to(BF)
        what = f"{call} M={M}"
        if call in ("o_proj", "down"):
            h0 = randn((M, 4096), g).to(BF)
            h = h0.clone()
            engine_call(ops, w, call, x_view(x), h=h)
            plan = nf4_plan(M, W.n, W.k)
            (ref, tol), (ref_e, tol_e) = gemv_ref(x, W, plan, residual=h0)
            close(h, ref, tol, "decode projections", what)
            close(h, ref_e, tol_e, "decode projections vs W_eff", what)
            assert torch.equal(ops.gemm(x, W.w, residual=h0), h), f"{what}: in-place residual differs"
        else:
            glu = ops.GLU_SWIGLU if call == "gate_up" else 0
            kscale = w["g1"] if call == "qkv" else w["g2"]
            run_gemv(cuda, x, W, "decode projections", what, glu=glu, rms_eps=EPS, kscale=kscale)


# ---------------------------------------------------------------------------------------------------- B: every epilogue
def epilogues(g, M, N, K):
    """name -> ops.gemm keyword arguments, for an [N, K] weight without GLU."""
    from vitron_b200 import ops
    b = lambda: randn((N,), g, 0.5).to(BF)
    ks = lambda: (torch.exp2(torch.rand((K,), device=g.device, generator=g) * 2 - 1)).contiguous()
    return {
        "plain": {},
        "gelu": dict(bias=b(), act=ops.ACT_GELU),
        "quick_gelu": dict(bias=b(), act=ops.ACT_QUICK_GELU),
        "relu": dict(bias=b(), act=ops.ACT_RELU),
        "silu": dict(act=ops.ACT_SILU),
        "rowbias1": dict(rowbias=randn((M, N), g, 0.5).to(BF), rowbias_rows=1),
        "rowbias3+gelu": dict(rowbias=randn((-(-M // 3), N), g, 0.5).to(BF), rowbias_rows=3, act=ops.ACT_GELU),
        "rowscale": dict(rowscale=(torch.rand((M,), device=g.device, generator=g) * 2 + 0.25)),
        "alpha": dict(alpha=-0.75, bias=b()),
        "alpha+residual": dict(alpha=0.5, residual=randn((M, N), g).to(BF)),
        "fp32": dict(bias=b(), out_fp32=True),
        "rms+kscale+fp32+residual": dict(rms_eps=EPS, kscale=ks(), residual=randn((M, N), g).to(BF), out_fp32=True),
        "rms+kscale+silu": dict(rms_eps=EPS, kscale=ks(), act=ops.ACT_SILU),
    }


def glu_epilogues(g, M, N, K):
    from vitron_b200 import ops
    return {
        "swiglu": dict(glu=ops.GLU_SWIGLU, bias=randn((N,), g, 0.5).to(BF)),
        "geglu": dict(glu=ops.GLU_GEGLU, bias=randn((N,), g, 0.5).to(BF)),
        "swiglu+rms+kscale": dict(glu=ops.GLU_SWIGLU, rms_eps=EPS,
                                  kscale=(torch.rand((K,), device=g.device, generator=g) + 0.5).contiguous()),
        "geglu+rowbias3+residual": dict(glu=ops.GLU_GEGLU, rowbias=randn((-(-M // 3), N), g, 0.5).to(BF), rowbias_rows=3,
                                        residual=randn((M, N // 2), g).to(BF), alpha=2.0),
        "swiglu+rowscale+fp32": dict(glu=ops.GLU_SWIGLU, rowscale=torch.rand((M,), device=g.device, generator=g) + 0.5,
                                     out_fp32=True),
    }


@pytest.mark.parametrize("K", EDGE_K)
@pytest.mark.parametrize("nname", EDGE_N)
def test_every_epilogue_at_edge_shapes(cuda, nname, K):
    """Every activation, rowbias with 1 and 3 rows per bias row, an explicit rowscale, alpha with and without a
    residual, fp32 out and the fused RMS scale with kscale, at N in {37, 200, 16 (6 SMs + 1)} (the last one on 32-row
    tiles without GLU) and K with one to 65 blocks; each epilogue at another row count; scales spread over 2^12."""
    N = edge_n(nname)
    g = gen(cuda, 7 * N + K)
    W = rand_w4(g, N, K, spread=6.0)
    for i, (name, epi) in enumerate(epilogues(g, 32, N, K).items()):
        M = MS[(i + EDGE_K.index(K) + 3 * EDGE_N.index(nname)) % len(MS)]
        for k in ("rowscale", "residual"):
            if k in epi:
                epi[k] = epi[k][:M].contiguous()
        if "rowbias" in epi:
            epi["rowbias"] = epi["rowbias"][:-(-M // max(epi["rowbias_rows"], 1))].contiguous()
        x = randn((M, K), g, 2.0).to(BF)
        out_fp32 = epi.pop("out_fp32", False)
        run_gemv(cuda, x, W, "epilogues", f"{name} M={M} N={N} K={K}", out_fp32=out_fp32, **epi)


@pytest.mark.parametrize("nname", ["32", "224", "many"])
@pytest.mark.parametrize("K", [64, 192, 4160])
def test_glu_epilogues(cuda, nname, K):
    """SwiGLU and GEGLU on the packed [16 a | 16 b] layout with bias, rowbias, residual, rowscale, fp32 out and the RMS
    scale, at one tile, seven tiles and 4 SMs + 1 tiles (three on one CTA)."""
    N = 32 * (4 * sms() + 1) if nname == "many" else int(nname)
    g = gen(cuda, 3 * N + K)
    W = rand_w4(g, N, K, spread=4.0)
    for i, (name, epi) in enumerate(glu_epilogues(g, 32, N, K).items()):
        M = MS[(5 * i + K) % len(MS)]
        for k in ("rowscale", "residual"):
            if k in epi:
                epi[k] = epi[k][:M].contiguous()
        if "rowbias" in epi:
            epi["rowbias"] = epi["rowbias"][:-(-M // epi["rowbias_rows"])].contiguous()
        x = randn((M, K), g, 2.0).to(BF)
        out_fp32 = epi.pop("out_fp32", False)
        run_gemv(cuda, x, W, "glu epilogues", f"{name} M={M} N={N} K={K}", out_fp32=out_fp32, **epi)


@pytest.mark.parametrize("M", [1, 9, 25, 32])
def test_region_mlp_and_loc_encoder(cuda, vicuna, M):
    """RegionExtractor.forward on NF4 weights (adapters.py): the MLP's ReLU + bias layers, its last bias layer, and the
    location encoder's second layer with bias + residual."""
    from vitron_b200 import ops
    w = vicuna
    g = gen(cuda, 500 + M)
    h = randn((M, 1024), g).to(BF)
    # h is a clone of the guarded out= view: at M = 1 it keeps that view's row stride (4109), which is not a multiple of 8
    for i, name in enumerate(("region0", "region1")):
        h = run_gemv(cuda, h, w[name], "region / loc", f"{name} M={M}", bias=w["bias"][name], act=ops.ACT_RELU).clone()
    hr = run_gemv(cuda, h, w["region1"], "region / loc", f"region2 M={M}", bias=w["bias"]["region1"]).clone()
    loc = F.relu(randn((M, 2048), g)).to(BF)
    run_gemv(cuda, loc, w["loc1"], "region / loc", f"loc1 M={M}", bias=w["bias"]["loc1"], residual=hr)


# ---------------------------------------------------------------------------------------------------- C: probes
def probe_blocks(plan):
    """Blocks at the first and last superchunk of every k-slice, the first and the last block, and the odd tail."""
    blocks = {0, plan["chunks"] - 1}
    for s in plan["slices"]:
        if s["s1"] > s["s0"]:
            for sc in (s["s0"], s["s1"] - 1):
                blocks.update(b for b in (2 * sc, 2 * sc + 1) if b < plan["chunks"])
    return sorted(blocks)


@pytest.mark.parametrize("case", ["ks8", "ks4", "glu-b"])
def test_single_live_block(cuda, case):
    """All scales zero but one (row, block): the output is that block's product in that row's column and exactly zero
    elsewhere. The block sits at the first and last superchunk of each k-slice, the first, the last and the odd tail
    block; the row at tile rows 0, 7, 8, 15, 16, 31 and N - 1, and (glu-b) in the b half of the packed GLU layout."""
    from vitron_b200 import ops
    N, K, glu = {"ks8": (4096, 4160, 0), "ks4": (edge_n("rows32"), 4160, 0), "glu-b": (2048, 4160, ops.GLU_SWIGLU)}[case]
    g = gen(cuda, len(case) + N)
    base = W4(rand_codes(g, N, K), torch.zeros((N, K // 64), dtype=torch.float16, device=cuda), g)
    rows = [0, 7, 8, 15, 16, 31, N - 1]
    if glu:
        rows = [16, 23, 24, 31, 48, 63, N - 1]      # rows 16..31 of a 32-row tile: the b half
    plan = nf4_plan(32, N, K, bool(glu))
    assert plan["ks"] == (4 if glu or case == "ks4" else 8)
    blocks = probe_blocks(plan)
    assert K // 64 - 1 in blocks and (K // 64) % 2 == 1
    bias = torch.ones((N,), dtype=BF, device=cuda) if glu else None
    for i, b in enumerate(blocks):
        r = rows[i % len(rows)]
        M = MS[(3 * i) % len(MS)]
        sc = torch.zeros((N, K // 64), dtype=torch.float16, device=cuda)
        sc[r, b] = 0.5 + i / 7
        W = base.with_scales(sc)
        x = randn((M, K), g).to(BF)
        what = f"{case} row {r} block {b} M={M}"
        out = run_gemv(cuda, x, W, "single live block", what, glu=glu, bias=bias)
        col = (r // 32) * 16 + r % 16 if glu else r
        others = torch.ones(out.shape[1], dtype=torch.bool, device=cuda)
        others[col] = False
        rest = F.silu(torch.ones((), dtype=F64, device=cuda)).to(BF) if glu else torch.zeros((), dtype=BF, device=cuda)
        assert bool((out[:, others] == rest).all()), f"{what}: a column without a live block is not {float(rest)}"
        assert bool((out[:, col] != rest).any()), f"{what}: the live block left no trace"


@pytest.mark.parametrize("K", [128, 192])
def test_every_byte_value(cuda, K):
    """Byte (n + 7 p) mod 256 at byte position p of row n: every position holds all 256 values over the rows. One-hot x
    at every k, even and odd (the low and the high nibble of a byte), picks single products T[c] s that an fp32 output
    must return exactly."""
    N = 256
    g = gen(cuda, K)
    p = torch.arange(K // 2 if K % 128 == 0 else (K + 64) // 2, device=cuda)
    packed = ((torch.arange(N, device=cuda)[:, None] + 7 * p[None, :]) % 256).to(torch.uint8).contiguous()
    codes = nf4.unpack_codes(packed, K)
    sc = (torch.rand((N, K // 64), device=cuda, generator=g) * 3 + 0.25).to(torch.float16)
    W = nf4.NF4Weight(packed, sc, K)
    t64 = nf4.NF4.to(BF).to(F64).to(cuda)
    from vitron_b200 import ops
    for k0 in range(0, K, 32):
        ks = torch.arange(k0, k0 + 32, device=cuda)
        x = torch.zeros((32, K), dtype=BF, device=cuda)
        x[torch.arange(32, device=cuda), ks] = 1
        out = ops.gemm(x_view(x), W, out_fp32=True)
        want = (t64[codes[:, ks].long()] * sc[:, ks // 64].to(F64)).t()
        bad = int((out.to(F64) != want).sum())
        assert bad == 0, f"K={K} k {k0}..{k0 + 31}: {bad} of {out.numel()} products differ"


@pytest.mark.parametrize("M", [9, 17, 32])
def test_one_live_token_row(cuda, vicuna, M):
    """X zero but one token row at 0, 7, 8, 15, 16, 24, 31 or M - 1: every other row of the output is exactly zero (qkv
    with the RMS scale and kscale, o_proj with bias through the region weights)."""
    w = vicuna
    g = gen(cuda, 700 + M)
    for t in sorted({t for t in (0, 7, 8, 15, 16, 24, 31, M - 1) if t < M}):
        x = torch.zeros((M, 4096), dtype=BF, device=cuda)
        x[t] = randn((4096,), g, 3.0).to(BF)
        out = run_gemv(cuda, x, w["qkv"], "one live row", f"qkv row {t} M={M}", rms_eps=EPS, kscale=w["g1"])
        rest = torch.ones(M, dtype=torch.bool, device=cuda)
        rest[t] = False
        assert bool((out[rest] == 0).all()) and bool((out[t] != 0).any()), f"row {t} M={M}"


@pytest.mark.parametrize("rows", [16, 32])
def test_rms_probes(cuda, rows):
    """Token rows whose energy sits only in the last 64-block, only in the odd tail block, or only in one k-slice (one
    row per slice): an RMS sum that misses a block or a slice is off by orders of magnitude."""
    N = 4096 if rows == 16 else edge_n("rows32")
    for K in (4096, 4160):
        g = gen(cuda, rows + K)
        W = rand_w4(g, N, K, spread=2.0)
        plan = nf4_plan(32, N, K)
        assert plan["rows"] == rows
        x = randn((32, K), g, 0.01).to(BF)
        x[0, -64:] = randn((64,), g, 5.0).to(BF)
        x[1, -128:-64] = randn((64,), g, 5.0).to(BF)
        for j, s in enumerate(plan["slices"]):
            x[2 + j, 128 * s["s0"]:min(128 * s["s1"], K)] = randn((min(128 * s["s1"], K) - 128 * s["s0"],), g, 5.0).to(BF)
        for M in (8, 16, 32):
            run_gemv(cuda, x[:M].contiguous(), W, "rms probes", f"rows {rows} K={K} M={M}", rms_eps=EPS)
            ks = (torch.rand((K,), device=cuda, generator=g) + 0.5).contiguous()
            run_gemv(cuda, x[:M].contiguous(), W, "rms probes", f"rows {rows} K={K} M={M} kscale", rms_eps=EPS, kscale=ks)


def test_kscale_probes(cuda):
    """kscale one-hot per block (zero elsewhere) at the probe blocks of 16- and 32-row plans, and kscale spanning
    2^-8 .. 2^8 with one octave per 8 consecutive k (both halves of each lane's 64-block)."""
    for N in (4096, edge_n("rows32")):
        K = 4160
        g = gen(cuda, N)
        W = rand_w4(g, N, K, spread=2.0)
        plan = nf4_plan(17, N, K)
        x = randn((17, K), g).to(BF)
        for b in probe_blocks(plan):
            ks = torch.zeros((K,), device=cuda)
            ks[64 * b:64 * b + 64] = 1.5
            out = run_gemv(cuda, x, W, "kscale probes", f"N={N} block {b}", kscale=ks)
            assert bool((out != 0).any()), f"N={N} block {b}: zero output"
        e = (torch.arange(K, device=cuda) // 8) % 17 - 8
        ks = torch.exp2(e.float()).contiguous()
        run_gemv(cuda, x, W, "kscale probes", f"N={N} octaves", kscale=ks)
        run_gemv(cuda, x, W, "kscale probes", f"N={N} octaves rms", kscale=ks, rms_eps=EPS)
        run_gemv(cuda, x, W, "kscale probes", f"N={N} octaves reversed", kscale=ks.flip(0).contiguous())


# ---------------------------------------------------------------------------------------------------- D: prefill (M > 32)
PREFILL_ROWS = [33, 48, 64, 65, 77, 256, 768]


def run_prefill(cuda, x, W, kscale, group, what, rs=None, **epi):
    """ops.gemm(x, NF4, M > 32) against float64 over the dequantised bf16 weight, and bit-identical to ops.gemm over
    that bf16 weight."""
    from vitron_b200 import ops
    M, K = x.shape
    wd = ((nf4.dequantize(W.w) * kscale[None, :]) if kscale is not None else nf4.dequantize(W.w)).to(BF)
    glu = epi.get("glu", 0)
    buf, out = guarded(M, W.n // 2 if glu else W.n, BF, cuda)
    res = ops.gemm(x_view(x), W.w, kscale=kscale, out=out, **epi)
    assert res.data_ptr() == out.data_ptr()
    check_guards(buf, out, what)
    assert torch.equal(ops.gemm(x, wd, **epi), out), f"{what}: differs from the bf16 GEMM over the dequantised weight"
    a64, w64 = x.to(F64), wd.to(F64)
    r = dict(epi)
    rsx = torch.ones((M, 1), dtype=F64, device=cuda)
    if r.pop("rms_eps", 0.0):
        rsx = rs.to(F64)[:, None]
    v = (a64 @ w64.t()) * rsx
    e = (math.ceil(K / 16) + 8) * U23 * (a64.abs() @ w64.abs().t()) * rsx.abs()
    ref, tol = epi64(v, e, **r)
    close(out, ref, tol, group, what)


@pytest.mark.parametrize("M", PREFILL_ROWS)
def test_prefill_projections(cuda, vicuna, M):
    """The LLaMA prefill calls on NF4 weights (kscale folded by the dequantiser, RMS scale from row_rstd), the
    mm_projector's GELU + bias layer and the region MLP's ReLU + bias layer, rows scaled x1 .. x30."""
    from vitron_b200 import ops
    w = vicuna
    g = gen(cuda, 900 + M)
    for call in ("qkv", "gate_up", "o_proj", "down", "region0", "region1"):
        W = w[call]
        x = (randn((M, W.k), g) * (1 + 29 * torch.rand((M, 1), device=cuda, generator=g))).to(BF)
        what = f"{call} M={M}"
        if call in ("qkv", "gate_up"):
            rs = ops.row_rstd(x, EPS)
            rs64 = torch.rsqrt(x.to(F64).pow(2).mean(-1) + EPS)
            assert bool(((rs.to(F64) - rs64).abs() <= 2.0 ** -16 * rs64).all()), f"{what}: row_rstd"
            run_prefill(cuda, x, W, w["g1"] if call == "qkv" else w["g2"], "prefill", what, rs=rs, rms_eps=EPS,
                        glu=ops.GLU_SWIGLU if call == "gate_up" else 0)
        elif call in ("o_proj", "down"):
            run_prefill(cuda, x, W, None, "prefill", what, residual=randn((M, 4096), g).to(BF))
        else:
            act = ops.ACT_GELU if call == "region0" else ops.ACT_RELU     # mm_projector: GELU; region MLP: ReLU
            run_prefill(cuda, x, W, None, "prefill", what, bias=w["bias"][call], act=act)


@pytest.fixture(scope="module")
def big_nf4(cuda):
    """An NF4 weight whose dequantisation needs more than the current "nf4" workspace (built on first use)."""
    from vitron_b200 import ops
    made = {}

    def get():
        cur = ops._ws.get((torch.cuda.current_device(), "nf4"))
        need = 0 if cur is None else cur.numel()
        K = 4096
        if "w" not in made or 2 * made["w"].n * K <= need:
            N = (need // (2 * K) // 16 + 2) * 16
            made["w"] = rand_w4(gen(cuda, N), N, K, spread=1.0)
        return made["w"]
    return get


def test_prefill_workspace_growth(cuda, vicuna, big_nf4):
    """Two NF4 weights of different sizes alternate at M = 96; the larger one outgrows the workspace. Every result stays
    bit-identical to the first one of its weight."""
    from vitron_b200 import ops
    g = gen(cuda, 1234)
    small = vicuna["region0"]
    big = big_nf4()
    key = (torch.cuda.current_device(), "nf4")
    xs, xb = randn((96, small.k), g).to(BF), randn((96, big.k), g).to(BF)
    first_s = ops.gemm(xs, small.w, act=ops.ACT_RELU, bias=vicuna["bias"]["region0"])
    ws0 = ops._ws[key].data_ptr()
    first_b = ops.gemm(xb, big.w)
    assert ops._ws[key].data_ptr() != ws0, "the larger weight did not grow the workspace"
    for _ in range(2):
        assert torch.equal(ops.gemm(xs, small.w, act=ops.ACT_RELU, bias=vicuna["bias"]["region0"]), first_s)
        assert torch.equal(ops.gemm(xb, big.w), first_b)
    run_prefill(cuda, xb[:40].contiguous(), big, None, "prefill", "grown workspace M=40")


# ---------------------------------------------------------------------------------------------------- E: graphs and PDL
def layer_chain(ops, w, h):
    """qkv -> o_proj (its input: the first 4096 columns of qkv, lda 12288) with the residual in place -> gate / up
    SwiGLU -> down with the residual in place."""
    qkv = engine_call(ops, w, "qkv", h)
    engine_call(ops, w, "o_proj", qkv[:, :4096], h=h)
    act = engine_call(ops, w, "gate_up", h)
    engine_call(ops, w, "down", act, h=h)
    return qkv, h


@pytest.mark.parametrize("M", [8, 17, 32, 33, 64])
def test_graph_pdl_layer_chain(cuda, vicuna, big_nf4, M):
    """The layer chain captured in a CUDA graph under PDL replays bit-identically to an eager run with PDL off, over new
    inputs, and again after the "nf4" workspace has grown (the graph keeps its retired buffer). At M > 32 a capture
    after reserve_nf4_workspace does not move the workspace."""
    from vitron_b200 import ops
    w = vicuna
    key = (torch.cuda.current_device(), "nf4")
    ops.reserve_nf4_workspace([w[n].w for n in ("qkv", "o_proj", "gate_up", "down")], cuda)
    g = gen(cuda, 40 + M)
    inputs = [randn((M, 4096), g).to(BF) for _ in range(3)]

    def eager(h):
        with ops.pdl(False):
            qkv, out = layer_chain(ops, w, h.clone())
        return qkv.clone(), out.clone()

    static = inputs[0].clone()
    s = torch.cuda.Stream(device=cuda)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        layer_chain(ops, w, static.clone())
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    ws = ops._ws.get(key)
    ws_ptr = None if ws is None else ws.data_ptr()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), ops.pdl(True):
        g_qkv, g_h = layer_chain(ops, w, static)
    if M > 32:
        assert ops._ws[key].data_ptr() == ws_ptr, "capture moved the nf4 workspace"
    for x in inputs[1:] + inputs[:1]:
        static.copy_(x)
        graph.replay()
        want_qkv, want_h = eager(x)
        assert torch.equal(g_qkv, want_qkv) and torch.equal(g_h, want_h), f"M={M}: replay differs from eager"
    big = big_nf4()
    ops.gemm(randn((40, big.k), g).to(BF), big.w)         # grows the workspace: the graph keeps the retired one
    assert ops._ws[key].data_ptr() != ws_ptr
    static.copy_(inputs[1])
    graph.replay()
    want_qkv, want_h = eager(inputs[1])
    assert torch.equal(g_qkv, want_qkv) and torch.equal(g_h, want_h), f"M={M}: replay after workspace growth differs"
    if M <= 32:
        (ref, tol), _ = gemv_ref(inputs[1], w["qkv"], nf4_plan(M, 12288, 4096), kscale=w["g1"], rms_eps=EPS)
        close(want_qkv, ref, tol, "graph chain qkv", f"M={M}")


MIDSIZE = dict(hidden_size=512, intermediate_size=1408, num_hidden_layers=2, num_attention_heads=4, vocab_size=2000,
               rms_norm_eps=1e-5, rope_theta=10000.0)


def test_graphed_decode_above_32_rows(cuda):
    """An NF4 LlamaEngine with max_batch = 64 reserves the "nf4" workspace at load; its graphed decode at B = 33 and 64
    (the dequantise + GEMM path inside the captured step, PDL on) gives the token log of the eager step, and the
    capture leaves the workspace where it was."""
    from vitron_b200 import ops
    from vitron_b200.llama import LlamaEngine
    eng = LlamaEngine(MIDSIZE, cuda, max_batch=64, max_seq_len=64).init_random(seed=3, nf4=True)
    assert eng.nf4
    key = (torch.cuda.current_device(), "nf4")
    need = max(2 * w.shape[0] * w.shape[1] for L in eng.layers for w in (L["wqkv"], L["wo"], L["wgu"], L["wdown"]))
    assert ops._ws[key].numel() >= need
    NEW = 8
    for B in (33, 64):
        ids = torch.randint(3, 2000, (B, 12), generator=torch.Generator().manual_seed(B)).to(cuda)
        logs = []
        for use_graph in (True, False, True):
            logits = eng.prefill(eng.embed[ids])
            eng.start_decode(ops.argmax_rows(logits), NEW)
            ptr = ops._ws[key].data_ptr()
            eng.decode_steps(B, NEW - 1, use_graph=use_graph)
            assert ops._ws[key].data_ptr() == ptr, (B, use_graph)
            logs.append(eng.token_log[:B, :NEW].clone())
        assert torch.equal(logs[0], logs[1]) and torch.equal(logs[0], logs[2]), B


# ---------------------------------------------------------------------------------------------------- F: which kernel ran
def check_trace_cases(cuda):
    """Each family launches the gemv_nf4_kernel<ROWS, NT> its plan predicts; M > 32 launches the dequantiser and the
    wgmma GEMM and no GEMV."""
    from vitron_b200 import ops
    g = gen(cuda, 77)
    cases = []
    for M in (1, 8, 9, 16, 17, 32):
        for N, K, glu in [(4096, 4096, 0), (12288, 4096, 0), (edge_n("rows32"), 192, 0), (200, 4160, 0), (224, 64, ops.GLU_SWIGLU)]:
            cases.append((M, N, K, glu))
    for M in (33, 64, 256):
        cases.append((M, 4096, 1024, 0))
        cases.append((M, 224, 192, ops.GLU_GEGLU))
    fails = []
    for M, N, K, glu in cases:
        W = nf4.NF4Weight(torch.randint(0, 256, (N, -(-K // 128) * 64), device=cuda, dtype=torch.int32).to(torch.uint8),
                          torch.full((N, K // 64), 0.01, dtype=torch.float16, device=cuda), K)
        x = randn((M, K), g).to(BF)
        names = kernels_of(lambda: ops.gemm(x, W, glu=glu, rms_eps=EPS))
        vb = sorted(n for n in names if "vb::" in n)
        if M <= 32:
            plan = nf4_plan(M, N, K, bool(glu))
            want, absent = [plan["kernel"]], ["nf4_dequant_kernel", "gemm_v2_kernel"]
            others = [f"gemv_nf4_kernel<{r},{t}>" for r in (16, 32) for t in (1, 2, 4)]
            absent += [o for o in others if o != plan["kernel"]]
        else:
            want, absent = ["nf4_dequant_kernel", "gemm_v2_kernel"], ["gemv_nf4_kernel"]
        for p in want:
            if not launched(names, p):
                fails.append((M, N, K, glu, "missing", p, vb))
        for p in absent:
            if launched(names, p):
                fails.append((M, N, K, glu, "unexpected", p, vb))
    assert not fails, fails
    print(f"trace ok: {len(cases)} calls")


def test_dispatch_branches_in_trace(cuda):
    """check_trace_cases in a fresh Python process: a profiler session in a process that has already captured a CUDA
    graph can come back without kernel records."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import sys; sys.path.insert(0, {root!r}); import torch; import tests.test_nf4_kernels_gpu as t; "
            "t.check_trace_cases(torch.device('cuda:0'))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "trace ok" in r.stdout, (r.stdout[-4000:] + r.stderr[-4000:])


def test_report(cuda):
    """Prints the largest err / tol per group seen in this file."""
    for group, r in sorted(RATIOS.items()):
        print(f"max err/tol {group}: {r:.3f}")
