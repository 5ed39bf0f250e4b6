"""GPU: the row norms, the row softmax and the FocalNet / ViT glue kernels against float64 references, on the branches the
CLIP ViT / text, UNet, GLIGEN, SEEM, FocalNet, VAE and LLaMA prefill paths take:
- `ops.layernorm` / `ops.rmsnorm` on every branch of launch_rownorm (`rownorm_warp4_kernel<L>`, `rownorm_warp_kernel<L>`,
  `rownorm_kernel<T, V, L>`), `ops.row_rstd`, `ops.layernorm_add` (`layernorm_add_kernel<MAXV, ROWS>`), `ops.vit_embed_ln`;
- `ops.softmax_rows`, including rows with -inf entries;
- the FocalNet modulation: `ops.dwconv_nhwc` under every `set_dwconv_impl`, `ops.colmean`, `ops.focal_modulate`,
  `ops.mul_rows`; and the one-rounding glue `ops.add`, `ops.add_rowgroup`, `ops.upsample2x_nhwc`;
- Python statements of the host dispatch (launch_rownorm, vb200_layernorm_add, vb200_dwconv_nhwc, colsum_chunks), shown to
  be reached by the cases and checked against the library's workspace sizes and, in a profiler trace, against the kernels
  launched.

References are float64 over the exact bf16 (or fp32) inputs. u = 2^-24 is the fp32 unit roundoff; one fp32 operation
rounded to nearest is off by at most u times its result. A chain of n fp32 additions whose partial sums are bounded by S
is off by at most n u S. The bf16 rounding of an output y' is off by at most 2^-8 |y'|, written below as
2 * 2^-9 |ref| + (1 + 2^-8) E, where E bounds the fp32 error |y' - ref|.

Row norms. Each kernel sums a row in chains of known length n_c: `rownorm_kernel<T, V>` V * 8 per thread, then 5 shuffle
steps and 5 more in the block sum (block_sum: a warp_sum over the T / 32 warp partials padded to 32 lanes), so V * 8 + 10;
`rownorm_warp_kernel` 32 + 5; `rownorm_warp4_kernel` 16 + 5; `layernorm_add_kernel<MAXV, .>` MAXV * 8 + 5;
`vit_embed_ln_kernel` 16 + 5 + 4 (three adds of the warp partials and the division). For LayerNorm:
- mean: mu' = mu + dmu, |dmu| <= (n_c + 1) u mean|x| (the chain and the division);
- variance: sum (x - mu')^2 = sum (x - mu)^2 + d dmu^2 (the cross term vanishes), so dmu enters only to second order; the
  subtraction, the square and the chain cost (n_c + 3) u relative, the division and + eps one more, the square root halves
  it, and rsqrtf is within 2 ulp (4 u): |drstd| <= ((n_c + 4) / 2 + 4) u rstd;
- output (x - mu') rstd w + b: the subtraction, two products and the bias add cost 4 roundings more.
With C = (n_c + 12) u, which covers both (n_c + 1) u and (n_c / 2 + 10) u,
    |y - y_ref| <= 2 * 2^-9 |y_ref| + (1 + 2^-8) (C (mean|x| rstd + |x - mu| rstd + 1) |w| + 2^-22 |b| + 1e-6),
RMSNorm the same with mu = 0 and no mean term. `layernorm_add` adds the residual in fp32 (2^-23 (|res| + |y| + |b|) more).
Between the biased variance the kernels compute and the unbiased one, 1 / (2 d) relative: at d = 64 that is 2^-7, past the
bf16 bound of 2^-8. Dropping or duplicating one element of a random row of 4096 moves rstd by about 2^-13, below the bf16
rounding, so every branch also runs probes: rows where one element dominates the sum of squares (RMS: one element of
sqrt(d - 1) among +-1, so losing it moves rstd by sqrt 2; LN: one outlier on a constant row, whose loss makes the variance
zero), with that element at lane, chunk and VPT boundaries and in the last vector.

row_rstd (fp32 out). A lane adds 4 terms per 8-element vector, ceil(d / 256) vectors, then 5 shuffle steps and the
division: n_c = 4 ceil(d / 256) + 8 roundings relative to the sum of squares, halved by the square root, and rsqrtf's 2 ulp
(2^-22 relative): |r - r_ref| <= ((n_c + 2) 2^-25 + 2^-22) r_ref. At d = 4096 that is 2.4e-6, against 1.2e-4 for one
dropped element of a random row.

softmax_rows. __expf(x) is within 2 + floor(1.17 |x|) ulps (2^-23 relative each). Every probability is the element's own
exponential times the rescale factors of the online maximum (thread loop, 5 shuffle merges, the 8-warp merge: their
arguments sum to at most R, the row's finite range, within each of the 3 stages), summed over k = ceil(n / 256) steps per
thread, 5 shuffle and 8 warp steps, then __expf(x - max) / sum. Counting 1 ulp for every fp32 multiply, add and division,
2 + 1.17 * arg ulps for every __expf and u * R for the rounding of each exponent argument:
    |p - p_ref| <= 2 * 2^-9 |p_ref| + (1 + 2^-8) (4 k + 38 + 8 R) 2^-23 |p_ref| + 2^-126,
where 2^-126 covers the flush to zero of ex2.approx.ftz. One key that wins by 30 nats, dropped from the first pass, moves
every probability by a factor e^30; pairs ln 3 apart among -inf entries must come out as 0.75 / 0.25 within the bf16 ulp.

dwconv. Each output is K^2 fp32 FMAs in tap order, each off by at most u times a partial sum bounded by S = sum |x w| over
the in-bounds taps: tau = (K^2 + 2) 2^-23 (twice the rounding, as the GEMM bound of the sister file) times S. GELU
(gelu_erf_fast: A&S 7.1.26, |erf error| <= 1.5e-7, with rcp.approx and ex2.approx (2^-22) and ~6 FMA roundings inside,
together <= 7.5e-7 < 2^-20, and two more roundings in 0.5 x + 0.5 |x| erf): |gelu' - gelu(v)| <= 1.13 tau S + 0.5 |v| 2^-19,
an absolute error for v << 0, where the result is a cancellation. Impulse images (one non-zero pixel per channel, no GELU)
make every output a single exact product, so it must equal bf16(w * v) bit for bit: a flipped, transposed or shifted tap
fails exactly.

colmean (fp32 out). colsum_partial_kernel adds ceil(rows_per_chunk / nrl) rows per row lane, the finalise adds nrl lanes,
then ceil(nchunks / 32) chunks per lane and 32 lanes: n_c = ceil(rpc / nrl) + nrl + ceil(nchunks / 32) + 32 additions,
then * (1 / t) (two roundings): |m - m_ref| <= (n_c + 3) u mean|x|; with GELU (erff, 2 ulp, and three products):
1.13 E + |m| 2^-21.

focal_modulate. nlev FMAs on top of glob * g_L, then * scale: (nlev + 3) u scale sum_l |ctx_l g_l| + |glob g_L|, then bf16.
mul_rows (a bf16 x bf16 product is exact in fp32), add and add_rowgroup (an fp32 add rounded once to bf16, as torch does)
and upsample2x (a copy) must be bit-identical to torch.

No bound here was widened after a run: each is the expression above."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
U23 = 2.0 ** -23
BF_REL = 2.0 ** -8            # 2 * 2^-9
L_ACT = 1.13
RATIOS = {}                   # test group -> largest err / tol seen


# ---------------------------------------------------------------------------------------------------- helpers
def gen(cuda, seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, device=g.device, generator=g, dtype=F32) * scale + shift


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


def exact(out, ref, group, what):
    """Bit-identical (NaN where ref is NaN)."""
    same = (out == ref) | (out.isnan() & ref.isnan())
    RATIOS[group] = max(RATIOS.get(group, 0.0), 0.0 if bool(same.all()) else float("inf"))
    if not bool(same.all()):
        idx = [int(i) for i in torch.nonzero(~same)[0]]
        raise AssertionError(f"{what}: {int((~same).sum())}/{same.numel()} elements differ; first at {idx}: "
                             f"got {float(out[tuple(idx)])!r}, want {float(ref[tuple(idx)])!r}")


def kernels_of(fn):
    """Names (spaces removed) of the CUDA kernels `fn` launches, from a torch.profiler trace kept in memory; a trace that
    came back without any of this library's kernels is taken again."""
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


def guarded(rows, cols, dtype, device, col_off=8, pad=24):
    """A NaN-filled buffer with a guard row above and below and `pad` guard columns around an out= view [rows, cols]
    starting at column col_off (row stride cols + pad > cols)."""
    buf = torch.full((rows + 2, cols + pad), float("nan"), dtype=dtype, device=device)
    return buf, buf[1:1 + rows, col_off:col_off + cols]


def check_guards(buf, view, what):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    r0 = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    keep.view(-1)[torch.as_strided(torch.arange(buf.numel(), device=buf.device), view.shape, view.stride(), r0).reshape(-1)] = False
    n = int((~buf[keep].isnan()).sum())
    assert n == 0, f"{what}: {n} elements written outside the out= view"


def strided_rows(x, poison=1000.0, off=8, pad=16):
    """x [rows, d] as a view at column `off` of a wider buffer holding `poison` in the other columns."""
    rows, d = x.shape
    big = torch.full((rows, d + pad), poison, dtype=x.dtype, device=x.device)
    big[:, off:off + d] = x
    return big[:, off:off + d]


# ---------------------------------------------------------------------------------------------------- dispatch statements
MAX_ROWNORM_D = 512 * 8 * 4


def rownorm_plan(rows, d):
    """Statement of launch_rownorm (norm.cu): (kernel-name prefix, template args before L, n_c) or None (unsupported)."""
    if d <= 512 and rows >= 1024:
        return "rownorm_warp4_kernel", "", 16 + 5
    if d <= 1024 and rows >= 64:
        return "rownorm_warp_kernel", "", 32 + 5
    for t, v in ((128, 1), (256, 1), (256, 2), (256, 4), (512, 4)):
        if d <= t * 8 * v:
            return "rownorm_kernel", f"{t},{v},", v * 8 + 10
    return None


def rownorm_kernel_name(rows, d, layer):
    name, args, _ = rownorm_plan(rows, d)
    return f"{name}<{args}{'true' if layer else 'false'}>"


def lnadd_plan(d):
    """Statement of vb200_layernorm_add's dispatch: (MAXV, ROWS)."""
    return (1, 4) if d <= 256 else (2, 4) if d <= 512 else (4, 2) if d <= 1024 else (8, 1)


def dwconv_plan(impl, k):
    """Statement of vb200_dwconv_nhwc's dispatch: (kernel name, S)."""
    if impl >= 2 or (impl == 0 and k >= 7):
        s = 32 if impl == 3 else 16
        return f"dwconv_gelu_pair_kernel<{k},{s}>", s
    s = 8 if k <= 5 else 4
    return f"dwconv_gelu_kernel<{k},{s}>", s


def colsum_chunks(t):
    """Statement of colsum_chunks (focal.cu)."""
    return max(1, min(-(-t // 16), 2 * sms()))


def colmean_chain(t, c):
    nch = colsum_chunks(t)
    rpc = -(-t // nch)
    nrl = 256 // (c // 8)
    return -(-rpc // nrl) + nrl + -(-nch // 32) + 32


# ---------------------------------------------------------------------------------------------------- A: row norms
def norm_ref(x, w, b, eps, layer, n_c):
    """float64 LayerNorm / RMSNorm of bf16 x [rows, d] and the bound of the module docstring."""
    x64, w64 = x.to(F64), w.to(F64)
    b64 = b.to(F64) if b is not None else torch.zeros_like(w64)
    mu = x64.mean(-1, keepdim=True) if layer else torch.zeros_like(x64[:, :1])
    xc = x64 - mu
    rstd = 1.0 / torch.sqrt((xc * xc).mean(-1, keepdim=True) + eps)
    y = xc * rstd * w64 + b64
    C = (n_c + 12) * U
    mean_term = x64.abs().mean(-1, keepdim=True) * rstd if layer else 0.0
    err = C * (mean_term + xc.abs() * rstd + 1.0) * w64.abs() + 2.0 ** -22 * b64.abs() + 1e-6
    return y, BF_REL * y.abs() + (1 + BF_REL) * err


def norm_operands(g, rows, d, shift=0.0, bias=True):
    x = randn((rows, d), g, 1.0, shift).to(BF)
    w = randn((d,), g, 0.5, 1.0).to(BF)
    b = randn((d,), g, 0.5).to(BF) if bias else None
    return x, w, b


def run_norm(cuda, x, w, b, eps, layer, group, what, strided_x=True):
    """ops.layernorm / ops.rmsnorm of x (optionally as a poisoned strided view) into a guarded out= view; checks the
    guards, the bound, a bit-identical repeat and a bit-identical in-place run."""
    from vitron_b200 import ops
    rows, d = x.shape
    _, _, n_c = rownorm_plan(rows, d)
    xin = strided_rows(x) if strided_x else x
    buf, out = guarded(rows, d, BF, cuda)
    if layer:
        ops.layernorm(xin, w, b, eps, out=out)
    else:
        ops.rmsnorm(xin, w, eps, out=out)
    check_guards(buf, out, what)
    ref, tol = norm_ref(x, w, b, eps, layer, n_c)
    close(out, ref, tol, group, what)
    again = ops.layernorm(x, w, b, eps) if layer else ops.rmsnorm(x, w, eps)
    assert torch.equal(again, out), f"{what}: repeat / contiguous run differs"
    xi = x.clone()
    if layer:
        ops.layernorm(xi, w, b, eps, out=xi)
    else:
        ops.rmsnorm(xi, w, eps, out=xi)
    assert torch.equal(xi, out), f"{what}: in place differs"
    return out


# (rows, d) per branch: ragged d, d = 8, small d, the branch edges (rows 63 / 64 and 1023 / 1024; d 512 / 520, 1024 / 1032,
# 2048 / 2056, 4096 / 4104, 8192 / 8200) and the model calls
ROWNORM_CASES = {
    "warp4": [(1024, 8), (1024, 64), (1024, 264), (1025, 512), (4099, 320), (2048, 192), (1100, 384), (1031, 504),
              (40960, 320), (4096, 512)],
    "warp": [(64, 8), (64, 64), (1023, 512), (1024, 520), (64, 1024), (77, 1024), (101, 512), (257 * 8, 1024),
             (300, 640), (65, 768), (200, 1000), (1024, 1024), (99, 264)],
    "cta128": [(63, 1024), (1, 8), (8, 1000), (63, 64), (2, 264), (8, 512)],
    "cta256x1": [(1, 1032), (100, 1280), (40, 1536), (7, 2048), (3, 1000 + 1000)],
    "cta256x2": [(3, 2056), (40, 4096), (5, 3000)],
    "cta256x4": [(3, 4104), (2, 8192), (2, 6000)],
    "cta512x4": [(2, 8200), (2, 16384), (3, 10000)],
}
BRANCH_OF = {"warp4": "rownorm_warp4_kernel", "warp": "rownorm_warp_kernel", "cta128": "rownorm_kernel128,1,",
             "cta256x1": "rownorm_kernel256,1,", "cta256x2": "rownorm_kernel256,2,", "cta256x4": "rownorm_kernel256,4,",
             "cta512x4": "rownorm_kernel512,4,"}


def branch_key(rows, d):
    name, args, _ = rownorm_plan(rows, d)
    return name + args


@pytest.mark.parametrize("layer", [True, False], ids=["ln", "rms"])
@pytest.mark.parametrize("branch", list(ROWNORM_CASES))
def test_rownorm_branches(cuda, branch, layer):
    """Every case of the branch, at row means 0, 16 and 200 spreads from zero, with and without a bias."""
    g = gen(cuda, 10 + len(branch) * 7 + layer)
    for i, (rows, d) in enumerate(ROWNORM_CASES[branch]):
        assert branch_key(rows, d) == BRANCH_OF[branch], (rows, d)
        for shift in (0.0, 16.0, 200.0) if layer else (0.0, 16.0):
            x, w, b = norm_operands(g, rows, d, shift, bias=layer and (i + int(shift)) % 2 == 0)
            run_norm(cuda, x, w, b, 1e-5 if layer else 1e-6, layer, f"rownorm {'ln' if layer else 'rms'}",
                     f"{branch} {rows}x{d} shift {shift} bias {b is not None}")


def probe_positions(rows, d):
    """Element positions where a dropped or duplicated vector shows: the first and last element, lane ends of the
    first pass, the first element of every later pass (VPT / chunk boundaries) and the last vector."""
    name, args, _ = rownorm_plan(rows, d)
    stride = 256 if "warp" in name else int(args.split(",")[0]) * 8
    ps = {0, 7, 8, d - 8, d - 1, min(d - 1, 8 * 31), min(d - 1, 8 * 31 + 7), min(d - 1, 8 * 32)}
    ps |= {p for p in range(stride, d, stride)} | {p - 1 for p in range(stride, d, stride)}
    return sorted(p for p in ps if 0 <= p < d)


@pytest.mark.parametrize("layer", [True, False], ids=["ln", "rms"])
@pytest.mark.parametrize("branch", list(ROWNORM_CASES))
def test_rownorm_probes(cuda, branch, layer):
    """One element dominating the row's sum of squares, at each boundary position, for every d of the branch."""
    g = gen(cuda, 70 + len(branch) + layer)
    for rows0, d in ROWNORM_CASES[branch]:
        ps = probe_positions(rows0, d)
        rows = max(rows0, len(ps))
        if branch_key(rows, d) != BRANCH_OF[branch]:
            continue
        w = randn((d,), g, 0.5, 1.0).to(BF)
        b = randn((d,), g, 0.5).to(BF) if layer else None
        if layer:
            x = torch.full((rows, d), 3.0, device=cuda)
            a = 64.0
        else:
            x = torch.where(torch.rand((rows, d), device=cuda, generator=g) < 0.5, -1.0, 1.0)
            a = float(torch.tensor(math.sqrt(d - 1)).to(BF))
        for r in range(rows):
            x[r, ps[r % len(ps)]] = (3.0 + a) if layer else a
        run_norm(cuda, x.to(BF), w, b, 1e-5 if layer else 1e-6, layer, f"rownorm probes {'ln' if layer else 'rms'}",
                 f"{branch} probes {rows}x{d}", strided_x=False)


def test_rownorm_unsupported_and_3d_out(cuda):
    """d > 16384 is refused; a 3-D out= view whose rows share one stride is written in place."""
    from vitron_b200 import ops
    g = gen(cuda, 90)
    x = randn((2, 16392), g).to(BF)
    w = torch.ones((16392,), dtype=BF, device=cuda)
    with pytest.raises(RuntimeError):
        ops.layernorm(x, w, None, 1e-5)
    with pytest.raises(RuntimeError):
        ops.rmsnorm(x, w, 1e-6)
    for B, S, d in ((2, 77, 1024), (3, 500, 320), (1, 9, 4096)):
        xs, wt, bs = norm_operands(g, B * S, d, 1.0)
        big = torch.full((B, S, d + 16), float("nan"), dtype=BF, device=cuda)
        out = big[:, :, 8:8 + d]
        ops.layernorm(xs.view(B, S, d), wt, bs, 1e-5, out=out)
        ref, tol = norm_ref(xs, wt, bs, 1e-5, True, rownorm_plan(B * S, d)[2])
        close(out.reshape(B * S, d), ref, tol, "rownorm ln", f"3-D out {B}x{S}x{d}")
        assert bool(big[:, :, :8].isnan().all() and big[:, :, 8 + d:].isnan().all())
        if B > 1:
            with pytest.raises(ValueError):
                ops.layernorm(xs.view(B, S, d)[:, :S - 1], wt, bs, 1e-5,
                              out=torch.empty((B, S + 1, d), dtype=BF, device=cuda)[:, :S - 1])


# ---------------------------------------------------------------------------------------------------- B: row_rstd
def rstd_ref(x, eps):
    d = x.shape[1]
    r = 1.0 / torch.sqrt((x.to(F64) ** 2).mean(-1) + eps)
    n_c = 4 * -(-d // 256) + 8
    return r, ((n_c + 2) * 2.0 ** -25 + 2.0 ** -22) * r


@pytest.mark.parametrize("rows,d", [(1, 4096), (40, 4096), (2113 * 2, 4096), (7, 264), (33, 1000), (5, 8), (9, 4104),
                                    (3, 16384)])
def test_row_rstd(cuda, rows, d):
    """The prefill token counts at d = 4096, ragged d, and ldx > d with poisoned padding columns."""
    from vitron_b200 import ops
    g = gen(cuda, rows + d)
    x = randn((rows, d), g, 1.0, 0.3).to(BF)
    for xin, what in ((x, "contiguous"), (strided_rows(x, 1e4), "ldx > d")):
        r = ops.row_rstd(xin, 1e-5)
        ref, tol = rstd_ref(x, 1e-5)
        close(r, ref, tol, "row_rstd", f"{rows}x{d} {what}")


# ---------------------------------------------------------------------------------------------------- C: layernorm_add
LNADD_CASES = [(8, 5), (192, 4097), (192, 1), (264, 6), (384, 1027), (512, 3), (520, 7), (768, 1025), (1024, 2),
               (1032, 9), (1536, 257), (2048, 3)]


def lnadd_ref(x, w, b, res, eps):
    d = x.shape[1]
    maxv, _ = lnadd_plan(d)
    y, tol = norm_ref(x, w, b, eps, True, maxv * 8 + 5)
    if res is None:
        return y, tol
    r64 = res.to(F64)
    b64 = b.to(F64).abs() if b is not None else 0.0
    ref = r64 + y
    return ref, BF_REL * ref.abs() + (tol - BF_REL * y.abs()) + (1 + BF_REL) * U23 * (r64.abs() + y.abs() + b64)


@pytest.mark.parametrize("d,rows", LNADD_CASES)
def test_layernorm_add(cuda, d, rows):
    """All four instantiations, ROWS tails, residual / bias None, in place on the residual, mean offsets."""
    from vitron_b200 import ops
    g = gen(cuda, 300 + d + rows)
    for shift, use_res, use_b in ((0.0, True, True), (16.0, True, False), (200.0, False, True), (3.0, False, False)):
        x, w, b = norm_operands(g, rows, d, shift, bias=use_b)
        res = randn((rows, d), g, 2.0).to(BF) if use_res else None
        xin = strided_rows(x)
        rin = strided_rows(res, 7.0, off=16, pad=24) if use_res else None
        buf, out = guarded(rows, d, BF, cuda)
        ops.layernorm_add(xin, w, b, rin, 1e-5, out=out)
        check_guards(buf, out, f"layernorm_add {rows}x{d}")
        ref, tol = lnadd_ref(x, w, b, res, 1e-5)
        close(out, ref, tol, "layernorm_add", f"{rows}x{d} shift {shift} res {use_res} bias {use_b}")
        if use_res:
            ri = res.clone()
            ops.layernorm_add(x, w, b, ri, 1e-5, out=ri)
            assert torch.equal(ri, out), f"layernorm_add in place {rows}x{d}"


# ---------------------------------------------------------------------------------------------------- D: vit_embed_ln
@pytest.mark.parametrize("d", [8, 1000, 1024, 2048])
def test_vit_embed_ln(cuda, d):
    """nb in {1, 8}, npatch in {1, 255, 256}, distinct position rows; the reference rounds src + pos to bf16 first."""
    from vitron_b200 import ops
    g = gen(cuda, 500 + d)
    for nb in (1, 8):
        for npatch in (1, 255, 256):
            po = randn((nb * npatch, d), g, 1.0, 0.5).to(BF)
            cls = randn((d,), g).to(BF)
            pos = randn((npatch + 1, d), g, 2.0).to(BF)
            w, b = randn((d,), g, 0.5, 1.0).to(BF), randn((d,), g, 0.5).to(BF)
            out = ops.vit_embed_ln(po, cls, pos, w, b, nb, npatch, 1e-5)
            src = torch.cat([cls.view(1, 1, d).expand(nb, 1, d), po.view(nb, npatch, d)], 1)
            h = (src + pos.view(1, npatch + 1, d)).reshape(-1, d)          # bf16 + bf16: one rounding, as HF
            ref, tol = norm_ref(h, w, b, 1e-5, True, 16 + 5 + 4)
            close(out.reshape(-1, d), ref, tol, "vit_embed_ln", f"nb {nb} npatch {npatch} d {d}")


# ---------------------------------------------------------------------------------------------------- E: softmax_rows
SOFTMAX_N = [1, 7, 255, 256, 257, 2560, 4096]


def softmax_ref(x):
    """float64 softmax of fp32 x [rows, n] and the bound of the module docstring (R over each row's finite entries)."""
    x64 = x.to(F64)
    p = torch.softmax(x64, -1)
    fin = torch.isfinite(x64)
    hi = torch.where(fin, x64, torch.full_like(x64, -math.inf)).amax(-1, keepdim=True)
    lo = torch.where(fin, x64, torch.full_like(x64, math.inf)).amin(-1, keepdim=True)
    R = (hi - lo).clamp_min(0).nan_to_num(0.0)
    k = -(-x.shape[1] // 256)
    eps = (4 * k + 38 + 8 * R) * U23
    return p, BF_REL * p.abs() + (1 + BF_REL) * eps * p.abs() + 2.0 ** -126


def run_softmax(cuda, x, group, what):
    from vitron_b200 import ops
    rows, n = x.shape
    xin = strided_rows(x, 1000.0, off=5, pad=13)                          # +1000 in the padding wins the row if read
    buf, out = guarded(rows, n, BF, cuda, col_off=3, pad=11)
    ops.softmax_rows(xin, out=out)
    check_guards(buf, out, what)
    ref, tol = softmax_ref(x)
    close(out, ref, tol, group, what)
    return out


@pytest.mark.parametrize("n", SOFTMAX_N)
def test_softmax_rows(cuda, n):
    """Random rows (range ~ 30 nats) and probe rows: one key winning by 30 nats at i % 256 in {0, 255}, at n - 1 and in
    the last partial pass."""
    g = gen(cuda, 700 + n)
    x = randn((37, n), g, 4.0, -3.0)
    run_softmax(cuda, x, "softmax", f"random n {n}")
    ps = sorted({p for p in (0, 255, 256, 511, n - 1, (n - 1) // 256 * 256, n - 2, 300, 2559) if 0 <= p < n})
    xp = randn((len(ps), n), g, 1.0)
    for r, p in enumerate(ps):
        xp[r, p] = float(xp[r].max()) + 30.0
    run_softmax(cuda, xp, "softmax", f"probes n {n}")


@pytest.mark.parametrize("n", SOFTMAX_N)
def test_softmax_rows_inf(cuda, n):
    """Rows with -inf entries: at every thread's first position, everywhere but two entries ln 3 apart in different
    threads or warps (p = 0.75 / 0.25), and everywhere (NaN, as torch)."""
    from vitron_b200 import ops
    g = gen(cuda, 800 + n)
    rows = []
    x = randn((4, n), g, 2.0)
    x[:, : min(n, 256)] = -math.inf
    if n > 256:
        rows.append(x)
    pairs = [(i, j) for i, j in ((0, 1), (0, 33), (5, 200), (255, n - 1), (31, 32), (0, 256), (100, n - 1)) if i < j < n]
    if pairs:
        y = torch.full((len(pairs), n), -math.inf, device=cuda)
        for r, (i, j) in enumerate(pairs):
            y[r, i] = 0.5
            y[r, j] = 0.5 + math.log(3.0)
        rows.append(y)
    z = randn((3, n), g, 2.0)
    z[:, ::3] = -math.inf
    if n > 1:
        rows.append(z)
    first = randn((2, n), g)
    first[:, 0] = -math.inf
    if n > 1:
        rows.append(first)
    if rows:
        xi = torch.cat(rows)
        out = run_softmax(cuda, xi, "softmax -inf", f"-inf rows n {n}")
        assert not bool(out.isnan().any())
        if pairs:
            y_out = out[-len(pairs) - (3 + 2 if n > 1 else 0):][:len(pairs)]
            for r, (i, j) in enumerate(pairs):
                assert float(y_out[r, i]) == 0.25 and float(y_out[r, j]) == 0.75, (n, i, j)
    allinf = torch.full((2, n), -math.inf, device=cuda)
    assert bool(ops.softmax_rows(allinf).isnan().all()) and bool(torch.softmax(allinf, -1).isnan().all())


# ---------------------------------------------------------------------------------------------------- F: dwconv
def dw_ref(x, wt, k, gelu):
    """float64 depthwise conv of x [nb, h, w, c] with wt [k*k, c], S = the same conv of |x| and |w|, and the bound."""
    c = x.shape[-1]
    xn = x.to(F64).permute(0, 3, 1, 2)
    wk = wt.to(F64).t().reshape(c, 1, k, k)
    v = F.conv2d(xn, wk, padding=k // 2, groups=c).permute(0, 2, 3, 1)
    S = F.conv2d(xn.abs(), wk.abs(), padding=k // 2, groups=c).permute(0, 2, 3, 1)
    E = (k * k + 2) * U23 * S
    if not gelu:
        return v, BF_REL * v.abs() + (1 + BF_REL) * E
    y = 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    return y, BF_REL * y.abs() + (1 + BF_REL) * (L_ACT * E + 0.5 * v.abs() * 2.0 ** -19) + 1e-30


def dw_input(x):
    """x [nb, h, w, c] as the [..., C:2C] slice of a 2C + 8-wide row (FocalNet's ctx), other columns poisoned."""
    nb, h, w, c = x.shape
    big = torch.full((nb, h, w, 2 * c + 8), 300.0, dtype=BF, device=x.device)
    big[..., c:2 * c] = x
    return big[..., c:2 * c]


DW_C = [8, 24, 192, 1536]


class dw_mode:
    def __init__(self, impl):
        self.impl = impl

    def __enter__(self):
        from vitron_b200 import ops
        self.prev = ops.set_dwconv_impl(self.impl)

    def __exit__(self, *exc):
        from vitron_b200 import ops
        ops.set_dwconv_impl(self.prev)
        return False


def dw_shapes(impl, k):
    """(h, w) pairs: w in {1, R, S - 1, S, S + 1, 2S + R}, h in {1, K - 1} (K + 2 for the widest)."""
    _, S = dwconv_plan(impl, k)
    R = k // 2
    ws = [1, R, S - 1, S, S + 1, 2 * S + R]
    return [(h, w) for w in ws for h in (1, k - 1)] + [(k + 2, 2 * S + R)]


@pytest.mark.parametrize("k", [3, 5, 7, 9, 11])
@pytest.mark.parametrize("impl", [0, 1, 2, 3])
def test_dwconv(cuda, impl, k):
    """nb = 3 (a batch-stride error reads the neighbouring image), c cycling through 8 / 24 / 192 / 1536, with and
    without GELU, input the ctx slice of the projection's rows."""
    from vitron_b200 import ops
    g = gen(cuda, 900 + 10 * impl + k)
    with dw_mode(impl):
        for i, (h, w) in enumerate(dw_shapes(impl, k)):
            c = DW_C[i % len(DW_C)]
            x = randn((3, h, w, c), g, 1.0, 0.2).to(BF)
            wt = randn((k * k, c), g, 0.3).to(BF)
            for gelu in (False, True):
                out = ops.dwconv_nhwc(dw_input(x), wt, k, act=ops.ACT_GELU if gelu else ops.ACT_NONE)
                ref, tol = dw_ref(x, wt, k, gelu)
                close(out, ref, tol, "dwconv", f"impl {impl} k {k} {h}x{w}x{c} gelu {gelu}")


@pytest.mark.parametrize("k", [3, 5, 7, 9, 11])
@pytest.mark.parametrize("impl", [0, 1, 2, 3])
def test_dwconv_impulses(cuda, impl, k):
    """One non-zero pixel per channel (corners, strip boundaries, the image centre), no GELU: every output is a single
    exact product and must equal bf16(w[ky, kx] * v) bit for bit."""
    from vitron_b200 import ops
    g = gen(cuda, 950 + 10 * impl + k)
    _, S = dwconv_plan(impl, k)
    R = k // 2
    with dw_mode(impl):
        for h, w, c in ((k + 2, 2 * S + R, 24), (1, S + 1, 8), (2 * k, 3 * S + 1, 192)):
            spots = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (h // 2, w // 2), (0, min(w - 1, S - 1)),
                     (h - 1, min(w - 1, S)), (h // 2, min(w - 1, 2 * S - 1)), (h // 2, min(w - 1, R))]
            x = torch.zeros((3, h, w, c), dtype=F32, device=cuda)
            vals = randn((3, c), g, 1.0, 0.1)
            for n in range(3):
                for ch in range(c):
                    y0, x0 = spots[(ch + n) % len(spots)]
                    x[n, y0, x0, ch] = vals[n, ch]
            x = x.to(BF)
            wt = randn((k * k, c), g).to(BF)
            out = ops.dwconv_nhwc(dw_input(x), wt, k)
            ref, _ = dw_ref(x, wt, k, False)
            exact(out, ref.to(BF), "dwconv impulses", f"impl {impl} k {k} {h}x{w}x{c}")


# ---------------------------------------------------------------------------------------------------- G: colmean, modulation
def colmean_cases():
    """(nb, t, c): t in {1, 15, 16, 17, 70000}, the chunk-count cap and one past it, rows_per_chunk / nrl edges."""
    cap = 2 * sms()
    return [(1, 1, 8), (3, 15, 192), (1, 16, 1536), (3, 17, 2048), (1, 70000, 8), (3, 70000, 192), (1, 16 * cap, 1536),
            (3, 16 * cap + 1, 2048), (1, 257, 8), (3, 255, 1536), (1, 4 * 16 * cap + 3, 192), (1, 4096, 768)]


def colmean_ref(x, act):
    nb, t, c = x.shape
    x64 = x.to(F64)
    m = x64.mean(1)
    E = (colmean_chain(t, c) + 3) * U * x64.abs().mean(1)
    if not act:
        return m, E + 1e-30
    y = 0.5 * m * (1.0 + torch.erf(m / math.sqrt(2.0)))
    return y, L_ACT * E + m.abs() * 2.0 ** -21 + 1e-30


@pytest.mark.parametrize("case", range(12))
def test_colmean(cuda, case):
    """Non-zero means, a single large row at the first and last row of a chunk and at t - 1, bit-identical repeats."""
    from vitron_b200 import ops
    nb, t, c = colmean_cases()[case]
    g = gen(cuda, 1000 + case)
    nch = colsum_chunks(t)
    rpc = -(-t // nch)
    x = randn((nb, t, c), g, 1.0, 0.7)
    spots = sorted({0, t - 1, min(t - 1, rpc - 1), min(t - 1, rpc), min(t - 1, (nch - 1) * rpc)})
    for n in range(nb):
        x[n, spots[n % len(spots)]] += 1000.0
        x[n, spots[-1 - n % len(spots)]] -= 500.0
    x = x.to(BF)
    for act in (ops.ACT_NONE, ops.ACT_GELU):
        out = ops.colmean(x, nb, act=act)
        ref, tol = colmean_ref(x, act == ops.ACT_GELU)
        close(out, ref, tol, "colmean", f"{nb}x{t}x{c} act {act}")
        assert torch.equal(ops.colmean(x, nb, act=act), out), "colmean repeat differs"


@pytest.mark.parametrize("nlev", [1, 2, 3, 4, 5, 6])
def test_focal_modulate_mul_rows(cuda, nlev):
    """focal_modulate with the gates as the projection's column-2C view, then mul_rows with the q view: bound, then
    bit-identical to torch's bf16 product."""
    from vitron_b200 import ops
    g = gen(cuda, 1100 + nlev)
    for nb, t, c in ((1, 33, 192), (3, 257, 384), (2, 64, 1536)):
        proj = randn((nb * t, 2 * c + 8), g).to(BF)                       # q | ctx | gates (+ padding)
        q, gates = proj[:, :c], proj[:, 2 * c:]
        levels = [randn((nb * t, c), g, 0.5, 0.1 * l).to(BF) for l in range(nlev)]
        glob = randn((nb, c), g, 0.3)
        scale = 1.0 / (nlev + 1)
        out = ops.focal_modulate(levels, gates, glob, nb, scale)
        gl = gates[:, :nlev + 1].to(F64)
        bidx = torch.arange(nb * t, device=cuda) // t
        terms = [levels[l].to(F64) * gl[:, l:l + 1] for l in range(nlev)] + [glob.to(F64)[bidx] * gl[:, nlev:nlev + 1]]
        ref = scale * sum(terms)
        S = scale * sum(t_.abs() for t_ in terms)
        close(out, ref, BF_REL * ref.abs() + (1 + BF_REL) * (nlev + 3) * U * S + 1e-30, "focal_modulate",
              f"nlev {nlev} {nb}x{t}x{c}")
        prod = ops.mul_rows(q, out)
        exact(prod, q * out, "mul_rows", f"{nb * t}x{c}")
        prod2 = ops.mul_rows(gates[:, :8], proj[:, c:c + 8])
        exact(prod2, gates[:, :8] * proj[:, c:c + 8], "mul_rows", f"gate view {nb * t}x8")


# ---------------------------------------------------------------------------------------------------- H: one-rounding glue
def test_add_upsample_bit_identical(cuda):
    """add (plain, broadcast period, in place), add_rowgroup (the video tower's temporal embedding, in place) and
    upsample2x against torch, bit for bit."""
    from vitron_b200 import ops
    g = gen(cuda, 1200)
    for n in (8, 1000, 257 * 1024, 4096 * 5 + 8):
        a, b = randn((n,), g, 3.0).to(BF), randn((n,), g).to(BF)
        exact(ops.add(a, b), a + b, "add", f"add {n}")
        ai = a.clone()
        ops.add(ai, b, out=ai)
        exact(ai, a + b, "add", f"add in place {n}")
    for rows, period in ((64, 320), (1024, 1024 * 3)):
        a, b = randn((rows, period), g).to(BF), randn((period,), g).to(BF)
        exact(ops.add(a, b), a + b, "add", f"broadcast {rows}x{period}")
    for nb, T, N, d in ((1, 8, 257, 1024), (2, 8, 50, 64), (3, 1, 7, 8)):
        x = randn((nb * T * N, d), g, 2.0).to(BF)
        table = randn((T, d), g).to(BF)
        ref = x + table[(torch.arange(nb * T * N, device=cuda) // N) % T]
        exact(ops.add_rowgroup(x, table, N, T), ref, "add_rowgroup", f"{nb}x{T}x{N}x{d}")
        xi = x.clone()
        ops.add_rowgroup(xi, table, N, T, out=xi)
        exact(xi, ref, "add_rowgroup", f"in place {nb}x{T}x{N}x{d}")
    for nb, h, w, c in ((1, 5, 8, 320), (2, 40, 64, 8), (3, 1, 1, 1280)):
        x = randn((nb, h, w, c), g).to(BF)
        exact(ops.upsample2x_nhwc(x), x.repeat_interleave(2, 1).repeat_interleave(2, 2), "upsample2x", f"{nb}x{h}x{w}x{c}")


# ---------------------------------------------------------------------------------------------------- I: dispatch reach
def test_case_list_reaches_every_branch(cuda):
    """The cases of this file reach every branch of the dispatch statements on this device, and colsum_chunks agrees
    with the library's workspace size."""
    from vitron_b200 import _lib
    lib = _lib.load()
    reached = {branch_key(r, d) for cases in ROWNORM_CASES.values() for r, d in cases}
    assert reached == set(BRANCH_OF.values()), reached
    assert rownorm_plan(1, MAX_ROWNORM_D + 8) is None and rownorm_plan(1, MAX_ROWNORM_D) is not None
    edges = {(r, d) for cases in ROWNORM_CASES.values() for r, d in cases}
    for r_lo, r_hi in ((63, 64), (1023, 1024)):
        assert any(r == r_lo for r, _ in edges) and any(r == r_hi for r, _ in edges)
    for d_lo in (512, 1024, 2048, 4096, 8192):
        assert any(d == d_lo for _, d in edges) and any(d == d_lo + 8 for _, d in edges), d_lo
    assert {lnadd_plan(d) for d, _ in LNADD_CASES} == {(1, 4), (2, 4), (4, 2), (8, 1)}
    assert {r % 4 for d, r in LNADD_CASES if lnadd_plan(d)[1] == 4} >= {1, 2, 3}
    dw = {dwconv_plan(impl, k)[0] for impl in range(4) for k in (3, 5, 7, 9, 11)}
    assert dw == {f"dwconv_gelu_kernel<{k},{8 if k <= 5 else 4}>" for k in (3, 5, 7, 9, 11)} | \
                 {f"dwconv_gelu_pair_kernel<{k},{s}>" for k in (3, 5, 7, 9, 11) for s in (16, 32)}
    cap = 2 * sms()
    chunks = {colsum_chunks(t) for _, t, _ in colmean_cases()}
    assert 1 in chunks and cap in chunks and any(1 < n < cap for n in chunks)
    assert any(-(-t // colsum_chunks(t)) % (4 * (256 // (c // 8))) for _, t, c in colmean_cases())   # tail loop runs
    for nb, t, c in colmean_cases():
        assert lib.vb200_colmean_workspace_size(nb, t, c) == nb * colsum_chunks(t) * c * 4, (nb, t, c)


# ---------------------------------------------------------------------------------------------------- J: which kernel ran
def check_trace_cases(cuda):
    """Each case family launches the instantiation the statements predict; every instantiation is launched."""
    from vitron_b200 import ops
    g = gen(cuda, 1900)
    want, seen = [], set()

    def case(fn, present, what):
        names = kernels_of(fn)
        want.append((names, present, what))

    for cases in ROWNORM_CASES.values():
        for layer in (True, False):
            rows, d = cases[0]
            x, w, b = norm_operands(g, rows, d)
            fn = (lambda x=x, w=w, b=b: ops.layernorm(x, w, b, 1e-5)) if layer else (lambda x=x, w=w: ops.rmsnorm(x, w, 1e-6))
            case(fn, [rownorm_kernel_name(rows, d, layer)], (rows, d, layer))
    x = randn((40, 4096), g).to(BF)
    case(lambda: ops.row_rstd(x, 1e-5), ["row_rstd_kernel"], "row_rstd")
    for d, rows in LNADD_CASES:
        x, w, b = norm_operands(g, rows, d)
        mv, rw = lnadd_plan(d)
        case(lambda x=x, w=w, b=b: ops.layernorm_add(x, w, b, x, 1e-5), [f"layernorm_add_kernel<{mv},{rw}>"], (d, rows))
    po, cls, pos = randn((256, 1024), g).to(BF), randn((1024,), g).to(BF), randn((257, 1024), g).to(BF)
    wv = torch.ones((1024,), dtype=BF, device=cuda)
    case(lambda: ops.vit_embed_ln(po, cls, pos, wv, wv, 1, 256, 1e-5), ["vit_embed_ln_kernel"], "vit_embed_ln")
    s = randn((4, 2560), g)
    case(lambda: ops.softmax_rows(s), ["softmax_rows_kernel"], "softmax")
    for impl in range(4):
        for k in (3, 5, 7, 9, 11):
            x = randn((1, 5, 40, 192), g).to(BF)
            wt = randn((k * k, 192), g).to(BF)

            def fn(x=x, wt=wt, impl=impl, k=k):
                with dw_mode(impl):
                    ops.dwconv_nhwc(x, wt, k, act=ops.ACT_GELU)
            case(fn, [dwconv_plan(impl, k)[0]], (impl, k))
    x = randn((2, 1000, 192), g).to(BF)
    case(lambda: ops.colmean(x, 2, act=ops.ACT_GELU), ["colsum_partial_kernel", "colmean_finalize_kernel"], "colmean")
    lv = [randn((64, 192), g).to(BF) for _ in range(3)]
    gt = randn((64, 8), g).to(BF)
    gb = randn((1, 192), g)
    case(lambda: ops.focal_modulate(lv, gt, gb, 1, 0.25), ["focal_modulate_kernel"], "focal_modulate")
    case(lambda: ops.mul_rows(lv[0], lv[1]), ["mul_rows_kernel"], "mul_rows")
    case(lambda: ops.add(lv[0], lv[1]), ["add_kernel"], "add")
    case(lambda: ops.add_rowgroup(lv[0], lv[1][:4], 16, 4), ["add_rowgroup_kernel"], "add_rowgroup")
    u = randn((1, 4, 4, 64), g).to(BF)
    case(lambda: ops.upsample2x_nhwc(u), ["upsample2x_kernel"], "upsample2x")
    for names, present, what in want:
        for p in present:
            assert launched(names, p), (what, p, sorted(n for n in names if "vb::" in n))
            seen.add(p)
        # no other instantiation of the same family
        fam = present[0].split("<")[0] + "<"
        others = [n for n in names if fam in n and not any(p.replace(" ", "") in n for p in present)]
        assert not others, (what, others)
    every = {rownorm_kernel_name(r, d, l) for cases in ROWNORM_CASES.values() for r, d in cases[:1] for l in (True, False)}
    every |= {f"layernorm_add_kernel<{a},{b}>" for a, b in ((1, 4), (2, 4), (4, 2), (8, 1))}
    every |= {dwconv_plan(i, k)[0] for i in range(4) for k in (3, 5, 7, 9, 11)}
    assert every <= seen, sorted(every - seen)
    print(f"trace ok: {len(want)} calls, {len(seen)} instantiations")


def test_dispatch_branches_in_trace(cuda):
    """check_trace_cases in a fresh Python process: a profiler session in a process that has already captured a CUDA
    graph (other test files do) can come back without kernel records."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import sys; sys.path.insert(0, {root!r}); import torch; import tests.test_norms_softmax_focal_gpu as t; "
            "t.check_trace_cases(torch.device('cuda:0'))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "trace ok" in r.stdout, (r.stdout[-4000:] + r.stderr[-4000:])


def test_report(cuda):
    """Prints the largest err / tol per group seen in this file."""
    for group, r in sorted(RATIOS.items()):
        print(f"max err/tol {group}: {r:.3f}")
