"""Kernel-level numerics: every C-ABI entry point against a plain torch fp32 reference of the same
op on the same seeded inputs (these are floating-point kernels: tolerance stated per test)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

BF = torch.bfloat16


def rnd(shape, dev, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(BF)


def close(a, b, atol, rtol, what=""):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    tol = atol + rtol * b.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


def act_ref(x, act):
    from vitron_b200 import ops
    return {ops.ACT_NONE: lambda t: t, ops.ACT_GELU: F.gelu, ops.ACT_QUICK_GELU: lambda t: t * torch.sigmoid(1.702 * t),
            ops.ACT_RELU: F.relu, ops.ACT_SILU: F.silu}[act](x)


@pytest.fixture(params=[0, 1], ids=["v2", "generic"])
def gemm_impl(request, cuda):
    """Every GEMM / convolution test runs on both epilogue forms of the ONE wgmma kernel body: the variants specialised by
    feature set (default) and the variants that resolve every epilogue feature at run time. This checks the template
    specialisation; the shared main loop and fragment mapping are checked against the torch references."""
    from vitron_b200 import ops
    prev = ops.set_gemm_impl(request.param)
    yield request.param
    ops.set_gemm_impl(prev)


GEMM_SHAPES = [
    (128, 128, 64), (128, 256, 128), (256, 512, 256), (200, 136, 72), (2056, 1024, 1024),
    (257, 3072, 1024), (1000, 4096, 1024), (6144, 1024, 4096), (101, 512, 512), (77, 1024, 1024),
    (4096, 32000, 128), (130, 8, 64), (300, 48, 128), (1000, 80, 320), (129, 2560, 64), (40960, 320, 320),
    # few tiles, long K: split-K on the v2 kernel
    (640, 1280, 3840), (200, 1280, 5120), (2560, 1280, 11520), (128, 256, 4096), (640, 336, 2048),
    # 17..64 rows with a small weight matrix: persistent kernel with a mostly empty 128-row tile (not the swap-AB path)
    (64, 512, 512), (33, 1024, 1024), (17, 512, 256), (60, 768, 768), (40, 2048, 512),
]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_plain(cuda, gemm_impl, M, N, K):
    from vitron_b200 import ops
    a, w = rnd((M, K), cuda, 1), rnd((N, K), cuda, 2, 0.05)
    out = ops.gemm(a, w)
    ref = a.float() @ w.float().t()
    close(out, ref, 2e-2 * math.sqrt(K / 64), 1.6e-2, f"gemm {M}x{N}x{K}")


@pytest.mark.parametrize("M", [1, 8, 16, 17, 33, 64])
@pytest.mark.parametrize("N,K", [(4096, 4096), (12288, 4096), (4096, 11008), (1000, 520)])
def test_gemm_swap_small_m(cuda, M, N, K):
    from vitron_b200 import ops
    a, w = rnd((M, K), cuda, 3), rnd((N, K), cuda, 4, 0.02)
    bias = rnd((N,), cuda, 5)
    res = rnd((M, N), cuda, 6)
    out = ops.gemm(a, w, bias=bias, residual=res, alpha=0.5)
    ref = res.float() + 0.5 * (a.float() @ w.float().t() + bias.float())
    close(out, ref, 3e-2, 1.6e-2, f"swap gemm {M}x{N}x{K}")


@pytest.mark.parametrize("act", [1, 2, 3, 4])
def test_gemm_bias_act_residual(cuda, gemm_impl, act):
    from vitron_b200 import ops
    M, N, K = 777, 1024, 512
    a, w, bias, res = rnd((M, K), cuda, 1), rnd((N, K), cuda, 2, 0.05), rnd((N,), cuda, 3), rnd((M, N), cuda, 4)
    out = ops.gemm(a, w, bias=bias, act=act)
    ref = act_ref(a.float() @ w.float().t() + bias.float(), act)
    close(out, ref, 3e-2, 1.6e-2, f"act {act}")
    out = ops.gemm(a, w, bias=bias, residual=res, alpha=-0.75)
    ref = res.float() - 0.75 * (a.float() @ w.float().t() + bias.float())
    close(out, ref, 3e-2, 1.6e-2, "residual")
    # in-place residual (out aliases residual)
    res2 = res.clone()
    ops.gemm(a, w, residual=res2, out=res2)
    close(res2, res.float() + a.float() @ w.float().t(), 3e-2, 1.6e-2, "inplace residual")
    out32 = ops.gemm(a, w, out_fp32=True)
    close(out32, a.float() @ w.float().t(), 2e-3, 2e-3, "fp32 out")


@pytest.mark.parametrize("M", [8, 300, 2048])
@pytest.mark.parametrize("glu", [1, 2])
def test_gemm_glu(cuda, gemm_impl, M, glu):
    from vitron_b200 import ops
    K, Fd = 512, 1376
    a = rnd((M, K), cuda, 1)
    wa, wb = rnd((Fd, K), cuda, 2, 0.05), rnd((Fd, K), cuda, 3, 0.05)
    ba, bb = rnd((Fd,), cuda, 4), rnd((Fd,), cuda, 5)
    w = ops.pack_glu_weight(wa, wb)
    b = ops.pack_glu_weight(ba, bb)
    out = ops.gemm(a, w, bias=b, glu=glu)
    xa = a.float() @ wa.float().t() + ba.float()
    xb = a.float() @ wb.float().t() + bb.float()
    ref = F.silu(xa) * xb if glu == 1 else xa * F.gelu(xb)
    close(out, ref, 4e-2, 2e-2, f"glu {glu} M={M}")


def test_gemm_v2_feature_matrix(cuda, gemm_impl):
    """rowscale (folded RMSNorm), rowscale + SwiGLU, residual / alpha through the split-K finaliser, fp32 output, bias-free
    residual, all on shapes that take the specialised variants (and the same calls on the generic kernel)."""
    from vitron_b200 import ops
    M, N, K = 6144, 512, 256
    a, w = rnd((M, K), cuda, 1), rnd((N, K), cuda, 2, 0.05)
    rsc = (torch.rand((M,), device=cuda) + 0.5).float()
    ref = (a.float() @ w.float().t()) * rsc[:, None]
    close(ops.gemm(a, w, rowscale=rsc), ref, 3e-2, 1.6e-2, "rowscale")
    wa, wb = rnd((N, K), cuda, 3, 0.05), rnd((N, K), cuda, 4, 0.05)
    out = ops.gemm(a, ops.pack_glu_weight(wa, wb), glu=1, rowscale=rsc)
    xa, xb = (a.float() @ wa.float().t()) * rsc[:, None], (a.float() @ wb.float().t()) * rsc[:, None]
    close(out, F.silu(xa) * xb, 4e-2, 2e-2, "rowscale + swiglu")
    close(ops.gemm(a, w, rowscale=rsc, out_fp32=True), ref, 2e-3, 2e-3, "rowscale fp32 out")
    # split-K shapes with the whole epilogue in the finaliser
    M, N, K = 640, 1280, 3840
    a, w = rnd((M, K), cuda, 5), rnd((N, K), cuda, 6, 0.02)
    bias, res = rnd((N,), cuda, 7), rnd((M, N), cuda, 8)
    rb = rnd((M // 40, N), cuda, 9)
    ref = a.float() @ w.float().t() + bias.float()
    close(ops.gemm(a, w, bias=bias, residual=res, alpha=0.5), res.float() + 0.5 * ref, 5e-2, 2e-2, "split residual")
    close(ops.gemm(a, w, bias=bias, act=4, rowbias=rb, rowbias_rows=40),
          F.silu(ref + rb.float().repeat_interleave(40, 0)), 5e-2, 2e-2, "split act rowbias")
    wa, wb = rnd((N // 2, K), cuda, 10, 0.02), rnd((N // 2, K), cuda, 11, 0.02)
    out = ops.gemm(a, ops.pack_glu_weight(wa, wb), glu=2)
    close(out, (a.float() @ wa.float().t()) * F.gelu(a.float() @ wb.float().t()), 5e-2, 2e-2, "split geglu")
    close(ops.gemm(a, w, bias=bias, out_fp32=True), ref, 5e-3, 3e-3, "split fp32 out")
    r2 = res.clone()
    ops.gemm(a, w, residual=r2, out=r2)
    close(r2, res.float() + a.float() @ w.float().t(), 5e-2, 2e-2, "split in-place residual")
    # repeated split launches reuse the self-zeroing counters
    for _ in range(3):
        close(ops.gemm(a, w, bias=bias), ref, 5e-2, 2e-2, "split repeat")


@pytest.mark.parametrize("M,N,K", [(40960, 320, 320), (8192, 960, 320), (5000, 640, 192), (4096, 2560, 320), (10240, 640, 640), (4224, 336, 128)])
def test_gemm_resident_b(cuda, M, N, K):
    """The small-K 'weight slab stays in shared memory' variant of the GEMM kernel (and the same call with it switched off):
    plain, residual (in place), GEGLU, activation; M with a ragged last tile, N with a ragged last chunk."""
    from vitron_b200 import ops
    a, w, bias = rnd((M, K), cuda, 1), rnd((N, K), cuda, 2, 0.05), rnd((N,), cuda, 3)
    res = rnd((M, N), cuda, 4)
    ref = a.float() @ w.float().t() + bias.float()
    for rb in (3, 0):
        prev = ops.set_gemm_debug(rb, 0)
        try:
            close(ops.gemm(a, w, bias=bias), ref, 3e-2 * math.sqrt(K / 64), 1.6e-2, f"resb={rb} plain")
            close(ops.gemm(a, w, bias=bias, act=4), F.silu(ref), 3e-2 * math.sqrt(K / 64), 1.6e-2, f"resb={rb} act")
            r2 = res.clone()
            ops.gemm(a, w, bias=bias, residual=r2, out=r2, alpha=0.5)
            close(r2, res.float() + 0.5 * ref, 3e-2 * math.sqrt(K / 64), 1.6e-2, f"resb={rb} residual in place")
            if N % 32 == 0:
                wa, wb = rnd((N // 2, K), cuda, 5, 0.05), rnd((N // 2, K), cuda, 6, 0.05)
                out = ops.gemm(a, ops.pack_glu_weight(wa, wb), glu=2)
                close(out, (a.float() @ wa.float().t()) * F.gelu(a.float() @ wb.float().t()), 4e-2 * math.sqrt(K / 64), 2e-2, f"resb={rb} geglu")
        finally:
            ops.set_gemm_debug(prev & 0xff, 0)


def test_gemm_rowbias_strided(cuda, gemm_impl):
    from vitron_b200 import ops
    M, N, K = 640, 320, 256
    big = rnd((M, K + 64), cuda, 1)
    a = big[:, 8:8 + K]  # strided view: lda = K + 64, base offset 16 bytes
    w = rnd((N, K), cuda, 2, 0.05)
    rb = rnd((M // 64, N), cuda, 3)
    out = ops.gemm(a, w, rowbias=rb, rowbias_rows=64)
    ref = a.float() @ w.float().t() + rb.float().repeat_interleave(64, 0)
    close(out, ref, 3e-2, 1.6e-2, "rowbias")


CONVS = [
    # nb, h, w, cin, cout, kh, kw, stride
    (2, 16, 16, 64, 64, 3, 3, 1), (16, 40, 64, 320, 320, 3, 3, 1), (16, 20, 32, 640, 1280, 3, 3, 1),
    (16, 5, 8, 1280, 1280, 3, 3, 1), (3, 10, 16, 320, 640, 1, 1, 1), (16, 40, 64, 320, 320, 3, 3, 2),
    (4, 9, 13, 128, 96, 3, 3, 2), (2, 16, 2560 // 16, 320, 320, 3, 1, 1), (1, 64, 64, 512, 512, 3, 3, 1),
    (1, 33, 200, 192, 512, 1, 1, 1), (2, 12, 12, 8, 320, 3, 3, 1), (2, 12, 12, 320, 8, 3, 3, 1),
    # few pixel tiles, long K (UNet 1280-channel levels, temporal Conv3d (3,1,1) as kh=3 kw=1): split-K on v2
    (16, 10, 16, 1280, 1280, 3, 3, 1), (1, 16, 40, 1280, 1280, 3, 1, 1), (1, 16, 160, 1280, 1280, 3, 1, 1),
    (16, 5, 8, 2560, 1280, 3, 3, 1), (2, 5, 8, 640, 48, 3, 3, 1),
]


@pytest.mark.parametrize("nb,h,w,cin,cout,kh,kw,stride", CONVS)
def test_conv_nhwc(cuda, gemm_impl, nb, h, w, cin, cout, kh, kw, stride):
    from vitron_b200 import ops
    x = rnd((nb, h, w, cin), cuda, 1)
    wt = rnd((cout, cin, kh, kw), cuda, 2, 0.03)
    bias = rnd((cout,), cuda, 3)
    out = ops.conv_nhwc(x, ops.pack_conv_weight(wt), kh, kw, stride=stride, bias=bias)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias.float(), stride=stride, padding=(kh // 2, kw // 2))
    close(out, ref.permute(0, 2, 3, 1), 4e-2 * math.sqrt(cin * kh * kw / 576), 2e-2, "conv")


def test_conv_epilogue(cuda, gemm_impl):
    from vitron_b200 import ops
    nb, h, w, cin, cout = 4, 20, 32, 128, 256
    x, wt = rnd((nb, h, w, cin), cuda, 1), rnd((cout, cin, 3, 3), cuda, 2, 0.03)
    bias, rb, res = rnd((cout,), cuda, 3), rnd((nb, cout), cuda, 4), rnd((nb, h, w, cout), cuda, 5)
    out = ops.conv_nhwc(x, ops.pack_conv_weight(wt), 3, 3, bias=bias, rowbias=rb, rowbias_rows=h * w, residual=res)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias.float(), padding=1).permute(0, 2, 3, 1)
    ref = res.float() + ref + rb.float()[:, None, None, :]
    close(out, ref, 5e-2, 2e-2, "conv epilogue")
    d = ops.conv_nhwc_direct(x, wt.permute(0, 2, 3, 1).reshape(cout, 9, cin).contiguous(), bias, 3, 3)
    ref2 = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias.float(), padding=1).permute(0, 2, 3, 1)
    close(d, ref2, 5e-2, 2e-2, "direct conv")
    # few-tile convolution (split-K on v2) with the ResBlock epilogue: bias + time-embedding rowbias + residual
    nb, h, w, cin, cout = 16, 5, 8, 1280, 1280
    x, wt = rnd((nb, h, w, cin), cuda, 6), rnd((cout, cin, 3, 3), cuda, 7, 0.01)
    bias, rb, res = rnd((cout,), cuda, 8), rnd((1, cout), cuda, 9), rnd((nb, h, w, cout), cuda, 10)
    out = ops.conv_nhwc(x, ops.pack_conv_weight(wt), 3, 3, bias=bias, rowbias=rb, rowbias_rows=nb * h * w, residual=res)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias.float(), padding=1).permute(0, 2, 3, 1)
    close(out, res.float() + ref + rb.float()[0], 8e-2, 2e-2, "split conv epilogue")


@pytest.mark.parametrize("rows,d", [(7, 4096), (300, 1024), (33, 320), (5, 1280), (3, 11008), (9, 512),
                                    (2001, 320), (1025, 512), (4099, 64), (40960, 320)])
def test_norms(cuda, rows, d):
    from vitron_b200 import ops
    x, w, b = rnd((rows, d), cuda, 1, 2.0), rnd((d,), cuda, 2), rnd((d,), cuda, 3)
    xf = x.float()
    ref = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * w.float()
    close(ops.rmsnorm(x, w, 1e-5), ref, 2e-2, 1e-2, "rmsnorm")
    close(ops.layernorm(x, w, b, 1e-5), F.layer_norm(xf, (d,), w.float(), b.float(), 1e-5), 2e-2, 1e-2, "layernorm")


@pytest.mark.parametrize("n,sp,c,act", [(2, 40960, 320, 4), (32, 2560, 320, 0), (3, 40960, 320, 4), (32, 2560, 640, 4), (8, 128, 64, 4), (8, 128, 64, 0), (8, 128, 64, 3), (16, 40 * 64, 320, 4), (2, 16 * 100, 640, 0), (3, 77, 1280, 4), (1, 64 * 64, 512, 3),
                                        (2, 50, 2560, 4), (2, 33, 960, 4),
                                        (1, 16 * 2560, 320, 4), (1, 16 * 640, 640, 4), (2, 5000, 1920, 0),
                                        # UNet temporal layouts
                                        (1, 16 * 160, 1280, 4), (1, 16 * 40, 1280, 0), (16, 20 * 32, 640, 4),
                                        # narrow groups (VAE: 4 channels per group), fewer rows than a CTA pass, one row
                                        (2, 300, 128, 4), (3, 3, 320, 0), (4, 1, 64, 3), (16, 5 * 8, 2560, 4)])
def test_groupnorm(cuda, n, sp, c, act):
    from vitron_b200 import ops
    x, w, b = rnd((n, sp, c), cuda, 1, 1.5), rnd((c,), cuda, 2), rnd((c,), cuda, 3)
    ref = F.group_norm(x.float().permute(0, 2, 1), 32, w.float(), b.float(), 1e-5).permute(0, 2, 1)
    ref = act_ref(ref, act)
    y1 = ops.groupnorm_nhwc(x, w, b, 32, 1e-5, act=act)
    close(y1, ref, 3e-2, 2e-2, "groupnorm")
    # the workspace hands itself back zeroed: a second call (and an in-place one) must give the same result, bit for bit
    # (the statistics are reduced in a fixed order, never by atomics)
    y2 = ops.groupnorm_nhwc(x, w, b, 32, 1e-5, act=act)
    close(y2, ref, 3e-2, 2e-2, "groupnorm (second call)")
    assert torch.equal(y1, y2), "groupnorm is not bit-reproducible"
    xi = x.clone()
    close(ops.groupnorm_nhwc(xi, w, b, 32, 1e-5, act=act, out=xi), ref, 3e-2, 2e-2, "groupnorm (in place)")


def sdpa_ref(q, k, v, scale, causal=False, kv_len=None, mask=None):
    # q [B,Sq,H,D] -> fp32 eager attention
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    s = qf @ kf.transpose(-1, -2) * scale
    B, H, Sq, Skv = s.shape
    dead = torch.zeros((B, 1, Sq, Skv), dtype=torch.bool, device=q.device)
    lens = kv_len if kv_len is not None else torch.full((B,), Skv, device=q.device)
    kk = torch.arange(Skv, device=q.device)
    dead = dead | (kk[None, None, None, :] >= lens[:, None, None, None])
    if causal:
        qi = torch.arange(Sq, device=q.device)
        dead = dead | (kk[None, None, None, :] > (qi[None, None, :, None] + (Skv - Sq)))
    if mask is not None:
        dead = dead | mask.bool()
    s = s.masked_fill(dead, float("-inf"))
    p = torch.softmax(s, -1).nan_to_num(0.0)
    return (p @ vf).permute(0, 2, 1, 3)


ATT = [
    # B, H, Sq, Skv, D, causal
    (2, 4, 768, 768, 128, True), (8, 16, 257, 257, 64, False), (2, 5, 2560, 2560, 64, False),
    (2, 5, 640, 145, 64, False), (1, 8, 101, 1024, 64, False), (2, 8, 1054, 1054, 40, False),
    (1, 8, 286, 286, 80, False), (1, 8, 94, 94, 160, False), (3, 2, 70, 200, 128, True), (1, 2, 1, 130, 128, True),
]


@pytest.mark.parametrize("B,H,Sq,Skv,D,causal", ATT)
def test_attention(cuda, B, H, Sq, Skv, D, causal):
    from vitron_b200 import ops
    q, k, v = rnd((B, Sq, H, D), cuda, 1), rnd((B, Skv, H, D), cuda, 2), rnd((B, Skv, H, D), cuda, 3)
    out = ops.attention(q, k, v, causal=causal)
    close(out, sdpa_ref(q, k, v, 1 / math.sqrt(D), causal), 2e-2, 2e-2, "attention")


ATT_TC = [
    # B, H, Sq, Skv, D, causal — shapes of the prefill (hd 128, causal), ViT (257, hd 64), UNet spatial (hd 64)
    (2, 4, 768, 768, 128, True), (8, 16, 257, 257, 64, False), (2, 5, 2560, 2560, 64, False),
    (2, 5, 640, 145, 64, False), (1, 8, 101, 1024, 64, False), (3, 2, 70, 200, 128, True),
    (1, 2, 1, 130, 128, True), (1, 3, 130, 1, 64, False), (2, 2, 129, 63, 128, False), (1, 32, 1728, 1728, 128, True),
    # GLIGEN gated self-attention (visual + 30 grounding tokens; heads x 40 / 80 / 160): zero-padded by the TMA unit
    (2, 8, 1054, 1054, 80, False), (2, 8, 286, 286, 160, False), (1, 8, 4126, 4126, 40, False), (2, 3, 200, 77, 40, True),
    # few queries over a long memory: split over the keys + merge kernel (SEEM cross-attention levels)
    (1, 8, 101, 16384, 64, False), (1, 8, 101, 4096, 64, False), (2, 2, 130, 2000, 128, False), (1, 4, 100, 1100, 80, False),
]


@pytest.mark.parametrize("B,H,Sq,Skv,D,causal", ATT_TC)
@pytest.mark.parametrize("amp", [1.0, 6.0])
def test_attention_tcgen05(cuda, B, H, Sq, Skv, D, causal, amp):
    """wgmma flash-attention kernel pinned (impl 2) against the fp32 reference and against the mma.sync kernel; amp 6
    makes row maxima jump by orders of magnitude between key blocks so the running-max rescale of O is exercised."""
    from vitron_b200 import ops
    q, k, v = rnd((B, Sq, H, D), cuda, 1) * amp, rnd((B, Skv, H, D), cuda, 2) * amp, rnd((B, Skv, H, D), cuda, 3)
    ref = sdpa_ref(q, k, v, 1 / math.sqrt(D), causal)
    try:
        ops.set_attention_impl(2)
        out = ops.attention(q, k, v, causal=causal)
        ops.set_attention_impl(1)
        out_mma = ops.attention(q, k, v, causal=causal)
    finally:
        ops.set_attention_impl(0)
    close(out, ref, 2e-2, 2e-2, "wgmma attention")
    close(out, out_mma, 2e-2, 2e-2, "wgmma vs mma.sync")


@pytest.mark.parametrize("B,H,Sq,Skv,D", [(1, 8, 101, 1024, 64), (2, 8, 101, 4096, 64), (2, 4, 300, 1000, 64), (1, 2, 130, 77, 128),
                                          (2, 8, 286, 286, 160)])
def test_attention_tcgen05_bool_mask(cuda, B, H, Sq, Skv, D):
    """SEEM masked cross-attention (101 queries over 32^2 / 64^2 memories, mask shared by the heads) and general
    per-head masks on the wgmma kernel: 16-byte mask rows (Skv % 16 == 0) and the byte-wise path (Skv = 1000, 77)."""
    from vitron_b200 import ops
    q, k, v = rnd((B, Sq, H, D), cuda, 1), rnd((B, Skv, H, D), cuda, 2), rnd((B, Skv, H, D), cuda, 3)
    g = torch.Generator().manual_seed(5)
    for shape in ((B, 1, Sq, Skv), (B, H, Sq, Skv), (1, 1, Sq, Skv)):
        mask = (torch.rand(shape, generator=g) < 0.6).to(cuda)
        mask[0, 0, 5] = True          # a fully masked row -> zeros
        mask[0, 0, 7, :64] = True     # a fully masked first key block followed by live keys
        ref = sdpa_ref(q, k, v, 1 / math.sqrt(D), mask=mask)
        try:
            ops.set_attention_impl(2)
            out = ops.attention(q, k, v, mask=mask)
            ops.set_attention_impl(1)
            out_mma = ops.attention(q, k, v, mask=mask)
        finally:
            ops.set_attention_impl(0)
        close(out, ref, 2e-2, 2e-2, f"wgmma masked attention {shape}")
        close(out, out_mma, 2e-2, 2e-2, "wgmma vs mma.sync (masked)")


def test_attention_tcgen05_layouts(cuda):
    from vitron_b200 import ops
    B, S, H, D = 3, 300, 4, 128
    qkv = rnd((B, S, 3 * H * D), cuda, 1)
    q, k, v = (qkv[..., i * H * D:(i + 1) * H * D].view(B, S, H, D) for i in range(3))
    lens = torch.tensor([300, 17, 129], dtype=torch.int32, device=cuda)
    try:
        ops.set_attention_impl(2)
        out = ops.attention(q, k, v, causal=False, kv_len=lens)
        close(out, sdpa_ref(q, k, v, 1 / math.sqrt(D), False, lens), 2e-2, 2e-2, "kv_len")
        out = ops.attention(q, k, v, causal=True, kv_len=lens)
        ref = sdpa_ref(q, k, v, 1 / math.sqrt(D), True, lens)
        for b, l in enumerate(lens.tolist()):
            close(out[b, :l], ref[b, :l], 2e-2, 2e-2, "causal + kv_len")
        # output written through a strided view ([B, S, H*D] slice of a wider buffer)
        wide = torch.zeros((B, S, 2 * H * D), dtype=torch.bfloat16, device=cuda)
        o = wide[..., H * D:].view(B, S, H, D)
        ops.attention(q, k, v, out=o)
        close(o, sdpa_ref(q, k, v, 1 / math.sqrt(D)), 2e-2, 2e-2, "strided out")
        assert float(wide[..., :H * D].abs().max()) == 0.0
        # head-major [B, H, S, D] storage viewed as [B, S, H, D]
        qh = rnd((B, H, S, D), cuda, 7).permute(0, 2, 1, 3)
        kh = rnd((B, H, S, D), cuda, 8).permute(0, 2, 1, 3)
        vh = rnd((B, H, S, D), cuda, 9).permute(0, 2, 1, 3)
        close(ops.attention(qh, kh, vh), sdpa_ref(qh, kh, vh, 1 / math.sqrt(D)), 2e-2, 2e-2, "head-major")
    finally:
        ops.set_attention_impl(0)


def test_attention_fused_qkv_layout_kvlen_mask(cuda):
    from vitron_b200 import ops
    B, S, H, D = 3, 300, 4, 128
    qkv = rnd((B, S, 3 * H * D), cuda, 1)
    q, k, v = (qkv[..., i * H * D:(i + 1) * H * D].view(B, S, H, D) for i in range(3))
    lens = torch.tensor([300, 17, 129], dtype=torch.int32, device=cuda)
    out = ops.attention(q, k, v, causal=False, kv_len=lens)
    close(out, sdpa_ref(q, k, v, 1 / math.sqrt(D), False, lens), 2e-2, 2e-2, "kv_len")
    out = ops.attention(q, k, v, causal=True, kv_len=lens)  # right-padded prefill
    ref = sdpa_ref(q, k, v, 1 / math.sqrt(D), True, lens)
    for b, l in enumerate(lens.tolist()):
        close(out[b, :l], ref[b, :l], 2e-2, 2e-2, "causal + kv_len")
    g = torch.Generator().manual_seed(5)
    mask = (torch.rand((B, H, S, S), generator=g) < 0.6).to(cuda)
    mask[0, 1, 5] = True  # a fully masked row -> zeros
    out = ops.attention(q, k, v, mask=mask)
    close(out, sdpa_ref(q, k, v, 1 / math.sqrt(D), mask=mask), 2e-2, 2e-2, "bool mask")
    m2 = mask[:1, :1]
    out = ops.attention(q, k, v, mask=m2)
    close(out, sdpa_ref(q, k, v, 1 / math.sqrt(D), mask=m2), 2e-2, 2e-2, "broadcast mask")


@pytest.mark.parametrize("nseq,S,H", [(257 * 2, 8, 16), (640, 16, 5), (100, 16, 8), (7, 32, 3), (5, 3, 2)])
def test_attention_short(cuda, nseq, S, H):
    from vitron_b200 import ops
    # strided "frames-major" layout: tensor [S, nseq, H*64], sequences run along dim 0
    base = rnd((S, nseq, 3, H, 64), cuda, 1)
    q, k, v = (base[:, :, i].permute(1, 0, 2, 3) for i in range(3))
    out = ops.attention_short(q, k, v)
    close(out, sdpa_ref(q, k, v, 1 / 8.0), 2e-2, 2e-2, "short attention")


def test_attention_short_unaligned_rows(cuda):
    """Row pieces that are only 4-byte aligned take the scalar kernel instead of the 16-byte / mma.sync one."""
    from vitron_b200 import ops
    base = rnd((16, 50, 3, 4, 66), cuda, 3)
    q, k, v = (base[:, :, i, :, 2:].permute(1, 0, 2, 3) for i in range(3))
    out = ops.attention_short(q, k, v)
    close(out, sdpa_ref(q, k, v, 1 / 8.0), 2e-2, 2e-2, "short attention (unaligned)")


def rope_ref(x, pos, theta):
    # x [T, H, D] fp32, rotate_half convention
    D = x.shape[-1]
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, device=x.device, dtype=torch.float32) / D))
    ang = pos.float()[:, None] * inv[None, :]
    cos, sin = torch.cat([ang.cos()] * 2, -1)[:, None, :], torch.cat([ang.sin()] * 2, -1)[:, None, :]
    rot = torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1)
    return x * cos + rot * sin


def test_rope_kv_append_and_decode(cuda):
    from vitron_b200 import ops
    B, H, D, PS = 3, 32, 128, 64
    lens = [130, 64, 777]
    max_pages = 16
    npages = B * max_pages
    g = torch.Generator().manual_seed(0)
    perm = torch.randperm(npages, generator=g).to(torch.int32).view(B, max_pages).to(cuda)
    kp = torch.zeros((npages, H, PS, D), dtype=BF, device=cuda)
    vp = torch.zeros_like(kp)
    toks = sum(lens)
    qkv = rnd((toks, 3 * H * D), cuda, 1)
    pos = torch.cat([torch.arange(l) for l in lens]).to(torch.int32).to(cuda)
    bot = torch.cat([torch.full((l,), i) for i, l in enumerate(lens)]).to(torch.int32).to(cuda)
    ref_in = qkv.clone().float().view(toks, 3, H, D)
    ops.rope_kv_append(qkv, pos, H, D, 10000.0, kp, vp, perm, bot, None, PS)
    out = qkv.float().view(toks, 3, H, D)
    close(out[:, 0], rope_ref(ref_in[:, 0], pos, 10000.0), 2e-2, 1e-2, "rope q")
    kref = rope_ref(ref_in[:, 1], pos, 10000.0)
    close(out[:, 1], kref, 2e-2, 1e-2, "rope k")
    close(out[:, 2], ref_in[:, 2], 0, 0, "v untouched")
    # cache content
    off = 0
    for b, l in enumerate(lens):
        for t in (0, l // 2, l - 1):
            page, o = perm[b, t // PS].item(), t % PS
            close(kp[page, :, o], out[off + t, 1], 0, 0, "k cache")
            close(vp[page, :, o], out[off + t, 2], 0, 0, "v cache")
        off += l
    # decode attention over the cache vs dense reference
    qd = rnd((B, 3 * H * D), cuda, 7)
    kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
    o = ops.attn_decode_paged(qd, kp, vp, perm, kvl, H, D, PS, max(lens))
    off = 0
    for b, l in enumerate(lens):
        kk = out[off:off + l, 1].unsqueeze(0).to(BF)
        vv = out[off:off + l, 2].unsqueeze(0).to(BF)
        ref = sdpa_ref(qd[b, :H * D].view(1, 1, H, D), kk, vv, 1 / math.sqrt(D))
        close(o[b].view(H, D), ref[0, 0], 2e-2, 2e-2, f"decode attn b={b}")
        off += l
    # single-split path
    o1 = ops.attn_decode_paged(qd, kp, vp, perm, torch.tensor([100, 64, 1], dtype=torch.int32, device=cuda), H, D, PS, 100)
    kk = out[:100, 1].unsqueeze(0).to(BF); vv = out[:100, 2].unsqueeze(0).to(BF)
    close(o1[0].view(H, D), sdpa_ref(qd[0, :H * D].view(1, 1, H, D), kk, vv, 1 / math.sqrt(D))[0, 0], 2e-2, 2e-2, "decode 1 split")
    # ONE workspace, calls of different batch sizes / head counts in turn (what one engine's per-batch-size graphs do): the
    # partial results a small call leaves behind must never be read as arrival counters by a larger one
    for rep in range(2):
        for bsub, hsub in ((1, 4), (3, 32), (2, 8), (3, 32)):
            kvs = kvl[:bsub].contiguous()
            qs = qd[:bsub].contiguous()
            os_ = ops.attn_decode_paged(qs[:, :3 * hsub * D].contiguous(), kp[:, :hsub].contiguous(), vp[:, :hsub].contiguous(),
                                        perm[:bsub].contiguous(), kvs, hsub, D, PS, max(lens))
            off = 0
            for b in range(bsub):
                l = lens[b]
                kk = out[off:off + l, 1, :hsub].unsqueeze(0).to(BF)
                vv = out[off:off + l, 2, :hsub].unsqueeze(0).to(BF)
                ref = sdpa_ref(qs[b, :hsub * D].view(1, 1, hsub, D), kk, vv, 1 / math.sqrt(D))
                close(os_[b].view(hsub, D), ref[0, 0], 2e-2, 2e-2, f"decode attn shared workspace B={bsub} H={hsub} b={b} rep={rep}")
                off += l


def test_splice_argmax(cuda):
    from vitron_b200 import ops
    V, d = 1000, 4096
    emb, feats = rnd((V, d), cuda, 1), rnd((300, d), cuda, 2)
    src = torch.tensor([[5, 999, -1, -300, -2147483648, 0]], dtype=torch.int32, device=cuda)
    out = ops.splice_multimodal(emb, feats, src)
    ref = torch.stack([emb[5], emb[999], feats[0], feats[299], torch.zeros(d, device=cuda, dtype=BF), emb[0]])
    close(out[0], ref, 0, 0, "splice")
    g = torch.Generator().manual_seed(3)
    logits = torch.randn((9, 32001), generator=g).to(cuda)
    logits[2, 777] = 50.0; logits[2, 31000] = 50.0  # tie -> first index
    assert torch.equal(ops.argmax_rows(logits), logits.argmax(-1)) or ops.argmax_rows(logits)[2].item() == 777
    assert ops.argmax_rows(logits)[2].item() == 777
    lb = logits.to(BF)
    idx = ops.argmax_rows(lb)
    assert torch.equal(lb.float().gather(1, idx[:, None]), lb.float().max(-1, keepdim=True).values)


def test_vision_glue(cuda):
    from vitron_b200 import ops
    px = rnd((3, 3, 224, 224), cuda, 1).float()
    w = rnd((1024, 3, 14, 14), cuda, 2, 0.03)
    A = ops.patchify(px, 14, 640)
    wk = torch.zeros((1024, 640), dtype=BF, device=cuda); wk[:, :588] = w.reshape(1024, 588)
    po = ops.gemm(A, wk)
    ref = F.conv2d(px.to(BF).float(), w.float(), stride=14).flatten(2).transpose(1, 2)
    close(po.view(3, 256, 1024), ref, 4e-2, 2e-2, "patch embed")
    cls, pos, lw, lb = rnd((1024,), cuda, 3), rnd((257, 1024), cuda, 4), rnd((1024,), cuda, 5), rnd((1024,), cuda, 6)
    h = ops.vit_embed_ln(po, cls, pos, lw, lb, 3, 256, 1e-5)
    e = torch.cat([cls.float().expand(3, 1, 1024), po.float().view(3, 256, 1024)], 1) + pos.float()
    close(h, F.layer_norm(e.to(BF).float(), (1024,), lw.float(), lb.float(), 1e-5), 4e-2, 2e-2, "vit embed ln")
    x = rnd((2, 5, 8, 64), cuda, 7)
    up = ops.upsample2x_nhwc(x)
    close(up, F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1), 0, 0, "upsample")
    a, b = rnd((4, 16, 64), cuda, 8), rnd((16, 64), cuda, 9)
    close(ops.add(a, b), (a.float() + b.float()), 1e-2, 1e-2, "add bcast")
    y, u = torch.randn(1000, device=cuda), torch.randn(1000, device=cuda)
    close(ops.cfg_combine(y, u, 9.0), u + 9.0 * (y - u), 1e-5, 1e-5, "cfg")


def test_region_pool_and_seem_mask(cuda):
    from vitron_b200 import ops
    feats = rnd((4, 256, 1024), cuda, 1)
    boxes = torch.tensor([[16., 32., 160., 200.], [0., 0., 224., 224.], [100.5, 3.2, 101.9, 220.], [50., 60., 50., 60.]], device=cuda)
    out = ops.region_mask_pool(feats, boxes, 224)
    for b in range(4):
        m = torch.zeros((224, 224), device=cuda)
        x1, y1, x2, y2 = boxes[b].tolist()
        m[int(x1):int(x2), int(y1):int(y2)] = 1
        m = F.interpolate(m[None, None], size=(16, 16), mode="bilinear", align_corners=False)
        m = (m > 0).float()
        den = m.sum() + 1e-8
        ref = torch.einsum("chw,hw->c", feats[b].float().view(16, 16, 1024).permute(2, 0, 1), (m / den)[0, 0])
        close(out[b], ref, 2e-2, 2e-2, f"region pool {b}")
    lg = torch.randn((7, 64, 64), device=cuda)
    lg[3] = -5.0  # everything masked -> cleared
    mk = ops.seem_attn_mask(lg, 16, 16)
    r = F.interpolate(lg[None], size=(16, 16), mode="bilinear", align_corners=False)[0]
    refm = (r.sigmoid() < 0.5).flatten(1)
    refm[refm.sum(-1) == refm.shape[-1]] = False
    assert torch.equal(mk.bool(), refm)
    mk_same = ops.seem_attn_mask(lg, 64, 64)   # same size: threshold + fully-masked-row reset only
    refs = (lg < 0).flatten(1)
    refs[refs.all(-1)] = False
    assert torch.equal(mk_same.bool(), refs)


@pytest.mark.parametrize("nb,H,W,C,h2,w2", [(1, 256, 256, 512, 32, 32), (1, 256, 256, 512, 128, 128), (2, 36, 52, 64, 9, 13),
                                            (1, 37, 50, 128, 18, 26), (1, 16, 16, 8, 16, 16), (1, 10, 14, 64, 20, 28)])
def test_resize_bilinear_nhwc(cuda, nb, H, W, C, h2, w2):
    """F.interpolate(bilinear, align_corners=False) on NHWC bf16 (SEEM: mask_features resized once per level); also the
    linearity the decoder relies on: resize(E . F) == E . resize(F)."""
    from vitron_b200 import ops
    x = rnd((nb, H, W, C), cuda, 1)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), size=(h2, w2), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    close(ops.resize_bilinear_nhwc(x, h2, w2), ref, 1e-2, 8e-3, "bilinear resize")
    e = rnd((5, C), cuda, 2).float()
    full = torch.einsum("qc,nhwc->nqhw", e, x.float())
    lhs = F.interpolate(full, size=(h2, w2), mode="bilinear", align_corners=False)
    rhs = torch.einsum("qc,nhwc->nqhw", e, ref)
    assert (lhs - rhs).abs().max() < 1e-3 * max(1.0, float(full.abs().max()))


@pytest.mark.parametrize("M", [1, 8, 13, 16, 40, 300])
def test_gemm_fused_rmsnorm(cuda, M):
    """LlamaRMSNorm -> Linear as ONE GEMM on gain-folded weights with a 1/rms row scale."""
    from vitron_b200 import ops
    K, N = 4096, 1024
    x, w, g = rnd((M, K), cuda, 1, 3.0), rnd((N, K), cuda, 2, 0.02), rnd((K,), cuda, 3)
    wf = (w.float() * g.float()[None, :]).to(BF)
    xf = x.float()
    ref = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * g.float()) @ w.float().t()
    close(ops.gemm(x, wf, rms_eps=1e-5), ref, 3e-2, 2e-2, f"fused rms gemm M={M}")
    ga, gb = rnd((512, K), cuda, 4, 0.02), rnd((512, K), cuda, 5, 0.02)
    wp = ops.pack_glu_weight((ga.float() * g.float()).to(BF), (gb.float() * g.float()).to(BF))
    xn = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * g.float()
    refg = F.silu(xn @ ga.float().t()) * (xn @ gb.float().t())
    close(ops.gemm(x, wp, glu=ops.GLU_SWIGLU, rms_eps=1e-5), refg, 3e-2, 3e-2, f"fused rms swiglu M={M}")
    rs = ops.row_rstd(x, 1e-5)
    close(rs, torch.rsqrt(xf.pow(2).mean(-1) + 1e-5), 1e-5, 1e-4, "row_rstd")


def test_attn_decode_rope_fused_equals_unfused(cuda):
    from vitron_b200 import ops
    B, H, D, PS = 4, 32, 128, 64
    lens = [130, 65, 777, 1]          # kv_len INCLUDING the new token
    max_pages = 16
    g = torch.Generator().manual_seed(0)
    perm = torch.randperm(B * max_pages, generator=g).to(torch.int32).view(B, max_pages).to(cuda)
    kp = rnd((B * max_pages, H, PS, D), cuda, 1)
    vp = rnd((B * max_pages, H, PS, D), cuda, 2)
    kp2, vp2 = kp.clone(), vp.clone()
    qkv = rnd((B, 3 * H * D), cuda, 3)
    kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
    pos = kvl - 1
    bot = torch.arange(B, dtype=torch.int32, device=cuda)
    # unfused: rope + append, then paged attention
    q1 = qkv.clone()
    ops.rope_kv_append(q1, pos, H, D, 10000.0, kp, vp, perm, bot, None, PS)
    o1 = ops.attn_decode_paged(q1, kp, vp, perm, kvl, H, D, PS, 1024)
    # fused
    o2 = ops.attn_decode_rope(qkv.clone(), ops.rope_table(pos, D, 10000.0), kp2, vp2, perm, kvl, H, D, PS, 1024)
    close(o2, o1, 1e-2, 1e-2, "fused decode attention")
    close(kp2, kp, 1e-2, 1e-2, "k cache append")
    assert torch.equal(vp2, vp)
