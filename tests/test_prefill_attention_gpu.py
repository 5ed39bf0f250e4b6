"""GPU: the attention kernels off the decode path against float64 references, on the branches the models take:
- `ops.attention` on the wgmma kernel (`flash_attn_tc_kernel<64|128|192, TcAttnParams>`): head dims 40-160, tile and block
  edges, the model sizes (ViT, LLaMA prefill, UNet spatial, GLIGEN, SEEM), causal with Skv != Sq, right-padded kv_len,
  boolean masks, GLIGEN's fused qkv rows;
- its split-KV path with `attn_split_merge_kernel`, on every branch of the split policy;
- `ops.attention_paged` (`<128, TcPagedParams>`) over shuffled, poisoned pages, split and unsplit;
- the mma.sync kernel (`flash_attn_kernel<48|64|80|128|160>`): the UNet cross-attention call with stride-0 K / V, LLaMA
  prefill below 96 tokens, CLIP text, masks;
- `ops.attention_short` in the 4-D and the 5-D layouts of the UNet and the video tower, on both kernels;
- probes (one or two keys that dominate a row) at block edges, causal diagonals, split boundaries and kv_len, padding
  columns that hold 1000, NaN-filled output buffers around strided `out=` views, and a trace of the launched kernels.

Tolerance. The kernels round P to bf16 before P·V while l is summed from the unrounded fp32 p, then round O to bf16.
Each rounding is at most 2^-8 relative, so per output element
    |O - O_ref| <= C_TOL * 2^-9 * (|O_ref| + sum_j p_j |v_j|) + 1e-6,          C_TOL = 2,
with O_ref and sum_j p_j |v_j| from float64 attention over the same bf16 operands. The other error sources are orders of
magnitude below that term at the amplitudes used (|q| <= 6 (N(0, 1) + 0.5), |k|, |v| ~ N(0, 1)): an fp32 score of D <= 160
products is off by ~ D * 2^-24 * sum |q k| * scale < 1e-4 nats, which moves p by 1e-4 relative (2^-8 = 3.9e-3);
ex2.approx is within 2^-22 relative; fp32 accumulation of P·V adds ~ 2^-23 * sum p |v|. attn_short_kernel keeps P in fp32,
so its bound drops the sum p |v| term except for an fp32 allowance (__expf is within ~1e-5 relative at these scores)."""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

BF, F64 = torch.bfloat16, torch.float64
C_TOL = 2.0                       # see the module docstring; every kernel stays within it
U9 = 2.0 ** -9
FP32_SLOP = 2.0 ** -14            # attn_short_kernel: fp32 P, relative to sum p |v|
PAD, PAD_VAL = 64, 1000.0         # columns past D in every Q / K / V row, holding 1000
POISON_K, POISON_V = 1000.0, -50.0
RATIOS = {}                       # test group -> largest err / tol seen


# ---------------------------------------------------------------------------------------------------- helpers
def gen(cuda, seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, device=g.device, generator=g, dtype=torch.float32) * scale + shift


def padded(x, pad=PAD):
    """bf16 copy of x [..., D] as a view into rows of D + pad columns; the padding holds PAD_VAL, so a kernel that reads
    past D takes a 1000 into its dot products."""
    buf = torch.full(tuple(x.shape[:-1]) + (x.shape[-1] + pad,), PAD_VAL, dtype=BF, device=x.device)
    buf[..., :x.shape[-1]] = x.to(BF)
    return buf[..., :x.shape[-1]]


def sentinel_out(shape, device, grow=(0, 2, 1, 8)):
    """A NaN-filled buffer larger than `shape` in every dim by `grow`, and the out= view [:shape] of it."""
    buf = torch.full(tuple(s + e for s, e in zip(shape, grow)), float("nan"), dtype=BF, device=device)
    return buf, buf[tuple(slice(0, s) for s in shape)]


def check_sentinel(buf, shape, what):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    keep[tuple(slice(0, s) for s in shape)] = False
    n = int((~buf[keep].isnan()).sum())
    assert n == 0, f"{what}: {n} elements written outside the out= view"


class impl:
    """vb200_set_attention_impl for the duration of a block (0 = automatic afterwards)."""

    def __init__(self, n):
        self.n = n

    def __enter__(self):
        from vitron_b200 import ops
        ops.set_attention_impl(self.n)

    def __exit__(self, *exc):
        from vitron_b200 import ops
        ops.set_attention_impl(0)
        return False


def reference(q, k, v, scale, causal=False, kv_len=None, mask=None, probes=None):
    """float64 attention over the bf16 operands q [B, Sq, H, D], k / v [B, Skv, H, D] (any strides): key j is visible to
    query i iff j < kv_len[b], j <= i + Skv - Sq (causal) and mask[b, h, i, j] == 0; a row without visible keys is 0.
    Returns (O, A) with A = sum_j p_j |v_j|. probes {(b, h): [keys]}: asserts that in every row that sees a probe key, the
    probe keys outweigh every other key by >= 30 nats, and that a visible pair splits its weight 3:1."""
    B, Sq, H, D = q.shape
    Skv = k.shape[1]
    dev = q.device
    O = torch.zeros((B, Sq, H, D), dtype=F64, device=dev)
    A = torch.zeros_like(O)
    i = torch.arange(Sq, device=dev)[:, None]
    j = torch.arange(Skv, device=dev)[None, :]
    hc = max(1, int(2e8 // (Sq * Skv * 8 * 4)))           # heads per chunk: the score block stays under ~200 MB
    for b in range(B):
        kvl = Skv if kv_len is None else int(kv_len[b])
        vis = j < kvl
        if causal:
            vis = vis & (j <= i + (Skv - Sq))
        vis = vis.expand(Sq, Skv)
        for h0 in range(0, H, hc):
            hs = slice(h0, min(H, h0 + hc))
            qh = q[b, :, hs].to(F64).transpose(0, 1)
            kh = k[b, :, hs].to(F64).transpose(0, 1)
            vh = v[b, :, hs].to(F64).transpose(0, 1)
            ok = vis[None]
            if mask is not None:
                mb = mask[b if mask.shape[0] > 1 else 0]
                ok = ok & ~(mb[hs] if mb.shape[0] > 1 else mb).bool()
            s = (qh @ kh.transpose(1, 2)) * scale
            s = s.masked_fill(~ok, float("-inf"))
            m = s.amax(-1, keepdim=True)
            p = torch.exp(s - torch.where(torch.isinf(m), torch.zeros_like(m), m))
            l = p.sum(-1, keepdim=True)
            w = p / torch.where(l > 0, l, torch.ones_like(l))
            O[b, :, hs] = (w @ vh).transpose(0, 1)
            A[b, :, hs] = (w @ vh.abs()).transpose(0, 1)
            for (bb, h), keys in (probes or {}).items():
                if bb != b or not h0 <= h < hs.stop:
                    continue
                wh, okh = w[h - h0], ok[min(h - h0, ok.shape[0] - 1)]
                rows = okh[:, keys].any(-1)
                if not bool(rows.any()):
                    continue
                rest = wh[rows].clone()
                rest[:, keys] = 0
                top = wh[rows][:, keys].max(-1).values
                assert bool((rest.max(-1).values <= top * math.exp(-30)).all()), ("probe margin", b, h, keys)
                if len(keys) == 2:
                    both = okh[:, keys].all(-1)
                    if bool(both.any()):
                        pw = wh[both][:, keys]
                        assert bool(((pw[:, 0] - 0.75).abs() < 0.02).all() and ((pw[:, 1] - 0.25).abs() < 0.02).all()), \
                            ("pair weights", b, h, keys)
    return O, A


def check(out, ref, absum, group, what, short=False):
    """The bound of the module docstring, element by element; records the largest err / tol of the group."""
    ref = ref.to(out.device)
    if short:
        tol = C_TOL * U9 * ref.abs() + FP32_SLOP * absum + 1e-6
    else:
        tol = C_TOL * U9 * (ref.abs() + absum) + 1e-6
    ratio = ((out.to(F64) - ref).abs() / tol).nan_to_num(float("inf"))
    r = float(ratio.max()) if ratio.numel() else 0.0
    RATIOS[group] = max(RATIOS.get(group, 0.0), r)
    if r > 1:
        idx = [int(x) for x in torch.nonzero(ratio > 1)[0]]
        n = int((ratio > 1).sum())
        raise AssertionError(f"{what}: {n}/{ratio.numel()} elements over the bound, max err/tol {r:.3g}; first at "
                             f"{idx}: got {float(out[tuple(idx)]):.6g}, want {float(ref[tuple(idx)]):.6g}")


def operands(g, B, Sq, Skv, H, D, amp):
    """q = amp (N(0, 1) + 0.5): every row's component sum is positive, so a poisoned key (all components POISON_K) that
    is read takes the whole row; k, v ~ N(0, 1). Each a view into rows padded with PAD_VAL."""
    return (padded(randn((B, Sq, H, D), g, amp, 0.5 * amp)), padded(randn((B, Skv, H, D), g)),
            padded(randn((B, Skv, H, D), g)))


def poison(k, v, b, keys, h=slice(None)):
    k[b, keys, h] = POISON_K
    v[b, keys, h] = POISON_V


def run_attention(cuda, q, k, v, group, what, causal=False, kv_len=None, mask=None, use=0, probes=None):
    """ops.attention into the out= view of a NaN-filled buffer: checks the bound and the bytes around the view."""
    from vitron_b200 import ops
    B, Sq, H, D = q.shape
    buf, out = sentinel_out((B, Sq, H, D), cuda)
    kvl = None if kv_len is None else torch.tensor(kv_len, dtype=torch.int32, device=cuda)
    with impl(use):
        res = ops.attention(q, k, v, causal=causal, kv_len=kvl, mask=mask, out=out)
    assert res.data_ptr() == out.data_ptr()
    check_sentinel(buf, (B, Sq, H, D), what)
    ref, absum = reference(q, k, v, 1.0 / math.sqrt(D), causal, kv_len, mask, probes)
    check(out, ref, absum, group, what)
    return out


def tc_splits(B, H, Sq, Skv, causal):
    """Statement of tc_splits() (attention_tc.cu) on this device."""
    if causal:
        return 1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = -(-Sq // 128) * H * B
    nblk = -(-Skv // 64)
    if ctas * 2 > sms or nblk < 8:
        return 1
    s = min(-(-2 * sms // ctas), nblk // 4, 32)
    return 1 if s < 2 else s


def split_plan(B, H, Sq, Skv, causal=False):
    """splits, key blocks per split, and which bound set the split count."""
    s = tc_splits(B, H, Sq, Skv, causal)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nblk = -(-Skv // 64)
    raw = -(-2 * sms // (-(-Sq // 128) * H * B))
    per = -(-nblk // s)
    return dict(splits=s, per=per, nblk=nblk, quarter_cap=s > 1 and s == nblk // 4 and raw > s,
                cap32=s == 32 and raw > 32 and nblk // 4 > 32, empty=s > 1 and per * (s - 1) >= nblk)


def paged_splits(B, H, Sq, max_kv_len):
    """Statement of paged_splits() (attention_tc.cu) on this device."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = -(-Sq // 128) * H * B
    nblk = -(-max_kv_len // 64)
    if ctas * 2 > sms or nblk < 4:
        return 1
    s = min(2 * sms // ctas, nblk // 2, 32)
    return 1 if s < 2 else s


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


# ---------------------------------------------------------------------------------------------------- A: wgmma kernel
EDGES = [(1, 1), (1, 129), (63, 64), (64, 65), (65, 63), (127, 128), (128, 127), (129, 129), (129, 1), (200, 65)]


@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("D", [40, 64, 80, 128, 160])
def test_wgmma_edges(cuda, D, amp):
    """Sq / Skv at 1, 63, 64, 65, 127, 128, 129, causal and not (Skv < Sq leaves the first causal rows without keys: zeros),
    on the wgmma kernel (pinned: below 96 queries the automatic choice is the mma.sync kernel)."""
    g = gen(cuda, 10 * D + int(amp))
    for Sq, Skv in EDGES:
        q, k, v = operands(g, 2, Sq, Skv, 3, D, amp)
        for causal in (False, True):
            run_attention(cuda, q, k, v, "wgmma edges", f"D {D} amp {amp} Sq {Sq} Skv {Skv} causal {causal}",
                          causal=causal, use=2)


# name: (B, H, Sq, Skv, D, causal)
MODEL = {
    "vit-257": (2, 16, 257, 257, 64, False),
    "openclip-vit-257-d80": (1, 16, 257, 257, 80, False),
    "prefill-768": (1, 32, 768, 768, 128, True),
    "prefill-1728": (1, 8, 1728, 1728, 128, True),
    "chunk-200-over-457": (1, 8, 200, 457, 128, True),       # causal with Skv > Sq
    "unet-spatial-2560": (2, 5, 2560, 2560, 64, False),
    "gligen-1054-d80": (2, 8, 1054, 1054, 80, False),
    "gligen-286-d160": (2, 8, 286, 286, 160, False),
    "gligen-4126-d40": (1, 8, 4126, 4126, 40, False),
    "seem-101x1024": (1, 8, 101, 1024, 64, False),
    "seem-101x4096": (1, 8, 101, 4096, 64, False),
    "seem-101x16384": (1, 8, 101, 16384, 64, False),
}


@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("name", list(MODEL))
def test_wgmma_model_shapes(cuda, name, amp):
    """The models' attention shapes on the automatic kernel choice (wgmma; SEEM's few-query shapes split over the keys);
    repeated calls are bit-identical."""
    B, H, Sq, Skv, D, causal = MODEL[name]
    q, k, v = operands(gen(cuda, 100 + len(name)), B, Sq, Skv, H, D, amp)
    out = run_attention(cuda, q, k, v, "wgmma model shapes", f"{name} amp {amp}", causal=causal)
    from vitron_b200 import ops
    assert torch.equal(ops.attention(q, k, v, causal=causal), out), f"{name}: repeat differs"


KV_LENS = [0, 300, 64, 65, 63, 128, 1, 193]


@pytest.mark.parametrize("use", [0, 1])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [40, 128])
def test_kv_len_every_row(cuda, D, causal, use):
    """Right-padded rows (kv_len 0, Skv, 64, 65, 63, 128, 1, 193): keys at or past kv_len hold poison, and every query
    row is checked, including rows at or past kv_len (they attend to the first kv_len keys; kv_len 0 gives zeros)."""
    B, H, S = len(KV_LENS), 2, 300
    q, k, v = operands(gen(cuda, 300 + D), B, S, S, H, D, 1.0)
    for b, L in enumerate(KV_LENS):
        poison(k, v, b, slice(L, S))
    out = run_attention(cuda, q, k, v, "kv_len", f"D {D} causal {causal} impl {use}", causal=causal, kv_len=KV_LENS,
                        use=use)
    assert int(out[0].count_nonzero()) == 0, "kv_len 0 row is not zero"


def make_mask(g, shape, Skv, dev):
    """Random uint8 mask (1 = masked) of `shape` [Bm, Hm, Sq, Skv] with edge rows: row 0 fully masked, row 1 with its
    first 64-key block masked then random, row 2 with only the last key live; keys 100..163 are masked in every row (the
    caller poisons them)."""
    m = torch.rand(shape, generator=g, device=dev) < 0.5
    m[:, :, 0] = True
    m[:, :, 1, :64] = True
    m[:, :, 2] = True
    m[:, :, 2, -1] = False
    m[..., 100:164] = True
    return m


MASK_CASES = {   # name: (B, H, Sq, Skv, D, mask shape (1 = broadcast))
    "seem-cross-per-batch": (2, 8, 101, 1024, 64, "b1"),      # seem.py: [bs, 1, Q, HW]; few queries: split over the keys
    "seem-self-per-batch": (2, 8, 130, 130, 64, "b1"),
    "gligen-cross-per-batch-d40": (2, 8, 256, 286, 40, "b1"),  # gligen.py: [B, 1, N, M]
    "per-head-d80": (2, 4, 129, 300, 80, "bh"),
    "broadcast-d128": (3, 4, 200, 257, 128, "11"),
    "broadcast-d160": (2, 2, 97, 190, 160, "11"),
}


@pytest.mark.parametrize("use", [0, 1])
@pytest.mark.parametrize("name", list(MASK_CASES))
def test_bool_masks(cuda, name, use):
    """Boolean masks per batch, per head and broadcast, on the wgmma kernel (impl 0) and the mma.sync kernel (impl 1,
    which loads masked keys and must drop them): masked-everywhere keys hold poison."""
    B, H, Sq, Skv, D, kind = MASK_CASES[name]
    g = gen(cuda, 400 + len(name))
    q, k, v = operands(g, B, Sq, Skv, H, D, 1.0)
    shape = {"b1": (B, 1, Sq, Skv), "bh": (B, H, Sq, Skv), "11": (1, 1, Sq, Skv)}[kind]
    mask = make_mask(g, shape, Skv, cuda)
    for b in range(B):
        poison(k, v, b, slice(100, 164))
    out = run_attention(cuda, q, k, v, "masks", f"{name} impl {use}", mask=mask, use=use)
    assert int(out[:, 0].count_nonzero()) == 0, "fully masked row is not zero"


@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("nq,D", [(4096, 40), (1024, 80), (256, 160)])
def test_gligen_fused_qkv(cuda, nq, D, amp):
    """GLIGEN gated self-attention exactly as gligen.py calls it: q = qkv[:, :nq, 0] over k, v = qkv[:, :, 1|2] of a fused
    [B, nq + 30, 3, H, D] buffer. Heads are adjacent (no padding), so a read past D takes the next head's columns."""
    B, H, N = 2, 8, nq + 30
    qkv = randn((B, N, 3, H, D), gen(cuda, 500 + D), 1.0).to(BF)
    qkv[:, :, 0] = (qkv[:, :, 0].float() * amp + 0.5 * amp).to(BF)
    run_attention(cuda, qkv[:, :nq, 0], qkv[:, :, 1], qkv[:, :, 2], "gligen fused qkv", f"nq {nq} D {D} amp {amp}")


# ---------------------------------------------------------------------------------------------------- B: split-KV
# name: (B, H, Sq, Skv, D)
SPLIT_CASES = {
    "unsplit-256": (1, 8, 101, 256, 64),            # fewer than 8 key blocks
    "quarter-cap-1024": (1, 8, 101, 1024, 64),      # SEEM: 33 wanted, nblk / 4 = 4
    "uncapped-b3-4096": (3, 8, 101, 4096, 64),      # 2 * SMs / 24 CTAs = 11 splits
    "cap32-16384": (1, 8, 101, 16384, 64),          # SEEM's largest memory: 32-split cap
    "empty-splits-8300": (1, 8, 101, 8300, 64),     # 130 blocks over 32 splits of 5: the last 6 splits hold none
    "d40-1054": (1, 8, 101, 1054, 40),              # HD 64 != D in the workspace stride
    "d80-2100": (2, 4, 150, 2100, 80),              # HD 128 != D
}


def test_split_case_list_reaches_every_branch(cuda):
    """The split cases must reach each branch of tc_splits on this device; otherwise the numerical tests would silently
    stop covering one of them."""
    plans = {n: split_plan(B, H, Sq, Skv) for n, (B, H, Sq, Skv, D) in SPLIT_CASES.items()}
    assert any(p["splits"] == 1 for p in plans.values()), plans
    assert any(2 <= p["splits"] <= 31 and not p["quarter_cap"] for p in plans.values()), plans
    assert any(p["quarter_cap"] for p in plans.values()), plans
    assert any(p["cap32"] for p in plans.values()), plans
    assert any(p["empty"] for p in plans.values()), plans
    assert all(p["splits"] > 1 for n, p in plans.items() if n.startswith("d")), plans
    assert tc_splits(1, 8, 101, 16384, True) == 1


@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("name", list(SPLIT_CASES))
def test_split_random(cuda, name, amp):
    """Random operands on every split branch, with a per-batch mask on the same shape (split + mask)."""
    B, H, Sq, Skv, D = SPLIT_CASES[name]
    g = gen(cuda, 600 + len(name))
    q, k, v = operands(g, B, Sq, Skv, H, D, amp)
    run_attention(cuda, q, k, v, "split", f"{name} amp {amp}")
    mask = make_mask(g, (B, 1, Sq, Skv), Skv, cuda)
    for b in range(B):
        poison(k, v, b, slice(100, 164))
    run_attention(cuda, q, k, v, "split", f"{name} amp {amp} masked", mask=mask)


def test_split_kv_len_runs_unsplit(cuda):
    """kv_len turns the split path off (its workspace sizing ignores kv_len; the trace test shows no merge kernel for this
    call): the unsplit result over the first 5000 of 16384 keys is right, with the rest poisoned."""
    B, H, Sq, Skv, D = SPLIT_CASES["cap32-16384"]
    q, k, v = operands(gen(cuda, 700), B, Sq, Skv, H, D, 1.0)
    poison(k, v, 0, slice(5000, Skv))
    run_attention(cuda, q, k, v, "split", "kv_len 5000 of 16384", kv_len=[5000])


def test_split_repeat_and_shared_workspace(cuda):
    """Split calls are bit-identical on repeat, and when interleaved with other split shapes on the one "attn" workspace
    (and with a paged split call, which shares it)."""
    from vitron_b200 import ops
    calls = {}
    for i, n in enumerate(["quarter-cap-1024", "uncapped-b3-4096", "cap32-16384", "empty-splits-8300", "d40-1054"]):
        B, H, Sq, Skv, D = SPLIT_CASES[n]
        calls[n] = operands(gen(cuda, 800 + i), B, Sq, Skv, H, D, 6.0)
    alone = {}
    for n, (q, k, v) in calls.items():
        alone[n] = ops.attention(q, k, v)
        assert torch.equal(ops.attention(q, k, v), alone[n]), f"{n}: repeat differs"
    pc = PagedCase(cuda, PAGED["split-nblk-half-cap"], 6.0, seed=5)
    paged_alone = pc.run()
    order = list(calls) + list(calls)[::-1] + list(calls)[::2]
    for n in order:
        q, k, v = calls[n]
        assert torch.equal(ops.attention(q, k, v), alone[n]), f"{n}: differs after other shapes used the workspace"
        assert torch.equal(pc.run(), paged_alone), f"paged call differs after {n}"


# ---------------------------------------------------------------------------------------------------- C: paged prefill
# name: (H, q_start per row, q_len per row); D = 128, pages of 64 keys
PAGED = {
    "unsplit-b8": (32, [0, 1, 63, 64, 65, 700, 2047, 128], [17, 2, 64, 128, 129, 1, 33, 64]),
    "split-nblk-half-cap": (32, [640], [77]),               # 32 CTAs: 8 splits wanted, 717 keys = 12 blocks -> 6
    "split-uncapped-b2": (8, [3000, 300], [64, 17]),        # 16 CTAs: 16 splits of 48 blocks
    "split-cap32": (4, [4200], [17]),                       # 4 CTAs: 66 wanted, 66 blocks -> 32
    "ragged-b3-split": (8, [0, 700, 129], [128, 17, 1]),
    "chunk-ends-on-page": (8, [64, 100, 192], [64, 28, 128]),   # q_start + q_len a multiple of 64: next page is NaN
}
N_POISON = 3


class PagedCase:
    """A paged cache with shuffled page ids. Poison (K = 1000, V = -50): page 0 and pages no row owns, the block-table
    entries past ceil(max_kv_len / 64), and the slots past q_start + q_len inside each row's last page. Entries between a
    row's last page and ceil(max_kv_len / 64) point at NaN pages (K = 1000, V = NaN): the kernel never reads them (the
    header requires finite V only in pages a row reads), so a NaN in the output means it read one."""

    def __init__(self, cuda, spec, amp, seed):
        H, starts, lens = spec
        self.H, self.starts, self.lens = H, starts, lens
        B, D, P = len(starts), 128, 64
        self.max_kv = max(s + n for s, n in zip(starts, lens))
        self.Sq = max(lens)
        g, gc = gen(cuda, seed), torch.Generator().manual_seed(seed)
        read = [-(-(s + n) // P) for s, n in zip(starts, lens)]        # pages row b reads
        mp_kv = -(-self.max_kv // P)
        self.max_pages = mp_kv + 2                                     # 2 table entries past max_kv_len
        n_nan = max(1, sum(mp_kv - r for r in read))
        total = sum(read) + N_POISON + n_nan
        ids = torch.randperm(total - 1, generator=gc) + 1
        real = ids[:sum(read)]
        pois = torch.cat([torch.zeros(1, dtype=torch.long), ids[sum(read):sum(read) + N_POISON - 1]])
        nan_pages = ids[sum(read) + N_POISON - 1:]
        bt = pois[torch.randint(0, N_POISON, (B, self.max_pages), generator=gc)]
        off, noff = 0, 0
        for b, r in enumerate(read):
            bt[b, :r] = real[off:off + r]
            off += r
            for e in range(r, mp_kv):
                bt[b, e] = nan_pages[noff % len(nan_pages)]
                noff += 1
        self.bt_host, self.bt = bt, bt.to(torch.int32).to(cuda)
        self.kp = randn((total, H, P, D), g).to(BF)
        self.vp = randn((total, H, P, D), g).to(BF)
        self.kp[pois.to(cuda)] = POISON_K
        self.vp[pois.to(cuda)] = POISON_V
        self.kp[nan_pages.to(cuda)] = POISON_K
        self.vp[nan_pages.to(cuda)] = float("nan")
        for b, (s, n) in enumerate(zip(starts, lens)):
            for j in range(s + n, read[b] * P):
                p = int(bt[b, j // P])
                self.kp[p, :, j % P] = POISON_K
                self.vp[p, :, j % P] = POISON_V
        qkv = randn((B, self.Sq, 3, H, D), g).to(BF)
        qkv[:, :, 0] = (qkv[:, :, 0].float() * amp + 0.5 * amp).to(BF)
        self.q = qkv[:, :, 0]
        self.qs = torch.tensor(starts, dtype=torch.int32, device=cuda)
        self.ql = torch.tensor(lens, dtype=torch.int32, device=cuda)

    def run(self, out=None):
        from vitron_b200 import ops
        return ops.attention_paged(self.q, self.kp, self.vp, self.bt, self.qs, self.ql, self.max_kv, out=out)

    def gather(self, b, T):
        j = torch.arange(T, device=self.bt.device)
        pages = self.bt[b, j // 64].long()
        return (self.kp[pages, :, j % 64].unsqueeze(0), self.vp[pages, :, j % 64].unsqueeze(0))   # [1, T, H, D]


def test_paged_case_list_reaches_every_branch(cuda):
    """The paged cases reach each branch of paged_splits on this device: unsplit, the nblk / 2 cap, the 32 cap and an
    uncapped split."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    plans = {}
    for n, (H, starts, lens) in PAGED.items():
        B, Sq, mkv = len(starts), max(lens), max(s + l for s, l in zip(starts, lens))
        ctas, nblk = -(-Sq // 128) * H * B, -(-mkv // 64)
        plans[n] = (paged_splits(B, H, Sq, mkv), nblk, 2 * sms // ctas if 2 * ctas <= sms else 0)
    assert any(s == 1 for s, _, _ in plans.values()), plans
    assert any(s > 1 and s == nb // 2 and raw > s for s, nb, raw in plans.values()), plans
    assert any(s == 32 and raw > 32 and nb // 2 > 32 for s, nb, raw in plans.values()), plans
    assert any(1 < s < 32 and s == raw for s, nb, raw in plans.values()), plans


@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("name", list(PAGED))
def test_paged_poisoned(cuda, name, amp):
    """Paged prefill over poisoned pages against float64 over the keys gathered through the block table; query rows past
    q_len are exact zeros; the out= view of a NaN buffer is the only thing written; repeats are bit-identical."""
    pc = PagedCase(cuda, PAGED[name], amp, seed=len(name) + int(amp))
    B, Sq, H, D = len(pc.starts), pc.Sq, pc.H, 128
    buf, out = sentinel_out((B, Sq, H, D), cuda)
    pc.run(out=out)
    check_sentinel(buf, (B, Sq, H, D), name)
    for b, (s, n) in enumerate(zip(pc.starts, pc.lens)):
        K, V = pc.gather(b, s + n)
        ref, absum = reference(pc.q[b:b + 1, :n], K, V, 1.0 / math.sqrt(D), causal=True)
        check(out[b:b + 1, :n], ref, absum, "paged", f"{name} amp {amp} row {b} (q_start {s}, q_len {n})")
        assert int(out[b, n:].count_nonzero()) == 0, f"{name} row {b}: rows past q_len are not zero"
    assert torch.equal(pc.run(), out), f"{name}: repeat differs"


# ---------------------------------------------------------------------------------------------------- D: mma.sync kernel
def test_unet_cross_attention_stride0(cuda):
    """UNet cross-attention exactly as unet_i2vgen.py calls it: q[bi] [f, hw, H, 64] over kv[bi:bi+1].expand(f, 77, H, 64)
    (K / V with batch stride 0, which the wgmma kernel refuses), written into att[bi] of a NaN buffer: the other sample's
    frames stay untouched."""
    from vitron_b200 import ops
    b, f, hw, H, hd, L = 2, 16, 2560, 5, 64, 77
    g = gen(cuda, 900)
    q = randn((b, f, hw, H, hd), g, 1.0, 0.5).to(BF)
    kv = randn((b, L, 2, H, hd), g).to(BF)
    att = torch.full((b, f, hw, H, hd), float("nan"), dtype=BF, device=cuda)
    for bi in range(b):
        kb, vb = kv[bi:bi + 1, :, 0].expand(f, L, H, hd), kv[bi:bi + 1, :, 1].expand(f, L, H, hd)
        ops.attention(q[bi], kb, vb, scale=hd ** -0.5, out=att[bi])
        assert bool(att[bi + 1:].isnan().all()), "wrote into the next sample"
        ref, absum = reference(q[bi], kb, vb, hd ** -0.5)
        check(att[bi], ref, absum, "mma.sync", f"unet cross sample {bi}")


@pytest.mark.parametrize("Sq", [1, 17, 77, 95])
def test_llama_short_prefill(cuda, Sq):
    """LLaMA prefill below 96 tokens (automatic choice: mma.sync), causal, ragged kv_len, head dim 128, q / k / v the
    thirds of fused qkv rows; keys past kv_len hold poison and every row is checked."""
    B, H, D = 4, 8, 128
    qkv = randn((B, Sq, 3, H, D), gen(cuda, 1000 + Sq)).to(BF)
    qkv[:, :, 0] = (qkv[:, :, 0].float() + 0.5).to(BF)
    lens = [Sq, 1, (Sq + 1) // 2, 0]
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    for b, L in enumerate(lens):
        poison(k, v, b, slice(L, Sq))
    run_attention(cuda, q, k, v, "mma.sync", f"llama prefill Sq {Sq}", causal=True, kv_len=lens)


def test_clip_text_causal(cuda):
    """CLIP text: 77 tokens, causal, head dim 64, fused qkv rows, amp 1 and 6."""
    B, H, S, D = 2, 12, 77, 64
    for amp in (1.0, 6.0):
        qkv = randn((B, S, 3, H, D), gen(cuda, 1100 + int(amp))).to(BF)
        qkv[:, :, 0] = (qkv[:, :, 0].float() * amp + 0.5 * amp).to(BF)
        run_attention(cuda, qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], "mma.sync", f"clip text amp {amp}", causal=True)


@pytest.mark.parametrize("D", [40, 64, 80, 128, 160])
def test_mma_sync_edges(cuda, D):
    """The mma.sync kernel pinned (impl 1) at its 64-row / 64-key tile edges, causal and not, every head dim."""
    g = gen(cuda, 1200 + D)
    for Sq, Skv in [(1, 1), (63, 65), (64, 64), (65, 129), (129, 63), (300, 300)]:
        q, k, v = operands(g, 2, Sq, Skv, 2, D, 6.0)
        for causal in (False, True):
            run_attention(cuda, q, k, v, "mma.sync", f"D {D} Sq {Sq} Skv {Skv} causal {causal}", causal=causal, use=1)


# ---------------------------------------------------------------------------------------------------- E: probes
# name: (B, H, Sq, Skv, D, causal, kv_len, impl)
PROBE_CASES = {
    "wg-causal-300": (2, 8, 300, 300, 64, True, None, 0),
    "wg-causal-200-over-457": (1, 8, 200, 457, 128, True, None, 0),
    "wg-kvlen": (4, 4, 300, 300, 128, False, [300, 64, 65, 193], 0),
    "wg-kvlen-causal-d80": (4, 4, 300, 300, 80, True, [300, 64, 65, 193], 0),
    "split-quarter-cap": (1, 8, 101, 1024, 64, False, None, 0),
    "split-uncapped": (3, 8, 101, 4096, 64, False, None, 0),
    "split-empty": (1, 8, 101, 8300, 64, False, None, 0),
    "split-d40": (1, 8, 101, 1054, 40, False, None, 0),
    "mma-causal-77": (2, 8, 77, 77, 128, True, [77, 40], 0),
    "mma-causal-95-over-200": (1, 4, 95, 200, 64, True, None, 1),
    "mma-causal-300": (1, 8, 300, 300, 64, True, [300], 1),
    "mma-kvlen-d160": (2, 4, 130, 130, 160, False, [130, 65], 1),
}
DIAG_ROWS = [0, 5, 63, 64, 70, 127, 128, 129, 191, 255]   # both consumer warpgroups' rows of the first tiles


def probe_options(spec, b, kind):
    B, H, Sq, Skv, D, causal, kv_len, use = spec
    L = Skv if kv_len is None else kv_len[b]
    single = {63, 64, 127, 128, L - 1, L}
    if causal:
        off = Skv - Sq
        for i in DIAG_ROWS + [Sq - 1]:
            single |= {i + off, i + off + 1}
    pl = split_plan(B, H, Sq, Skv)
    if not causal and kv_len is None and pl["splits"] > 1:
        for s in range(1, pl["splits"]):
            single |= {s * pl["per"] * 64 - 1, s * pl["per"] * 64}
    if kind == "single":
        return sorted(j for j in single if 0 <= j < Skv)
    pairs = [(63, 64), (127, 128), (0, L - 1), (64, L - 1)]
    if not causal and kv_len is None and pl["splits"] > 1:
        e = pl["per"] * 64
        pairs += [(e - 1, e), (0, Skv - 1), (e, (pl["splits"] - 1) * e)]
    return [(a, c) for a, c in pairs if 0 <= a < c < min(L, Skv)]


@pytest.mark.parametrize("kind", ["single", "pair"])
@pytest.mark.parametrize("name", list(PROBE_CASES))
def test_probes(cuda, name, kind):
    """One key per (batch, head) that beats every other by >= 30 nats (the output is that key's V), or two keys ln 3
    apart (0.75 V1 + 0.25 V2), at block edges, causal diagonals (rows in both consumer warpgroups), split boundaries,
    kv_len - 1 (must win) and kv_len (must have no effect). Every query row of a (batch, head) is the same vector u, so
    the probe dominates every row that sees it."""
    spec = PROBE_CASES[name]
    B, H, Sq, Skv, D, causal, kv_len, use = spec
    g = gen(cuda, 1300 + len(name))
    scale = 1.0 / math.sqrt(D)
    u = randn((B, 1, H, D), g, 1.0, 1.0).to(BF).to(F64)
    opts = [probe_options(spec, b, kind) for b in range(B)]
    rounds = max(-(-len(o) // H) for o in opts)
    for rnd in range(rounds):
        q = padded(u.expand(B, Sq, H, D))
        k, v = padded(randn((B, Skv, H, D), g, 0.25)), padded(randn((B, Skv, H, D), g))
        probes = {}
        for b in range(B):
            for h in range(H):
                sel = opts[b][(h + b + rnd * H) % len(opts[b])]
                keys = [sel] if kind == "single" else list(sel)
                k1 = u[b, 0, h] * (40.0 / (float((u[b, 0, h] ** 2).sum()) * scale))
                s1 = float((bf_(k1) * u[b, 0, h]).sum()) * scale
                for n, j in enumerate(keys):
                    k[b, j, h] = (k1 if n == 0 else bf_(k1) * (1.0 - math.log(3.0) / s1)).to(BF)
                probes[(b, h)] = keys
        run_attention(cuda, q, k, v, "probes", f"{name} {kind} round {rnd}", causal=causal, kv_len=kv_len, use=use,
                      probes=probes)


def bf_(x):
    return x.to(BF).to(F64)


# ---------------------------------------------------------------------------------------------------- F: short sequences
def run_short(cuda, q, k, v, group, what, out=None, sentinel=None):
    from vitron_b200 import ops
    res = ops.attention_short(q, k, v, out=out)
    if sentinel is not None:
        check_sentinel(*sentinel, what)
    shp = q.shape
    flat = lambda t: t.reshape(-1, *t.shape[-3:])
    ref, absum = reference(flat(q), flat(k), flat(v), 1.0 / 8.0)
    check(flat(res), ref, absum, group, what, short=group.endswith("fp32"))
    assert res.shape == shp
    return res


@pytest.mark.parametrize("S", [1, 2, 7, 8, 15, 16])
def test_short_mma(cuda, S):
    """attn_short_mma_kernel<4>: 4-D [nseq, S, H, 64] views padded with 1000, output through a NaN buffer, amp 1 and 6."""
    for amp in (1.0, 6.0):
        q, k, v = operands(gen(cuda, 1400 + S), 37, S, S, 3, 64, amp)
        buf, out = sentinel_out((37, S, 3, 64), cuda)
        run_short(cuda, q, k, v, "short mma", f"S {S} amp {amp}", out=out, sentinel=(buf, (37, S, 3, 64)))


@pytest.mark.parametrize("S,aligned", [(17, True), (31, True), (32, True), (3, False), (8, False), (9, False),
                                       (16, False), (32, False)])
def test_short_fp32(cuda, S, aligned):
    """attn_short_kernel<8|16|32, .>: S > 16, or rows only 4-byte aligned (base offset by 2 elements); P stays fp32."""
    nseq, H = 29, 3
    for amp in (1.0, 6.0):
        g = gen(cuda, 1500 + S)
        ops_ = []
        for t in range(3):
            x = randn((nseq, S, H, 64), g, amp if t == 0 else 1.0, 0.5 * amp if t == 0 else 0.0)
            base = torch.full((nseq, S, H, 72), PAD_VAL, dtype=BF, device=cuda)
            view = base[..., 0:64] if aligned else base[..., 2:66]
            view.copy_(x.to(BF))
            ops_.append(view)
        run_short(cuda, *ops_, "short fp32", f"S {S} aligned {aligned} amp {amp}")


def test_short_5d_unet_and_video_tower(cuda):
    """The 5-D layouts: unet_i2vgen.py (qkv [b, f=16, hw, 3, H, 64] permuted to [3, b, hw, f, H, 64], out= the permuted
    view of att [b, f, hw, H, 64]) and vision_tower.py (T = 8 frames, N = 257 tokens, H = 16)."""
    from vitron_b200 import ops
    for (b, f, hw, H), group in [((2, 16, 96, 5), "short mma"), ((2, 8, 257, 16), "short mma")]:
        for amp in (1.0, 6.0):
            qkv = randn((b, f, hw, 3, H, 64), gen(cuda, 1600 + f), 1.0).to(BF)
            qkv[:, :, :, 0] = (qkv[:, :, :, 0].float() * amp + 0.5 * amp).to(BF)
            q5 = qkv.view(b, f, hw, 3, H, 64).permute(3, 0, 2, 1, 4, 5)
            att = torch.full((b, f, hw, H, 64), float("nan"), dtype=BF, device=cuda)
            ops.attention_short(q5[0], q5[1], q5[2], scale=0.125, out=att.permute(0, 2, 1, 3, 4))
            assert not bool(att.isnan().any()), "unwritten output"
            flat = lambda t: t.reshape(b * hw, f, H, 64)
            ref, absum = reference(flat(q5[0]), flat(q5[1]), flat(q5[2]), 0.125)
            check(flat(att.permute(0, 2, 1, 3, 4)), ref, absum, group, f"5-D f {f} hw {hw} H {H} amp {amp}")


@pytest.mark.parametrize("S,aligned", [(1, True), (8, True), (16, True), (5, False), (16, False), (17, True),
                                       (32, True)])
def test_short_probe_last_key(cuda, S, aligned):
    """Amp 6 probe on the last key: every query row of a (sequence, head) is u and key S - 1 is a multiple of u that wins
    by >= 30 nats, so the output is V[S - 1] in every row."""
    nseq, H = 11, 4
    g = gen(cuda, 1700 + S)
    u = (randn((nseq, 1, H, 64), g, 6.0, 6.0)).to(BF).to(F64)
    k = randn((nseq, S, H, 64), g, 0.25).to(F64)
    k[:, S - 1] = u[:, 0] * (50.0 / ((u[:, 0] ** 2).sum(-1, keepdim=True) * 0.125))
    views = []
    for t, x in enumerate([u.expand(nseq, S, H, 64), k, randn((nseq, S, H, 64), g).to(F64)]):
        base = torch.full((nseq, S, H, 72), PAD_VAL, dtype=BF, device=cuda)
        view = base[..., 0:64] if aligned else base[..., 2:66]
        view.copy_(x.to(BF))
        views.append(view)
    from vitron_b200 import ops
    res = ops.attention_short(*views)
    ref, absum = reference(*views, 0.125, probes={(s, h): [S - 1] for s in range(nseq) for h in range(H)})
    short = not (aligned and S <= 16)
    check(res, ref, absum, "short fp32" if short else "short mma", f"probe S {S} aligned {aligned}", short=short)


# ---------------------------------------------------------------------------------------------------- G: branch coverage
def check_trace_cases(cuda):
    """Each family of cases above runs the kernel instantiation it was written for (the dispatch is asserted per call)."""
    from vitron_b200 import ops
    g = gen(cuda, 1800)

    def att(B, H, Sq, Skv, D, use=0, **kw):
        q, k, v = operands(g, B, Sq, Skv, H, D, 1.0)
        if "kv_len" in kw:
            kw["kv_len"] = torch.tensor(kw["kv_len"], dtype=torch.int32, device=cuda)

        def fn():
            with impl(use):
                ops.attention(q, k, v, **kw)
        return kernels_of(fn)

    tc = "flash_attn_tc_kernel<{}, vb::TcAttnParams>"
    want = [  # (names, present, absent)
        (att(2, 16, 257, 257, 64), [tc.format(64)], ["attn_split_merge_kernel", "flash_attn_kernel<"]),
        (att(1, 8, 768, 768, 128, causal=True), [tc.format(128)], ["attn_split_merge_kernel"]),
        (att(1, 8, 286, 286, 160), [tc.format(192)], ["flash_attn_kernel<"]),
        (att(1, 8, 1054, 1054, 40), [tc.format(64)], ["flash_attn_kernel<"]),
        (att(1, 8, 1054, 1054, 80), [tc.format(128)], ["flash_attn_kernel<"]),
        (att(1, 8, 63, 64, 40, use=2), [tc.format(64)], ["flash_attn_kernel<"]),
        (att(1, 8, 101, 16384, 64), [tc.format(64), "attn_split_merge_kernel"], []),
        (att(1, 8, 101, 16384, 64, kv_len=[5000]), [tc.format(64)], ["attn_split_merge_kernel"]),
        (att(1, 8, 101, 1054, 40), [tc.format(64), "attn_split_merge_kernel"], []),
        (att(2, 4, 150, 2100, 80), [tc.format(128), "attn_split_merge_kernel"], []),
        (att(1, 8, 101, 256, 64), [tc.format(64)], ["attn_split_merge_kernel"]),
        (att(2, 8, 77, 77, 128, causal=True), ["flash_attn_kernel<128>"], ["flash_attn_tc_kernel"]),
        (att(2, 12, 77, 77, 64, causal=True), ["flash_attn_kernel<64>"], ["flash_attn_tc_kernel"]),
        (att(2, 2, 95, 95, 40), ["flash_attn_kernel<48>"], ["flash_attn_tc_kernel"]),
        (att(2, 2, 95, 95, 80), ["flash_attn_kernel<80>"], ["flash_attn_tc_kernel"]),
        (att(2, 2, 95, 95, 160), ["flash_attn_kernel<160>"], ["flash_attn_tc_kernel"]),
        (att(2, 2, 300, 300, 64, use=1), ["flash_attn_kernel<64>"], ["flash_attn_tc_kernel"]),
    ]
    # UNet cross-attention: stride-0 K / V over the frames
    q = randn((16, 2560, 5, 64), g).to(BF)
    kv = randn((1, 77, 2, 5, 64), g).to(BF)
    want.append((kernels_of(lambda: ops.attention(q, kv[:, :, 0].expand(16, 77, 5, 64), kv[:, :, 1].expand(16, 77, 5, 64))),
                 ["flash_attn_kernel<64>"], ["flash_attn_tc_kernel"]))
    # paged: unsplit and split
    for name, merge in [("unsplit-b8", False), ("split-cap32", True), ("split-nblk-half-cap", True)]:
        pc = PagedCase(cuda, PAGED[name], 1.0, seed=3)
        want.append((kernels_of(pc.run), ["flash_attn_tc_kernel<128, vb::TcPagedParams>"] + (["attn_split_merge_kernel"] if merge else []),
                     [] if merge else ["attn_split_merge_kernel"]))
    # short sequences
    for S, aligned, kern in [(16, True, "attn_short_mma_kernel<4>"), (1, True, "attn_short_mma_kernel<4>"),
                             (8, False, "attn_short_kernel<8, 4>"), (16, False, "attn_short_kernel<16, 4>"),
                             (17, True, "attn_short_kernel<32, 2>"), (32, False, "attn_short_kernel<32, 2>")]:
        base = torch.zeros((7, S, 2, 72), dtype=BF, device=cuda)
        x = base[..., 0:64] if aligned else base[..., 2:66]
        want.append((kernels_of(lambda: ops.attention_short(x, x, x)), [kern],
                     ["attn_short_kernel" if kern.startswith("attn_short_mma") else "attn_short_mma_kernel"]))
    for i, (names, present, absent) in enumerate(want):
        for p in present:
            assert launched(names, p), (i, p, sorted(names))
        for a in absent:
            assert not launched(names, a), (i, a, sorted(names))
    print(f"trace ok: {len(want)} calls")


def test_dispatch_branches_in_trace(cuda):
    """check_trace_cases in a fresh Python process. A torch.profiler session tears CUPTI down when it ends, and CUPTI
    re-initialised after a CUDA graph capture in the same process (other test files capture graphs) can return traces
    without any GPU kernel record; a new process has neither."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import sys; sys.path.insert(0, {root!r}); import torch; import tests.test_prefill_attention_gpu as t; "
            "t.check_trace_cases(torch.device('cuda:0'))")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "trace ok" in r.stdout, (r.stdout[-4000:] + r.stderr[-4000:])


def test_watchdog_clear_and_report(cuda):
    """No wgmma attention wait timed out in this file; prints the largest err / tol per group."""
    from vitron_b200 import ops
    assert ops.attention_watchdog()[0] == 0
    for group, r in sorted(RATIOS.items()):
        print(f"max err/tol {group}: {r:.3f}")
