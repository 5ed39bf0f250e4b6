"""GPU: the decode step's kernels against float64 references, on the branches their host-side policies pick at serving
shapes:
- split-KV decode attention (`attn_decode_paged`, `attn_decode_rope`, `attn_decode_rope_beam`): one split, the 4-trip
  and the 8-trip kernel, the 32-split cap, splits with no keys, over shuffled pages with poisoned pages and slots, with
  probes that make one or two chosen keys dominate, the fused RoPE + KV append, the beam indirection, a shared
  workspace and CUDA-graph replay;
- the GEMM at decode row counts (`ops.gemm`): the weight-streaming GEMV (16- and 32-row CTAs, one and two token tiles),
  the swap-AB + split-K path of 17-64 rows and the persistent kernel at 65, with the epilogues the engine's layer and
  lm_head use, at Vicuna-7B widths and ragged vocabularies;
- a trace of the launched kernel names, so that a change of dispatch policy fails here instead of quietly moving these
  cases off the branch they were written for."""
import copy
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

BF, F64 = torch.bfloat16, torch.float64
D, PS, THETA, EPS = 128, 64, 10000.0, 1e-5
SCALE = 1.0 / math.sqrt(D)
POISON_K, POISON_V = 1000.0, -50.0     # a read of a poisoned key takes the whole softmax and returns -50
N_POISON = 3                           # poisoned pages; page id 0 is always one of them


# ---------------------------------------------------------------------------------------------------- helpers
def close(a, b, atol, rtol, what=""):
    """|a - b| <= atol + rtol |b| everywhere; NaN counts as a mismatch."""
    a, b = a.double(), b.double()
    err = (a - b).abs()
    bad = ~(err <= atol + rtol * b.abs())
    n = int(bad.sum())
    assert n == 0, f"{what}: {n}/{a.numel()} mismatches, max err {err.nan_to_num(float('inf')).max().item():.4g}"


def gen(cuda, seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, device=g.device, generator=g, dtype=torch.float32) * scale + shift


def decode_plan(cap, bh):
    """Statement of decode_splits() and the trip choice of launch_attn_decode() (llm.cu) for a capacity of `cap` keys and
    B * H = bh: splits, keys per split (`per`), the kernel's trip count, and whether the 32-split cap bound."""
    keys = os.environ.get("VB200_DEC_SPLIT_KEYS", "")
    keys = int(keys) if keys.isdigit() else 0
    if keys in (128, 256, 512):
        raw = -(-cap // keys)
    else:
        s_min, s_max = -(-cap // 512), -(-cap // 128)
        raw = max(min(4 * torch.cuda.get_device_properties(0).multi_processor_count // max(bh, 1), s_max), s_min)
    splits = min(max(raw, 1), 32)
    per = -(-cap // splits)
    per = -(-per // 64) * 64
    return dict(splits=splits, per=per, trips=4 if per <= 256 else 8, capped=raw > 32)


def rope64(x, pos):
    """rotate_half RoPE in float64: x [..., D], pos broadcastable to x[..., 0]."""
    half = x.shape[-1] // 2
    inv = THETA ** (-torch.arange(half, dtype=F64, device=x.device) / half)
    ang = torch.as_tensor(pos, dtype=F64, device=x.device)[..., None] * inv
    c, s = ang.cos(), ang.sin()
    lo, hi = x[..., :half], x[..., half:]
    return torch.cat([lo * c - hi * s, hi * c + lo * s], -1)


def bf(x):
    return x.to(BF).to(F64)


# name: (B, H, capacity, short): lengths take the edge values first (capacity, per + 1, 1, capacity - 1, per, 65,
# per - 1, 64, 63), the remaining rows draw from 1..capacity (1..300 when short: most splits of those rows hold no key)
CASES = {
    "one-page": (3, 32, 64, False),
    "per128": (3, 8, 1024, False),
    "per256": (4, 32, 1024, False),
    "per320": (8, 32, 640, False),
    "b8-cap960": (8, 32, 960, False),        # the headline decode configuration
    "b8-cap4096": (8, 32, 4096, False),
    "b64-cap4096": (64, 32, 4096, True),
    "h4-b64-cap1024": (64, 4, 1024, True),
    "splits32-cap4096": (2, 8, 4096, False),
    "capped-cap8192": (2, 8, 8192, False),
    "capped-cap16384": (1, 8, 16384, False),
}


def case_lengths(name, g):
    B, H, cap, short = CASES[name]
    per = decode_plan(cap, B * H)["per"]
    lens = []
    for l in (cap, per + 1, 1, cap - 1, per, 65, per - 1, 64, 63):
        if 1 <= l <= cap and l not in lens:
            lens.append(l)
    hi = min(cap, 300) if short else cap
    rest = torch.randint(1, hi + 1, (max(B - len(lens), 0),), generator=g).tolist()
    return (lens + rest)[:B]


class PagedCache:
    """K / V pages [pages, H, 64, 128] with shuffled page ids and a block table [B (+ pad_rows), capacity / 64]. Every
    entry past a row's pages, every pad row, page 0, and every slot past a row's length inside its last page hold
    poison: a key the kernel should not read dominates the softmax and turns the output into POISON_V."""

    def __init__(self, cuda, H, cap, lens, seed, key_scale=1.0, pad_rows=0):
        g, gc = gen(cuda, seed), torch.Generator().manual_seed(seed)
        self.H, self.cap, self.lens = H, cap, list(lens)
        self.max_pages = -(-cap // PS)
        need = [-(-l // PS) for l in lens]
        total = sum(need) + N_POISON
        ids = torch.randperm(total - 1, generator=gc) + 1
        real, self.poison = ids[:sum(need)], torch.cat([torch.zeros(1, dtype=torch.long), ids[sum(need):]])
        bt = self.poison[torch.randint(0, N_POISON, (len(lens) + pad_rows, self.max_pages), generator=gc)]
        off = 0
        for b, n in enumerate(need):
            bt[b, :n] = real[off:off + n]
            off += n
        self.bt_host, self.bt = bt, bt.to(torch.int32).to(cuda)
        self.kp = randn((total, H, PS, D), g, key_scale).to(BF)
        self.vp = randn((total, H, PS, D), g).to(BF)
        self.kp[self.poison.to(cuda)] = POISON_K
        self.vp[self.poison.to(cuda)] = POISON_V
        for b, l in enumerate(lens):
            self.poison_slot(b, l, PS * need[b])

    def slot(self, b, j):
        return int(self.bt_host[b, j // PS]), j % PS

    def copy(self):
        c = copy.copy(self)
        c.kp, c.vp = self.kp.clone(), self.vp.clone()
        return c

    def poison_slot(self, b, j0, j1):
        """Poison key slots [j0, j1) of row b (inside its pages)."""
        for j in range(j0, j1):
            p, s = self.slot(b, j)
            self.kp[p, :, s] = POISON_K
            self.vp[p, :, s] = POISON_V

    def gather(self, b, L, src=None):
        """float64 K, V [L, H, D] of row b's keys 0..L-1; src [L] int (optional): the row whose pages hold key j."""
        j = torch.arange(L, device=self.bt.device)
        rows = torch.full_like(j, b) if src is None else src.to(self.bt.device).long()
        pages = self.bt[rows, j // PS].long()
        return self.kp[pages, :, j % PS].to(F64), self.vp[pages, :, j % PS].to(F64)

    def set_key(self, b, j, h, k=None, v=None):
        p, s = self.slot(b, j)
        if k is not None:
            self.kp[p, h, s] = k.to(BF)
        if v is not None:
            self.vp[p, h, s] = v.to(BF)


def attend(q, K, V):
    """float64 attention of one row: q [H, D] (already rotated), K / V [L, H, D] -> (out [H, D], weights [H, L])."""
    p = torch.softmax(torch.einsum("hd,lhd->hl", q, K) * SCALE, -1)
    return torch.einsum("hl,lhd->hd", p, V), p


def q_for(g, B, H, amp, pos=None, spread=1.0):
    """Query rows whose (rotated, when pos is given) vectors are spread * N(0, 1) + 1: every per-head sum is positive, so a
    poisoned key (all components POISON_K) always wins. Returns (the bf16 input rows [B, H*D], their rotated float64
    form as the kernel sees it: bf16-rounded)."""
    target = randn((B, H, D), g, spread * amp, amp).to(F64)
    if pos is None:
        q = bf(target)
        return q.to(BF).view(B, H * D), q
    q = bf(rope64(target, -pos.to(F64)[:, None]))
    return q.to(BF).view(B, H * D), bf(rope64(q, pos.to(F64)[:, None]))


def attn_tol(amp, rope):
    # bf16 output rounding (2^-8 relative) and fp32 scores; with RoPE the kernel's fp32 rotation of q may round a few
    # components to the neighbouring bf16 value, which moves peaked (amp 6) scores by ~1e-2
    return (3e-2, 1e-2) if rope and amp > 1 else (1e-2, 1e-2)


def ulp_bf16(x):
    a = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


# ---------------------------------------------------------------------------------------------------- the case list
def test_case_list_reaches_every_branch(cuda):
    """The shapes below must reach each branch of the split policy on this device; otherwise the numerical tests would
    silently stop covering one of them."""
    plans = {n: decode_plan(cap, B * H) for n, (B, H, cap, _) in CASES.items()}
    assert any(p["splits"] == 1 for p in plans.values())
    assert {p["per"] for p in plans.values() if p["trips"] == 4} >= {64, 128, 256}
    assert any(p["trips"] == 8 and p["per"] < 512 for p in plans.values())
    assert any(p["trips"] == 8 and p["per"] == 512 and p["splits"] > 1 for p in plans.values())
    assert any(p["capped"] for p in plans.values()) and any(p["splits"] == 32 for p in plans.values())
    assert plans["b8-cap960"]["trips"] == 8 and plans["b8-cap960"]["splits"] > 1


# ---------------------------------------------------------------------------------------------------- A: decode attention
@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("name", list(CASES))
def test_attn_decode_paged_random(cuda, name, amp):
    """Random keys over shuffled, poisoned pages against float64 attention over the keys gathered through the block
    table; repeated calls are bit-identical."""
    from vitron_b200 import ops
    B, H, cap, _ = CASES[name]
    g = gen(cuda, 100 + len(name))
    lens = case_lengths(name, torch.Generator().manual_seed(len(name)))
    c = PagedCache(cuda, H, cap, lens, seed=7 + len(name))
    q, q64 = q_for(g, B, H, amp)
    qrow = torch.cat([q, randn((B, 2 * H * D), g).to(BF)], 1)      # the fused q | k | v row of the engine
    kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
    out = ops.attn_decode_paged(qrow, c.kp, c.vp, c.bt, kvl, H, D, PS, cap)
    assert torch.equal(out, ops.attn_decode_paged(qrow, c.kp, c.vp, c.bt, kvl, H, D, PS, cap)), "repeat differs"
    for b, L in enumerate(lens):
        ref, _ = attend(q64[b], *c.gather(b, L))
        close(out[b].view(H, D), ref, *attn_tol(amp, False), f"{name} amp {amp} row {b} (kv_len {L})")


def probe_positions(L, plan):
    """Keys worth isolating in a row of length L: first and last key of every split, page boundaries, the last key."""
    per, pos = plan["per"], {0, 63, 64, L - 1}
    for s in range(1, plan["splits"]):
        pos |= {s * per - 1, s * per}
    return sorted(p for p in pos if 0 <= p < L)


def probe_pairs(L, plan):
    """Two keys in different splits (or, inside one split, in different lane groups: a lane group takes keys j % 16)."""
    per = plan["per"]
    pairs = [(0, L - 1), (per - 1, per), (63, 64), (per, L - 1)]
    return [(a, b) for a, b in pairs if 0 <= a < b < L and (a // per != b // per or a % 16 != b % 16)]


def probe_options(lens, plan, kind):
    return [probe_positions(L, plan) if kind == "single" else probe_pairs(L, plan) for L in lens]


def probe_rounds(lens, plan, kind, H):
    """Calls needed for every row to place every one of its probes on some head."""
    return max(-(-len(o) // H) for o in probe_options(lens, plan, kind))


def build_probes(c, B, H, lens, plan, kind, qrot, rnd=0, rope_new=None):
    """Plant dominant keys: head h of row b gets one key (kind 'single') equal to its rotated query, or two keys
    (kind 'pair') whose scores differ by ln 3; round `rnd` takes the next H options of each row. Returns
    {(b, h): [positions]}. rope_new(b, h, k): called instead of writing the cache when the position is the new token's
    slot (the fused-RoPE kernel writes that key itself)."""
    planted = {}
    for b, (L, opts) in enumerate(zip(lens, probe_options(lens, plan, kind))):
        if not opts:
            continue
        for h in range(H):
            sel = opts[(h + b + rnd * H) % len(opts)]
            keys = [sel] if kind == "single" else list(sel)
            k1 = qrot[b, h]
            s1 = float((k1 * k1).sum()) * SCALE
            for i, j in enumerate(keys):
                k = k1 if i == 0 else k1 * (1.0 - math.log(3.0) / s1)
                if rope_new is not None and j == L - 1:
                    rope_new(b, h, k)
                else:
                    c.set_key(b, j, h, k=k)
            planted[(b, h)] = keys
    return planted


def check_probe_weights(planted, b, w, kind, what):
    """The test data must do what the probe claims: the planted keys score >= 30 nats above every other key, and a pair
    splits its weight 3:1."""
    for (bb, h), keys in planted.items():
        if bb != b:
            continue
        rest = w[h].clone()
        rest[keys] = 0
        assert float(rest.max()) <= float(w[h, keys].min()) * math.exp(-30), (what, h, keys)
        if kind == "pair":
            assert abs(float(w[h, keys[0]]) - 0.75) < 0.02 and abs(float(w[h, keys[1]]) - 0.25) < 0.02, (what, h, keys)


@pytest.mark.parametrize("kind", ["single", "pair"])
@pytest.mark.parametrize("name", list(CASES))
def test_attn_decode_paged_probes(cuda, name, kind):
    """One key per head that beats all others by >= 30 nats (output = that key's V to bf16 rounding), at split edges,
    page boundaries and kv_len - 1; or two keys in different splits at ln 3 apart (output = 0.75 V1 + 0.25 V2): the
    merge weights across lane groups and across splits."""
    from vitron_b200 import ops
    B, H, cap, _ = CASES[name]
    plan = decode_plan(cap, B * H)
    g = gen(cuda, 200 + len(name))
    lens = case_lengths(name, torch.Generator().manual_seed(len(name)))
    base = PagedCache(cuda, H, cap, lens, seed=9 + len(name), key_scale=0.25)
    q, q64 = q_for(g, B, H, 1.0, spread=2.0)
    kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
    for rnd in range(probe_rounds(lens, plan, kind, H)):
        c = base.copy()
        planted = build_probes(c, B, H, lens, plan, kind, q64, rnd)
        out = ops.attn_decode_paged(q, c.kp, c.vp, c.bt, kvl, H, D, PS, cap)
        for b, L in enumerate(lens):
            ref, w = attend(q64[b], *c.gather(b, L))
            check_probe_weights(planted, b, w, kind, f"{name} row {b}")
            close(out[b].view(H, D), ref, 2e-3, 8e-3, f"{name} {kind} probe round {rnd} row {b} (kv_len {L})")


def rope_call(cuda, c, B, H, lens, qkv, beam=None):
    """attn_decode_rope (or the beam variant) on the cache, with the new token at slot kv_len - 1 poisoned beforehand.
    Returns (out, snapshot of the pages before the call)."""
    from vitron_b200 import ops
    for b, L in enumerate(lens):
        c.poison_slot(b, L - 1, L)
    snap = (c.kp.clone(), c.vp.clone())
    kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
    tab = ops.rope_table(kvl - 1, D, THETA)
    if beam is None:
        out = ops.attn_decode_rope(qkv, tab, c.kp, c.vp, c.bt, kvl, H, D, PS, c.cap)
    else:
        src, gstart = beam
        out = ops.attn_decode_rope_beam(qkv, tab, c.kp, c.vp, c.bt, kvl, src, gstart, H, D, PS, c.cap)
    return out, snap


def check_append(c, B, H, lens, qkv, snap, what):
    """The new token's K is float64 RoPE of the input within one bf16 ulp (plus the rounding of the kernel's fp32
    rotation angle, a few fp32 ulps of pos * inv_freq); its V is a bit copy; no other byte of the cache changed."""
    kp, vp = c.kp.clone(), c.vp.clone()
    for b, L in enumerate(lens):
        p, s = c.slot(b, L - 1)
        x = qkv[b, H * D:2 * H * D].view(H, D).to(F64)
        ref = rope64(x, float(L - 1))
        hyp = torch.cat([x[:, :D // 2].hypot(x[:, D // 2:])] * 2, -1)
        tol = ulp_bf16(ref) + (4e-7 * (L - 1) + 1e-6) * hyp
        err = (kp[p, :, s].to(F64) - ref).abs()
        assert bool((err <= tol).all()), f"{what}: new K of row {b} off by {float((err / tol).max()):.3g} x tolerance"
        assert torch.equal(vp[p, :, s], qkv[b, 2 * H * D:].view(H, D)), f"{what}: new V of row {b}"
        kp[p, :, s], vp[p, :, s] = snap[0][p, :, s], snap[1][p, :, s]
    assert torch.equal(kp, snap[0]) and torch.equal(vp, snap[1]), f"{what}: the call wrote outside the new token's slot"


def rope_ref(c, B, H, lens, qkv, q64, src=None):
    """float64 reference of the fused call: cached keys, then the new token (RoPE of its k, rounded like the cache)."""
    refs, ws = [], []
    for b, L in enumerate(lens):
        K, V = c.gather(b, L - 1, None if src is None else src[b, :L - 1])
        knew = bf(rope64(qkv[b, H * D:2 * H * D].view(1, H, D).to(F64), float(L - 1)))
        vnew = qkv[b, 2 * H * D:].view(1, H, D).to(F64)
        r, w = attend(q64[b], torch.cat([K, knew]), torch.cat([V, vnew]))
        refs.append(r)
        ws.append(w)
    return refs, ws


@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("name", list(CASES))
def test_attn_decode_rope_random(cuda, name, amp):
    """Fused RoPE + KV append + attention: output against float64, the appended K / V, and nothing else written."""
    B, H, cap, _ = CASES[name]
    g = gen(cuda, 300 + len(name))
    lens = case_lengths(name, torch.Generator().manual_seed(len(name)))
    c = PagedCache(cuda, H, cap, lens, seed=11 + len(name))
    pos = torch.tensor(lens, device=cuda) - 1
    q, q64 = q_for(g, B, H, amp, pos=pos)
    qkv = torch.cat([q, randn((B, 2 * H * D), g).to(BF)], 1)
    out, snap = rope_call(cuda, c, B, H, lens, qkv)
    check_append(c, B, H, lens, qkv, snap, f"{name} amp {amp}")
    refs, _ = rope_ref(c, B, H, lens, qkv, q64)
    for b, L in enumerate(lens):
        close(out[b].view(H, D), refs[b], *attn_tol(amp, True), f"{name} amp {amp} row {b} (kv_len {L})")


@pytest.mark.parametrize("kind", ["single", "pair"])
@pytest.mark.parametrize("name", ["one-page", "per256", "b8-cap960", "b64-cap4096", "capped-cap8192"])
def test_attn_decode_rope_probes(cuda, name, kind):
    """Probes through the fused kernel: a dominant cached key is the float64 RoPE of q at the step's position, rounded to
    bf16; a probe on the new token sets its k equal to q before rotation."""
    B, H, cap, _ = CASES[name]
    plan = decode_plan(cap, B * H)
    g = gen(cuda, 400 + len(name))
    lens = case_lengths(name, torch.Generator().manual_seed(len(name)))
    base = PagedCache(cuda, H, cap, lens, seed=13 + len(name), key_scale=0.25)
    pos = torch.tensor(lens, device=cuda) - 1
    q, q64 = q_for(g, B, H, 1.0, pos=pos, spread=2.0)
    kv0 = randn((B, 2, H, D), g)
    kv0[:, 0] *= 0.25
    for rnd in range(probe_rounds(lens, plan, kind, H)):
        c, kv = base.copy(), kv0.clone()

        def new_token(b, h, k):   # k = q before rotation (times the pair's factor): the kernel rotates both alike
            kv[b, 0, h] = q.view(B, H, D)[b, h].float() * float(k.norm() / q64[b, h].norm())

        planted = build_probes(c, B, H, lens, plan, kind, q64, rnd, rope_new=new_token)
        qkv = torch.cat([q, kv.view(B, 2 * H * D).to(BF)], 1)
        out, snap = rope_call(cuda, c, B, H, lens, qkv)
        check_append(c, B, H, lens, qkv, snap, f"{name} {kind}")
        refs, ws = rope_ref(c, B, H, lens, qkv, q64)
        # a pair's weights follow the difference of two ~56-nat scores: the kernel's fp32 rotation may round a few
        # components of q or of the new k to the neighbouring bf16 value, which moves that difference by up to ~0.03
        atol = 2e-3 if kind == "single" else 2e-2
        for b, L in enumerate(lens):
            check_probe_weights(planted, b, ws[b], kind, f"{name} row {b}")
            close(out[b].view(H, D), refs[b], atol, 8e-3, f"{name} {kind} probe round {rnd} row {b} (kv_len {L})")


@pytest.mark.parametrize("amp", [1.0, 6.0])
def test_attn_decode_rope_beam_vs_float64(cuda, amp):
    """8-trip beam shape (8 rows = 2 requests x 4 beams, capacity 960): keys at or past the prompt are read through
    beam_src from the source row's pages; checked against float64 attention over exactly those keys."""
    H, cap, k = 32, 960, 4
    lens, gstart = [960] * 4 + [513] * 4, [700] * 4 + [450] * 4
    R = len(lens)
    assert decode_plan(cap, R * H)["trips"] == 8
    g, gc = gen(cuda, 500), torch.Generator().manual_seed(5)
    c = PagedCache(cuda, H, cap, lens, seed=17, pad_rows=1)
    src = torch.arange(R, dtype=torch.int32)[:, None].repeat(1, cap + 8)
    for b in range(R):
        lo = (b // k) * k
        src[b, gstart[b]:lens[b] - 1] = torch.randint(lo, lo + k, (lens[b] - 1 - gstart[b],), generator=gc,
                                                      dtype=torch.int32)
    pos = torch.tensor(lens, device=cuda) - 1
    q, q64 = q_for(g, R, H, amp, pos=pos)
    qkv = torch.cat([q, randn((R, 2 * H * D), g).to(BF)], 1)
    src_d, gs_d = src.to(cuda), torch.tensor(gstart, dtype=torch.int32, device=cuda)
    out, snap = rope_call(cuda, c, R, H, lens, qkv, beam=(src_d, gs_d))
    check_append(c, R, H, lens, qkv, snap, f"beam amp {amp}")
    eff = torch.where(torch.arange(cap + 8)[None, :] < torch.tensor(gstart)[:, None], torch.arange(R)[:, None], src)
    refs, _ = rope_ref(c, R, H, lens, qkv, q64, src=eff)
    for b in range(R):
        close(out[b].view(H, D), refs[b], *attn_tol(amp, True), f"beam amp {amp} row {b}")
    again, _ = rope_call(cuda, c, R, H, lens, qkv, beam=(src_d, gs_d))
    assert torch.equal(out, again)


def test_attn_decode_shared_workspace_interleaved(cuda):
    """Calls with different (B, H, capacity), so different split counts, interleaved on the one "dec" workspace: each is
    bit-identical to the same call made alone."""
    from vitron_b200 import ops
    names = ["b8-cap960", "one-page", "splits32-cap4096", "per256", "b64-cap4096"]
    ops.reserve_decode_workspace(max(CASES[n][0] for n in names), 32, D, cuda)
    calls = {}
    for i, n in enumerate(names):
        B, H, cap, _ = CASES[n]
        lens = case_lengths(n, torch.Generator().manual_seed(len(n)))
        c = PagedCache(cuda, H, cap, lens, seed=19 + i)
        q, _ = q_for(gen(cuda, 600 + i), B, H, 6.0)
        kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
        calls[n] = (q, c, kvl, H, cap)
    run = lambda n: ops.attn_decode_paged(calls[n][0], calls[n][1].kp, calls[n][1].vp, calls[n][1].bt, calls[n][2],
                                          calls[n][3], D, PS, calls[n][4])
    alone = {}
    for n in names:          # each call right after the same call: no other shape has used the workspace in between
        run(n)
        alone[n] = run(n)
    order = names + names[::-1] + names[::2] + names[1::2]
    outs = [(n, run(n)) for n in order]
    for n, o in outs:
        assert torch.equal(o, alone[n]), n


def test_attn_decode_rope_graph_replay(cuda):
    """One attn_decode_rope call captured in a CUDA graph with the device-side advance of kv_len and positions, as the
    engine's decode step runs it, replayed for 3 steps: each replay equals the eager call bit for bit and the float64
    reference."""
    from vitron_b200 import ops
    name, steps = "b8-cap960", 3
    B, H, cap, _ = CASES[name]
    lens0 = [l - steps for l in case_lengths(name, torch.Generator().manual_seed(len(name)))]
    lens0 = [max(l, 1) for l in lens0]
    ops.reserve_decode_workspace(B, H, D, cuda)
    g = gen(cuda, 700)
    c = PagedCache(cuda, H, cap, [l + steps - 1 for l in lens0], seed=23)
    ce = c.copy()
    qkvs, eager, refs = [], [], []
    for s in range(steps):
        lens = [l + s for l in lens0]
        pos = torch.tensor(lens, device=cuda) - 1
        q, q64 = q_for(g, B, H, 1.0, pos=pos)
        qkv = torch.cat([q, randn((B, 2 * H * D), g).to(BF)], 1)
        kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
        eager.append(ops.attn_decode_rope(qkv, ops.rope_table(kvl - 1, D, THETA), ce.kp, ce.vp, ce.bt, kvl, H, D, PS,
                                          cap))
        refs.append(rope_ref(ce, B, H, lens, qkv, q64)[0])
        qkvs.append(qkv)
    kvl.add_(1)                                      # the device-side advance below, run once before capture
    # the graph: rope table, fused attention, then kv_len / positions advanced on the device
    s_qkv = torch.empty_like(qkvs[0])
    s_pos = torch.tensor(lens0, dtype=torch.int32, device=cuda) - 1
    s_len = torch.tensor(lens0, dtype=torch.int32, device=cuda)
    s_tab = torch.empty((B, D), dtype=torch.float32, device=cuda)
    s_out = torch.empty((B, H * D), dtype=BF, device=cuda)
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side), ops.pdl(True):
        ops.rope_table(s_pos, D, THETA, out=s_tab)
        ops.attn_decode_rope(s_qkv, s_tab, c.kp, c.vp, c.bt, s_len, H, D, PS, cap, out=s_out)
        s_pos.add_(1)
        s_len.add_(1)
    torch.cuda.current_stream().wait_stream(side)
    for s in range(steps):
        s_qkv.copy_(qkvs[s])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(s_out, eager[s]), f"replay {s} differs from the eager call"
        for b in range(B):
            close(s_out[b].view(H, D), refs[s][b], 1e-2, 1e-2, f"replay {s} row {b}")
    assert torch.equal(c.kp, ce.kp) and torch.equal(c.vp, ce.vp)
    assert s_len.tolist() == [l + steps for l in lens0]


def test_attn_decode_refusals(cuda):
    """Host-side refusals, before any launch: more than 4096 (batch, head) pairs with more than one split, and a capacity
    whose split would exceed 512 keys, raise VitronB200Error instead of returning a truncated result."""
    from vitron_b200 import ops
    from vitron_b200._lib import VitronB200Error
    page = torch.zeros((1, 32, PS, D), dtype=BF, device=cuda)        # every table entry is page 0: a valid address
    B, H, cap = 129, 32, 1024
    assert decode_plan(cap, B * H)["splits"] > 1
    q = torch.zeros((B, 3 * H * D), dtype=BF, device=cuda)
    bt = torch.zeros((B, cap // PS), dtype=torch.int32, device=cuda)
    kvl = torch.ones((B,), dtype=torch.int32, device=cuda)
    with pytest.raises(VitronB200Error, match="VB_ERR_UNSUPPORTED"):
        ops.attn_decode_paged(q, page, page, bt, kvl, H, D, PS, cap)
    with pytest.raises(VitronB200Error, match="VB_ERR_UNSUPPORTED"):
        ops.attn_decode_rope(q, ops.rope_table(kvl - 1, D, THETA), page, page, bt, kvl, H, D, PS, cap)
    B, H, cap = 1, 8, 16384 + 64
    assert decode_plan(cap, B * H)["per"] > 512
    q = torch.zeros((B, 3 * H * D), dtype=BF, device=cuda)
    bt = torch.zeros((B, cap // PS), dtype=torch.int32, device=cuda)
    kvl = torch.ones((B,), dtype=torch.int32, device=cuda)
    with pytest.raises(VitronB200Error, match="VB_ERR_ARG"):
        ops.attn_decode_paged(q, page[:, :H].contiguous(), page[:, :H].contiguous(), bt, kvl, H, D, PS, cap)
    with pytest.raises(VitronB200Error, match="VB_ERR_ARG"):
        ops.attn_decode_rope(q, ops.rope_table(kvl - 1, D, THETA), page[:, :H].contiguous(), page[:, :H].contiguous(),
                             bt, kvl, H, D, PS, cap)


# ---------------------------------------------------------------------------------------------------- B: decode GEMMs
GEMM_ROWS = [1, 2, 7, 8, 9, 15, 16,        # GEMV, one (M <= 8) and two token tiles
             17, 24, 32, 33, 48, 64,       # swap-AB + split-K, 32- and 64-column tiles
             65]                           # persistent kernel
CALLS = ["qkv", "o_proj", "gate_up", "down", "lm_head-32000", "lm_head-32001", "lm_head-32002"]


@pytest.fixture(scope="module")
def vicuna(cuda):
    """Vicuna-7B layer and lm_head weights (bf16, 0.02 N(0, 1)) and their float64 copies."""
    from vitron_b200 import ops
    g = gen(cuda, 31)
    w = {n: randn(s, g, 0.02).to(BF) for n, s in (("qkv", (12288, 4096)), ("o_proj", (4096, 4096)),
                                                   ("gate", (11008, 4096)), ("up", (11008, 4096)),
                                                   ("down", (4096, 11008)), ("lm_head", (32002, 4096)))}
    w["gate_up"] = ops.pack_glu_weight(w["gate"], w["up"])
    return w, {n: t.to(F64) for n, t in w.items() if n != "gate_up"}


def engine_call(ops, w, call, M, x, h=None, out=None):
    """The call exactly as LlamaEngine issues it (_layer / _decode_graph_body), with `out` where the engine lets the
    library allocate (prefilled by the test, so an unwritten element shows)."""
    if call == "qkv":
        return ops.gemm(x, w["qkv"], rms_eps=EPS, out=out)
    if call in ("o_proj", "down"):
        return ops.gemm(x, w[call], residual=h, out=h if out is None else out)
    if call == "gate_up":
        return ops.gemm(x, w["gate_up"], glu=ops.GLU_SWIGLU, rms_eps=EPS, out=out)
    return ops.gemm(x, w["lm_head"][:int(call.split("-")[1])], out=out, out_fp32=True, rms_eps=EPS)


@pytest.mark.parametrize("call", CALLS)
@pytest.mark.parametrize("M", GEMM_ROWS)
def test_gemm_decode_rows(cuda, vicuna, M, call):
    """The engine's projections and lm_head at decode row counts against float64 from the same bf16 operands (RMS row
    scale included); the last two columns and the last row are asserted on their own; repeats are bit-identical, and so
    is the in-place residual form against the out-of-place one."""
    from vitron_b200 import ops
    w, w64 = vicuna
    g = gen(cuda, 1000 * M + CALLS.index(call))
    K = 11008 if call == "down" else 4096
    x = randn((M, K), g, 1.0 if call in ("o_proj", "down") else 3.0).to(BF)
    x64 = x.to(F64)
    rstd = torch.rsqrt(x64.pow(2).mean(-1, keepdim=True) + EPS)
    if call in ("o_proj", "down"):
        h0 = randn((M, 4096), g).to(BF)
        h = h0.clone()
        got = engine_call(ops, w, call, M, x, h=h)
        assert got.data_ptr() == h.data_ptr()
        ref = h0.to(F64) + x64 @ w64[call].t()
        assert torch.equal(ops.gemm(x, w[call], residual=h0), h), "in-place residual differs from out of place"
        h2 = h0.clone()
        assert torch.equal(engine_call(ops, w, call, M, x, h=h2), h), "repeat differs"
    elif call.startswith("lm_head"):
        V = int(call.split("-")[1])
        buf = torch.full((M + 3, V), float("nan"), device=cuda)   # the engine's [max_batch, V] logits, rows [:B] written
        engine_call(ops, w, call, M, x, out=buf[:M])
        got = buf[:M]
        assert bool(buf[M:].isnan().all()), "lm_head wrote past its rows"
        ref = (x64 @ w64["lm_head"][:V].t()) * rstd
        again = torch.full_like(buf, float("nan"))
        engine_call(ops, w, call, M, x, out=again[:M])
        assert torch.equal(again[:M], got), "repeat differs"
    else:
        n = 12288 if call == "qkv" else 11008
        got = torch.full((M, n), float("nan"), dtype=BF, device=cuda)
        engine_call(ops, w, call, M, x, out=got)
        if call == "qkv":
            ref = (x64 @ w64["qkv"].t()) * rstd
        else:
            ref = F.silu((x64 @ w64["gate"].t()) * rstd) * ((x64 @ w64["up"].t()) * rstd)
        again = torch.full_like(got, float("nan"))
        engine_call(ops, w, call, M, x, out=again)
        assert torch.equal(again, got), "repeat differs"
    tol = (2e-3, 2e-3) if got.dtype == torch.float32 else (2e-3 * math.sqrt(K / 64), 1.6e-2)
    close(got[:, -2:], ref[:, -2:], *tol, f"{call} M={M}: last two columns")
    close(got[-1], ref[-1], *tol, f"{call} M={M}: last row")
    close(got, ref, *tol, f"{call} M={M}")


# ---------------------------------------------------------------------------------------------------- C: branch coverage
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


def test_dispatch_branches_in_trace(cuda, vicuna):
    """Each case of this file runs the kernel instantiation it was written for: the 8- and 4-trip decode kernels (plain,
    fused RoPE, beam), the 32-row GEMV of lm_head with one and two token tiles, the 16-row GEMV of the qkv projection, and
    the swap-AB tiles with the split-K reduce for 17-64 rows."""
    from vitron_b200 import ops
    w, _ = vicuna

    def decode(name, kernel):
        B, H, cap, _ = CASES[name]
        lens = case_lengths(name, torch.Generator().manual_seed(len(name)))
        c = PagedCache(cuda, H, cap, lens, seed=29)
        q, _ = q_for(gen(cuda, 800), B, H, 1.0)
        qkv = torch.cat([q, q, q], 1)
        kvl = torch.tensor(lens, dtype=torch.int32, device=cuda)
        tab = ops.rope_table(kvl - 1, D, THETA)
        src = torch.arange(B, dtype=torch.int32, device=cuda)[:, None].repeat(1, cap)
        run = {"paged": lambda: ops.attn_decode_paged(qkv, c.kp, c.vp, c.bt, kvl, H, D, PS, cap),
               "rope": lambda: ops.attn_decode_rope(qkv, tab, c.kp, c.vp, c.bt, kvl, H, D, PS, cap),
               "beam": lambda: ops.attn_decode_rope_beam(qkv, tab, c.kp, c.vp, c.bt, kvl, src, kvl, H, D, PS, cap)}
        return kernels_of(run[kernel])

    want = {("b8-cap960", "paged"): "attn_decode_kernel<false, 8, false>",
            ("b8-cap960", "rope"): "attn_decode_kernel<true, 8, false>",
            ("b8-cap960", "beam"): "attn_decode_kernel<true, 8, true>",
            ("capped-cap16384", "rope"): "attn_decode_kernel<true, 8, false>",
            ("b64-cap4096", "rope"): "attn_decode_kernel<true, 8, false>",
            ("per320", "rope"): "attn_decode_kernel<true, 8, false>",
            ("per256", "paged"): "attn_decode_kernel<false, 4, false>",
            ("per256", "rope"): "attn_decode_kernel<true, 4, false>",
            ("one-page", "rope"): "attn_decode_kernel<true, 4, false>",
            ("splits32-cap4096", "rope"): "attn_decode_kernel<true, 4, false>"}
    for (name, kernel), pattern in want.items():
        names = decode(name, kernel)
        assert launched(names, pattern), (name, kernel, sorted(names))
        other = pattern.replace(", 8,", ", 4,") if ", 8," in pattern else pattern.replace(", 4,", ", 8,")
        assert not launched(names, other), (name, kernel, sorted(names))

    def gemm(call, M):
        g = gen(cuda, 900 + M)
        x = randn((M, 11008 if call == "down" else 4096), g).to(BF)
        h = randn((M, 4096), g).to(BF)
        return kernels_of(lambda: engine_call(ops, w, call, M, x, h=h))

    qkv_rows = 32 if 12288 // 16 > 6 * torch.cuda.get_device_properties(0).multi_processor_count else 16   # 16 on SXM
    for M, call, pattern in [(8, "lm_head-32000", "gemv_bf16_kernel<32, 1>"), (1, "lm_head-32001", "gemv_bf16_kernel<32, 1>"),
                             (16, "lm_head-32002", "gemv_bf16_kernel<32, 2>"), (9, "lm_head-32000", "gemv_bf16_kernel<32, 2>"),
                             (8, "o_proj", "gemv_bf16_kernel<16, 1>"), (16, "down", "gemv_bf16_kernel<16, 2>"),
                             (8, "qkv", f"gemv_bf16_kernel<{qkv_rows}, 1>"), (16, "qkv", f"gemv_bf16_kernel<{qkv_rows}, 2>"),
                             (16, "gate_up", "gemv_bf16_kernel<32, 2>")]:
        names = gemm(call, M)
        assert launched(names, pattern), (call, M, sorted(names))
        assert not launched(names, "gemm_v2_kernel"), (call, M, sorted(names))
    for M in (17, 24, 32, 33, 48, 64):
        for call in ("qkv", "o_proj", "gate_up", "down", "lm_head-32001"):
            names = gemm(call, M)
            assert launched(names, f"gemm_v2_kernel<{32 if M <= 32 else 64},"), (call, M, sorted(names))
            assert launched(names, "splitk_reduce_kernel"), (call, M, sorted(names))
            assert not launched(names, "gemv_bf16_kernel"), (call, M, sorted(names))
    names = gemm("qkv", 65)
    assert launched(names, "gemm_v2_kernel") and not launched(names, "gemm_v2_kernel<32,"), sorted(names)
