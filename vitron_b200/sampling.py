"""float64 statement of the vb200_sample_advance contract (include/vitron_b200.h): temperature, top-k, top-p and the
Philox4x32-10 draw, vectorised over rows with torch / numpy on the host.

It is what a CPU-resident LlamaEngine runs for its sampled step: such an engine runs no kernels of this library (its
host logic is checked with the kernels replaced by torch statements), and the sampler has no other CPU form. On a CUDA
engine the step is always the kernel (ops.sample_advance); the GPU tests compare the kernel with this statement.
"""
import numpy as np
import torch


def philox4x32_10(counter, key):
    """Random123 philox4x32-10 in integer arithmetic, vectorised over leading dims: counter [..., 4] and key [..., 2]
    hold uint32 values -> numpy uint64 [..., 4]."""
    m32 = np.uint64(0xFFFFFFFF)
    c = [np.asarray(counter, dtype=np.uint64)[..., i] for i in range(4)]
    k0, k1 = np.asarray(key, dtype=np.uint64)[..., 0], np.asarray(key, dtype=np.uint64)[..., 1]
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]     # < 2^64: exact
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m32, (k1 + np.uint64(0xBB67AE85)) & m32
    return np.stack(c, -1)


def sample_support(logits, temperature, top_k, top_p, min_keep=1):
    """Steps 1-4 of the contract in float64 for logits [B, V]: (kept bool [B, V], p float64 [B, V] zero outside the kept
    set, near_cut bool [B]: a kept token's top-p fraction lies within 1e-5 of top_p). min_keep = 2 (beam sampling) also
    keeps, through top-p, every token with fewer than 2 strictly larger z among the tokens top-k kept."""
    l = logits.detach().double().cpu()
    B, V = l.shape
    neg_inf = torch.tensor(float("-inf"), dtype=torch.float64)
    valid = ~torch.isnan(l)
    z = l / float(temperature)
    zk = torch.where(valid, z, neg_inf)
    zmax = zk.max(1, keepdim=True).values
    kept = valid.clone()
    nvalid = valid.sum(1)
    if top_k > 0:
        k = min(int(top_k), V)
        kth = zk.sort(1, descending=True).values[:, k - 1:k]
        on = (nvalid > int(top_k))[:, None]
        kept &= ~on | (z >= kth)
    p = torch.where(z == zmax, torch.ones_like(z), torch.exp(z - zmax))
    p = torch.where(kept, p, torch.zeros_like(p))
    near = torch.zeros(B, dtype=torch.bool)
    kept_k = kept.clone()
    if top_p < 1.0:
        if top_p <= 0.0:
            kept &= z == zmax
        else:
            total = p.sum(1, keepdim=True)
            zs, order = torch.where(kept, z, neg_inf).sort(dim=1, descending=True, stable=True)
            ps = p.gather(1, order)
            excl = ps.cumsum(1) - ps
            first = torch.searchsorted(-zs.contiguous(), -zs.contiguous(), right=False).clamp(max=V - 1)   # tie-group start
            above = torch.empty_like(excl).scatter_(1, order, excl.gather(1, first))     # kept mass of strictly larger z
            frac = above / total
            near |= (kept & ((frac - float(top_p)).abs() < 1e-5)).any(1)
            kept &= (frac < float(top_p)) | (z == zmax)
        if min_keep > 1:
            zs0 = torch.where(kept_k, z, neg_inf).sort(dim=1, descending=True).values
            larger = torch.searchsorted(-zs0.contiguous(), -z.contiguous(), right=False)   # kept z strictly above
            kept |= kept_k & (larger < min_keep)
        p = torch.where(kept, p, torch.zeros_like(p))
    return kept, p, near


def sample_reference(logits, temperature, top_k, top_p, seed, step):
    """The contract for the rows b of logits [B, V] at draw step `step` (int or [B]). Returns (tokens int64 [B], near
    bool [B]); `near` marks rows whose draw u * Z lies within 1e-5 * Z of a CDF boundary, or whose top-p cut has a token
    within 1e-5 of top_p: there float32 device arithmetic may legitimately pick the neighbouring token."""
    kept, p, near = sample_support(logits, temperature, top_k, top_p)
    B = p.shape[0]
    nvalid = (~torch.isnan(logits.detach().cpu())).sum(1)
    cdf = p.cumsum(1)
    total = cdf[:, -1:]
    steps = np.broadcast_to(np.asarray(step, dtype=np.int64), (B,)).astype(np.uint64) & np.uint64(0xFFFFFFFF)
    ctr = np.stack([steps, np.arange(B, dtype=np.uint64), np.zeros(B, np.uint64), np.zeros(B, np.uint64)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint64), (B, 2))
    x = philox4x32_10(ctr, key)[:, 0]
    u = torch.from_numpy((x >> np.uint64(8)).astype(np.float64) / 2.0 ** 24)[:, None]
    target = u * total
    tok = (cdf > target).to(torch.int8).argmax(1)
    near |= (kept & ((cdf - target).abs() < 1e-5 * total)).any(1)
    dead = nvalid == 0
    tok[dead] = 0
    near[dead] = False
    return tok.long(), near


def sample_advance(logits, params, out_idx=None, next_src=None, positions=None, kv_len=None, token_log=None,
                   prompt_len=None):
    """Same arguments and bookkeeping as ops.sample_advance, on host tensors."""
    from .ops import SAMPLE_PARAMS
    temperature, top_k, top_p, _, seed = SAMPLE_PARAMS.unpack(params.cpu().numpy().tobytes())
    step = (kv_len.long() - prompt_len.long()).cpu().numpy() if kv_len is not None and prompt_len is not None else 0
    idx, _ = sample_reference(logits, temperature, top_k, top_p, seed, step)
    if out_idx is None:
        out_idx = torch.empty((logits.shape[0],), dtype=torch.int64)
    out_idx.copy_(idx)
    if next_src is not None:
        next_src.copy_(idx.to(next_src.dtype))
    if token_log is not None:
        for b in range(idx.shape[0]):
            s = int(kv_len[b]) - int(prompt_len[b])
            if 0 <= s < token_log.shape[1]:
                token_log[b, s] = idx[b]
    if positions is not None:
        positions.add_(1)
    if kv_len is not None:
        kv_len.add_(1)
    return out_idx
