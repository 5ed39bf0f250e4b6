"""Appending a chunk to the paged KV cache against re-prefilling the whole sequence, on one GPU: random-init Vicuna-7B,
B = 1 (one chat user) and B = 8, a cached past P in {768, 2113} and chunks S in {1, 32, 128, 512}.

Two legs, timed with CUDA events after a warm-up of the card and of every configuration (best of REPEATS, alternating):
  engine:  LlamaEngine.append(S tokens after P cached) against LlamaEngine.prefill(P + S tokens);
  kernel:  vb200_attention_paged (S queries over P + S cached keys, pages shuffled) against vb200_attention at the equal
           causal shape (q [B, S, 32, 128], contiguous k / v [B, P + S, 32, 128]), and the paged kernel without split-KV;
           mean over ITERS launches replayed from one CUDA graph.
Reads the card's name and power limit in the same run. Prints one JSON line (and writes it to --out if given)."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import ops  # noqa: E402
from vitron_b200.llama import LlamaEngine  # noqa: E402

VICUNA_7B = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)
BATCHES, PASTS, CHUNKS = (1, 8), (768, 2113), (1, 32, 128, 512)
REPEATS, ITERS, WARMUP, WARM_PREFILLS = 5, 50, 3, 20


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[-1] if r.returncode == 0 else f"nvidia-smi failed: {r.stderr.strip()}"


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def engine_leg(dev):
    eng = LlamaEngine(VICUNA_7B, dev, max_batch=max(BATCHES), max_seq_len=max(PASTS) + max(CHUNKS)).init_random(seed=0)
    out = {}
    with torch.no_grad():
        # bring the card to its sustained clock before the first timed configuration (a few seconds of prefills)
        warm = eng.embed[torch.randint(3, 32000, (max(BATCHES), max(PASTS)), generator=torch.Generator().manual_seed(1))
                         .to(dev)]
        for _ in range(WARM_PREFILLS):
            eng.prefill(warm)
        torch.cuda.synchronize()
        for B in BATCHES:
            for P in PASTS:
                ids = torch.randint(3, 32000, (B, P + max(CHUNKS)), generator=torch.Generator().manual_seed(P)).to(dev)
                emb = eng.embed[ids]
                eng.prefill(emb[:, :P])
                for S in CHUNKS:
                    chunk, whole = emb[:, P:P + S].contiguous(), emb[:, :P + S].contiguous()
                    append = lambda: eng.append(chunk, [S] * B, all_logits=False, past_lens=[P] * B)
                    prefill = lambda: eng.prefill(whole)
                    for _ in range(WARMUP):                # workspaces, tensor maps, allocator, clocks
                        for f in (prefill, append):
                            f()
                    ta, tp = [], []
                    for _ in range(REPEATS):
                        tp.append(timed(prefill))
                        ta.append(timed(append))        # branches from the same P cached tokens every time
                    out[f"B={B} P={P} S={S}"] = {"append_ms": round(min(ta), 3), "prefill_P+S_ms": round(min(tp), 3),
                                                 "speedup": round(min(tp) / min(ta), 2)}
    del eng
    torch.cuda.empty_cache()
    return out


def us_per_call(fn):
    """Mean time of ITERS launches replayed from one CUDA graph (no host launch overhead in the window)."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(ITERS):
            fn()
    g.replay()
    return timed(g.replay) * 1e3 / ITERS


def kernel_leg(dev):
    lib = ops._lib.load()
    H, D, PG = 32, 128, 64
    out = {}
    g = torch.Generator(device="cpu").manual_seed(3)
    for B in BATCHES:
        for P in PASTS:
            for S in CHUNKS:
                T = P + S
                npg = (T + PG - 1) // PG
                table = torch.randperm(B * npg, generator=g).view(B, npg).to(torch.int32).to(dev)
                kp = torch.randn((B * npg, H, PG, D), device=dev).to(torch.bfloat16)
                vp = torch.randn((B * npg, H, PG, D), device=dev).to(torch.bfloat16)
                qkv = torch.randn((B * S, 3 * H * D), device=dev).to(torch.bfloat16)
                q = qkv.view(B, S, 3, H, D)[:, :, 0]
                qs = torch.full((B,), P, dtype=torch.int32, device=dev)
                ql = torch.full((B,), S, dtype=torch.int32, device=dev)
                k = torch.randn((B, T, H, D), device=dev).to(torch.bfloat16)
                v = torch.randn((B, T, H, D), device=dev).to(torch.bfloat16)
                o = torch.empty((B, S, H, D), dtype=torch.bfloat16, device=dev)
                paged = lambda: ops.attention_paged(q, kp, vp, table, qs, ql, T, out=o)
                dense = lambda: ops.attention(q, k, v, causal=True, out=o)
                unsplit = lambda: ops.check(lib.vb200_attention_paged(   # the same kernel without a workspace: unsplit
                    q.data_ptr(), *q.stride()[:3], kp.data_ptr(), vp.data_ptr(), kp.shape[0], table.data_ptr(), npg,
                    qs.data_ptr(), ql.data_ptr(), o.data_ptr(), *o.stride()[:3], B, H, S, D, PG, T, D ** -0.5, None, 0,
                    torch.cuda.current_stream().cuda_stream), "vb200_attention_paged")
                t = {name: min(us_per_call(f) for _ in range(REPEATS))
                     for name, f in (("paged", paged), ("attention", dense), ("paged_unsplit", unsplit))}
                flops = 4.0 * B * H * D * S * (P + (S + 1) / 2)   # QK^T and PV over the visible keys
                out[f"B={B} P={P} S={S}"] = {"paged_us": round(t["paged"], 2), "attention_us": round(t["attention"], 2),
                                             "paged_unsplit_us": round(t["paged_unsplit"], 2),
                                             "paged_TFLOPs": round(flops / (t["paged"] * 1e-6) * 1e-12, 1),
                                             "split_kv": lib.vb200_attention_paged_workspace_size(B, H, S, D, T) > 0}
                del kp, vp, k, v, qkv
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv_append.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"what": "random-init Vicuna-7B: append(S after P cached) vs prefill(P + S); paged attention kernel vs "
                   "vb200_attention at the equal causal shape (H=32, hd=128); best of 5",
           "gpu": gpu_info(), "engine_ms": engine_leg(dev), "kernel_us": kernel_leg(dev)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
