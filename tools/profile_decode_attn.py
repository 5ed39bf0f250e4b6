"""Decode attention at the benchmark's shape (B = 8, 32 heads x 128, 896-token cache capacity, 832 tokens held): a CUDA-event
timing of `attn_decode_rope` launches replayed from a graph over enough layers' worth of distinct KV pages (> 200 MB) that
every launch reads its pages from HBM, not from the 50 MB L2 of an H100.

    python tools/profile_decode_attn.py            # the headline shape, one JSON line
    python tools/profile_decode_attn.py --sweep    # also B in {1, 2, 4, 8, 16, 32} and the beam kernel at B*k = 8, 32

The beam rows (k = 4 beams per request, 768 prompt keys shared by the beams of a request, 64 generated keys read through
beam_src from a sibling beam's pages) time `attn_decode_rope_beam`. Prints the GPU name and power limit."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
BF = torch.bfloat16
H, D, PS, CAP, LEN, PROMPT = 32, 128, 64, 896, 832, 768
max_pages = CAP // PS


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[-1] if r.returncode == 0 else f"nvidia-smi failed: {r.stderr.strip()}"


def time_attn(B, beam_k=0):
    layer_bytes = B * max_pages * H * PS * D * 2 * 2
    layers = max(2, -(-200_000_000 // layer_bytes))
    g = torch.Generator().manual_seed(0)
    n_pages = B * max_pages
    perm = torch.randperm(n_pages, generator=g).to(torch.int32).view(B, max_pages)
    if beam_k:   # the beams of a request share the prompt's pages (as LlamaEngine.start_beam forks them)
        for b in range(B):
            perm[b, :PROMPT // PS] = perm[b - b % beam_k, :PROMPT // PS]
        src = torch.arange(B, dtype=torch.int32)[:, None].repeat(1, CAP)
        sib = torch.randint(0, beam_k, (B, CAP), generator=g, dtype=torch.int32)
        src = (src - src % beam_k + sib).to(dev)
        gen = torch.full((B,), PROMPT, dtype=torch.int32, device=dev)
    perm = perm.to(dev)
    kps = [torch.randn((n_pages, H, PS, D), device=dev).to(BF) for _ in range(layers)]
    vps = [torch.randn((n_pages, H, PS, D), device=dev).to(BF) for _ in range(layers)]
    qkv = torch.randn((B, 3 * H * D), device=dev).to(BF)
    kvl = torch.full((B,), LEN, dtype=torch.int32, device=dev)
    table = ops.rope_table(kvl - 1, D, 10000.0)

    def run():
        for l in range(layers):
            if beam_k:
                ops.attn_decode_rope_beam(qkv, table, kps[l], vps[l], perm, kvl, src, gen, H, D, PS, CAP)
            else:
                ops.attn_decode_rope(qkv, table, kps[l], vps[l], perm, kvl, H, D, PS, CAP)
    run(); run()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr), ops.pdl(True):
        run()
    for _ in range(3):
        gr.replay()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    reps = max(20, 2000 // (layers * B))
    a.record()
    for _ in range(reps):
        gr.replay()
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) / reps / layers * 1e3
    bytes_ = B * LEN * 2 * H * D * 2
    del kps, vps, gr
    torch.cuda.empty_cache()
    return {"B": B, "beam_k": beam_k, "us_per_launch": round(us, 2), "algorithmic_MB": round(bytes_ / 1e6, 1),
            "achieved_GBs": round(bytes_ / us / 1e3, 1), "frac_of_h100_datasheet_hbm": round(bytes_ / us / 1e3 / 3350.0, 3)}


def main():
    with torch.no_grad():
        head = time_attn(8)
        res = {"gpu": gpu_info(), "shape": {"B": 8, "heads": H, "head_dim": D, "kv_len": LEN, "capacity": CAP}, **head}
        if "--sweep" in sys.argv:
            res["sweep"] = [time_attn(b) for b in (1, 2, 4, 8, 16, 32)] + [time_attn(b, beam_k=4) for b in (8, 32)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
