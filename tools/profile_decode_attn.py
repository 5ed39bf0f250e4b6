"""Decode attention at the benchmark's shape (B = 8, 32 heads x 128, 896-token cache capacity, 832 tokens held) over several
layers' worth of distinct KV pages, for `ncu --set full -k regex:attn_decode -s 4 -c 2` (steady-state launches), and a
CUDA-event timing of the same launches replayed from a graph with L2 flushed by the page set (8 layers x 109 MB > 126 MB)."""
import os, sys, json
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
BF = torch.bfloat16
B, H, D, PS, CAP, LEN, LAYERS = 8, 32, 128, 64, 896, 832, 8
max_pages = CAP // PS
with torch.no_grad():
    g = torch.Generator().manual_seed(0)
    perm = torch.randperm(B * max_pages, generator=g).to(torch.int32).view(B, max_pages).to(dev)
    kps = [torch.randn((B * max_pages, H, PS, D), device=dev).to(BF) for _ in range(LAYERS)]
    vps = [torch.randn((B * max_pages, H, PS, D), device=dev).to(BF) for _ in range(LAYERS)]
    qkv = torch.randn((B, 3 * H * D), device=dev).to(BF)
    kvl = torch.full((B,), LEN, dtype=torch.int32, device=dev)
    table = ops.rope_table(kvl - 1, D, 10000.0)

    def run():
        for l in range(LAYERS):
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
    a.record()
    for _ in range(20):
        gr.replay()
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) / 20 / LAYERS * 1e3
    bytes_ = B * LEN * 2 * H * D * 2
    print(json.dumps({"shape": {"B": B, "heads": H, "head_dim": D, "kv_len": LEN, "capacity": CAP}, "us_per_launch": round(us, 2),
                      "algorithmic_MB": round(bytes_ / 1e6, 1), "achieved_GBs": round(bytes_ / us / 1e3, 1),
                      "frac_of_h100_datasheet_hbm": round(bytes_ / us / 1e3 / 3350.0, 3)}))
