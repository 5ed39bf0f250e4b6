"""Quick GPU check of the wgmma attention kernel against fp32 eager attention + timing vs mma.sync / SDPA."""
import math, sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vitron_b200 import ops

dev = torch.device("cuda:0")
BF = torch.bfloat16


def ref(q, k, v, causal):
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    s = qf @ kf.transpose(-1, -2) / math.sqrt(q.shape[-1])
    if causal:
        Sq, Skv = s.shape[-2:]
        m = torch.arange(Skv, device=dev)[None, :] > (torch.arange(Sq, device=dev)[:, None] + Skv - Sq)
        s = s.masked_fill(m, float("-inf"))
    return (torch.softmax(s, -1) @ vf).permute(0, 2, 1, 3)


def timed(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


from vitron_b200 import _lib
print("occupancy hd64/hd128:", _lib.load().vb200_attention_tc_occupancy(64), _lib.load().vb200_attention_tc_occupancy(128), flush=True)
cases = [(1, 2, 128, 64, 64, False), (1, 2, 128, 64, 128, False), (1, 1, 128, 128, 64, False), (2, 4, 300, 300, 128, True),
         (8, 16, 257, 257, 64, False), (1, 32, 1728, 1728, 128, True), (2, 5, 2560, 2560, 64, False), (16, 5, 2560, 2560, 64, False),
         (16, 10, 640, 640, 64, False), (16, 5, 2560, 77, 64, False)]
for B, H, Sq, Skv, D, causal in cases:
    g = torch.Generator(device=dev).manual_seed(1)
    q, k, v = (torch.randn((B, s, H, D), device=dev, generator=g).to(BF) for s in (Sq, Skv, Skv))
    r = ref(q, k, v, causal)
    out = {}
    for impl in (2, 1):
        ops.set_attention_impl(impl)
        o = ops.attention(q, k, v, causal=causal)
        wd = ops.attention_watchdog()
        if wd[0]:
            print("WATCHDOG", wd, "case", (B, H, Sq, Skv, D, causal), "impl", impl, flush=True)
            sys.exit(1)
        err = float((o.float() - r).abs().max())
        ms = timed(lambda: ops.attention(q, k, v, causal=causal))
        out[impl] = (err, ms)
    ops.set_attention_impl(0)
    qs, ks, vs = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    ms_sdpa = timed(lambda: torch.nn.functional.scaled_dot_product_attention(qs, ks, vs, is_causal=causal))
    fl = 4.0 * B * H * Sq * Skv * D * (0.5 if causal else 1.0)
    print(json.dumps({"case": [B, H, Sq, Skv, D, causal], "tc_err": round(out[2][0], 5), "mma_err": round(out[1][0], 5),
                      "tc_ms": round(out[2][1], 4), "mma_ms": round(out[1][1], 4), "sdpa_ms": round(ms_sdpa, 4),
                      "tc_tflops": round(fl / out[2][1] / 1e9, 1)}), flush=True)
