"""NF4 against bf16 weights at BASELINE.json configs[1]'s LLM shapes on one GPU: random-init Vicuna-7B, B = 8, a 768-token
prompt, 128 new tokens (the first from the prefill logits, then 127 graphed decode steps). Both engines live in one
process and are timed with CUDA events, alternating, after a warm-up, 3 repeats. Prints decode tokens/s and step time,
prefill time, streamed weight bytes, device memory, achieved bytes/s (weight bytes + KV bytes per step, from shapes, over
the step time), and a kernel leg: the NF4 GEMV against the bf16 GEMV per Vicuna projection shape at M = 1, 8 and 32
(CUDA-graph replay, weights rotated through more than the L2). Prints one JSON line."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import nf4, ops  # noqa: E402
from vitron_b200.llama import LlamaEngine  # noqa: E402

VICUNA_7B = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)
B, PROMPT, NEW, REPEATS = 8, 768, 128, 3
SHAPES = {"qkv": (12288, 4096), "o": (4096, 4096), "gate_up (SwiGLU)": (22016, 4096), "down": (4096, 11008)}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[-1] if r.returncode == 0 else f"nvidia-smi failed: {r.stderr.strip()}"


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def run(eng, emb):
    """(prefill ms, decode ms of the 127 graphed steps)."""
    t_pre, logits = timed(lambda: eng.prefill(emb))
    eng.start_decode(ops.argmax_rows(logits), NEW)
    t_dec, _ = timed(lambda: eng.decode_steps(B, NEW - 1))
    return t_pre, t_dec


def kv_bytes_per_step(c):
    """K and V of every layer read over the mean attended length of the 127 steps, plus the new token's K/V written."""
    mean_keys = PROMPT + 1 + (NEW - 2) / 2
    per_key = 2 * c["num_hidden_layers"] * c["hidden_size"] * 2
    return B * per_key * (mean_keys + 1)


def us_per_call(fn, n=20, reps=5):
    fn(0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), ops.pdl(True):
        for i in range(n):
            fn(i)
    g.replay()
    ms, _ = timed(lambda: [g.replay() for _ in range(reps)])
    return ms * 1e3 / (n * reps)


def kernel_leg(dev):
    res = {}
    gen = torch.Generator(device=dev).manual_seed(5)
    for name, (n, k) in SHAPES.items():
        copies = max(2, int(200e6 // (2 * n * k)) + 1)           # > L2 of bf16 weights per replay cycle
        w16 = [(torch.randn((n, k), generator=gen, device=dev) * 0.02).to(torch.bfloat16) for _ in range(copies)]
        w4 = [nf4.quantize(w) for w in w16]
        ks = torch.ones((k,), dtype=torch.float32, device=dev)
        glu = ops.GLU_SWIGLU if "SwiGLU" in name else ops.GLU_NONE
        for m in (1, 8, 32):
            x = torch.randn((m, k), generator=gen, device=dev).to(torch.bfloat16)
            t16 = us_per_call(lambda i: ops.gemm(x, w16[i % copies], glu=glu))
            t4 = us_per_call(lambda i: ops.gemm(x, w4[i % copies], glu=glu, kscale=ks))
            b4 = w4[0].nbytes
            res[f"{name} {n}x{k} M={m}"] = {"bf16_us": round(t16, 2), "nf4_us": round(t4, 2), "speedup": round(t16 / t4, 3),
                                            "bf16_weight_GBps": round(2 * n * k / t16 * 1e-3, 1),
                                            "nf4_weight_GBps": round(b4 / t4 * 1e-3, 1)}
        del w16, w4
        torch.cuda.empty_cache()
    return res


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_nf4.py needs a CUDA device")
    dev = torch.device("cuda:0")
    engines, mem = {}, {}
    for name, q in (("bf16", False), ("nf4", True)):
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated(dev)
        engines[name] = LlamaEngine(VICUNA_7B, dev, max_batch=B, max_seq_len=PROMPT + NEW).init_random(seed=0, nf4=q)
        torch.cuda.synchronize()
        mem[name] = torch.cuda.memory_allocated(dev) - m0
    ids = torch.randint(3, 32000, (B, PROMPT), generator=torch.Generator().manual_seed(2)).to(dev)
    res = {name: {"prefill_ms": [], "decode_ms": []} for name in engines}
    with torch.no_grad():
        for name, eng in engines.items():        # capture + warm every graph and workspace before timing
            run(eng, eng.embed[ids])
        for _ in range(REPEATS):
            for name, eng in engines.items():
                t_pre, t_dec = run(eng, eng.embed[ids])
                res[name]["prefill_ms"].append(round(t_pre, 3))
                res[name]["decode_ms"].append(round(t_dec, 3))
        kv = kv_bytes_per_step(VICUNA_7B)
        out = {}
        for name, eng in engines.items():
            step_ms = min(res[name]["decode_ms"]) / (NEW - 1)
            wb = eng.weight_bytes()
            out[name] = {"decode_tokens_per_s": round(B / (step_ms * 1e-3), 1), "step_ms": round(step_ms, 4),
                         "prefill_ms": min(res[name]["prefill_ms"]), "launches_per_step": eng.launches_per_step,
                         "weight_bytes_streamed_per_step": wb, "engine_device_bytes": mem[name],
                         "achieved_TBps": round((wb + kv) / (step_ms * 1e-3) * 1e-12, 3), "all_repeats": res[name]}
        for eng in engines.values():
            eng._graphs = {}
        del engines
        torch.cuda.empty_cache()
        kern = kernel_leg(dev)
    print(json.dumps({
        "what": "random-init Vicuna-7B, B=8, 768-token prompt, 127 graphed decode steps; best of 3 alternating repeats",
        "gpu": gpu_info(),
        "kv_bytes_per_step": int(kv),
        "engines": out,
        "decode_speedup_nf4_over_bf16": round(out["bf16"]["step_ms"] / out["nf4"]["step_ms"], 3),
        "kernels_us_graph_replay": kern,
    }))


if __name__ == "__main__":
    main()
