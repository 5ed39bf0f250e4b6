"""Per-kernel, in-situ breakdown of one graphed decode step at BASELINE.json configs[1]'s LLM shape: random-init Vicuna-7B,
B = 8, a 768-token prompt, KV capacity 896. The engine is run to mid-decode (64 steps), then STEPS replays of the step
graph are taken with torch.profiler (CUDA activities). Per kernel name: total time, launches, us per launch; GB/s for
`attn_decode_kernel` (K and V bytes of every row's attended keys, from the row lengths) and for each GEMV projection
(weight bytes from shapes; the GEMV launches of a step are qkv, o, gate_up, down per layer, then lm_head). Prints the GPU
name, power limit and max SM clock read in the same run. Under PDL a kernel's duration includes the time it waits for its
predecessor, so the per-kernel sum exceeds the step time.
Usage: python tools/kineto_decode.py [tag] [--out FILE]   (--out also writes the full breakdown as JSON)"""
import collections
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200.llama import LlamaEngine  # noqa: E402

VICUNA_7B = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)
B, PROMPT, CAP, WARM_STEPS, STEPS = 8, 768, 896, 64, 4
D, L = VICUNA_7B["hidden_size"], VICUNA_7B["num_hidden_layers"]
PROJ = [("qkv", 3 * D * D), ("o", D * D), ("gate_up", 2 * VICUNA_7B["intermediate_size"] * D),
        ("down", VICUNA_7B["intermediate_size"] * D)]


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[-1] if r.returncode == 0 else f"nvidia-smi failed: {r.stderr.strip()}"


def main():
    if not torch.cuda.is_available():
        raise SystemExit("kineto_decode.py needs a CUDA device")
    args = [a for a in sys.argv[1:]]
    out_file = None
    if "--out" in args:
        i = args.index("--out")
        out_file = args[i + 1]
        del args[i:i + 2]
    tag = args[0] if args else "run"
    dev = torch.device("cuda:0")
    eng = LlamaEngine(VICUNA_7B, dev, max_batch=B, max_seq_len=CAP).init_random(seed=0)
    ids = torch.randint(3, 32000, (B, PROMPT), generator=torch.Generator().manual_seed(2)).to(dev)
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        logits = eng.prefill(eng.embed[ids])
        eng.start_decode(logits.argmax(-1), CAP - PROMPT)
        eng.decode_steps(B, WARM_STEPS)
        torch.cuda.synchronize()
        lens = eng.d_len[:B].tolist()           # attended keys of the first profiled step; +1 per step after it
        a, b = torch.cuda.Event(True), torch.cuda.Event(True)
        a.record()
        eng.decode_steps(B, STEPS)
        b.record()
        torch.cuda.synchronize()
        step_ms = a.elapsed_time(b) / STEPS
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.decode_steps(B, STEPS)
            torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    dur = lambda e: e.device_time if hasattr(e, "device_time") else e.cuda_time
    name = lambda e: e.name.split("(")[0].replace("void ", "")[:80]
    agg = collections.defaultdict(lambda: [0, 0.0])
    for e in evs:
        agg[name(e)][0] += 1
        agg[name(e)][1] += dur(e)
    # bytes per launch kind: KV over the profiled steps' row lengths; weights by the GEMV's place in the step
    kv_bytes = sum(2 * (n + s) * D * 2 for s in range(STEPS) for n in lens) * L
    gemv = [e for e in evs if "gemv" in e.name]
    per_step = len(gemv) // STEPS
    proj = collections.defaultdict(lambda: [0, 0.0, 0])
    if per_step == 4 * L + 1:
        for i, e in enumerate(gemv):
            j = i % per_step
            nm, wb = PROJ[j % 4] if j < 4 * L else ("lm_head", VICUNA_7B["vocab_size"] * D)
            proj[nm][0] += 1
            proj[nm][1] += dur(e)
            proj[nm][2] += 2 * wb
    tot = sum(v[1] for v in agg.values())
    rows = sorted(agg.items(), key=lambda kv: -kv[1][1])
    attn = [v for k, v in agg.items() if "attn_decode_kernel" in k]
    attn_us = sum(v[1] for v in attn)
    attn_n = sum(v[0] for v in attn)
    out = {"tag": tag, "gpu": gpu_info(), "shape": {"B": B, "prompt": PROMPT, "capacity": CAP, "first_profiled_len": lens[0]},
           "step_ms_graph": round(step_ms, 4), "kernel_sum_ms_per_step": round(tot / 1e3 / STEPS, 4),
           "attn_decode": {"us_per_launch": round(attn_us / max(attn_n, 1), 2), "share_of_kernel_time": round(attn_us / tot, 4),
                           "GBps": round(kv_bytes / attn_us * 1e-3, 1) if attn_us else None},
           "gemv": {k: {"launches": v[0], "us_per_launch": round(v[1] / v[0], 2), "GBps": round(v[2] / v[1] * 1e-3, 1)}
                    for k, v in proj.items()},
           "kernels": {k: {"launches": v[0], "total_us": round(v[1], 1), "us_per_launch": round(v[1] / v[0], 2)}
                       for k, v in rows}}
    print(json.dumps({k: out[k] for k in ("tag", "gpu", "shape", "step_ms_graph", "kernel_sum_ms_per_step", "attn_decode",
                                          "gemv")}))
    for k, v in rows[:20]:
        print(f"{v[1] / 1e3 / STEPS:8.3f} ms/step  {100 * v[1] / tot:5.1f}%  n={v[0] // STEPS:4d}/step  {v[1] / v[0]:7.1f} us  {k}")
    if out_file:
        with open(out_file, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
