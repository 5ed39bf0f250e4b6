"""Sampled against greedy graphed decode on one GPU at BASELINE.json configs[1]'s LLM shapes: random-init Vicuna-7B,
B = 8, a 768-token prompt, 128 new tokens (the first from the prefill logits, then 127 graphed decode steps). Modes are
timed with CUDA events in one process, alternating, 3 repeats. Also times sample_advance against argmax_advance per
launch from a CUDA graph of back-to-back launches on [8, 32000] fp32 logits. Prints one JSON line."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import ops, param_shapes as PS  # noqa: E402
from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM  # noqa: E402

VICUNA_7B = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)
B, PROMPT, NEW, REPEATS = 8, 768, 128, 3
MODES = {"greedy": None, "T0.2_top_p0.9": (0.2, None, 0.9), "top_k50": (1.0, 50, None), "T1": (1.0, None, None)}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[-1] if r.returncode == 0 else f"nvidia-smi failed: {r.stderr.strip()}"


def time_decode(eng, emb, mode):
    """ms of the 127 graphed decode steps after a prefill (the prefill is outside the timed window)."""
    logits = eng.prefill(emb)
    if mode is None:
        first = ops.argmax_rows(logits)
    else:
        eng.set_sampling(*mode, seed=1234)
        first = ops.sample_advance(logits, eng.d_sample)
    eng.start_decode(first, NEW)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    eng.decode_steps(B, NEW - 1, sampled=mode is not None)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def us_per_launch(fn, n=200, reps=5):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (n * reps)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling.py needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = VitronConfig(llm=VICUNA_7B, vision=None, video=None, tokenizer_model_max_length=4096)
    model = VitronLlamaForCausalLM(cfg, dev, max_batch=B, max_seq_len=PROMPT + NEW)
    sd = PS.random_state_dict(PS.vitron_shapes(cfg), dev, seed=0)
    model.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    eng = model.engine
    ids = torch.randint(3, 32000, (B, PROMPT), generator=torch.Generator().manual_seed(2)).to(dev)
    with torch.no_grad():
        emb = model.model.embed_tokens(ids)
        launches = {}
        for name, mode in MODES.items():            # capture + warm every graph before timing
            time_decode(eng, emb, mode)
            launches[name] = eng.launches_per_step
        ms = {name: [] for name in MODES}
        for _ in range(REPEATS):
            for name, mode in MODES.items():
                ms[name].append(time_decode(eng, emb, mode))
        logits = torch.randn((B, 32000), generator=torch.Generator().manual_seed(3)).to(dev) * 3
        params = ops.sample_params(1.0, 50, 0.9, 7).to(dev)
        idx = torch.empty((B,), dtype=torch.int64, device=dev)
        us_sample = us_per_launch(lambda: ops.sample_advance(logits, params, idx))
        us_argmax = us_per_launch(lambda: ops.argmax_advance(logits, idx))
    best = {name: min(v) for name, v in ms.items()}
    tps = {name: B * (NEW - 1) / (t * 1e-3) for name, t in best.items()}
    print(json.dumps({
        "what": "graphed decode tokens/s (127 steps after the prefill, best of 3 alternating repeats), "
                "random-init Vicuna-7B, B=8, 768-token prompt",
        "gpu": gpu_info(),
        "tokens_per_s": {k: round(v, 1) for k, v in tps.items()},
        "ratio_to_greedy": {k: round(v / tps["greedy"], 4) for k, v in tps.items()},
        "ms_all_repeats": {k: [round(x, 3) for x in v] for k, v in ms.items()},
        "launches_per_step": launches,
        "us_per_launch_B8_V32000": {"sample_advance(top_k=50, top_p=0.9)": round(us_sample, 2),
                                    "argmax_advance": round(us_argmax, 2)},
    }))


if __name__ == "__main__":
    main()
