"""Logits processors on one GPU: graphed decode steps with processors off against on (repetition_penalty = 1.1,
no_repeat_ngram_size = 3, min_new_tokens = 8) at BASELINE.json configs[1]'s LLM shapes (random-init Vicuna-7B, 768-token
prompt, 128 new tokens with EOS disabled: the first from the prefill logits, then 127 graphed steps). Greedy and sampled
(T = 0.7, top_p = 0.9) at B = 8, beam search and beam sampling at B = 8 requests x k = 4 beams; off and on alternate, best
of 3 repeats, timed with CUDA events. Also launches per step, and logits_process alone in µs per launch at [8, 32000] and
[32, 32000] with a 513-token prompt + 127 generated ids of history (raw and LOGPROBS mode), back to back in a CUDA graph.
Prints the GPU name and power limit and one JSON line."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import beam, ops, processors, param_shapes as PS  # noqa: E402
from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM  # noqa: E402
from tools.bench_beam import VICUNA_7B, gpu_info, timed  # noqa: E402

PROMPT, NEW, REPEATS, B, K = 768, 128, 3, 8, 4
PROC = dict(repetition_penalty=1.1, no_repeat_ngram_size=3, min_new_tokens=8)


def step_ms(eng, emb, ids, mode, proc):
    """ms per graphed step of one 127-step decode; the prefill and the first token are outside the timed window."""
    rows = emb.shape[0] * (K if mode.startswith("beam") else 1)
    if proc:
        eng.set_processors(ids.cpu().repeat_interleave(rows // ids.shape[0], 0), eos_ids=[-1], **PROC)
    else:
        eng.clear_processors()
    logits = eng.prefill(emb)
    if mode.startswith("beam"):
        prm = beam.pack_params(1.0, False, 0, PROMPT, PROMPT + NEW, [-1]).to(emb.device)
        eng.start_beam(logits, K, NEW, prm, sample=mode == "beam_sample")
    else:
        if proc:
            eng.process_logits(logits)
        first = eng.sample_advance(logits) if mode == "sample" else ops.argmax_rows(logits)
        eng.start_decode(first, NEW)
    sampled = {"greedy": False, "sample": True}.get(mode, mode)
    ms = timed(lambda: eng.decode_steps(rows, NEW - 1, sampled=sampled)) / (NEW - 1)
    return ms, eng.launches_per_step


def process_us(R, logprobs, dev):
    """µs per launch of logits_process at [R, 32000]: history = 513 prompt ids + 127 generated ids per row."""
    g = torch.Generator().manual_seed(R)
    V, n_in, t, P = 32000, 513, 127, 700
    logits = torch.randn((R, V), generator=g).to(dev)
    prompt = torch.randint(0, V, (R, n_in), generator=g, dtype=torch.int32).to(dev)
    token_log = torch.randint(0, V, (R, 1024), generator=g).to(dev)
    beam_src = torch.arange(R, dtype=torch.int32)[:, None].repeat(1, 1024).to(dev) if logprobs else None
    kv_len = torch.full((R,), P + t, dtype=torch.int32, device=dev)
    prompt_len = torch.full((R,), P, dtype=torch.int32, device=dev)
    prm = processors.pack_params(input_len=n_in, eos_ids=[2], **PROC).to(dev)
    call = lambda: ops.logits_process(logits, prm, prompt, token_log=token_log, kv_len=kv_len, prompt_len=prompt_len,
                                      beam_src=beam_src, logprobs=logprobs)
    call()
    n = 50
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), ops.pdl(True):
        for _ in range(n):
            call()
    return min(timed(graph.replay) * 1e3 / n for _ in range(5))


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_processors.py needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = VitronConfig(llm=VICUNA_7B, vision=None, video=None, tokenizer_model_max_length=4096)
    model = VitronLlamaForCausalLM(cfg, dev, max_batch=B * K, max_seq_len=PROMPT + NEW)
    sd = PS.random_state_dict(PS.vitron_shapes(cfg), dev, seed=0)
    model.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    eng = model.engine
    out = {"what": "ms per graphed decode step (127 steps after the prefill, best of 3 alternating repeats), processors "
                   "off vs on (repetition_penalty 1.1, no_repeat_ngram_size 3, min_new_tokens 8), random-init Vicuna-7B, "
                   "768-token prompt, EOS disabled, B = 8 (beam modes: 8 requests x 4 beams); sampling T = 0.7, top_p 0.9",
           "gpu": gpu_info(), "modes": {}}
    eng.set_sampling(0.7, None, 0.9, 1234)
    ids = torch.randint(3, 32000, (B, PROMPT), generator=torch.Generator().manual_seed(B)).to(dev)
    with torch.no_grad():
        emb = model.model.embed_tokens(ids)
        for mode in ("greedy", "sample", "beam", "beam_sample"):
            l_off = step_ms(eng, emb, ids, mode, False)[1]      # capture + warm both graphs
            l_on = step_ms(eng, emb, ids, mode, True)[1]
            off, on = [], []
            for _ in range(REPEATS):
                off.append(step_ms(eng, emb, ids, mode, False)[0])
                on.append(step_ms(eng, emb, ids, mode, True)[0])
            out["modes"][mode] = {"rows": B * (K if mode.startswith("beam") else 1),
                                  "off_ms_per_step": round(min(off), 3), "on_ms_per_step": round(min(on), 3),
                                  "on_over_off": round(min(on) / min(off), 4),
                                  "ms_all_repeats": {"off": [round(x, 3) for x in off], "on": [round(x, 3) for x in on]},
                                  "launches_per_step": {"off": l_off, "on": l_on}}
        eng.clear_processors()
        out["logits_process_us_per_launch"] = {f"R{R}_{'logprobs' if lp else 'raw'}": round(process_us(R, lp, dev), 2)
                                               for R in (8, 32) for lp in (False, True)}
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
