"""Beam search and beam sampling against greedy graphed decode on one GPU: random-init Vicuna-7B, B in {1, 8} requests,
k in {2, 4} beams, a 768-token prompt and 128 new tokens with EOS disabled (the first from the prefill logits, then 127
graphed steps). Beam-search, beam-sampling (do_sample with T = 0.7, top_p = 0.9) and greedy steps are compared at the
same number of rows (B * k), alternating, best of 3 repeats, timed with CUDA events. Also times beam_advance and
beam_sample_advance per launch on the [B * k, 32000] logits of the step, and the prompt prefill once per request against
the reference's prefill of B * k expanded rows. Prints one JSON line."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import beam, ops, param_shapes as PS  # noqa: E402
from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM  # noqa: E402

VICUNA_7B = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, vocab_size=32000,
                 rms_norm_eps=1e-5, rope_theta=10000.0)
PROMPT, NEW, REPEATS = 768, 128, 3
CASES = [(1, 2), (1, 4), (8, 2), (8, 4)]


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


def greedy_ms(eng, emb_rows):
    R = emb_rows.shape[0]
    eng.start_decode(ops.argmax_rows(eng.prefill(emb_rows)), NEW)
    return timed(lambda: eng.decode_steps(R, NEW - 1)) / (NEW - 1), eng.launches_per_step


def beam_ms(eng, emb, k, prm, sample=False):
    mode = "beam_sample" if sample else "beam"
    eng.start_beam(eng.prefill(emb), k, NEW, prm, sample=sample)
    return timed(lambda: eng.decode_steps(emb.shape[0] * k, NEW - 1, sampled=mode)) / (NEW - 1), eng.launches_per_step


def step_us(eng, emb, k, prm, sample):
    """µs per launch of the beam step alone, back to back in a CUDA graph, on the state start_beam leaves (step 0 on the
    prefill logits done) and the logits of the step."""
    R = emb.shape[0] * k
    eng.start_beam(eng.prefill(emb), k, NEW, prm, sample=sample)
    st = {n: t[:R] for n, t in eng.beam.items()}
    book = dict(next_src=eng.d_src[:R], positions=eng.d_pos[:R], kv_len=eng.d_len[:R], token_log=eng.token_log[:R],
                prompt_len=eng.d_prompt[:R])
    saved = [t.clone() for t in list(st.values()) + list(book.values())]
    if sample:
        step = lambda: ops.beam_sample_advance(eng.d_logits[:R], k, prm, eng.d_sample, **st, **book)
    else:
        step = lambda: ops.beam_advance(eng.d_logits[:R], k, prm, **st, **book)
    graph = torch.cuda.CUDAGraph()
    n = 20                                      # 20 launches move kv_len by 20 < the reserved 128 positions
    with torch.cuda.graph(graph):
        for _ in range(n):
            step()
    us = []
    for _ in range(5):
        for t, sv in zip(list(st.values()) + list(book.values()), saved):
            t.copy_(sv)
        us.append(timed(graph.replay) * 1e3 / n)
    for t, sv in zip(list(st.values()) + list(book.values()), saved):
        t.copy_(sv)
    return min(us)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_beam.py needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = VitronConfig(llm=VICUNA_7B, vision=None, video=None, tokenizer_model_max_length=4096)
    Rmax = max(b * k for b, k in CASES)
    model = VitronLlamaForCausalLM(cfg, dev, max_batch=Rmax, max_seq_len=PROMPT + NEW)
    sd = PS.random_state_dict(PS.vitron_shapes(cfg), dev, seed=0)
    model.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    eng = model.engine
    out = {"what": "ms per graphed decode step (127 steps after the prefill, best of 3 alternating repeats), "
                   "random-init Vicuna-7B, 768-token prompt, EOS disabled; beam sampling at T = 0.7, top_p = 0.9",
           "gpu": gpu_info(), "cases": {}}
    eng.set_sampling(0.7, None, 0.9, 1234)
    with torch.no_grad():
        for B, k in CASES:
            ids = torch.randint(3, 32000, (B, PROMPT), generator=torch.Generator().manual_seed(B)).to(dev)
            emb = model.model.embed_tokens(ids)
            emb_rows = emb.repeat_interleave(k, 0)
            prm = beam.pack_params(1.0, False, 0, PROMPT, PROMPT + NEW, [-1]).to(dev)
            g_l = greedy_ms(eng, emb_rows)[1]          # capture + warm the three graphs
            b_l = beam_ms(eng, emb, k, prm)[1]
            s_l = beam_ms(eng, emb, k, prm, sample=True)[1]
            g, bm, bs, pf1, pfk = [], [], [], [], []
            for _ in range(REPEATS):
                g.append(greedy_ms(eng, emb_rows)[0])
                bm.append(beam_ms(eng, emb, k, prm)[0])
                bs.append(beam_ms(eng, emb, k, prm, sample=True)[0])
                pf1.append(timed(lambda: eng.prefill(emb)))
                pfk.append(timed(lambda: eng.prefill(emb_rows)))
            R = B * k
            us, us_s = [], []
            for _ in range(2):                          # the two step kernels alternate on the logits of a decode step
                us.append(step_us(eng, emb, k, prm, False))
                us_s.append(step_us(eng, emb, k, prm, True))
            out["cases"][f"B{B}_k{k}"] = {
                "rows": R, "greedy_ms_per_step": round(min(g), 3), "beam_ms_per_step": round(min(bm), 3),
                "beam_sample_ms_per_step": round(min(bs), 3), "beam_over_greedy": round(min(bm) / min(g), 4),
                "beam_sample_over_beam": round(min(bs) / min(bm), 4),
                "ms_all_repeats": {"greedy": [round(x, 3) for x in g], "beam": [round(x, 3) for x in bm],
                                   "beam_sample": [round(x, 3) for x in bs]},
                "launches_per_step": {"greedy": g_l, "beam": b_l, "beam_sample": s_l},
                "beam_advance_us_per_launch": round(min(us), 2),
                "beam_sample_advance_us_per_launch": round(min(us_s), 2),
                "prefill_ms": {"once_per_request": round(min(pf1), 2), "expanded_B_x_k_rows": round(min(pfk), 2)},
            }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
