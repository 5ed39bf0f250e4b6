#!/usr/bin/env python
"""bench.py — headline benchmark of the Vitron multimodal forward path on an H100 (sm_90a).

Workload (BASELINE.json configs[1]): batch-8 images -> LanguageBind ViT-L/14 encode + mlp2x_gelu
projector + splice -> Vicuna-7B prefill over 256 vision + 512 text tokens -> 128 greedy decode
tokens, bf16, random-init weights, synthetic pixels / ids. One "step" = that whole pass for one
batch. `value` = generated tokens / s of the whole job (all ranks) with inputs resident in HBM;
`e2e` = same through VitronLlamaForCausalLM.generate() with HOST (pinned) inputs and the ids read
back. N > 1: one process per GPU (torchrun), independent request batches (weak scaling), one NCCL
all_gather of the generated ids at the end of every step.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]

--steps K sets the timed steps of every leg (tokens/s, e2e, video, UNet). --dump-outputs DIR writes what the timed path
returned in its last step as DIR/<name>.npy (token ids as float64, latents as float32): the inputs are seeded, so two
builds run with the same arguments can be compared output for output.
"""
import argparse
import json
import os
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "Vicuna-7B generated tokens/s, batch-8 x (256 vision + 512 text) prefill + 128-token greedy decode, incl. ViT-L/14 encode"
VICUNA_7B = dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                 vocab_size=32000, rms_norm_eps=1e-5, rope_theta=10000.0)
VIT_L14 = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
               image_size=224, patch_size=14, hidden_act="gelu")
BATCH, TEXT, VISION, NEW = 8, 512, 256, 128


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return d.get("hbm_gbs", 3350.0), d.get("bf16_tflops", 989.0), "measured"
    return 3350.0, 989.0, "H100 SXM data sheet (dense bf16, 700 W)"


class ClockSampler(threading.Thread):
    """Samples SM clock / throttle reasons of one GPU with NVML while the timed region runs."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.samples, self.reasons, self.stop_flag, self.max_mhz = index, [], set(), False, None

    def run(self):
        try:
            import pynvml as N
            N.nvmlInit()
            h = N.nvmlDeviceGetHandleByIndex(self.index)
            self.max_mhz = N.nvmlDeviceGetMaxClockInfo(h, N.NVML_CLOCK_SM)
            names = {"hw_slowdown": getattr(N, "nvmlClocksThrottleReasonHwSlowdown", 0x8),
                     "hw_thermal_slowdown": getattr(N, "nvmlClocksThrottleReasonHwThermalSlowdown", 0x40),
                     "sw_thermal_slowdown": getattr(N, "nvmlClocksThrottleReasonSwThermalSlowdown", 0x20),
                     "sw_power_cap": getattr(N, "nvmlClocksThrottleReasonSwPowerCap", 0x4)}
            while not self.stop_flag:
                self.samples.append(N.nvmlDeviceGetClockInfo(h, N.NVML_CLOCK_SM))
                try:
                    r = N.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                    for k, bit in names.items():
                        if r & bit:
                            self.reasons.add(k)
                except Exception:
                    pass
                time.sleep(0.1)
        except Exception as e:  # NVML unavailable: report it rather than invent numbers
            self.reasons.add(f"nvml_unavailable:{type(e).__name__}")

    def result(self):
        s = sorted(self.samples)
        return {"sm_mhz": s[len(s) // 2] if s else None, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons)}


def synth_inputs(seed_px=1, seed_ids=2, batch=BATCH):
    g = torch.Generator().manual_seed(seed_px)
    pixels = torch.randn((batch, 3, 224, 224), generator=g)
    g = torch.Generator().manual_seed(seed_ids)
    ids = torch.randint(3, 32000, (batch, TEXT + 1), generator=g)
    ids[:, 0] = 1
    ids[:, 1] = -200  # <image> right after BOS; 513 ids -> 768 positions
    return pixels, ids


# =============================================================================== CPU (reference arm)
CPU_LLM_LAYERS, CPU_VIT_LAYERS, CPU_DECODE_STEPS = 8, 6, 3


def _cpu_weights():
    """fp32 random-init weights of the timed slice: CPU_LLM_LAYERS LLaMA-7B layers + embeddings + lm_head,
    CPU_VIT_LAYERS ViT-L/14 layers (built once per process)."""
    if "w" in _CPU_CACHE:
        return _CPU_CACHE["w"]
    g = torch.Generator().manual_seed(0)
    rn = lambda *s: torch.randn(s, generator=g) * 0.02
    d, f, V = 4096, 11008, 32000
    sd = {"model.embed_tokens.weight": rn(V, d), "lm_head.weight": rn(V, d), "model.norm.weight": torch.ones(d)}
    for i in range(CPU_LLM_LAYERS):
        p = f"model.layers.{i}."
        for n in "qkvo":
            sd[p + f"self_attn.{n}_proj.weight"] = rn(d, d)
        sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"], sd[p + "mlp.down_proj.weight"] = rn(f, d), rn(f, d), rn(d, f)
        sd[p + "input_layernorm.weight"] = torch.ones(d)
        sd[p + "post_attention_layernorm.weight"] = torch.ones(d)
    cfg = dict(VICUNA_7B, num_hidden_layers=CPU_LLM_LAYERS)
    vd, vf = 1024, 4096
    vp = "v."
    vsd = {vp + "embeddings.class_embedding": rn(vd), vp + "embeddings.patch_embedding.weight": rn(vd, 3, 14, 14),
           vp + "embeddings.position_embedding.weight": rn(257, vd), vp + "pre_layrnorm.weight": torch.ones(vd),
           vp + "pre_layrnorm.bias": torch.zeros(vd)}
    for i in range(CPU_VIT_LAYERS):
        p = vp + f"encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            vsd[p + f"self_attn.{n}.weight"], vsd[p + f"self_attn.{n}.bias"] = rn(vd, vd), torch.zeros(vd)
        for n in ("layer_norm1", "layer_norm2"):
            vsd[p + n + ".weight"], vsd[p + n + ".bias"] = torch.ones(vd), torch.zeros(vd)
        vsd[p + "mlp.fc1.weight"], vsd[p + "mlp.fc1.bias"] = rn(vf, vd), torch.zeros(vf)
        vsd[p + "mlp.fc2.weight"], vsd[p + "mlp.fc2.bias"] = rn(vd, vf), torch.zeros(vd)
    vcfg = dict(VIT_L14, num_hidden_layers=CPU_VIT_LAYERS, layer_norm_eps=1e-5)
    _CPU_CACHE["w"] = (sd, cfg, vsd, vcfg, vp, rn, g)
    return _CPU_CACHE["w"]


def cpu_sample(batch=BATCH):
    """One BOUNDED sample of the workload on the host cores with the oracle port of the reference (oracle/restate_llm.py,
    fp32, KV cache grown by torch.cat like HF 4.31): every stage at its REAL shape and context —
      * ViT-L/14 encode of 1 image, CPU_VIT_LAYERS of the 23 layers the path needs,
      * LLaMA-7B prefill of ONE sequence at the full S = 768, CPU_LLM_LAYERS of 32 layers,
      * CPU_DECODE_STEPS cached decode steps at batch `batch` on the real 768+ token context (the prefill KV replicated
        over the batch), same layer count, + the full-size final norm / lm_head.
    The layers of both stacks are identical, so the full-depth time is the per-layer time x depth; per-sequence stages
    scale with the batch (they are compute-bound on a CPU). Returns (tokens_per_s_of_the_full_workload, info) where
    info['sample_s'] is the wall time this sample actually took."""
    import torch.nn.functional as F
    from oracle import restate_llm as R
    threads = _pick_threads()
    torch.set_num_threads(threads)
    sd, cfg, vsd, vcfg, vp, rn, g = _cpu_weights()
    d = 4096
    with torch.no_grad():
        t_all = time.perf_counter()
        t0 = time.perf_counter()
        R.clip_vit_hidden(vsd, vp, vcfg, torch.randn((1, 3, 224, 224), generator=g), select_layer=-1)
        t_vit = time.perf_counter() - t0
        m = R.LlamaCPU(sd, cfg)
        t0 = time.perf_counter()
        m.prefill(rn(1, VISION + TEXT, d))
        t_pre = time.perf_counter() - t0
        m.kv = [(k.expand(batch, -1, -1, -1).contiguous(), v.expand(batch, -1, -1, -1).contiguous()) for k, v in m.kv]
        h = rn(batch, 1, d)
        t0 = time.perf_counter()
        for _ in range(CPU_DECODE_STEPS):
            m._layers(h, m.pos)
            m.pos += 1
        t_lay = (time.perf_counter() - t0) / CPU_DECODE_STEPS
        t0 = time.perf_counter()
        F.linear(R.rms_norm(h, sd["model.norm.weight"], 1e-5), sd["lm_head.weight"])
        t_head = time.perf_counter() - t0
        sample_s = time.perf_counter() - t_all
    t_dec_full = (32 / CPU_LLM_LAYERS) * t_lay + t_head
    full = batch * (23 / CPU_VIT_LAYERS) * t_vit + batch * (32 / CPU_LLM_LAYERS) * t_pre + NEW * t_dec_full
    info = {"sample_s": round(sample_s, 3), f"t_vit_{CPU_VIT_LAYERS}of23_layers_1img_s": round(t_vit, 3),
            f"t_prefill_{CPU_LLM_LAYERS}of32_layers_b1_s768_s": round(t_pre, 3),
            f"t_decode_{CPU_LLM_LAYERS}of32_layers_b{batch}_ctx{VISION + TEXT}_s": round(t_lay, 4), f"t_lm_head_b{batch}_s": round(t_head, 4),
            "threads": threads, "batch": batch, "full_depth_decode_step_s": round(t_dec_full, 3), "full_workload_step_s": round(full, 2)}
    return batch * NEW / full, info


CPU_SAMPLE_TEXT = (f"oracle port (fp32 torch restatement of the reference path, KV cache by torch.cat): per step ViT-L/14 "
                   f"{CPU_VIT_LAYERS}/23 layers on 1 image + LLaMA-7B {CPU_LLM_LAYERS}/32 layers: prefill of ONE sequence at S=768 and "
                   f"{CPU_DECODE_STEPS} cached decode steps at the full batch on the real 768-token context + full lm_head; value = "
                   "batch x 128 tokens / (per-layer times x depth, per-sequence stages x batch); ms_per_step = wall time of the sample itself")

_CPU_CACHE = {}


def _host_cores():
    try:
        return len(os.sched_getaffinity(0))
    except AttributeError:
        return os.cpu_count() or 1


def _pick_threads():
    """torch's intra-op pool does not always scale to every hardware thread of a large host (SMT siblings,
    cgroup quotas): probe a prefill-shaped fp32 GEMM at a few thread counts once and keep the fastest."""
    if "threads" in _CPU_CACHE:
        return _CPU_CACHE["threads"]
    avail = _host_cores()
    x, w = torch.randn(768, 4096), torch.randn(4096, 4096)
    best, best_t = avail, None
    for th in sorted({avail, max(1, avail // 2), min(avail, 64), min(avail, 32), min(avail, 16)}, reverse=True):
        torch.set_num_threads(th)
        torch.nn.functional.linear(x, w)
        t0 = time.perf_counter()
        for _ in range(3):
            torch.nn.functional.linear(x, w)
        t = time.perf_counter() - t0
        if best_t is None or t < best_t * 0.95:
            best, best_t = th, t
    _CPU_CACHE["threads"] = best
    return best


def run_reference(args, rank):
    """`--impl reference`: the reference's CPU path (oracle port) on this box's host cores, K bounded samples after W
    warm-up samples; the batch follows the GPU arm's global batch (8 x N)."""
    if rank != 0:
        return
    batch = BATCH * max(1, args.gpus)
    vals, secs, info = [], [], {}
    for i in range(args.warmup + args.steps):
        v, info = cpu_sample(batch)
        if i >= args.warmup:
            vals.append(v)
            secs.append(info["sample_s"])
    v = sum(vals) / len(vals)
    line = {"impl": "reference", "metric": METRIC, "value": v, "unit": "tokens/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1000.0 * sum(secs) / len(secs),
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(args.gpus),
            "cpu_baseline": {"value": v, "unit": "tokens/s", "cores": info.get("threads"), "host_cores": _host_cores(), "kind": "port",
                             "sample": CPU_SAMPLE_TEXT, **info},
            "e2e": {"value": v, "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def workload_config(n):
    return {"workload": "BASELINE.json configs[1]: batch-8 336x336 images (processor output 224x224), ViT-L/14 encode + "
                        "Vicuna-7B 256-vision + 512-text prefill + 128-token greedy decode, bf16",
            "global_batch": BATCH * n, "prompt_tokens": VISION + TEXT, "new_tokens": NEW, "parallelism": f"dp{n}",
            "l2": "inputs_larger_than_L2 (13.5 GB of weights streamed per decode step)", "kv_cache": "paged, 64-token pages"}


# =============================================================================== GPU (ours)
def build_model(device):
    from vitron_b200 import param_shapes as PS
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    cfg = VitronConfig(llm=VICUNA_7B, vision=VisionConfig(**VIT_L14), tokenizer_model_max_length=4096, eos_token_id=None)
    model = VitronLlamaForCausalLM(cfg, device, max_batch=BATCH, max_seq_len=VISION + TEXT + NEW)
    sd = PS.random_state_dict(PS.vitron_shapes(cfg), device, seed=0)
    model.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    return model


def dump_outputs(directory, arrays):
    """--dump-outputs: one DIR/<name>.npy per array; integer results (token ids) as float64, which holds them exactly."""
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    for name, t in arrays.items():
        t = t.detach().cpu()
        a = t.float().numpy() if t.is_floating_point() else t.double().numpy()
        np.save(os.path.join(directory, name + ".npy"), a)


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def roofline_decode_gemm(model, hbm_peak, peak_kind):
    """Dominant kernel of the step = gemv_bf16_kernel streaming the decoder weights at M=8 (128 of the
    ~290 launches and ~60% of the time of a decode token, 127 tokens per step). Timed live: all 128
    decode GEMMs of one token (4 per layer x 32 layers = 12.95 GB of distinct weights, >> L2),
    captured in one CUDA graph and replayed back to back."""
    from vitron_b200 import ops
    eng = model.engine
    d, f = eng.cfg.hidden_size, eng.cfg.intermediate_size
    x = torch.randn((BATCH, d), device=eng.device).to(torch.bfloat16)
    a = torch.randn((BATCH, f), device=eng.device).to(torch.bfloat16)

    def one_token():
        for L in eng.layers:
            ops.gemm(x, L["wqkv"])
            ops.gemm(x, L["wo"])
            ops.gemm(x, L["wgu"], glu=ops.GLU_SWIGLU)
            ops.gemm(a, L["wdown"])
    for _ in range(3):
        one_token()
    # replay through a CUDA graph so that the CUDA-event time is device time, not Python launch rate
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        one_token()
    g.replay()
    ms = timed(g.replay, 10)
    n_launch = 4 * len(eng.layers)
    wbytes = sum(L[k].numel() * 2 for L in eng.layers for k in ("wqkv", "wo", "wgu", "wdown"))
    abytes = len(eng.layers) * BATCH * 2 * (d * 3 + f + (3 * d + d + f + d))  # activations in + out
    per_launch = (wbytes + abytes) / n_launch
    achieved = per_launch / (ms * 1e-3 / n_launch) / 1e9
    traffic = None
    pj = os.path.join(ROOT, "profiles", "dominant_kernel.json")
    if os.path.exists(pj):
        with open(pj) as fh:
            traffic = json.load(fh).get("traffic_bytes_per_launch")
    return {"bound": "hbm", "kernel": "gemv_bf16_kernel<16|32,1> (weight-streaming M=8 decode GEMMs, epilogue fused)",
            "achieved": achieved, "peak": hbm_peak, "unit": "GB/s", "frac": achieved / hbm_peak,
            "peak_source": f"MEASURED_PEAKS.json hbm_gbs ({peak_kind})", "traffic": traffic,
            "algorithmic_bytes_per_launch": per_launch, "avg_launch_us": ms * 1e3 / n_launch}


def run_profile():
    """Same step as the benchmark but short and without the CUDA graph, so that
    `ncu --metrics gpu__time_duration.sum` lists every kernel once: ViT + projector, prefill
    (B=8, S=768), then 4 decode tokens (the benchmark runs 127; scale the decode rows by 127/4)."""
    from vitron_b200 import ops
    device = torch.device("cuda:0")
    model = build_model(device)
    pixels, ids = synth_inputs()
    pixels, ids = pixels.to(device), ids.to(device)
    _, _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids, None, torch.ones_like(ids), None, None, pixels)
    eng = model.engine
    first = ops.argmax_rows(eng.prefill(emb))
    eng.start_decode(first, NEW)
    eng.decode_steps(BATCH, 4, use_graph=False)
    torch.cuda.synchronize()
    print(json.dumps({"profile": "ok", "tokens": eng.token_log[:BATCH, :5].tolist()}))


UNET_CFG = dict(in_dim=4, concat_dim=4, dim=320, y_dim=1024, context_dim=1024, out_dim=4, dim_mult=[1, 2, 4, 4], num_heads=8,
                head_dim=64, num_res_blocks=2, attn_scales=[1.0, 0.5, 0.25], num_tokens=4)
UNET_TFLOP_PER_FORWARD = 12.67  # algorithmic FLOPs of the reference class at f=16, 40x64 latent (BASELINE.md §2)
UNET_METRIC = "i2vgen-xl UNet3D DDIM steps/s (conditional + unconditional UNet evaluation + CFG per step), latent [1,4,16,40,64] = 16 frames of 320x512 px"
UNET_LATENT = (1, 4, 16, 40, 64)


def _unet_inputs(device, seed=4):
    g = torch.Generator(device=device).manual_seed(seed)
    rn = lambda *s: torch.randn(s, generator=g, device=device)
    noise, local = rn(*UNET_LATENT), rn(*UNET_LATENT)
    cond = dict(y=rn(1, 77, 1024), image=rn(1, 1, 1024), local_image=local, fps=torch.tensor([16], device=device))
    unc = dict(y=rn(1, 77, 1024), image=torch.zeros((1, 1, 1024), device=device), local_image=local,
               fps=torch.tensor([16], device=device))
    return noise, cond, unc


def unet_gemm_roofline(unet, noise, cond, tf_peak, peak_kind, t_steps=None):
    """Dominant kernel family of a UNet forward = the wgmma GEMM / implicit-GEMM conv kernel (gemm_v2_kernel<BN,...>,
    ~70 % of the forward). Every ops.gemm / ops.conv_nhwc call of ONE forward is recorded with its live operands, then
    exactly those calls are replayed back to back from a CUDA graph and timed with CUDA events: achieved = their
    algorithmic FLOPs (2*M*N*K, conv 2*pixels*cout*cin*taps) / that time. `noise` / `cond` are what the timed step feeds the
    UNet: the batch-2 [cond | uncond] tensors of the graphed CFG denoiser."""
    from vitron_b200 import ops
    calls = []
    real_gemm, real_conv = ops.gemm, ops.conv_nhwc

    def rec_gemm(a, w, *args, **kw):
        out = real_gemm(a, w, *args, **kw)
        if a.numel() // a.shape[-1] > 16:
            kw2 = dict(kw)
            kw2["out"] = out if kw.get("out") is None else kw["out"]
            if kw2.get("residual") is not None and kw2["residual"].data_ptr() == kw2["out"].data_ptr():
                kw2["residual"] = kw2["residual"].clone()  # replay must not accumulate in place
                kw2["out"] = torch.empty_like(kw2["residual"])
            calls.append((real_gemm, (a, w) + args, kw2, 2.0 * (a.numel() // a.shape[-1]) * a.shape[-1] * w.shape[0]))
        return out

    def rec_conv(x, wt, kh, kw_, *args, **kw):
        out = real_conv(x, wt, kh, kw_, *args, **kw)
        calls.append((real_conv, (x, wt, kh, kw_) + args, dict(kw, out=out),
                      2.0 * out.shape[0] * out.shape[1] * out.shape[2] * wt.shape[0] * wt.shape[1] * x.shape[-1]))
        return out
    ops.gemm, ops.conv_nhwc = rec_gemm, rec_conv
    import vitron_b200.unet_i2vgen as U
    try:
        unet(noise, torch.full((noise.shape[0],), 981, dtype=torch.long, device=noise.device), **cond)
    finally:
        ops.gemm, ops.conv_nhwc = real_gemm, real_conv
    torch.cuda.synchronize()
    flops = sum(c[3] for c in calls)

    def replay():
        for fn, a, kw, _ in calls:
            fn(*a, **kw)
    s = torch.cuda.Stream(device=noise.device)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        replay()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), ops.pdl(True):   # same launch mode as the benchmarked step
        replay()
    for _ in range(2):
        g.replay()
    ms = timed(g.replay, 5)
    traffic = None
    pj = os.path.join(ROOT, "profiles", "dominant_kernel_unet.json")
    if os.path.exists(pj):
        with open(pj) as fh:
            traffic = json.load(fh).get("traffic_bytes_per_launch")
    ach = flops / (ms * 1e-3) / 1e12
    return {"bound": "tensor", "kernel": "gemm_v2_kernel<BN,STAGES,EPI> (wgmma GEMM + implicit-GEMM conv: every Linear / Conv2d / Conv3d of the forward)",
            "achieved": ach, "peak": tf_peak, "unit": "TFLOP/s", "frac": ach / tf_peak,
            "peak_source": f"MEASURED_PEAKS.json bf16_tflops ({peak_kind}, burst)", "traffic": traffic,
            "launches": len(calls), "algorithmic_tflop": flops / 1e12, "avg_launch_us": ms * 1e3 / len(calls), "replay_ms": ms}


def unet_cpu_baseline():
    """CPU baseline of the UNet half: the oracle port (oracle/restate_unet.py, fp32, the reference class's arithmetic) with
    the full 1.42 B-parameter weights on a REDUCED latent [1,4,4,24,32] (3/40 of the frames x pixels), one forward timed;
    steps/s = 1 / (2 forwards x 13.3 x t): convolutions / linears scale with frames x pixels (BASELINE.md §3 prescribes the
    FLOP-ratio scaling; the quadratic attention terms shrink faster, so this slightly FAVOURS the CPU)."""
    from oracle import restate_unet as RU
    from vitron_b200 import param_shapes as PS
    threads = _pick_threads()
    torch.set_num_threads(threads)
    sd = {k: v.float() for k, v in PS.random_state_dict(PS.unet_shapes(UNET_CFG), torch.device("cpu"), seed=4).items()}
    g = torch.Generator().manual_seed(4)
    rn = lambda *sh: torch.randn(sh, generator=g)
    f, h, w = 4, 24, 32  # h, w divisible by 8 (three stride-2 levels)
    x, local = rn(1, 4, f, h, w), rn(1, 4, f, h, w)
    with torch.no_grad():
        t0 = time.perf_counter()
        RU.unet_forward(sd, UNET_CFG, x, torch.tensor([981]), y=rn(1, 77, 1024), image=rn(1, 1, 1024), local_image=local,
                        fps=torch.tensor([16]))
        t = time.perf_counter() - t0
    scale = (16 * 40 * 64) / (f * h * w)
    return {"value": 1.0 / (2 * scale * t), "unit": "steps/s", "cores": threads, "host_cores": _host_cores(), "kind": "port",
            "sample": f"oracle port fp32, full weights, ONE forward at latent [1,4,{f},{h},{w}] ({t:.2f} s), scaled x{scale:.0f} "
                      "(frames x pixels) to the [1,4,16,40,64] latent, 2 forwards per step"}


def bench_unet(device, tf_peak, peak_kind, steps=10, rank=0, world=1, with_cpu=True, outputs=None):
    """Second half of BASELINE.json's metric: i2vgen-xl UNet3D denoise steps/s (configs[4] at the primary latent reading
    16 x (40x64) = 320x512 px; DDIM step = the conditional and the unconditional UNet evaluation of classifier-free guidance 9.0
    — run as ONE batch-2 forward [cond | uncond], GraphedCFGDenoiser — + the v-prediction update),
    bf16, random-init 1.42 B-parameter UNetSD_I2VGen, CUDA-graphed.
    N = 1: one request. N > 1 (SURVEY §8e): `value` = N independent requests (replicas, no collective); `cfg_split` =
    the cond / uncond branches of ONE request on a GPU pair, one NCCL all_gather of the two [1,4,16,40,64] fp32 branch
    outputs per step (N/2 requests in flight, each step ~2x faster)."""
    from vitron_b200 import ops
    from vitron_b200 import param_shapes as PS
    from vitron_b200.unet_i2vgen import CFGSplitDenoiser, DiffusionDDIM, GraphedBranch, GraphedCFGDenoiser, UNetSD_I2VGen
    dist = None
    if world > 1:
        import torch.distributed as dist
    unet = UNetSD_I2VGen(**UNET_CFG, device=device)
    sd = PS.random_state_dict(PS.unet_shapes(UNET_CFG), device, seed=4)
    unet.load_state_dict(sd)
    del sd
    noise, cond, unc = _unet_inputs(device)
    diff = DiffusionDDIM()
    tz = torch.zeros((1,), dtype=torch.long, device=device)
    den = GraphedCFGDenoiser(unet, cond, unc, 9.0, noise, tz)
    ts = [int(v) for v in (1 + torch.arange(0, 1000, 20)).clamp(0, 999).flip(0)]  # the DDIM-50 schedule

    def run_steps(model, xt, tvals):
        for tv in tvals:
            xt, _ = diff.ddim_sample(xt, torch.full((1,), tv, dtype=torch.long, device=device), model, None, 9.0, 50)
        return xt

    def time_steps(model, x0, n):
        xt = run_steps(model, x0, ts[:3])  # warm-up + capture
        if world > 1:
            dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        xt = run_steps(model, xt, [ts[3 + i % (len(ts) - 3)] for i in range(n)])   # --steps beyond the schedule wrap around
        e1.record()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        t = torch.tensor([e0.elapsed_time(e1) / n], device=device, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t), xt

    l0 = ops.launch_count()
    ms, xt = time_steps(den, noise, steps)
    launches = (ops.launch_count() - l0) // (steps + 3)
    if outputs is not None:
        outputs["unet_latent"] = xt
    finite = bool(torch.isfinite(xt).all())
    tfs = 2 * UNET_TFLOP_PER_FORWARD / (ms * 1e-3)
    out = {"metric": UNET_METRIC, "value": world * 1000.0 / ms, "unit": "steps/s", "n_gpus": world, "steps": steps, "warmup": 3,
           "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "dtype": "bf16", "data": "synthetic",
           "config": {"workload": "BASELINE.json configs[4], primary latent reading [1,4,16,40,64]; DDIM-50 schedule, guide 9.0",
                      "parallelism": f"{world} request replica(s)", "requests_in_flight": world,
                      "cfg_evaluation": "one batch-2 forward [cond | uncond]" if den.batched else "two batch-1 forwards",
                      "l2": "2.8 GB of weights + ~0.6 GB of activations streamed per forward (> 50 MB L2)"},
           "latent": list(UNET_LATENT), "guide_scale": 9.0, "gpu_launches": launches,
           "achieved_tflops_per_gpu": tfs, "frac_of_bf16_peak": tfs / tf_peak, "finite": finite,
           "algorithmic_tflop_per_step": 2 * UNET_TFLOP_PER_FORWARD}

    if world == 1:
        # ---- e2e: the latent of each step arrives from / returns to pinned host memory
        x_pin = noise.cpu().pin_memory()
        out_pin = torch.empty_like(x_pin).pin_memory()

        def e2e_step(i=[0]):
            xt = x_pin.to(device, non_blocking=True)
            xt = run_steps(den, xt, [ts[3 + i[0] % 40]])
            out_pin.copy_(xt, non_blocking=True)
            torch.cuda.synchronize()
            i[0] += 1
        e2e_step()
        ms_e2e = timed(e2e_step, steps)
        nb = x_pin.numel() * 4
        out["e2e"] = {"value": 1000.0 / ms_e2e, "unit": "steps/s", "ms_per_step": ms_e2e, "h2d_bytes_per_step": nb,
                      "d2h_bytes_per_step": nb, "input": "x_t fp32 [1,4,16,40,64] from pinned host memory, x_{t-1} read back"}
        if den.batched:   # the forward the timed step runs: ONE batch-2 evaluation [cond | uncond]
            out["roofline"] = unet_gemm_roofline(unet, den.xt2, den.both, tf_peak, peak_kind)
            out["roofline"]["forward"] = "batch-2 [cond | uncond] (one CFG evaluation)"
        else:
            out["roofline"] = unet_gemm_roofline(unet, noise, cond, tf_peak, peak_kind)
        if with_cpu:
            out["cpu_baseline"] = unet_cpu_baseline()
    elif world % 2 == 0:
        # ---- CFG-branch split over GPU pairs
        groups = [dist.new_group([2 * i, 2 * i + 1]) for i in range(world // 2)]
        role = rank % 2
        branch = GraphedBranch(unet, cond if role == 0 else unc, noise, tz)
        split = CFGSplitDenoiser(branch, role, 9.0, group=groups[rank // 2])
        ms2, xt2 = time_steps(split, noise, steps)
        ref = run_steps(den, noise, ts[:3 + steps])
        out["cfg_split"] = {"value": (world // 2) * 1000.0 / ms2, "unit": "steps/s", "ms_per_step": ms2, "requests_in_flight": world // 2,
                            "speedup_per_request_vs_1gpu": ms / ms2, "collective": "NCCL all_gather of 2 x 655 KB per step inside each pair",
                            "max_abs_diff_vs_single_gpu_cfg": float((xt2 - ref).abs().max()), "finite": bool(torch.isfinite(xt2).all())}
    del unet, den
    torch.cuda.empty_cache()
    return out


# 32 clips: the KV cache of 32 x 2145 positions (36 GB) + the 13.5 GB of weights fit one 80 GB H100
VIDEO_CLIPS, VIDEO_FRAMES, VIDEO_TEXT, VIDEO_NEW = 32, 8, 64, 32


def bench_video(device, rank, world, steps=2, outputs=None):
    """BASELINE.json configs[2] at a global batch of VIDEO_CLIPS: 8-frame 224x224 clips -> LanguageBind video tower (temporal
    attention) + projector + Vicuna-7B prefill over 8 x 256 vision + 65 text tokens + 32 greedy tokens, data-parallel over N
    GPUs: the clips are SHARDED VIDEO_CLIPS/N per rank (strong scaling), inputs start in pinned host memory (H2D inside the
    timed region), one NCCL all_gather of the generated ids. value = VIDEO_CLIPS clips / max-over-ranks step time."""
    from vitron_b200 import ops, param_shapes as PS
    from vitron_b200.dist import gather_results, shard_range
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    dist = None
    if world > 1:
        import torch.distributed as dist
    lo, hi = shard_range(VIDEO_CLIPS, rank, world)
    clips = hi - lo
    T = VIDEO_FRAMES
    S = T * 256 + VIDEO_TEXT + 1
    vcfg = VisionConfig(**VIT_L14, add_time_attn=True, num_frames=T)
    cfg = VitronConfig(llm=VICUNA_7B, vision=None, video=vcfg, tokenizer_model_max_length=4096, eos_token_id=None)
    model = VitronLlamaForCausalLM(cfg, device, max_batch=clips, max_seq_len=S + VIDEO_NEW)
    sd = PS.random_state_dict(PS.vitron_shapes(cfg), device, seed=0)
    model.load_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    g = torch.Generator().manual_seed(100 + rank)
    vids = [torch.randn((3, T, 224, 224), generator=g).pin_memory() for _ in range(clips)]
    ids = torch.cat([torch.ones((clips, 1), dtype=torch.long), torch.full((clips, T), -200, dtype=torch.long),
                     torch.randint(3, 32000, (clips, VIDEO_TEXT), generator=g)], 1).pin_memory()

    def step():
        out = model.generate(ids.to(device, non_blocking=True), images=[v.to(device, non_blocking=True) for v in vids],
                             max_new_tokens=VIDEO_NEW, do_sample=False, sync_every=VIDEO_NEW)
        new = out[:, -VIDEO_NEW:].contiguous()
        if world > 1:
            new = gather_results(new, VIDEO_CLIPS)
        new = new.cpu()
        if outputs is not None:
            outputs["video_tokens"] = new
        return new
    step()
    if world > 1:
        dist.barrier()
    l0 = ops.launch_count()
    ms = timed(step, steps)
    launches = (ops.launch_count() - l0) // steps
    t = torch.tensor([ms], device=device, dtype=torch.float64)
    if world > 1:
        dist.barrier()
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t)
    out = {"metric": f"video clips/s: 8-frame LanguageBind video tower + Vicuna-7B prefill (2113 tokens) + 32 greedy tokens, global batch {VIDEO_CLIPS}",
           "value": VIDEO_CLIPS / (ms * 1e-3), "unit": "clips/s", "n_gpus": world, "steps": steps, "warmup": 1, "ms_per_step": ms,
           "higher_is_better": True, "scaling": "strong", "dtype": "bf16", "data": "synthetic",
           "config": {"workload": f"BASELINE.json configs[2] at {VIDEO_CLIPS} clips, sharded {VIDEO_CLIPS}/N per GPU", "clips_per_gpu": clips, "frames": T,
                      "prompt_tokens": S, "new_tokens": VIDEO_NEW, "parallelism": f"dp{world}"},
           "generated_tokens_per_s": VIDEO_CLIPS * VIDEO_NEW / (ms * 1e-3), "gpu_launches": launches,
           "h2d_bytes_per_step": clips * 3 * T * 224 * 224 * 4 + ids.numel() * 8, "d2h_bytes_per_step": VIDEO_CLIPS * VIDEO_NEW * 8}
    del model
    torch.cuda.empty_cache()
    return out


def run_ours(args, rank, world):
    from vitron_b200 import _lib, ops
    lib = _lib.load()
    device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(device)
    if not lib.vb200_device_ok():
        raise RuntimeError("vitron_b200 needs an sm_90 (H100) device")
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    model = build_model(device)
    pixels_h, ids_h = synth_inputs(seed_px=1 + rank, seed_ids=2 + rank)
    pixels_pin, ids_pin = pixels_h.pin_memory(), ids_h.pin_memory()
    pixels_d, ids_d = pixels_h.to(device), ids_h.to(device)
    from vitron_b200.dist import gather_results

    def step(px, ids):
        out = model.generate(ids, images=px, do_sample=False, max_new_tokens=NEW, use_cache=True, sync_every=NEW)
        new = out[:, ids.shape[1]:]
        if world > 1:  # the only collective on the path: per-request results, NCCL all_gather
            return gather_results(new.contiguous(), world * BATCH)
        return new

    outputs = {}   # what the timed path returned in its last step (--dump-outputs)

    def step_resident():
        outputs["tokens"] = step(pixels_d, ids_d)
        return outputs["tokens"]

    # e2e starts from what the reference's caller holds: decoded uint8 336x336 RGB images (BASELINE.json configs[1]) in
    # pinned host memory. They cross PCIe as uint8 and the LanguageBind transform (resize 224 bicubic, crop, normalise —
    # processing_image.py:15-25) runs on the device (vitron_b200.processing, one fused kernel per image).
    raw_pin = torch.randint(0, 256, (BATCH, 336, 336, 3), generator=torch.Generator().manual_seed(11 + rank),
                            dtype=torch.uint8).pin_memory()
    from vitron_b200.processing import LanguageBindImageProcessor
    processor = LanguageBindImageProcessor(device=device, dtype=torch.bfloat16)

    def step_e2e():
        if args.e2e_input == "raw":
            raw = raw_pin.to(device, non_blocking=True)
            px = processor.preprocess(raw)["pixel_values"]
        else:
            px = pixels_pin.to(device, non_blocking=True)
        ids = ids_pin.to(device, non_blocking=True)
        outputs["e2e_tokens"] = step(px, ids).cpu()
        return outputs["e2e_tokens"]

    for _ in range(max(args.warmup, 3)):
        step_resident()
    sampler = ClockSampler(device.index or 0)
    sampler.start()
    if world > 1:
        dist.barrier()
    l0 = ops.launch_count()
    ms = timed(step_resident, args.steps)
    launches = (ops.launch_count() - l0) // args.steps
    dumped = {"tokens": outputs["tokens"]}
    if world > 1:
        dist.barrier()
    step_e2e()
    ms_e2e = timed(step_e2e, args.steps)
    dumped["e2e_tokens"] = outputs["e2e_tokens"]
    sampler.stop_flag = True
    sampler.join(timeout=2)
    t = torch.tensor([ms, ms_e2e], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ms_e2e = t.tolist()
    # guard on what was timed: the generated ids must be valid vocabulary entries, identical from run to run (greedy,
    # deterministic kernels) and identical between the HBM-resident and the host-input arms' code path
    tok_a, tok_b = step_resident()[:BATCH], step_resident()[:BATCH]
    tokens_check = {"in_vocab": bool(((tok_a >= 0) & (tok_a < VICUNA_7B["vocab_size"])).all()),
                    "deterministic": bool((tok_a == tok_b).all()), "distinct_ids": int(tok_a.unique().numel()),
                    "shape": list(tok_a.shape)}

    line = None
    if rank == 0:
        hbm_peak, tf_peak, kind = measured_peaks()
        # phase breakdown (diagnostic, separate short loops)
        eng = model.engine
        t_vit = timed(lambda: model.encode_images(pixels_d), 3)
        _, _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids_d, None, torch.ones_like(ids_d), None, None, pixels_d)
        t_pre = timed(lambda: eng.prefill(emb), 3)
        logits0 = eng.prefill(emb)
        tokens_check["prefill_logits_finite"] = bool(torch.isfinite(logits0).all())
        first = ops.argmax_rows(logits0)
        eng.start_decode(first, NEW)
        eng.decode_steps(BATCH, 2)
        t_dec = timed(lambda: eng.decode_steps(BATCH, 1), 64)
        S = VISION + TEXT
        pre_flops = BATCH * (12.95e9 * S + 2 * 4096 * 32000 + 32 * 4 * S * S * 4096 / 2)
        dec_bytes = eng.weight_bytes() + 2 * 32 * 4096 * 2 * (S + NEW / 2) * BATCH
        roof = roofline_decode_gemm(model, hbm_peak, kind)
        roof["decode_step"] = {"ms": t_dec, "achieved_gbs": dec_bytes / (t_dec * 1e-3) / 1e9,
                               "frac": dec_bytes / (t_dec * 1e-3) / 1e9 / hbm_peak}
        roof["prefill"] = {"ms": t_pre, "achieved_tflops": pre_flops / (t_pre * 1e-3) / 1e12,
                           "frac_of_bf16_peak": pre_flops / (t_pre * 1e-3) / 1e12 / tf_peak}
        cpu_v, cpu_info = (None, {})
        if world == 1:
            cpu_v, cpu_info = cpu_sample()
        h2d = (raw_pin.numel() if args.e2e_input == "raw" else pixels_pin.numel() * 4) + ids_pin.numel() * 8
        d2h = BATCH * NEW * 8
        line = {"metric": METRIC, "value": world * BATCH * NEW / (ms * 1e-3), "unit": "tokens/s", "n_gpus": world,
                "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms, "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
                "config": workload_config(world),
                "e2e": {"value": world * BATCH * NEW / (ms_e2e * 1e-3), "unit": "tokens/s", "h2d_bytes_per_step": h2d,
                        "d2h_bytes_per_step": d2h, "ms_per_step": ms_e2e,
                        "input": ("uint8 336x336 images, device-side LanguageBind transform" if args.e2e_input == "raw"
                                  else "pre-processed fp32 224x224 pixels")},
                "gpu_launches": launches, "clocks": sampler.result(), "roofline": roof, "tokens_check": tokens_check,
                "phases": {"vit_projector_ms": t_vit, "prefill_ms": t_pre, "decode_ms_per_token": t_dec,
                           "prefill_tokens_per_s": BATCH * S / (t_pre * 1e-3),
                           "decode_tokens_per_s": BATCH / (t_dec * 1e-3)}}
        if cpu_v is not None:
            line["cpu_baseline"] = {"value": cpu_v, "unit": "tokens/s", "cores": cpu_info.get("threads"),
                                    "host_cores": _host_cores(), "kind": "port", "sample": CPU_SAMPLE_TEXT, **cpu_info}
    # ---- configs[2]: the video job BASELINE.json names for 1/2/4/8 GPUs (strong scaling over a fixed batch of 64)
    video_line = None
    if not args.no_video:
        del model
        model = None
        torch.cuda.empty_cache()
        video_line = bench_video(device, rank, world, steps=args.steps, outputs=dumped)
    # ---- the UNet half of the metric (every rank takes part when N > 1)
    unet_line = None
    if not args.no_unet:
        del model
        torch.cuda.empty_cache()
        _, tf_peak_all, kind_all = measured_peaks()
        unet_line = bench_unet(device, tf_peak_all, kind_all, steps=args.steps, rank=rank, world=world,
                               with_cpu=(rank == 0), outputs=dumped)
    if rank == 0:
        if video_line is not None:
            line["video_cfg2"] = video_line
        if unet_line is not None:
            line["unet"] = unet_line
        if args.dump_outputs:
            dump_outputs(args.dump_outputs, dumped)
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5, help="timed steps of every leg")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--e2e-input", default="raw", choices=["raw", "processed"],
                    help="e2e arm input: raw uint8 336x336 images (device-side transform) or pre-processed fp32 pixels")
    ap.add_argument("--no-unet", action="store_true", help="skip the i2vgen-xl UNet3D steps/s measurement")
    ap.add_argument("--no-video", action="store_true", help="skip the configs[2] video batch-64 measurement")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's results (token ids, UNet latent) as DIR/<name>.npy")
    ap.add_argument("--profile", action="store_true",
                    help="ncu launch-list mode: one un-graphed step with 4 decode tokens, no timing loops")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    if args.impl == "reference":
        run_reference(args, rank)
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench.py --impl ours needs a CUDA device (there is no CPU fallback)")
    with torch.no_grad():
        if args.profile:
            run_profile()
        else:
            run_ours(args, rank, world)


if __name__ == "__main__":
    main()
