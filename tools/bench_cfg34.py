"""Measurements for BASELINE.json configs[2] and configs[3] (SURVEY.md §8d rows 3 and 4) on one GPU:

cfg3  8-frame 224x224 clips -> LanguageBind video tower (temporal attention over 8 frames) + projector +
      Vicuna-7B prefill over 8 x 256 vision + 65 text tokens + 32 greedy tokens. One GPU's share of the
      data-parallel batch-64 job at 8 GPUs is 8 clips; `--clips` changes it.
cfg4  SEEM pixel decoder + mask decoder (task 'seg'): backbone features of a 1024x1024 image, 101 queries.

Random-init weights of the reference shapes, synthetic inputs, bf16; CUDA-event timing through the public
drop-in entry points (generate / XDecoderHead.forward) with host inputs, i.e. H2D copies inside the timed region."""
import argparse, json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from vitron_b200 import ops, param_shapes as PS  # noqa: E402


def ev_time(fn, iters, warm):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def cfg3(dev, clips, new_tokens=32, text=64):
    from vitron_b200.vision_tower import VisionConfig
    from vitron_b200.vitron_model import VitronConfig, VitronLlamaForCausalLM
    T = 8
    vcfg = VisionConfig(**bench.VIT_L14, add_time_attn=True, num_frames=T)
    S = T * 256 + text + 1
    cfg = VitronConfig(llm=bench.VICUNA_7B, vision=None, video=vcfg, tokenizer_model_max_length=4096, eos_token_id=None)
    model = VitronLlamaForCausalLM(cfg, dev, max_batch=clips, max_seq_len=S + new_tokens)
    model.load_state_dict(PS.random_state_dict(PS.vitron_shapes(cfg), dev, seed=0))
    g = torch.Generator().manual_seed(1)
    vids = [torch.randn((3, T, 224, 224), generator=g).pin_memory() for _ in range(clips)]
    ids = torch.cat([torch.ones((clips, 1), dtype=torch.long), torch.full((clips, T), -200, dtype=torch.long),
                     torch.randint(3, 32000, (clips, text), generator=g)], 1).pin_memory()
    phases = {}

    def tower():
        model.encode_videos(torch.stack(vids).to(dev, non_blocking=True).to(torch.bfloat16))
    phases["video_tower_projector_ms"] = ev_time(tower, 3, 2)

    def run():
        out = model.generate(ids.to(dev, non_blocking=True), images=[v.to(dev, non_blocking=True) for v in vids],
                             max_new_tokens=new_tokens, do_sample=False)
        return out[:, -new_tokens:].cpu()
    l0 = ops.launch_count()
    ms = ev_time(run, 3, 2)
    return {"config": "BASELINE.json configs[2] (one GPU's share of the batch-64 job)", "clips": clips, "frames": T,
            "prompt_tokens": S, "new_tokens": new_tokens, "ms_per_batch": round(ms, 2),
            "clips_per_s": round(clips / (ms * 1e-3), 2), "generated_tokens_per_s": round(clips * new_tokens / (ms * 1e-3), 1),
            "prefill_tokens_per_s_incl_tower": None, **{k: round(v, 2) for k, v in phases.items()},
            "video_tower_tflops": round(clips * 1.71 / (phases["video_tower_projector_ms"] * 1e-3), 1),
            "launches_per_batch": (ops.launch_count() - l0) // 5}


def cfg4(dev):
    from vitron_b200.seem import MultiScaleMaskedTransformerDecoder, TransformerEncoderPixelDecoder, XDecoderHead
    in_ch = (192, 384, 768, 1536)
    sd = PS.random_state_dict(PS.seem_shapes(in_ch), dev, seed=3)
    head = XDecoderHead(TransformerEncoderPixelDecoder(in_ch, 512, 512, 8, 2048, 6, device=dev),
                        MultiScaleMaskedTransformerDecoder(512, 512, 101, 8, 2048, 9, 512, device=dev)).load_state_dict(sd)
    g = torch.Generator().manual_seed(3)
    feats = {f"res{i + 2}": torch.randn((1, c, 256 >> i, 256 >> i), generator=g).pin_memory() for i, c in enumerate(in_ch)}
    h2d = sum(v.numel() * 4 for v in feats.values())

    def run():
        out = head({k: v.to(dev, non_blocking=True) for k, v in feats.items()})
        return out["pred_masks"].float().cpu()
    l0 = ops.launch_count()
    ms = ev_time(run, 5, 2)
    launches = (ops.launch_count() - l0) // 7
    dfeats = {k: v.to(dev) for k, v in feats.items()}
    ms_pd = ev_time(lambda: head.pixel_decoder.forward_features(dfeats), 5, 2)
    ms_dev = ev_time(lambda: head(dfeats), 5, 2)             # features already in HBM, eager launches
    head.enable_graph(True)
    ms_graph = ev_time(lambda: head(dfeats), 10, 3)          # one CUDA graph replay per image
    bfeats = {k: v.to(torch.bfloat16) for k, v in dfeats.items()}
    ms_graph_bf16 = ev_time(lambda: head(bfeats), 10, 3)     # bf16 backbone features (what D2FocalNet hands over)
    head.enable_graph(False)
    head.predictor.aux_outputs = False   # inference mode: no per-layer full-resolution aux masks (evaluate() never reads them)
    head.enable_graph(True)
    ms_graph_noaux = ev_time(lambda: head(bfeats), 10, 3)
    head.enable_graph(False)
    head.predictor.aux_outputs = True
    return {"config": "BASELINE.json configs[3]: 1024x1024 image, 101 queries, pixel decoder + mask decoder, task seg",
            "device_resident_graph_bf16_feats_no_aux_ms": round(ms_graph_noaux, 2),
            "device_resident_eager_ms": round(ms_dev, 2), "device_resident_graph_ms": round(ms_graph, 2),
            "device_resident_graph_bf16_feats_ms": round(ms_graph_bf16, 2),
            "ms_per_image_e2e": round(ms, 2), "images_per_s": round(1e3 / ms, 2), "pixel_decoder_ms": round(ms_pd, 2),
            "mask_decoder_ms": round(ms - ms_pd, 2), "h2d_bytes": h2d, "d2h_bytes": 101 * 256 * 256 * 4,
            "achieved_tflops": round(0.95 / (ms * 1e-3), 1), "algorithmic_tflop_per_image": 0.95, "launches_per_image": launches}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=8)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    with torch.no_grad():
        if a.only in ("", "cfg4"):
            print(json.dumps({"cfg4_seem": cfg4(dev)}), flush=True)
            torch.cuda.empty_cache()
        if a.only in ("", "cfg3"):
            print(json.dumps({"cfg3_video": cfg3(dev, a.clips)}), flush=True)
