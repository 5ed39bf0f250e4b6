"""Measurements for SURVEY.md §8(f1): SEEM's FocalNet-L backbone (seem_focall_lang.yaml:29-47) on one GPU.

  * whole backbone at 1024x1024 (the BASELINE.json configs[3] image): ms / image with a pinned host image (H2D
    inside the timed region), achieved TFLOP/s on the algorithmic GEMM FLOPs;
  * the depthwise focal conv kernel alone (stage-0 shape, the four levels k = 3, 5, 7, 9): CUDA-event time per
    launch by CUDA-graph replay, achieved HBM GB/s on its algorithmic bytes (read ctx + write ctx: 2 * T * C * 2 B)
    and FP32 FMA rate (T * C * k^2 FMA) — the kernel is bound by whichever is lower;
  * images -> backbone -> pixel decoder -> mask decoder (configs[3] with the backbone included).
Random-init weights of the reference shapes, synthetic inputs, bf16. `--profile` runs ONE forward (for ncu)."""
import argparse, json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import ops, param_shapes as PS  # noqa: E402
from vitron_b200.focal import FOCAL_L_CFG, D2FocalNet  # noqa: E402

FOCAL_L = dict(embed_dim=192, depths=(2, 2, 18, 2), focal_levels=(4, 4, 4, 4), focal_windows=(3, 3, 3, 3), mlp_ratio=4.0,
               patch_size=4, use_conv_embed=True, use_postln=True, use_postln_in_modulation=False, scaling_modulator=True,
               use_layerscale=True, patch_norm=True, out_indices=(0, 1, 2, 3))


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


def graph_time(fn, iters=20):
    """Mean time of one fn() by CUDA-graph replay (no launch gaps)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    return ev_time(g.replay, 5, 2) / iters


def focal_flops(h, w, cfg=FOCAL_L):
    """Algorithmic FLOPs of one image: GEMMs (f, h, proj, fc1, fc2, stem, downsample) + depthwise convs."""
    E = cfg["embed_dim"]
    H, W = -(-h // 4), -(-w // 4)
    gemm = 2.0 * H * W * E * 147
    dw = 0.0
    for i, d in enumerate(cfg["depths"]):
        C, T, L = E * 2 ** i, H * W, cfg["focal_levels"][i]
        per_block = 2.0 * T * C * (2 * C + L + 1) + 2.0 * T * C * C * 2 + 2.0 * T * C * 4 * C * 2
        gemm += d * per_block
        dw += d * sum(2.0 * T * C * (2 * l + cfg["focal_windows"][i]) ** 2 for l in range(L))
        if i < len(cfg["depths"]) - 1:
            H, W = (H + 1) // 2, (W + 1) // 2
            gemm += 2.0 * H * W * (2 * C) * C * 9
    return gemm, dw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--no-seem", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = float(peaks.get("hbm_gbs", 3350.0))   # H100 SXM data sheet unless MEASURED_PEAKS.json says otherwise
    with torch.no_grad():
        net = D2FocalNet(FOCAL_L_CFG, device=dev).load_state_dict(PS.random_state_dict(PS.focalnet_shapes(FOCAL_L), dev, seed=5))
        img = torch.randn((1, 3, a.size, a.size), generator=torch.Generator().manual_seed(1)).pin_memory()
        if a.profile:
            net(img.to(dev))
            torch.cuda.synchronize()
            net(img.to(dev))
            torch.cuda.synchronize()
            return
        out = {}
        l0 = ops.launch_count()
        feats = net(img.to(dev))
        launches = ops.launch_count() - l0
        finite = all(bool(torch.isfinite(v.float()).all()) for v in feats.values())

        def run():
            f = net(img.to(dev, non_blocking=True))
            return f["res5"].float().cpu()
        ms = ev_time(run, 5, 3)
        gflop, dwflop = focal_flops(a.size, a.size)
        out["focalnet_l"] = {"image": [1, 3, a.size, a.size], "ms_per_image": round(ms, 3), "images_per_s": round(1e3 / ms, 2),
                             "launches_per_image": launches, "finite": finite, "gemm_tflop": round(gflop / 1e12, 3),
                             "dwconv_gflop": round(dwflop / 1e9, 1), "achieved_tflops_gemm_only": round(gflop / 1e12 / (ms * 1e-3), 1),
                             "h2d_bytes": img.numel() * 4, "shapes": {k: list(v.shape) for k, v in feats.items()}}
        # depthwise focal conv at the stage-0 and stage-2 shapes of a 1024^2 image, every kernel variant
        rows = []
        for (T_h, C) in ((a.size // 4, 192), (a.size // 16, 768)):
            T_w = T_h
            fo = torch.randn((1, T_h, T_w, 2 * C + 8), device=dev).to(torch.bfloat16)
            for k in (3, 5, 7, 9):
                wt = ops.pack_dwconv_weight(torch.randn((C, 1, k, k), device=dev) / k)
                src = fo[..., C:2 * C] if k == 3 else torch.randn((1, T_h, T_w, C), device=dev).to(torch.bfloat16)
                byts = 2.0 * T_h * T_w * C * 2
                fma = float(T_h * T_w * C * k * k)
                row = {"shape": [1, T_h, T_w, C], "k": k, "algorithmic_bytes": byts}
                for impl, name in ((0, "auto"), (1, "vec8"), (2, "pair16"), (3, "pair32")):
                    ops.set_dwconv_impl(impl)
                    t = graph_time(lambda: ops.dwconv_nhwc(src, wt, k, act=ops.ACT_GELU), 10)
                    row[name + "_us"] = round(t * 1e3, 2)
                ops.set_dwconv_impl(0)
                t = row["auto_us"] * 1e-3
                row.update({"achieved_gbs": round(byts / (t * 1e-3) / 1e9, 1), "frac_of_hbm_peak": round(byts / (t * 1e-3) / 1e9 / hbm, 3),
                            "tfma_per_s": round(fma / (t * 1e-3) / 1e12, 2)})
                rows.append(row)
        out["dwconv"] = {"hbm_peak_gbs": hbm, "fp32_fma_peak_tfma_s": round(148 * 128 * 1.965e9 / 1e12, 1), "levels": rows}
        x0 = torch.randn((1, 256 * 256, 192), device=dev).to(torch.bfloat16)
        x2 = torch.randn((1, 64 * 64, 768), device=dev).to(torch.bfloat16)
        out["colmean_us"] = {"stage0_65536x192": round(graph_time(lambda: ops.colmean(x0.view(-1, 192), 1, act=ops.ACT_GELU), 10) * 1e3, 2),
                             "stage2_4096x768": round(graph_time(lambda: ops.colmean(x2.view(-1, 768), 1, act=ops.ACT_GELU), 10) * 1e3, 2)}
        print(json.dumps(out), flush=True)
        if a.no_seem:
            return
        from vitron_b200.seem import MultiScaleMaskedTransformerDecoder, TransformerEncoderPixelDecoder, XDecoderHead
        in_ch = (192, 384, 768, 1536)
        head = XDecoderHead(TransformerEncoderPixelDecoder(in_ch, 512, 512, 8, 2048, 6, device=dev),
                            MultiScaleMaskedTransformerDecoder(512, 512, 101, 8, 2048, 9, 512, device=dev)).load_state_dict(
            PS.random_state_dict(PS.seem_shapes(in_ch), dev, seed=3))

        def e2e():
            o = head(net(img.to(dev, non_blocking=True)))
            return o["pred_masks"].float().cpu()
        l0 = ops.launch_count()
        ms2 = ev_time(e2e, 5, 2)
        print(json.dumps({"seem_with_backbone": {
            "config": "BASELINE.json configs[3] + FocalNet-L backbone: 1024x1024 image -> 101 mask logits [101,256,256]",
            "ms_per_image_e2e": round(ms2, 2), "images_per_s": round(1e3 / ms2, 2), "backbone_ms": round(ms, 2),
            "launches_per_image": (ops.launch_count() - l0) // 7, "h2d_bytes": img.numel() * 4, "d2h_bytes": 101 * 256 * 256 * 4,
            "achieved_tflops": round((gflop / 1e12 + 0.95) / (ms2 * 1e-3), 1)}}), flush=True)


if __name__ == "__main__":
    main()
