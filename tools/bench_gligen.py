"""Measurement for SURVEY.md §8(f2): GLIGEN's grounded SD-1.4 UNet (openaimodel.UNetModel, gatedSA fusers) on one GPU:
one denoising evaluation of a 512x512 image (latent [2, 4, 64, 64]: cond + uncond rows of classifier-free guidance,
77 text tokens, 30 grounding tokens), eager and CUDA-graph replay. Random-init weights, synthetic inputs, bf16; host
inputs (latents + conditioning in pinned memory) and the eps prediction read back inside the timed region."""
import argparse, json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import ops, param_shapes as PS  # noqa: E402
from vitron_b200.gligen_unet import SD14_GLIGEN_UNET, UNetModel  # noqa: E402


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


def unet_flops(net, B, H, W, n_ctx=77, n_obj=30):
    """Algorithmic FLOPs of one forward from the block plan (convs, linears, attention QK^T / PV)."""
    f = 0.0
    h, w = H, W
    conv = lambda px, cin, cout, k: 2.0 * px * cin * cout * k * k
    for layers in net.plan_in + [net.plan_mid] + net.plan_out:
        for kind, p, cin, cout in layers:
            px = B * h * w
            if kind == "conv":
                f += conv(px, cin, cout, 3)
            elif kind == "res":
                f += conv(px, cin, cout, 3) + conv(px, cout, cout, 3) + (conv(px, cin, cout, 1) if cin != cout else 0) + 2.0 * B * 1280 * cout
            elif kind == "st":
                c, T = cout, h * w
                per = 2.0 * px * c * c * 2                                  # proj_in / proj_out
                per += 2.0 * px * c * c * 4 + 4.0 * B * T * T * c            # attn1
                per += 2.0 * (px + B * n_obj) * c * c * 4 + 4.0 * B * T * (T + n_obj) * c + 2.0 * B * n_obj * 768 * c   # fuser attn
                per += 2.0 * px * c * 8 * c + 2.0 * px * 4 * c * c           # fuser ff (GEGLU)
                per += 2.0 * px * c * c * 2 + 2.0 * B * n_ctx * 768 * c * 2 + 4.0 * B * T * n_ctx * c   # attn2
                per += 2.0 * px * c * 8 * c + 2.0 * px * 4 * c * c           # ff
                f += per
            elif kind == "down":
                h, w = h // 2, w // 2
                f += conv(B * h * w, cin, cout, 3)
            elif kind == "up":
                h, w = h * 2, w * 2
                f += conv(B * h * w, cin, cout, 3)
    return f + conv(B * h * w, net.final_ch, net.out_channels, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    with torch.no_grad():
        net = UNetModel(**SD14_GLIGEN_UNET, device=dev).load_state_dict(PS.random_state_dict(PS.gligen_unet_shapes(SD14_GLIGEN_UNET), dev, seed=9))
        g = torch.Generator().manual_seed(4)
        B, L = 2, a.latent
        host = dict(x=torch.randn((B, 4, L, L), generator=g), timesteps=torch.tensor([500, 500]), context=torch.randn((B, 77, 768), generator=g),
                    boxes=torch.rand((B, 30, 4), generator=g), masks=(torch.rand((B, 30), generator=g) > 0.5).float(),
                    text_embeddings=torch.randn((B, 30, 768), generator=g))
        host = {k: v.pin_memory() for k, v in host.items()}
        if a.profile:
            net({k: v.to(dev) for k, v in host.items()})
            torch.cuda.synchronize()
            return
        l0 = ops.launch_count()
        out = net({k: v.to(dev) for k, v in host.items()})
        launches = ops.launch_count() - l0
        finite = bool(torch.isfinite(out).all())
        ms = ev_time(lambda: net({k: v.to(dev, non_blocking=True) for k, v in host.items()}).cpu(), 5, 3)
        # CUDA-graph replay of the same evaluation (what a sampler loop would do: static input buffers)
        stat = {k: v.to(dev) for k, v in host.items()}
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            net(stat)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            gout = net(stat)
        def replay():
            for k, v in host.items():
                stat[k].copy_(v, non_blocking=True)
            graph.replay()
            return gout.cpu()
        ms_g = ev_time(replay, 10, 3)
        fl = unet_flops(net, B, L, L)
        print(json.dumps({"gligen_unet_sd14": {
            "latent": [B, 4, L, L], "grounding_tokens": 30, "ms_eager_e2e": round(ms, 2), "ms_graph_e2e": round(ms_g, 2),
            "evals_per_s_graph": round(1e3 / ms_g, 2), "algorithmic_tflop": round(fl / 1e12, 3),
            "achieved_tflops_graph": round(fl / 1e12 / (ms_g * 1e-3), 1), "launches": launches, "finite": finite,
            "h2d_bytes": sum(v.numel() * v.element_size() for v in host.values()), "d2h_bytes": out.numel() * 4}}), flush=True)


if __name__ == "__main__":
    main()
