"""Measurement for SURVEY.md §8(f2): i2vgen-xl first-stage AutoencoderKL (SD-VAE, tools/modules/config.py:110-127) on
one GPU at the BASELINE.json configs[4] primary latent: decode of 16 frames [16, 4, 40, 64] -> [16, 3, 320, 512]
(the step after the 50 DDIM steps, inference_i2vgen_entrance.py:200-209) and encode of the conditioning image
[1, 3, 320, 512] (:172-173). Random-init weights, synthetic inputs, bf16; CUDA-event timing with host inputs / outputs."""
import argparse, json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vitron_b200 import ops, param_shapes as PS  # noqa: E402
from vitron_b200.autoencoder import SD_VAE_DDCONFIG, AutoencoderKL  # noqa: E402


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


def decode_flops(n, h, w, dd=SD_VAE_DDCONFIG):
    """Algorithmic FLOPs of Decoder.forward + post_quant_conv for n latents of h x w."""
    ch, mult, nrb, z = dd["ch"], dd["ch_mult"], dd["num_res_blocks"], dd["z_channels"]
    conv = lambda px, cin, cout, k: 2.0 * px * cin * cout * k * k
    c = ch * mult[-1]
    px = n * h * w
    f = conv(px, z, z, 1) + conv(px, z, c, 3)
    res = lambda px, cin, cout: conv(px, cin, cout, 3) + conv(px, cout, cout, 3) + (conv(px, cin, cout, 1) if cin != cout else 0)
    f += 2 * res(px, c, c) + 4 * conv(px, c, c, 1) + n * 4.0 * (h * w) ** 2 * c
    for i in reversed(range(len(mult))):
        co = ch * mult[i]
        for _ in range(nrb + 1):
            f += res(px, c, co)
            c = co
        if i != 0:
            px *= 4
            f += conv(px, c, c, 3)
    return f + conv(px, c, dd["out_ch"], 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    with torch.no_grad():
        ae = AutoencoderKL(SD_VAE_DDCONFIG, 4, device=dev).load_state_dict(PS.random_state_dict(PS.vae_shapes(SD_VAE_DDCONFIG), dev, seed=7))
        g = torch.Generator().manual_seed(2)
        z = torch.randn((a.frames, 4, 40, 64), generator=g).pin_memory()
        img = torch.randn((1, 3, 320, 512), generator=g).pin_memory()
        if a.profile:
            ae.decode(z[:2].to(dev))
            torch.cuda.synchronize()
            return
        l0 = ops.launch_count()
        out = ae.decode(z.to(dev))
        launches = ops.launch_count() - l0
        finite = bool(torch.isfinite(out).all())
        ms_dec = ev_time(lambda: ae.decode(z.to(dev, non_blocking=True)).cpu(), 3, 2)
        ms_enc = ev_time(lambda: ae.encode(img.to(dev, non_blocking=True)).mean.cpu(), 3, 2)
        fl = decode_flops(a.frames, 40, 64)
        print(json.dumps({"sd_vae": {
            "decode": {"latents": [a.frames, 4, 40, 64], "frames_out": list(out.shape), "ms": round(ms_dec, 2),
                       "frames_per_s": round(a.frames / (ms_dec * 1e-3), 1), "algorithmic_tflop": round(fl / 1e12, 2),
                       "achieved_tflops": round(fl / 1e12 / (ms_dec * 1e-3), 1), "launches": launches, "finite": finite,
                       "h2d_bytes": z.numel() * 4, "d2h_bytes": out.numel() * 4},
            "encode": {"image": [1, 3, 320, 512], "ms": round(ms_enc, 2)}}}), flush=True)


if __name__ == "__main__":
    main()
