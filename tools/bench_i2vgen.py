"""End-to-end i2vgen-xl sample on one GPU (BASELINE.json configs[4], primary latent reading 16 x 40 x 64 = 320 x 512 px,
50 DDIM steps, guidance 9): OpenCLIP ViT-H-14 text + image embedders -> SD-VAE encode of the conditioning image ->
50 x (2 UNetSD_I2VGen forwards + CFG), one CUDA graph replayed per step -> SD-VAE decode of 16 frames, through
vitron_b200.i2vgen_pipeline (the inner part of inference_i2vgen_entrance.worker, :118-209). Random-init weights of
the reference shapes (UNet 1.42 B, ViT-H-14, SD VAE), synthetic inputs in pinned host memory, decoded video read back."""
import argparse, json, os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from vitron_b200 import ops, param_shapes as PS  # noqa: E402
from vitron_b200.autoencoder import SD_VAE_DDCONFIG, AutoencoderKL  # noqa: E402
from vitron_b200.clip_embedder import VIT_H_14, FrozenOpenCLIPTtxtVisualEmbedder  # noqa: E402
from vitron_b200.i2vgen_pipeline import I2VGenXLPipeline  # noqa: E402
from vitron_b200.unet_i2vgen import UNetSD_I2VGen  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--samples", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    with torch.no_grad():
        unet = UNetSD_I2VGen(**bench.UNET_CFG, device=dev)
        unet.load_state_dict(PS.random_state_dict(PS.unet_shapes(bench.UNET_CFG), dev, seed=4))
        vae = AutoencoderKL(SD_VAE_DDCONFIG, 4, device=dev).load_state_dict(PS.random_state_dict(PS.vae_shapes(SD_VAE_DDCONFIG), dev, seed=7))
        clip = FrozenOpenCLIPTtxtVisualEmbedder(None, device=dev, layer="penultimate").load_state_dict(
            PS.random_state_dict(PS.openclip_shapes(VIT_H_14), dev, seed=8))
        pipe = I2VGenXLPipeline(unet, vae, clip, ddim_timesteps=a.steps, guide_scale=9.0, max_frames=16, decoder_bs=8)
        g = torch.Generator().manual_seed(3)
        img_vit = torch.randn((1, 3, 224, 224), generator=g).pin_memory()
        img_vae = torch.randn((1, 3, 320, 512), generator=g).pin_memory()
        tok = torch.randint(1, 49407, (1, 77), generator=g)
        tok[0, 12], tok[0, 13:] = 49407, 0
        neg = torch.randint(1, 49407, (1, 77), generator=g)
        neg[0, 30], neg[0, 31:] = 49407, 0
        tok, neg = tok.pin_memory(), neg.pin_memory()
        noise = torch.randn((1, 4, 16, 40, 64), generator=g).pin_memory()

        def sample():
            v = pipe(img_vit, img_vae, tok, neg, noise=noise)
            return v.cpu()
        l0 = ops.launch_count()
        v = sample()                         # first sample: graph capture + workspaces
        launches = ops.launch_count() - l0
        finite = bool(torch.isfinite(v).all())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        for _ in range(a.samples):
            sample()
        e1.record()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) / a.samples
        ms = e0.elapsed_time(e1) / a.samples
        tflop = a.steps * 2 * bench.UNET_TFLOP_PER_FORWARD + 25.0
        print(json.dumps({"i2vgen_xl_sample": {
            "config": "BASELINE.json configs[4] (primary latent [1,4,16,40,64]): CLIP ViT-H-14 + VAE encode + %d DDIM steps x 2 UNet forwards + VAE decode" % a.steps,
            "video": list(v.shape), "s_per_video": round(ms / 1e3, 3), "wall_s_per_video": round(wall, 3),
            "videos_per_min": round(60e3 / ms, 2), "denoise_steps_per_s_incl_everything": round(a.steps / (ms * 1e-3), 2),
            "algorithmic_tflop": round(tflop, 1), "achieved_tflops": round(tflop / (ms * 1e-3), 1), "launches_first_sample": launches,
            "finite": finite, "h2d_bytes": (img_vit.numel() + img_vae.numel() + noise.numel()) * 4 + 2 * 77 * 8,
            "d2h_bytes": v.numel() * 4}}), flush=True)


if __name__ == "__main__":
    main()
