"""GPU: GLIGEN's sampling chain (grounded_generation_box sampler call + decode, task_grounded_generation.py:241-263) through
vitron_b200.gligen_sampler.grounded_sample — PLMS with the scheduled gate over the CUDA UNetModel, AutoencoderKL decode —
against the same chain built from the CPU oracles (the sampler arithmetic itself is pinned against the unmodified reference
PLMSSampler on the CPU: tests/test_oracle_cpu.py::test_gligen_plms_sampler_matches_reference_sampler). Tiny widths, 5 steps,
mild guidance; <= 10 % inf / 8 % L2 on the decoded images."""
import os
from functools import partial

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_grounded_sample_vs_oracle_chain(cuda):
    from oracle import restate_gligen_unet as G, restate_vae as V
    from oracle.weights import seeded_state_dict
    from vitron_b200 import gligen_sampler as GS
    from vitron_b200.autoencoder import AutoencoderKL
    from vitron_b200.gligen_unet import UNetModel
    ufx = torch.load(os.path.join(GOLD, "gligen_unet_tiny.pt"), weights_only=False)
    vfx = torch.load(os.path.join(GOLD, "vae_tiny.pt"), weights_only=False)
    usd = seeded_state_dict(ufx["shapes"], ufx["seed"], ufx["gain"])
    vsd = seeded_state_dict(vfx["shapes"], vfx["seed"], 0.8)
    cfg = dict(ufx["cfg"], image_size=16)
    unet = UNetModel(**cfg, device=cuda).load_state_dict(usd)
    vae = AutoencoderKL(vfx["ddconfig"], 4, device=cuda).load_state_dict(vsd)
    inp = {k: v for k, v in ufx["inputs"].items() if k not in ("x", "timesteps")}
    g = torch.Generator().manual_seed(1)
    start = torch.randn((2, 4, 16, 16), generator=g)
    uc = torch.randn(inp["context"].shape, generator=g)
    steps, guide, atype = 5, 2.0, (0.4, 0.2, 0.4)
    dev_inp = {k: v.to(cuda) for k, v in inp.items()}
    img = GS.grounded_sample(unet, vae, GS.DDPM(device=cuda), dict(dev_inp, x=start.to(cuda), timesteps=None), uc.to(cuda),
                             guidance_scale=guide, steps=steps, alpha_type=atype)

    class OracleModel:
        scale = 1.0

        def __call__(self, d):
            return G.unet_forward(usd, cfg, d, alpha_scale=self.scale)
    sampler = GS.PLMSSampler(GS.DDPM(), OracleModel(), alpha_generator_func=partial(GS.alpha_generator, type=list(atype)),
                             set_alpha_scale=lambda m, a: setattr(m, "scale", float(a)))
    lat = sampler.sample(S=steps, shape=(2, 4, 16, 16), input=dict(inp, x=start.clone(), timesteps=None), uc=uc, guidance_scale=guide)
    ref = V.decode(vsd, lat / 0.18215, vfx["ddconfig"])  # GLIGEN decode = decoder(z / scale_factor), autoencoder.py:40-45
    got = img.float().cpu()
    assert got.shape == ref.shape and bool(torch.isfinite(got).all())
    e_inf = ((got - ref).abs().max() / (ref.abs().max() + 1e-6)).item()
    e_l2 = ((got - ref).norm() / (ref.norm() + 1e-6)).item()
    assert e_inf < 0.10 and e_l2 < 0.08, (e_inf, e_l2)
