"""GLIGEN's sampling loop around the grounded UNet (SURVEY.md §8 f2): diffusion schedule, PLMS sampler, the scheduled
gate of the grounding branch and the sampling part of `grounded_generation_box`.

Mirrors modules/GLIGEN/demo/gligen: `ldm/models/diffusion/ddpm.py::DDPM.register_schedule` (:20-58), `ldm/models/diffusion/
plms.py::PLMSSampler` (:13-178; eta = 0, uniform time steps `range(0, T, T // S) + 1`, pseudo improved Euler first step then
2nd-4th order Adams-Bashforth on the CFG-combined eps, inpainting blend `q_sample(x0, t) * mask + (1 - mask) * img`),
`task_grounded_generation.py::alpha_generator` (:23-55) and `evaluator.py::set_alpha_scale` (:35-39), and the sampler call of
`grounded_generation_box` (:241-263): `samples = PLMSSampler(diffusion, model, alpha_generator_func, set_alpha_scale).sample(
S=50, shape, input, uc, guidance_scale, mask, x0)` followed by `autoencoder.decode(samples)`.

All arithmetic here is fp32 torch on the device (elementwise on a [B, 4, 64, 64] latent: a few µs per step next to the two
UNet evaluations); the model is any callable with the reference's `model(input_dict) -> eps` contract —
`vitron_b200.gligen_unet.UNetModel` on the GPU. The gate schedule takes 2-3 distinct values over a run (alpha_type
[0.3, 0.0, 0.7] -> 1 ... 0), it is a Python float folded into GEMM epilogues, so a CUDA graph of the UNet evaluation has to be
captured per distinct value (not done here: the sampler calls the UNet eagerly).
"""
import numpy as np
import torch

from .gligen import GatedSelfAttentionDense


class DDPM:
    """Schedule holder (ddpm.py:11-58), `beta_schedule="linear"`: betas = linspace(sqrt(l0), sqrt(l1), T)^2 in float64."""

    def __init__(self, beta_schedule="linear", timesteps=1000, linear_start=1e-4, linear_end=2e-2, cosine_s=8e-3, device="cpu"):
        if beta_schedule != "linear":
            raise NotImplementedError("GLIGEN's diffusion config uses the linear schedule")
        betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
        alphas = 1.0 - betas
        ac = np.cumprod(alphas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        self.num_timesteps = int(timesteps)
        self.linear_start, self.linear_end = linear_start, linear_end
        t32 = lambda a: torch.tensor(a, dtype=torch.float32, device=device)
        self.betas, self.alphas_cumprod, self.alphas_cumprod_prev = t32(betas), t32(ac), t32(ac_prev)
        self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod = t32(np.sqrt(ac)), t32(np.sqrt(1.0 - ac))

    def to(self, device):
        for k, v in list(vars(self).items()):
            if torch.is_tensor(v):
                setattr(self, k, v.to(device))
        return self

    def q_sample(self, x_start, t, noise=None):
        """Standard forward process sample (used by the inpainting blend, plms.py:98)."""
        noise = torch.randn_like(x_start) if noise is None else noise
        a = self.sqrt_alphas_cumprod.to(x_start.device)[t].view(-1, 1, 1, 1)
        s = self.sqrt_one_minus_alphas_cumprod.to(x_start.device)[t].view(-1, 1, 1, 1)
        return a * x_start + s * noise


def alpha_generator(length, type=(1, 0, 0)):
    """task_grounded_generation.py:23-55: [1]*stage0 + linear decay + [0]*stage2."""
    assert len(type) == 3 and type[0] + type[1] + type[2] == 1
    s0, s1 = int(type[0] * length), int(type[1] * length)
    s2 = length - s0 - s1
    decay = list(np.arange(start=0, stop=1, step=1 / s1)[::-1]) if s1 != 0 else []
    alphas = [1] * s0 + decay + [0] * s2
    assert len(alphas) == length
    return alphas


def set_alpha_scale(model, alpha_scale):
    """evaluator.py:35-39 on the CUDA UNetModel: `scale` of every GatedSelfAttentionDense fuser."""
    w = getattr(model, "w", None)
    if w is None:
        raise RuntimeError("set_alpha_scale: load_state_dict() first")
    for entry in w.values():
        if isinstance(entry, dict) and "blocks" in entry:
            for blk in entry["blocks"]:
                if isinstance(blk.fuser, GatedSelfAttentionDense):
                    blk.fuser.scale = float(alpha_scale)


class PLMSSampler:
    def __init__(self, diffusion, model, schedule="linear", alpha_generator_func=None, set_alpha_scale=None):
        self.diffusion, self.model, self.schedule = diffusion, model, schedule
        self.device = diffusion.betas.device
        self.ddpm_num_timesteps = diffusion.num_timesteps
        self.alpha_generator_func, self.set_alpha_scale = alpha_generator_func, set_alpha_scale

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0.0, verbose=False):
        if ddim_eta != 0:
            raise ValueError("ddim_eta must be 0 for PLMS")
        if ddim_discretize != "uniform":
            raise NotImplementedError(ddim_discretize)
        c = self.ddpm_num_timesteps // ddim_num_steps
        self.ddim_timesteps = np.asarray(list(range(0, self.ddpm_num_timesteps, c))) + 1          # util.py:55-69
        ac = self.diffusion.alphas_cumprod.detach().cpu().numpy()
        self.ddim_alphas = ac[self.ddim_timesteps]                                                 # util.py:72-83
        self.ddim_alphas_prev = np.asarray([ac[0]] + ac[self.ddim_timesteps[:-1]].tolist())
        self.ddim_sigmas = np.zeros_like(self.ddim_alphas)                                         # eta = 0
        self.ddim_sqrt_one_minus_alphas = np.sqrt(1.0 - self.ddim_alphas)

    @torch.no_grad()
    def sample(self, S, shape, input, uc=None, guidance_scale=1, mask=None, x0=None):
        self.make_schedule(ddim_num_steps=S)
        return self.plms_sampling(shape, input, uc, guidance_scale, mask=mask, x0=x0)

    @torch.no_grad()
    def plms_sampling(self, shape, input, uc=None, guidance_scale=1, mask=None, x0=None):
        b = shape[0]
        img = input["x"]
        if img is None:
            img = torch.randn(shape if mask is None else (mask.shape[0], shape[1], mask.shape[-2], mask.shape[-1]), device=self.device)
            input["x"] = img
        time_range = np.flip(self.ddim_timesteps)
        total = self.ddim_timesteps.shape[0]
        old_eps = []
        alphas = self.alpha_generator_func(len(time_range)) if self.alpha_generator_func is not None else None
        for i, step in enumerate(time_range):
            if alphas is not None:
                self.set_alpha_scale(self.model, alphas[i])
            index = total - i - 1
            ts = torch.full((b,), int(step), device=self.device, dtype=torch.long)
            ts_next = torch.full((b,), int(time_range[min(i + 1, len(time_range) - 1)]), device=self.device, dtype=torch.long)
            if mask is not None:
                assert x0 is not None
                if img.size(2) != mask.size(2) or img.size(2) != x0.size(2):
                    raise NotImplementedError("mask / x0 at another resolution than the latent (plms.py:99-103)")
                img = self.diffusion.q_sample(x0, ts) * mask + (1.0 - mask) * img
                input["x"] = img
            img, _, e_t = self.p_sample_plms(input, ts, index=index, uc=uc, guidance_scale=guidance_scale, old_eps=old_eps, t_next=ts_next)
            input["x"] = img
            old_eps.append(e_t)
            if len(old_eps) >= 4:
                old_eps.pop(0)
        return img

    @torch.no_grad()
    def p_sample_plms(self, input, t, index, guidance_scale=1.0, uc=None, old_eps=None, t_next=None):
        x = input["x"].clone()

        def get_model_output(inp):
            e_t = self.model(inp).float()
            if uc is not None and guidance_scale != 1:
                un = dict(x=inp["x"], timesteps=inp["timesteps"], context=uc)
                if "inpainting_extra_input" in inp:
                    un["inpainting_extra_input"] = inp["inpainting_extra_input"]
                e_u = self.model(un).float()
                e_t = e_u + guidance_scale * (e_t - e_u)
            return e_t

        def get_x_prev_and_pred_x0(e_t, index):
            a_t, a_prev = float(self.ddim_alphas[index]), float(self.ddim_alphas_prev[index])
            sqrt_one_minus_at = float(self.ddim_sqrt_one_minus_alphas[index])
            pred_x0 = (x - sqrt_one_minus_at * e_t) / (a_t ** 0.5)
            dir_xt = ((1.0 - a_prev) ** 0.5) * e_t                     # sigma_t = 0
            torch.randn_like(x)   # plms.py:153 draws `sigma_t * randn_like(x)` even though sigma_t = 0: keeps the RNG stream
            #                       (start noise of later images, q_sample of the inpainting blend) aligned with the reference
            return (a_prev ** 0.5) * pred_x0 + dir_xt, pred_x0

        input["timesteps"] = t
        e_t = get_model_output(input)
        if len(old_eps) == 0:       # pseudo improved Euler (2nd order)
            x_prev, _ = get_x_prev_and_pred_x0(e_t, index)
            input["x"] = x_prev
            input["timesteps"] = t_next
            e_t_prime = (e_t + get_model_output(input)) / 2
        elif len(old_eps) == 1:     # Adams-Bashforth 2 / 3 / 4
            e_t_prime = (3 * e_t - old_eps[-1]) / 2
        elif len(old_eps) == 2:
            e_t_prime = (23 * e_t - 16 * old_eps[-1] + 5 * old_eps[-2]) / 12
        else:
            e_t_prime = (55 * e_t - 59 * old_eps[-1] + 37 * old_eps[-2] - 9 * old_eps[-3]) / 24
        x_prev, pred_x0 = get_x_prev_and_pred_x0(e_t_prime, index)
        return x_prev, pred_x0, e_t


class GligenAutoencoder:
    """GLIGEN's first stage (ldm/models/autoencoder.py:14-52): the SD AutoencoderKL with the latent scale folded into
    its interface — `encode` returns `posterior.sample() * scale_factor`, `decode` computes `decode(z / scale_factor)`
    (every GLIGEN config sets scale_factor 0.18215). Wraps the i2vgen-style `vitron_b200.autoencoder.AutoencoderKL`,
    whose encode / decode are unscaled."""

    def __init__(self, vae, scale_factor=0.18215):
        self.vae, self.scale_factor = vae, float(scale_factor)

    @torch.no_grad()
    def encode(self, x, generator=None, noise=None):
        return self.vae.encode(x).sample(generator=generator, noise=noise) * self.scale_factor

    @torch.no_grad()
    def decode(self, z):
        return self.vae.decode(z * (1.0 / self.scale_factor))


@torch.no_grad()
def grounded_sample(model, autoencoder, diffusion, input, uc, guidance_scale=7.5, steps=50, alpha_type=(0.3, 0.0, 0.7),
                    mask=None, x0=None, batch_size=None, scale_factor=0.18215):
    """The sampling part of `grounded_generation_box` (task_grounded_generation.py:241-263): PLMS over the grounded UNet with the
    scheduled gate, then VAE decode. `input` is the reference's dict (x=None draws the start noise), `uc` the unconditional context.
    `autoencoder` is either a `GligenAutoencoder` (scale already in its interface) or a bare `AutoencoderKL`, which is wrapped
    with `scale_factor` here: the reference decodes `1/scale_factor * z` (ldm/models/autoencoder.py:41) and its inpainting `x0`
    is `encode(image) = posterior.sample() * scale_factor` (:34-38) — pass x0 from `GligenAutoencoder.encode`."""
    from functools import partial
    b = batch_size or input["context"].shape[0]
    sampler = PLMSSampler(diffusion, model, alpha_generator_func=partial(alpha_generator, type=list(alpha_type)),
                          set_alpha_scale=set_alpha_scale)
    shape = (b, model.in_channels, model.image_size, model.image_size)
    latents = sampler.sample(S=steps, shape=shape, input=input, uc=uc, guidance_scale=guidance_scale, mask=mask, x0=x0)
    if not isinstance(autoencoder, GligenAutoencoder):
        autoencoder = GligenAutoencoder(autoencoder, scale_factor)
    return autoencoder.decode(latents)
