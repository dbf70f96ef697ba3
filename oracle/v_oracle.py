"""fp32 ground truth for v-prediction models (SD 2.x 768-v, v-parameterised SD1.5 / SDXL finetunes) and for the SD 2.x
text conditioning, built from the unchanged functions of oracle/sd_oracle.py and oracle/prompt_oracle.py.

  * SD 2.x conditioner (ldm FrozenOpenCLIPEmbedder, layer="penultimate", as sdwui's FrozenOpenCLIPEmbedderWithCustomWords
    drives it): the OpenCLIP ViT-H/14 text tower through all but its last resblock, then ln_final; prompts of k chunks are
    k separate 77-token sequences with EmphasisOriginal per chunk.
  * k-diffusion CompVisVDenoiser (sigma_data = 1) inside sdwui's CFGDenoiser, in the shape of sd_oracle.kdiff_model:
    c_skip = 1 / (sigma^2 + 1), c_out = -sigma / sqrt(sigma^2 + 1), c_in = 1 / sqrt(sigma^2 + 1);
    denoised = x c_skip + v(x c_in, t(sigma)) c_out.
  * sdwui CompVisTimestepsVDenoiser for DDIM and PLMS: eps = sqrt(a_t) v + sqrt(1 - a_t) x_t at the integer timestep
    (predict_eps_from_z_and_v), each UNet half converted before CFG combines them.
  * run_sampler: every sampler name of sd_oracle.run_sampler plus DDIM, for txt2img, the img2img half and masks.
"""
import math

import torch
import torch.nn.functional as F

from oracle import prompt_oracle as P
from oracle import sd_oracle as O

OPENCLIP_PREFIX = "cond_stage_model.model."

# SD 2.x (v2-inference-v.yaml) and its reduced-width test twin, in the oracle's config classes
SD21_UNET = O.UNetConfig(num_head_channels=64, context_dim=1024, linear_proj=True)
SD21_VAE = O.VAEConfig()
TINY21_UNET = O.UNetConfig(model_channels=64, num_head_channels=64, context_dim=64, linear_proj=True)
TINY21_VAE = O.VAEConfig(ch=64, ch_mult=(1, 2), num_res_blocks=1)


def _tower(cfg) -> O.CLIPConfig:
    """the OpenCLIP tower of an SD 2.x text config as sd_oracle.open_clip_text's xl_* fields describe one"""
    return O.CLIPConfig(vocab=cfg.vocab, width=cfg.width, layers=cfg.layers, heads=cfg.heads, xl_width=cfg.width,
                        xl_layers=cfg.layers, xl_heads=cfg.heads, xl_proj=cfg.width)


def sd21_text_encode(sd, cfg, tokens: torch.Tensor, prefix: str = OPENCLIP_PREFIX) -> torch.Tensor:
    """FrozenOpenCLIPEmbedder(layer="penultimate").encode_with_transformer: tokens [B, 77] -> ln_final(residual stream
    before the last resblock) [B, 77, width]"""
    pen, _ = O.open_clip_text(sd, _tower(cfg), tokens, prefix)
    return F.layer_norm(pen, (cfg.width,), sd[prefix + "ln_final.weight"], sd[prefix + "ln_final.bias"], 1e-5)


def encode_sd21(sd, cfg, ids: torch.Tensor, mults=None) -> torch.Tensor:
    """SD 2.x context [B, 77 * k, 1024] of token ids [B, 77 * k] with emphasis multipliers (None: unweighted)"""
    zs = []
    for _, t, m in P._chunks(ids, mults):
        z = sd21_text_encode(sd, cfg, t)
        zs.append(z if m is None else P.emphasis(z, m))
    return torch.cat(zs, dim=1)


def v_to_eps_unet(unet):
    """sdwui CompVisTimestepsVDenoiser around a v-prediction unet(x, t, c): eps = sqrt(a_t) v + sqrt(1 - a_t) x with
    a_t = alphas_cumprod[t] (integer timesteps: DDIM and PLMS)"""
    ac = O.alphas_cumprod().double()

    def eps_unet(x, t, c):
        a = ac[t.detach().cpu().round().long()].reshape(-1, 1, 1, 1)
        v = unet(x, t, c)
        return (a.sqrt().to(x) * v + (1 - a).sqrt().to(x) * x)
    return eps_unet


def kdiff_v_model(unet, cond, uncond, cfg_scale: float, log_sig: torch.Tensor, mask=None):
    """k-diffusion CompVisVDenoiser.forward inside sdwui's CFGDenoiser (sd_oracle.kdiff_model's shape): the CFG-combined v
    of the UNet at (x c_in, t(sigma)); denoised = x c_skip + v c_out.  `mask` = (init_latent, nmask) as kdiff_model."""
    def model(x, sigma: float):
        c_in = 1.0 / math.sqrt(sigma * sigma + 1.0)
        v = O.cfg_eps(unet, x * c_in, O.sigma_to_t(sigma, log_sig), cond, uncond, cfg_scale)
        den = x * (1.0 / (sigma * sigma + 1.0)) + v * (-sigma * c_in)
        if mask is not None:
            init, nmask = mask
            den = init * (1.0 - nmask) + nmask * den
        return den
    return model


def sample_ddim(unet, cond, uncond, cfg_scale: float, steps: int, noise0, init=None, denoising_strength=None, mask=None):
    """sdwui ddim (eta 0) on a v-prediction unet: txt2img from noise0, or the img2img half from `init`; `mask` =
    (init_latent, nmask): the model input is blended before every call (mask_before_denoising)"""
    eps_unet = v_to_eps_unet(unet)
    if init is None:
        rows, x = O.ddim_coefficients(steps), noise0
    else:
        sa, s1a, rows = O.ddim_img2img_coefficients(steps, denoising_strength)
        x = init * sa + noise0 * s1a
    for (t, c_sa, c_s1a, c_sap, c_s1ap) in rows:
        if mask is not None:
            x = mask[0] * (1.0 - mask[1]) + mask[1] * x
        e = O.cfg_eps(eps_unet, x, t, cond, uncond, cfg_scale)
        x = c_sap * ((x - c_s1a * e) / c_sa) + c_s1ap * e
    return x


def run_sampler(name: str, unet, cond, uncond, cfg_scale: float, steps: int, noise0, draws=None, init=None,
                denoising_strength=None, mask=None):
    """sd_oracle.run_sampler for a v-prediction unet(x, t, c) (plus "DDIM"): same schedules, starts and noise draws, the
    k-diffusion samplers around kdiff_v_model, the timestep samplers around v_to_eps_unet.  Returns the final latents
    (before the caller's final mask blend)."""
    karras = name.endswith(" Karras") or name == "DPM++ 2M"
    base = name[:-len(" Karras")] if name.endswith(" Karras") else name
    if base == "DDIM":
        return sample_ddim(unet, cond, uncond, cfg_scale, steps, noise0, init, denoising_strength, mask)
    if base == "PLMS":
        ts = O.ddim_timesteps(steps)
        x = noise0
        if init is not None:
            ac = O.alphas_cumprod().double()
            t_enc = max(1, min(int(min(denoising_strength, 0.999) * steps), len(ts) - 1))
            a = float(ac[ts[t_enc]])
            x = init * math.sqrt(a) + noise0 * math.sqrt(1 - a)
            ts = ts[:t_enc]
        return O.sample_plms(v_to_eps_unet(unet), x, cond, uncond, ts, cfg_scale, mask)
    sig, log_sig = O.sigmas_karras(steps) if karras else O.karras_sigmas_compvis(steps)
    if init is not None:
        sig = O.kdiff_img2img_sigmas(sig, steps, denoising_strength)
        x = init + noise0 * float(sig[0])
    else:
        x = noise0 * float(sig[0])
    model = kdiff_v_model(unet, cond, uncond, cfg_scale, log_sig, mask)
    fns = {"Euler": lambda: O.k_sample_euler(model, x, sig),
           "Euler a": lambda: O.k_sample_euler_ancestral(model, x, sig, draws),
           "Heun": lambda: O.k_sample_heun(model, x, sig),
           "DPM2": lambda: O.k_sample_dpm_2(model, x, sig),
           "DPM2 a": lambda: O.k_sample_dpm_2_ancestral(model, x, sig, draws),
           "DPM++ 2S a": lambda: O.k_sample_dpmpp_2s_ancestral(model, x, sig, draws),
           "DPM++ 2M": lambda: O.k_sample_dpmpp_2m(model, x, sig),
           "DPM++ SDE": lambda: O.k_sample_dpmpp_sde(model, x, sig, draws),
           "LMS": lambda: O.k_sample_lms(model, x, sig)}
    if base in fns:
        return fns[base]()
    if base in ("DPM fast", "DPM adaptive"):
        all_sig, _ = O.model_sigmas()
        lo, hi = (float(all_sig[0]), float(all_sig[-1])) if init is None else (float(sig[-2]), float(sig[0]))
        if base == "DPM fast":
            return O.k_sample_dpm_fast(model, x, lo, hi, len(sig) - 1)
        return O.k_sample_dpm_adaptive(model, x, lo, hi)[0]
    raise ValueError(name)


def cfg_unet(sd, unet_cfg, y=None):
    """unet(x, t, c) on one [cond | uncond] batch (equal context lengths); y: SDXL vector conditioning"""
    return lambda x, t, c: O.unet_forward(sd, unet_cfg, x, t, c, y=y)


def txt2img(sd, unet_cfg, vae_cfg, unet, cond, uncond, sampler: str, steps: int, cfg_scale: float, noises,
            hires=None):
    """whole v-prediction request from the contexts: noises [1 + draws, b, 4, h, w] (start noise, then the sampler's
    draws).  hires = (scale, steps, denoising strength, noises of the large shape): sdwui's hires fix with the "Latent"
    upscaler.  Returns (uint8 images [b, H, W, 3], final latents)."""
    z = run_sampler(sampler, unet, cond, uncond, cfg_scale, steps, noises[0], list(noises[1:]))
    if hires is not None:
        scale, hr_steps, d, nz2 = hires
        up = F.interpolate(z, size=(int(z.shape[2] * scale), int(z.shape[3] * scale)), mode="bilinear", antialias=False)
        z = run_sampler(sampler, unet, cond, uncond, cfg_scale, hr_steps or steps, nz2[0], list(nz2[1:]), init=up,
                        denoising_strength=d)
    return O.to_uint8(O.vae_decode(sd, vae_cfg, z / vae_cfg.scale_factor)), z


def img2img(sd, unet_cfg, vae_cfg, unet, cond, uncond, sampler: str, steps: int, cfg_scale: float, init_u8, d: float,
            noises, nmask=None):
    """v-prediction img2img (nmask [h, w]: inpainting, 1 = repaint) from uint8 init images; noises as txt2img.
    Returns (uint8 images, final latents)."""
    init = O.vae_encode_mean(sd, vae_cfg, O.image_to_model_input(init_u8)) * vae_cfg.scale_factor
    mask = None if nmask is None else (init, nmask[None, None].to(init))
    z = run_sampler(sampler, unet, cond, uncond, cfg_scale, steps, noises[0], list(noises[1:]), init=init,
                    denoising_strength=d, mask=mask)
    if mask is not None:
        z = z * mask[1] + init * (1 - mask[1])
    return O.to_uint8(O.vae_decode(sd, vae_cfg, z / vae_cfg.scale_factor)), z
