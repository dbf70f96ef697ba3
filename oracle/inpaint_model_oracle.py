"""fp32 oracle of inpainting checkpoints (9-channel UNets: sd-v1-5-inpainting, 512-inpainting-ema, SDXL inpainting), built
from the unchanged sd_oracle, v_oracle and controlnet_oracle functions.

Such a UNet is ldm's "hybrid" conditioning: its input is cat([x, c_concat]) along channels, c_concat = [mask at latent
size, VAE latents of the masked init image], the same for both CFG halves.  sdwui builds c_concat once per request:
  * txt2img_image_conditioning: a gray image (0.5 in [0, 1], so 0 in [-1, 1]) encoded, under an all-ones mask;
  * inpainting_image_conditioning (img2img, the hires fix's pixel upscalers): M = round(image_mask / 255) (all ones
    without a mask), the image torch.lerp(s, s * (1 - M), inpainting_mask_weight) encoded as init images are (posterior
    mean x scale_factor), the mask brought to latent size by F.interpolate (nearest).
The samplers run under a UNet shim: for the duration of `concat(c)` the `unet_forward` of sd_oracle and controlnet_oracle
see cat([x, c]) (c repeated over the [cond | uncond] batch), as tiling_oracle swaps their `F`.
"""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import controlnet_oracle as CN
from oracle import sd_oracle as O

VAE_CONV_IN = "first_stage_model.encoder.conv_in.weight"   # any encoder weight: where the oracle's tensors live


def processed_mask(mask_img, width: int, height: int, mask_blur: int = 4, invert: bool = False,
                   only_masked_padding=None):
    """sdwui StableDiffusionProcessingImg2Img.init's `image_mask` as uint8 [H, W] (mask_round True): the binary mask,
    inverted, blurred along x then y, at the processing size ("whole picture": resize_image(0), LANCZOS); with
    only_masked_padding ("Only masked") the padded crop region grown to the processing aspect, resize_image(2).
    None for an "Only masked" request with a blank mask (sdwui then runs plain img2img)."""
    import cv2
    from PIL import Image, ImageOps
    if mask_img.mode == "RGBA" and mask_img.getextrema()[-1] != (255, 255):
        m = mask_img.split()[-1].convert("L").point(lambda v: 255 if v > 128 else 0)
    else:
        m = mask_img.convert("L")
    if invert:
        m = ImageOps.invert(m)
    if mask_blur > 0:
        k = 2 * int(2.5 * mask_blur + 0.5) + 1
        m = Image.fromarray(cv2.GaussianBlur(cv2.GaussianBlur(np.array(m), (k, 1), mask_blur), (1, k), mask_blur))
    if only_masked_padding is None:
        if m.size != (width, height):
            m = m.resize((width, height), resample=Image.LANCZOS)
        return torch.from_numpy(np.array(m))
    if not np.array(m).any():
        return None
    region = O.expand_crop_region(O.get_crop_region(np.array(m), only_masked_padding), width, height, m.width, m.height)
    return torch.from_numpy(np.array(O.resize_image(2, m.crop(region), width, height).convert("L")))


def conditioning_mask(mask_u8, height: int, width: int, device="cpu") -> torch.Tensor:
    """M [1, 1, H, W] = round(image_mask / 255) (round half to even: 127 -> 0, 128 -> 1); None: all ones"""
    if mask_u8 is None:
        return torch.ones((1, 1, height, width), device=device)
    return torch.round(mask_u8.float()[None, None] / 255.0)


def image_conditioning(sd, vae_cfg, source: torch.Tensor, mask: torch.Tensor, weight: float) -> torch.Tensor:
    """sdwui inpainting_image_conditioning: source [b, 3, H, W] in [-1, 1], mask [1, 1, H, W] -> c_concat [b, 5, h, w]"""
    image = torch.lerp(source, source * (1.0 - mask), weight)
    z = O.vae_encode_mean(sd, vae_cfg, image) * vae_cfg.scale_factor
    m = F.interpolate(mask, size=z.shape[-2:])
    return torch.cat([m.expand(z.shape[0], -1, -1, -1), z], dim=1)


def img2img_image_conditioning(sd, vae_cfg, init_u8: torch.Tensor, mask_u8=None, weight: float = 1.0) -> torch.Tensor:
    """uint8 init images [b, H, W, 3] (after the fill) and image_mask uint8 [H, W] or None -> c_concat"""
    source = O.image_to_model_input(init_u8)
    return image_conditioning(sd, vae_cfg, source, conditioning_mask(mask_u8, *source.shape[-2:], source.device), weight)


def txt2img_image_conditioning(sd, vae_cfg, b: int, height: int, width: int) -> torch.Tensor:
    """sdwui txt2img_image_conditioning for an inpainting model: gray 0.5 -> 2 * 0.5 - 1 = 0, encoded; a mask channel of 1"""
    dev = sd[VAE_CONV_IN].device
    z = O.vae_encode_mean(sd, vae_cfg, torch.zeros((b, 3, height, width), device=dev)) * vae_cfg.scale_factor
    return torch.cat([torch.ones((b, 1, *z.shape[-2:]), device=dev), z], dim=1)


def hires_image_conditioning(sd, vae_cfg, upscaler: str, b: int, height: int, width: int, upscaled_u8=None,
                             weight: float = 1.0) -> torch.Tensor:
    """sdwui sample_hr_pass at the hires pixel size: "Latent ..." upscalers take txt2img's conditioning (weight 1; below 1
    sdwui conditions on the float decode of the upscaled latents, which is not restated), the pixel upscalers
    img2img's of the upscaled uint8 images without a mask"""
    if upscaler.startswith("Latent"):
        if weight < 1:
            raise NotImplementedError("Latent upscaler with inpainting_mask_weight < 1")
        return txt2img_image_conditioning(sd, vae_cfg, b, height, width)
    return img2img_image_conditioning(sd, vae_cfg, upscaled_u8, None, weight)


def _concat(fn, c_concat):
    def unet_forward(sd, cfg, x, *a, **k):
        c = c_concat.to(x)
        return fn(sd, cfg, torch.cat([x, c.repeat(x.shape[0] // c.shape[0], 1, 1, 1)], dim=1), *a, **k)
    return unet_forward


@contextlib.contextmanager
def concat(c_concat: torch.Tensor):
    """inside: sd_oracle.unet_forward and controlnet_oracle.unet_forward (what sd_oracle, v_oracle and controlnet_oracle
    sampling calls) take cat([x, c_concat]) for x; c_concat [b, 5, h, w] is repeated over x's [cond | uncond] batch"""
    saved = (O.unet_forward, CN.unet_forward)
    O.unet_forward, CN.unet_forward = _concat(saved[0], c_concat), _concat(saved[1], c_concat)
    try:
        yield
    finally:
        O.unet_forward, CN.unet_forward = saved


def run(fn, *a, c_concat: torch.Tensor, **k):
    """fn(*a, **k) — any sd_oracle / v_oracle / controlnet_oracle sampling entry point — on an inpainting UNet conditioned
    on c_concat"""
    with concat(c_concat):
        return fn(*a, **k)
