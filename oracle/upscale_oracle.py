"""fp32 oracle of sdwui's hires-fix upscalers, restated from sdwui >= 1.8 (processing.StableDiffusionProcessingTxt2Img.
sample_hr_pass, images.resize_image / split_grid / combine_grid, modules/upscaler.Upscaler.upscale,
upscaler_utils.upscale_with_model / upscale_pil_patch) and basicsr's RRDBNet, with PIL for every image operation.
sdwui itself is not vendored here, so this restatement is not pinned to its code (DESIGN §2: parity unpinned).

txt2img_hires is sd_oracle.txt2img_hires with the upscaler in the middle; it reuses sd_oracle's functions unchanged.
"""
import math
from collections import namedtuple

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image

from oracle import sd_oracle as O

LATENT_MODES = {"Latent": ("bilinear", False), "Latent (antialiased)": ("bilinear", True),
                "Latent (bicubic)": ("bicubic", False), "Latent (bicubic antialiased)": ("bicubic", True),
                "Latent (nearest)": ("nearest", False), "Latent (nearest-exact)": ("nearest-exact", False)}


# ------------------------------------------------------------------------------------------------ basicsr RRDBNet
def _conv(sd, key, x):
    return F.conv2d(x, sd[f"{key}.weight"], sd[f"{key}.bias"], padding=1)


def _lrelu(x):
    return F.leaky_relu(x, 0.2)


def rdb(sd, p, x):
    x1 = _lrelu(_conv(sd, f"{p}.conv1", x))
    x2 = _lrelu(_conv(sd, f"{p}.conv2", torch.cat((x, x1), 1)))
    x3 = _lrelu(_conv(sd, f"{p}.conv3", torch.cat((x, x1, x2), 1)))
    x4 = _lrelu(_conv(sd, f"{p}.conv4", torch.cat((x, x1, x2, x3), 1)))
    x5 = _conv(sd, f"{p}.conv5", torch.cat((x, x1, x2, x3, x4), 1))
    return x5 * 0.2 + x


def rrdbnet(sd, x):
    """basicsr RRDBNet(num_in_ch=3, num_out_ch=3, scale=4, num_feat=64, num_grow_ch=32) on BGR [N, 3, H, W] in [0, 1]"""
    nb = len({int(k.split(".")[1]) for k in sd if k.startswith("body.")})
    feat = _conv(sd, "conv_first", x)
    body = feat
    for i in range(nb):
        out = rdb(sd, f"body.{i}.rdb3", rdb(sd, f"body.{i}.rdb2", rdb(sd, f"body.{i}.rdb1", body)))
        body = out * 0.2 + body
    feat = feat + _conv(sd, "conv_body", body)
    feat = _lrelu(_conv(sd, "conv_up1", F.interpolate(feat, scale_factor=2, mode="nearest")))
    feat = _lrelu(_conv(sd, "conv_up2", F.interpolate(feat, scale_factor=2, mode="nearest")))
    return _conv(sd, "conv_last", _lrelu(_conv(sd, "conv_hr", feat)))


def pil_to_bgr(imgs):
    """upscaler_utils.pil_image_to_torch_bgr for a list of same-size images -> [N, 3, H, W] fp32 BGR / 255"""
    a = np.stack([np.array(im.convert("RGB")) for im in imgs])[..., ::-1]
    return torch.from_numpy(np.ascontiguousarray(a.transpose(0, 3, 1, 2)) / 255).float()


def bgr_to_pil(t):
    """upscaler_utils.torch_bgr_to_pil_image per image: clamp, x 255, round, uint8, BGR -> RGB"""
    arr = t.float().cpu().clamp_(0, 1).numpy()
    arr = (255.0 * np.moveaxis(arr, 1, 3)).round().astype(np.uint8)[..., ::-1]
    return [Image.fromarray(np.ascontiguousarray(a), "RGB") for a in arr]


# ------------------------------------------------------------------------------------------------ sdwui images.py
Grid = namedtuple("Grid", ["tiles", "tile_w", "tile_h", "image_w", "image_h", "overlap"])


def split_grid(image, tile_w=512, tile_h=512, overlap=64):
    w, h = image.size
    non_overlap_width = tile_w - overlap
    non_overlap_height = tile_h - overlap
    cols = math.ceil((w - overlap) / non_overlap_width)
    rows = math.ceil((h - overlap) / non_overlap_height)
    dx = (w - tile_w) / (cols - 1) if cols > 1 else 0
    dy = (h - tile_h) / (rows - 1) if rows > 1 else 0
    grid = Grid([], tile_w, tile_h, w, h, overlap)
    for row in range(rows):
        row_images = []
        y = int(row * dy)
        if y + tile_h >= h:
            y = h - tile_h
        for col in range(cols):
            x = int(col * dx)
            if x + tile_w >= w:
                x = w - tile_w
            tile = image.crop((x, y, x + tile_w, y + tile_h))
            row_images.append([x, tile_w, tile])
        grid.tiles.append([y, tile_h, row_images])
    return grid


def combine_grid(grid):
    def make_mask_image(r):
        r = r * 255 / grid.overlap
        r = r.astype(np.uint8)
        return Image.fromarray(r, 'L')

    mask_w = make_mask_image(np.arange(grid.overlap, dtype=np.float32).reshape((1, grid.overlap)).repeat(grid.tile_h, axis=0))
    mask_h = make_mask_image(np.arange(grid.overlap, dtype=np.float32).reshape((grid.overlap, 1)).repeat(grid.image_w, axis=1))
    combined_image = Image.new("RGB", (grid.image_w, grid.image_h))
    for y, h, row in grid.tiles:
        combined_row = Image.new("RGB", (grid.image_w, h))
        for x, w, tile in row:
            if x == 0:
                combined_row.paste(tile, (0, 0))
                continue
            combined_row.paste(tile.crop((0, 0, grid.overlap, h)), (x, 0), mask=mask_w)
            combined_row.paste(tile.crop((grid.overlap, 0, w, h)), (x + grid.overlap, 0))
        if y == 0:
            combined_image.paste(combined_row, (0, 0))
            continue
        combined_image.paste(combined_row.crop((0, 0, combined_row.width, grid.overlap)), (0, y), mask=mask_h)
        combined_image.paste(combined_row.crop((0, grid.overlap, combined_row.width, h)), (0, y + grid.overlap))
    return combined_image


def upscale_with_model(sd, img, tile_size=192, tile_overlap=8, device="cpu"):
    """upscaler_utils.upscale_with_model (tiles one at a time through upscale_pil_patch)"""
    net = lambda im: bgr_to_pil(rrdbnet(sd, pil_to_bgr([im]).to(device)))[0]  # noqa: E731
    if tile_size <= 0:
        return net(img)
    grid = split_grid(img, tile_size, tile_size, tile_overlap)
    newtiles = []
    scale_factor = 1
    for y, h, row in grid.tiles:
        newrow = []
        for x, w, tile in row:
            output = net(tile)
            scale_factor = output.width // tile.width
            newrow.append([x * scale_factor, w * scale_factor, output])
        newtiles.append([y * scale_factor, h * scale_factor, newrow])
    newgrid = Grid(newtiles, tile_w=grid.tile_w * scale_factor, tile_h=grid.tile_h * scale_factor,
                   image_w=grid.image_w * scale_factor, image_h=grid.image_h * scale_factor,
                   overlap=grid.overlap * scale_factor)
    return combine_grid(newgrid)


def upscaler_upscale(img, scale, do_upscale):
    """modules/upscaler.Upscaler.upscale"""
    dest_w = int((img.width * scale) // 8 * 8)
    dest_h = int((img.height * scale) // 8 * 8)
    for i in range(3):
        if img.width >= dest_w and img.height >= dest_h and (i > 0 or scale != 1):
            break
        shape = (img.width, img.height)
        img = do_upscale(img)
        if shape == (img.width, img.height):
            break
    if img.width != dest_w or img.height != dest_h:
        img = img.resize((int(dest_w), int(dest_h)), resample=Image.LANCZOS)
    return img


def resize_image(im, width, height, upscaler, esrgan_sd=None, tile=192, overlap=8, device="cpu"):
    """images.resize_image(0, im, width, height, upscaler_name=upscaler) for None / Lanczos / Nearest / an ESRGAN model
    given by its basicsr state dict"""
    if upscaler == "None":
        return im.resize((width, height), resample=Image.LANCZOS)
    scale = max(width / im.width, height / im.height)
    if scale > 1.0:
        if upscaler in ("Lanczos", "Nearest"):
            filt = Image.LANCZOS if upscaler == "Lanczos" else Image.NEAREST
            do = lambda i: i.resize((int(i.width * scale), int(i.height * scale)), resample=filt)  # noqa: E731
        else:
            do = lambda i: upscale_with_model(esrgan_sd, i, tile, overlap, device)  # noqa: E731
        im = upscaler_upscale(im, scale, do)
    if im.width != width or im.height != height:
        im = im.resize((width, height), resample=Image.LANCZOS)
    return im


# ------------------------------------------------------------------------------------------------ the hires request
def hires_upscale(dsd, vae_cfg, x, h2: int, w2: int, upscaler: str, esrgan_sd=None, tile: int = 192, overlap: int = 8,
                  device="cpu"):
    """sample_hr_pass's upscale of the first-pass latents x [b, 4, h, w] to [b, 4, h2, w2]: F.interpolate for the Latent
    modes, else decode, uint8, images.resize_image and VAE-encode (posterior mean x scale factor)"""
    if upscaler in LATENT_MODES:
        mode, aa = LATENT_MODES[upscaler]
        return F.interpolate(x, size=(h2, w2), mode=mode, antialias=aa)
    f = 2 ** (len(vae_cfg.ch_mult) - 1)   # the autoencoder's factor: 8 for kl-f8, where (w2, h2) * f = (W, H) * hr_scale
    low = O.to_uint8(O.vae_decode(dsd, vae_cfg, x / vae_cfg.scale_factor)).cpu().numpy()
    esd = None if esrgan_sd is None else {k: v.to(device) for k, v in esrgan_sd.items()}
    big = [np.array(resize_image(Image.fromarray(im), w2 * f, h2 * f, upscaler, esd, tile, overlap, device)) for im in low]
    x_in = O.image_to_model_input(torch.from_numpy(np.stack(big)).to(device))
    return O.vae_encode_mean(dsd, vae_cfg, x_in) * vae_cfg.scale_factor


def txt2img_hires(sd, unet_cfg, vae_cfg, clip_cfg, tokens, neg_tokens, seed: int, steps: int = 20,
                  cfg_scale: float = 7.0, height: int = 512, width: int = 512, hr_scale: float = 2.0, hr_steps: int = 0,
                  denoising_strength: float = 0.7, upscaler: str = "Latent", esrgan_sd=None, tile: int = 192,
                  overlap: int = 8, device="cpu"):
    """sd_oracle.txt2img_hires with sdwui's hr_upscaler: DDIM first pass -> hires_upscale -> DDIM img2img from t_enc ->
    decode.  Returns (uint8 images, final latents)."""
    b = tokens.shape[0]
    h, w = height // 8, width // 8
    h2, w2 = int(height * hr_scale) // 8, int(width * hr_scale) // 8
    dsd = {k: v.to(device) for k, v in sd.items()}
    cond = O.clip_text_encode(dsd, clip_cfg, tokens.to(device))
    uncond = O.clip_text_encode(dsd, clip_cfg, neg_tokens.to(device))
    unet = lambda a, tt, c: O.unet_forward(dsd, unet_cfg, a, tt, c)  # noqa: E731
    x = O.sample_ddim(unet, O.per_image_noise(seed, b, (4, h, w)).to(device), cond, uncond, steps, cfg_scale)
    up = hires_upscale(dsd, vae_cfg, x, h2, w2, upscaler, esrgan_sd, tile, overlap, device)
    noise = O.per_image_noise(seed, b, (4, h2, w2)).to(device)
    sa, s1a, rows = O.ddim_img2img_coefficients(hr_steps or steps, denoising_strength)
    x = up * sa + noise * s1a
    for (t, c_sa, c_s1a, c_sap, c_s1ap) in rows:
        e = O.cfg_eps(unet, x, t, cond, uncond, cfg_scale)
        x0 = (x - c_s1a * e) / c_sa
        x = c_sap * x0 + c_s1ap * e
    dec = O.vae_decode(dsd, vae_cfg, x / vae_cfg.scale_factor)
    return O.to_uint8(dec), x


def _noise_draws(seed: int, b: int, shape, draws: int):
    """sdwui ImageRNG (randn_source CPU): image k's generator seeded seed + k, `draws` successive tensors of `shape`
    -> [draws, b, *shape]"""
    out = torch.empty((draws, b, *shape))
    for k in range(b):
        g = torch.Generator().manual_seed(int(seed) + k)
        for d in range(draws):
            out[d, k] = torch.randn(shape, generator=g)
    return out


def txt2img_hires_xl(sd, unet_cfg, vae_cfg, clip_cfg, tokens, neg_tokens, seed: int, steps: int = 20,
                     cfg_scale: float = 7.0, height: int = 1024, width: int = 1024, hr_scale: float = 2.0,
                     hr_steps: int = 0, denoising_strength: float = 0.7, upscaler: str = "Latent", esrgan_sd=None,
                     tile: int = 192, overlap: int = 8, sampler: str = "Euler a", device="cpu"):
    """The SDXL hires fix on a k-diffusion sampler: sd_oracle.sdxl_conditioner (an all-empty negative prompt gets zero
    text embeddings, as sdwui's get_learned_conditioning does) and run_sampler for both passes, hires_upscale between
    them, the second pass conditioned on the large size (sdwui hr_c / hr_uc) and started from fresh noise of the large
    shape from the same seeds.  Returns (uint8 images, final latents)."""
    b = tokens.shape[0]
    h, w = height // 8, width // 8
    h2, w2 = int(height * hr_scale) // 8, int(width * hr_scale) // 8
    dsd = {k: v.to(device) for k, v in sd.items()}
    empty = bool((neg_tokens[:, 1:] == neg_tokens[:, -1:]).all())

    def run(hh, ww, n, init=None):
        ctx_c, y_c = O.sdxl_conditioner(dsd, clip_cfg, tokens.to(device), ww * 8, hh * 8)
        ctx_u, y_u = O.sdxl_conditioner(dsd, clip_cfg, neg_tokens.to(device), ww * 8, hh * 8, zero_txt=empty)
        y = torch.cat([y_c, y_u])
        unet = lambda a, tt, c: O.unet_forward(dsd, unet_cfg, a, tt, c, y=y)  # noqa: E731
        nz = _noise_draws(seed, b, (4, hh, ww), 1 + n).to(device)   # x_T, then at most one ancestral draw per step
        return O.run_sampler(sampler, unet, ctx_c, ctx_u, cfg_scale, n, nz[0], list(nz[1:]), init=init,
                             denoising_strength=None if init is None else denoising_strength)

    x = run(h, w, steps)
    up = hires_upscale(dsd, vae_cfg, x, h2, w2, upscaler, esrgan_sd, tile, overlap, device)
    x = run(h2, w2, hr_steps or steps, init=up)
    dec = O.vae_decode(dsd, vae_cfg, x / vae_cfg.scale_factor)
    return O.to_uint8(dec), x
