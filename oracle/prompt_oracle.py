"""fp32 ground truth for prompts with sdwui syntax, built from the pinned functions of oracle/sd_oracle.py.

  * Chunked, weighted text encoding (sdwui FrozenCLIPEmbedderWithCustomWordsBase.forward / process_tokens): a prompt of
    [B, 77 * k] token ids is k separate 77-token sequences through the tower, each chunk's output scaled by its emphasis
    multipliers as EmphasisOriginal does (z * m, then rescaled so the chunk's mean over 77 x width values is unchanged),
    concatenated along the tokens.  SDXL: per tower, the pooled vector is the first chunk's, unweighted.
  * CFG as sdwui's default evaluates it (pad_cond_uncond and pad_cond_uncond_v0 off): one UNet call on [cond | uncond]
    when the two contexts have the same length, otherwise two calls — cond alone on its own length, uncond alone on its.
"""
import torch

from oracle import sd_oracle as O

CHUNK = 77


def emphasis(z: torch.Tensor, mult: torch.Tensor) -> torch.Tensor:
    """sdwui EmphasisOriginal on one chunk: z [B, 77, W], mult [B, 77]; means per sequence (one chunk of one prompt), fp32"""
    zf = z.float()
    before = zf.mean(dim=(1, 2), keepdim=True)
    zf = zf * mult.to(zf)[:, :, None]
    return zf * (before / zf.mean(dim=(1, 2), keepdim=True))


def _chunks(ids: torch.Tensor, mults):
    n = ids.shape[1]
    assert n % CHUNK == 0, n
    for j in range(n // CHUNK):
        sl = slice(j * CHUNK, (j + 1) * CHUNK)
        yield j, ids[:, sl], None if mults is None else mults[:, sl]


def encode_sd1(sd, cfg, ids: torch.Tensor, mults=None) -> torch.Tensor:
    """SD1.x context [B, 77 * k, 768] of token ids [B, 77 * k] with emphasis multipliers (None: unweighted)"""
    zs = []
    for _, t, m in _chunks(ids, mults):
        z = O.clip_text_encode(sd, cfg, t)
        zs.append(z if m is None else emphasis(z, m))
    return torch.cat(zs, dim=1)


def encode_sdxl(sd, cfg, ids: torch.Tensor, mults, width: int, height: int, zero_txt: bool = False):
    """SDXL (context [B, 77 * k, 2048], vector conditioning [B, 2816]) as sdxl_conditioner, chunked and weighted per tower"""
    h0s, h1s, pooled = [], [], None
    for j, t, m in _chunks(ids, mults):
        h0 = O.clip_text_hidden(sd, cfg, t, cfg.layers - 1, "conditioner.embedders.0.transformer.text_model.")
        h1, p = O.open_clip_text(sd, cfg, t, "conditioner.embedders.1.model.")
        h0s.append(h0 if m is None else emphasis(h0, m))
        h1s.append(h1 if m is None else emphasis(h1, m))
        if j == 0:
            pooled = p
    ctx = torch.cat([torch.cat(h0s, dim=1), torch.cat(h1s, dim=1)], dim=-1)
    if zero_txt:
        ctx, pooled = torch.zeros_like(ctx), torch.zeros_like(pooled)
    # the size part of the vector conditioning does not depend on the text
    _, y = O.sdxl_conditioner(sd, cfg, ids[:, :CHUNK], width, height)
    return ctx, torch.cat([pooled, y[:, pooled.shape[1]:]], dim=-1)


def pad_pair(cond: torch.Tensor, uncond: torch.Tensor):
    """zero-pad two contexts to one length (so the samplers' torch.cat([cond, uncond]) works) -> (cond, uncond, lc, lu)"""
    lc, lu = cond.shape[1], uncond.shape[1]
    n = max(lc, lu)
    pad = lambda c: torch.cat([c, c.new_zeros((c.shape[0], n - c.shape[1], c.shape[2]))], dim=1)  # noqa: E731
    return pad(cond), pad(uncond), lc, lu


def cfg_unet(sd, unet_cfg, len_c: int, len_u: int, y=None):
    """the UNet callable the oracle samplers take (x, t, [cond | uncond] context padded to one length), evaluated as sdwui
    does by default: one call when len_c == len_u, otherwise cond and uncond as separate calls on their own lengths.
    y: SDXL vector conditioning [cond | uncond]."""
    def unet(x, t, c):
        if len_c == len_u:
            return O.unet_forward(sd, unet_cfg, x, t, c[:, :len_c], y=y)
        b = x.shape[0] // 2
        yc, yu = (None, None) if y is None else (y[:b], y[b:])
        return torch.cat([O.unet_forward(sd, unet_cfg, x[:b], t[:b], c[:b, :len_c], y=yc),
                          O.unet_forward(sd, unet_cfg, x[b:], t[b:], c[b:, :len_u], y=yu)])
    return unet


def sample(sd, unet_cfg, cond, uncond, sampler: str, steps: int, cfg_scale: float, noise0, draws=None, y=None, init=None,
           denoising_strength=None):
    """one sampling run (txt2img from noise0, or the img2img half from `init`) with sdwui's cond / uncond evaluation;
    returns the final latents"""
    cond, uncond, lc, lu = pad_pair(cond, uncond)
    unet = cfg_unet(sd, unet_cfg, lc, lu, y)
    if sampler != "DDIM":
        return O.run_sampler(sampler, unet, cond, uncond, cfg_scale, steps, noise0, draws, init, denoising_strength)
    if init is None:
        return O.sample_ddim(unet, noise0, cond, uncond, steps, cfg_scale)
    sa, s1a, rows = O.ddim_img2img_coefficients(steps, denoising_strength)
    x = init * sa + noise0 * s1a
    for (t, c_sa, c_s1a, c_sap, c_s1ap) in rows:
        e = O.cfg_eps(unet, x, t, cond, uncond, cfg_scale)
        x = c_sap * ((x - c_s1a * e) / c_sa) + c_s1ap * e
    return x
