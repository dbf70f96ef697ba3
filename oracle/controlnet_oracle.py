"""fp32 oracle of ControlNet as sd-webui-controlnet drives an ldm ControlNet in Balanced mode, built from the unchanged
sd_oracle functions (_run_block, _Prefixed, timestep_embedding).

  * the hint is image / 255 (RGB, NCHW, at the generation size); input_hint_block: 8 convs 3x3, SiLU between them
  * the ControlNet is the UNet's encoder + middle block under `control_model.`, evaluated on the same x, t and context;
    the hint block's output is added to its input block 0 output; output i = weight * zero_conv_i(h_i), the last one
    middle_block_out(middle result)
  * the controlled UNet adds output i to skip i when the decoder consumes it and the last one to the middle-block
    result; several units add up
  * a unit is active at sampler step i of n when guidance_start <= i / n <= guidance_end (run_sampler)
"""

import torch
import torch.nn.functional as F

from oracle import sd_oracle as O
from oracle import v_oracle as V

CONTROL_PREFIX = "control_model."
UNET_PREFIX = "model.diffusion_model."
HINT_STRIDES = (1, 1, 2, 1, 2, 1, 2, 1)   # ldm ControlNet.input_hint_block convs 0, 2, ..., 14


def hint_input(hint_u8: torch.Tensor) -> torch.Tensor:
    """uint8 [N, H, W, 3] -> float [N, 3, H, W] in [0, 1]"""
    return hint_u8.permute(0, 3, 1, 2).float() / 255.0


def _emb(sdp, cfg, t, dtype):
    emb = O.timestep_embedding(t, cfg.model_channels).to(dtype)
    emb = F.linear(emb, sdp["time_embed.0.weight"], sdp["time_embed.0.bias"])
    return F.linear(F.silu(emb), sdp["time_embed.2.weight"], sdp["time_embed.2.bias"])


def input_hint_block(csd, hint: torch.Tensor, prefix: str = CONTROL_PREFIX) -> torch.Tensor:
    sdp = O._Prefixed(csd, prefix)
    h = hint
    for j, stride in enumerate(HINT_STRIDES):
        h = F.conv2d(h, sdp[f"input_hint_block.{2 * j}.weight"], sdp[f"input_hint_block.{2 * j}.bias"], stride=stride,
                     padding=1)
        if j + 1 < len(HINT_STRIDES):
            h = F.silu(h)
    return h


def controlnet_forward(csd, cfg, x, hint, t, context, prefix: str = CONTROL_PREFIX, features: bool = False):
    """ldm ControlNet.forward -> [zero_conv_i(h_i) for every input block] + [middle_block_out(h_mid)] (features: the h_i
    and h_mid before their zero convs).  hint [1 or N, 3, H, W]."""
    sdp = O._Prefixed(csd, prefix)
    inputs, middle, _ = O.unet_layout(cfg)
    emb = _emb(sdp, cfg, t, x.dtype)
    guided = input_hint_block(csd, hint, prefix)
    h, outs, feats = x, [], []
    for i, blk in enumerate(inputs):
        h = O._run_block(sdp, cfg, f"input_blocks.{i}", blk, h, emb, context)
        if i == 0:
            h = h + guided
        feats.append(h)
        outs.append(F.conv2d(h, sdp[f"zero_convs.{i}.0.weight"], sdp[f"zero_convs.{i}.0.bias"]))
    h = O._run_block(sdp, cfg, "middle_block", middle, h, emb, context)
    feats.append(h)
    outs.append(F.conv2d(h, sdp["middle_block_out.0.weight"], sdp["middle_block_out.0.bias"]))
    return feats if features else outs


def unet_forward(sd, cfg, x, t, context, controls=(), prefix: str = UNET_PREFIX):
    """sd_oracle.unet_forward with ControlNet units added: controls = [(controlnet state_dict, hint [1|N, 3, H, W],
    weight)].  No units: the plain UNet."""
    sdp = O._Prefixed(sd, prefix)
    inputs, middle, outputs = O.unet_layout(cfg)
    adds = None
    for csd, hint, weight in controls:
        outs = [weight * o for o in controlnet_forward(csd, cfg, x, hint, t, context)]
        adds = outs if adds is None else [a + o for a, o in zip(adds, outs)]
    emb = _emb(sdp, cfg, t, x.dtype)
    hs, h = [], x
    for i, blk in enumerate(inputs):
        h = O._run_block(sdp, cfg, f"input_blocks.{i}", blk, h, emb, context)
        hs.append(h)
    h = O._run_block(sdp, cfg, "middle_block", middle, h, emb, context)
    if adds is not None:
        h = h + adds[-1]
    for i, blk in enumerate(outputs):
        skip = hs.pop()
        if adds is not None:
            skip = skip + adds[len(hs)]
        h = torch.cat([h, skip], dim=1)
        h = O._run_block(sdp, cfg, f"output_blocks.{i}", blk, h, emb, context)
    h = F.silu(O._gn(h, sdp, "out.0", 1e-5))
    return F.conv2d(h, sdp["out.2.weight"], sdp["out.2.bias"], padding=1)


class ControlledUNet:
    """unet(x, t, c) for the samplers: the units of `active` (indices into units) are applied.
    units = [(controlnet state_dict, hint uint8 [H, W, 3], weight, guidance_start, guidance_end)]"""

    def __init__(self, sd, cfg, units):
        self.sd, self.cfg = sd, cfg
        self.units = [(csd, hint_input(hint[None]), w, a, b) for csd, hint, w, a, b in units]
        self.active = ()

    def __call__(self, x, t, c):
        ctl = [(csd, hint, w) for k, (csd, hint, w, _, _) in enumerate(self.units) if k in self.active]
        return unet_forward(self.sd, self.cfg, x, t, c, ctl)


def _evals_per_step(name: str, steps: int, denoising_strength=None):
    """UNet evaluations of every sampler step as sdwui's samplers make them"""
    base = name[:-len(" Karras")] if name.endswith(" Karras") else name
    if base in ("DDIM", "PLMS"):
        ts = O.ddim_timesteps(steps)
        n = len(ts) - 1 if denoising_strength is None else \
            max(1, min(int(min(denoising_strength, 0.999) * steps), len(ts) - 1)) - 1
        return [2] + [1] * (n - 1) if base == "PLMS" and n else [1] * n
    karras = name.endswith(" Karras") or name == "DPM++ 2M"
    sig, _ = O.sigmas_karras(steps) if karras else O.karras_sigmas_compvis(steps)
    if denoising_strength is not None:
        sig = O.kdiff_img2img_sigmas(sig, steps, denoising_strength)
    n = len(sig) - 1
    if base in ("Heun", "DPM2", "DPM2 a", "DPM++ 2S a", "DPM++ SDE"):   # a second evaluation except on the step to 0
        return [2] * (n - 1) + [1]
    if base in ("Euler", "Euler a", "DPM++ 2M", "LMS"):
        return [1] * n
    raise ValueError(f"{name}: no ControlNet window rule in the oracle")


def run_sampler(name: str, unet: ControlledUNet, cond, uncond, cfg_scale: float, steps: int, noise0, draws=None,
                init=None, denoising_strength=None, mask=None, prediction: str = "eps"):
    """sd_oracle.run_sampler (v_oracle.run_sampler for prediction "v"; both with "DDIM") with the units of `unet` switched
    by their guidance windows: evaluation k belongs to sampler step i (the samplers' own evaluation counts per step) of n,
    and a unit is active there when guidance_start <= i / n <= guidance_end."""
    per = _evals_per_step(name, steps, denoising_strength)
    owner = [i for i, k in enumerate(per) for _ in range(k)]
    n = len(per)
    calls = [0]

    def counted(x, t, c):
        i = owner[min(calls[0], len(owner) - 1)]
        calls[0] += 1
        unet.active = tuple(k for k, (_, _, _, a, b) in enumerate(unet.units) if a <= i / n <= b)
        return unet(x, t, c)

    if prediction == "v" or name == "DDIM":
        if prediction == "v":
            out = V.run_sampler(name, counted, cond, uncond, cfg_scale, steps, noise0, draws, init, denoising_strength,
                                mask)
        else:   # eps DDIM: sd_oracle's rows, the img2img half and the mask blend before every call
            if init is None:
                rows, x = O.ddim_coefficients(steps), noise0
            else:
                sa, s1a, rows = O.ddim_img2img_coefficients(steps, denoising_strength)
                x = init * sa + noise0 * s1a
            for (t, c_sa, c_s1a, c_sap, c_s1ap) in rows:
                if mask is not None:
                    x = x * mask[1] + mask[0] * (1 - mask[1])
                e = O.cfg_eps(counted, x, t, cond, uncond, cfg_scale)
                x = c_sap * ((x - c_s1a * e) / c_sa) + c_s1ap * e
            out = x
    else:
        out = O.run_sampler(name, counted, cond, uncond, cfg_scale, steps, noise0, draws, init, denoising_strength, mask)
    assert calls[0] == len(owner), (name, calls[0], len(owner))
    return out
