"""Seeded synthetic weights with the exact SD1.5 / SDXL / SD 2.x parameter shapes and state_dict key names.

No checkpoint exists offline (SURVEY.md §8d): benchmarks, smoke and parity tests run on these.  Initialisation is
variance preserving (N(0, 1/fan_in)) so 20 sampler steps stay numerically sane in fp16, and nothing is zero-initialised
(ldm zero-inits proj_out / out convs) so every kernel does real work.
"""
import math
from typing import Dict

import torch

from .config import (CLIP_PREFIX, CONTROL_PREFIX, OPENCLIP_PREFIX, UNET_PREFIX, VAE_PREFIX, XL_PREFIX0, XL_PREFIX1,
                     CLIPConfig, UNetConfig, VAEConfig, controlnet_layout, unet_layout)


class _Init:
    def __init__(self, seed: int):
        self.g = torch.Generator(device="cpu").manual_seed(seed)
        self.sd: Dict[str, torch.Tensor] = {}

    def w(self, key, shape, gain=1.0):
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        self.sd[key] = torch.randn(shape, generator=self.g) * (gain / math.sqrt(fan_in))

    def b(self, key, n, std=0.05):
        self.sd[key] = torch.randn(n, generator=self.g) * std

    def norm(self, key, n):
        self.sd[key + ".weight"] = 1.0 + 0.05 * torch.randn(n, generator=self.g)
        self.sd[key + ".bias"] = 0.05 * torch.randn(n, generator=self.g)

    def conv(self, key, cout, cin, k, gain=1.0):
        self.w(key + ".weight", (cout, cin, k, k), gain)
        self.b(key + ".bias", cout)

    def lin(self, key, cout, cin, bias=True, gain=1.0):
        self.w(key + ".weight", (cout, cin), gain)
        if bias:
            self.b(key + ".bias", cout)


def _unet(i: _Init, cfg: UNetConfig, p: str = UNET_PREFIX, encoder_only: bool = False):
    ted = cfg.time_embed_dim
    i.lin(p + "time_embed.0", ted, cfg.model_channels)
    i.lin(p + "time_embed.2", ted, ted)
    if cfg.adm_in_channels:
        i.lin(p + "label_emb.0.0", ted, cfg.adm_in_channels)
        i.lin(p + "label_emb.0.2", ted, ted)

    def res(key, cin, cout):
        i.norm(key + ".in_layers.0", cin)
        i.conv(key + ".in_layers.2", cout, cin, 3)
        i.lin(key + ".emb_layers.1", cout, ted)
        i.norm(key + ".out_layers.0", cout)
        i.conv(key + ".out_layers.3", cout, cout, 3)
        if cin != cout:
            i.conv(key + ".skip_connection", cout, cin, 1)

    def attn(key, c, depth):
        i.norm(key + ".norm", c)
        if cfg.linear_proj:
            i.lin(key + ".proj_in", c, c)
        else:
            i.conv(key + ".proj_in", c, c, 1)
        for d in range(depth):
            t = f"{key}.transformer_blocks.{d}"
            for n in ("norm1", "norm2", "norm3"):
                i.norm(f"{t}.{n}", c)
            for a, ctx in (("attn1", c), ("attn2", cfg.context_dim)):
                i.lin(f"{t}.{a}.to_q", c, c, bias=False)
                i.lin(f"{t}.{a}.to_k", c, ctx, bias=False)
                i.lin(f"{t}.{a}.to_v", c, ctx, bias=False)
                i.lin(f"{t}.{a}.to_out.0", c, c)
            i.lin(f"{t}.ff.net.0.proj", 8 * c, c)
            i.lin(f"{t}.ff.net.2", c, 4 * c)
        if cfg.linear_proj:
            i.lin(key + ".proj_out", c, c)
        else:
            i.conv(key + ".proj_out", c, c, 1)

    def block(prefix, layers):
        for j, layer in enumerate(layers):
            key = f"{p}{prefix}.{j}"
            if layer[0] == "conv_in":
                i.conv(key, layer[2], layer[1], 3)
            elif layer[0] == "res":
                res(key, layer[1], layer[2])
            elif layer[0] == "attn":
                attn(key, layer[1], layer[2])
            elif layer[0] == "down":
                i.conv(key + ".op", layer[1], layer[1], 3)
            elif layer[0] == "up":
                i.conv(key + ".conv", layer[1], layer[1], 3)

    inputs, middle, outputs = unet_layout(cfg)
    for n, layers in enumerate(inputs):
        block(f"input_blocks.{n}", layers)
    block("middle_block", middle)
    if encoder_only:
        return
    for n, layers in enumerate(outputs):
        block(f"output_blocks.{n}", layers)
    i.norm(p + "out.0", cfg.model_channels)
    i.conv(p + "out.2", cfg.out_channels, cfg.model_channels, 3)


def make_controlnet_state_dict(unet: UNetConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """An ldm ControlNet for a UNet of config `unet`, with the key names of ControlNet checkpoints (control_model.*):
    time_embed, the UNet's input_blocks and middle_block, input_hint_block.{0,2,..,14}, zero_convs.i.0 and
    middle_block_out.0.  Zero convs are initialised like any other layer (ldm zero-inits them), so a synthetic unit
    changes the image."""
    i = _Init(seed)
    p = CONTROL_PREFIX
    _unet(i, unet, p, encoder_only=True)
    _, _, hint, zero_ch = controlnet_layout(unet)
    for j, (cin, cout, _) in enumerate(hint):
        i.conv(f"{p}input_hint_block.{2 * j}", cout, cin, 3)
    for j, c in enumerate(zero_ch):
        i.conv(f"{p}zero_convs.{j}.0", c, c, 1)
    mid = zero_ch[-1]
    i.conv(p + "middle_block_out.0", mid, mid, 1)
    return i.sd


def _vae(i: _Init, cfg: VAEConfig):
    p = VAE_PREFIX

    def res(key, cin, cout):
        i.norm(key + ".norm1", cin)
        i.conv(key + ".conv1", cout, cin, 3)
        i.norm(key + ".norm2", cout)
        i.conv(key + ".conv2", cout, cout, 3)
        if cin != cout:
            i.conv(key + ".nin_shortcut", cout, cin, 1)

    def attn(key, c):
        i.norm(key + ".norm", c)
        for n in ("q", "k", "v", "proj_out"):
            i.conv(f"{key}.{n}", c, c, 1)

    nlev = len(cfg.ch_mult)
    # encoder
    i.conv(p + "encoder.conv_in", cfg.ch, 3, 3)
    cin = cfg.ch
    for lvl in range(nlev):
        cout = cfg.ch * cfg.ch_mult[lvl]
        for b in range(cfg.num_res_blocks):
            res(f"{p}encoder.down.{lvl}.block.{b}", cin, cout)
            cin = cout
        if lvl != nlev - 1:
            i.conv(f"{p}encoder.down.{lvl}.downsample.conv", cin, cin, 3)
    res(p + "encoder.mid.block_1", cin, cin)
    attn(p + "encoder.mid.attn_1", cin)
    res(p + "encoder.mid.block_2", cin, cin)
    i.norm(p + "encoder.norm_out", cin)
    i.conv(p + "encoder.conv_out", 2 * cfg.z_channels, cin, 3)
    i.conv(p + "quant_conv", 2 * cfg.z_channels, 2 * cfg.z_channels, 1)
    # decoder
    i.conv(p + "post_quant_conv", cfg.z_channels, cfg.z_channels, 1)
    cin = cfg.ch * cfg.ch_mult[-1]
    i.conv(p + "decoder.conv_in", cin, cfg.z_channels, 3)
    res(p + "decoder.mid.block_1", cin, cin)
    attn(p + "decoder.mid.attn_1", cin)
    res(p + "decoder.mid.block_2", cin, cin)
    for lvl in reversed(range(nlev)):
        cout = cfg.ch * cfg.ch_mult[lvl]
        for b in range(cfg.num_res_blocks + 1):
            res(f"{p}decoder.up.{lvl}.block.{b}", cin, cout)
            cin = cout
        if lvl != 0:
            i.conv(f"{p}decoder.up.{lvl}.upsample.conv", cin, cin, 3)
    i.norm(p + "decoder.norm_out", cin)
    i.conv(p + "decoder.conv_out", cfg.out_ch, cin, 3, gain=0.7)  # keeps most pixels inside (-1, 1)


def _open_clip(i: _Init, cfg: CLIPConfig, p: str):
    """OpenCLIP text tower key names (sgm FrozenOpenCLIPEmbedder2.model for SDXL's second tower; ldm
    FrozenOpenCLIPEmbedder.model for SD 2.x, whose checkpoints also keep logit_scale)"""
    w, layers, proj = (cfg.xl_width, cfg.xl_layers, cfg.xl_proj) if cfg.xl_width else (cfg.width, cfg.layers, cfg.width)
    i.sd[p + "token_embedding.weight"] = 0.02 * torch.randn((cfg.vocab, w), generator=i.g)
    i.sd[p + "positional_embedding"] = 0.01 * torch.randn((cfg.ctx, w), generator=i.g)
    for l in range(layers):
        k = f"{p}transformer.resblocks.{l}"
        i.norm(k + ".ln_1", w)
        i.w(k + ".attn.in_proj_weight", (3 * w, w))
        i.b(k + ".attn.in_proj_bias", 3 * w)
        i.lin(k + ".attn.out_proj", w, w)
        i.norm(k + ".ln_2", w)
        i.lin(k + ".mlp.c_fc", 4 * w, w)
        i.lin(k + ".mlp.c_proj", w, 4 * w)
    i.norm(p + "ln_final", w)
    i.sd[p + "text_projection"] = torch.randn((w, proj), generator=i.g) / math.sqrt(w)
    if not cfg.xl_width:
        i.sd[p + "logit_scale"] = torch.tensor(math.log(1 / 0.07))


def _clip(i: _Init, cfg: CLIPConfig, p: str = CLIP_PREFIX):
    i.sd[p + "embeddings.token_embedding.weight"] = 0.02 * torch.randn((cfg.vocab, cfg.width), generator=i.g)
    i.sd[p + "embeddings.position_embedding.weight"] = 0.01 * torch.randn((cfg.ctx, cfg.width), generator=i.g)
    for l in range(cfg.layers):
        k = f"{p}encoder.layers.{l}"
        i.norm(k + ".layer_norm1", cfg.width)
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            i.lin(f"{k}.self_attn.{n}", cfg.width, cfg.width)
        i.norm(k + ".layer_norm2", cfg.width)
        i.lin(k + ".mlp.fc1", 4 * cfg.width, cfg.width)
        i.lin(k + ".mlp.fc2", cfg.width, 4 * cfg.width)
    i.norm(p + "final_layer_norm", cfg.width)


def make_state_dict(unet: UNetConfig, vae: VAEConfig, clip: CLIPConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """fp32 CPU tensors, deterministic in (configs, seed)."""
    i = _Init(seed)
    _unet(i, unet)
    _vae(i, vae)
    if clip.xl_width:      # SDXL: sgm conditioner key names, two towers
        _clip(i, clip, XL_PREFIX0)
        _open_clip(i, clip, XL_PREFIX1)
    elif getattr(clip, "open_clip", False):   # SD 2.x: one OpenCLIP tower (oracle configs lack the field)
        _open_clip(i, clip, OPENCLIP_PREFIX)
    else:
        _clip(i, clip)
    return i.sd


def _lora_unet_modules(cfg: UNetConfig):
    """(ldm module path, kind, out, in) of every UNet layer a kohya LoRA trains: kind "conv3" (LoCon 3x3), "conv1"
    (1x1 conv) or "linear"
    """
    ted = cfg.time_embed_dim
    mods = [("time_embed.0", "linear", ted, cfg.model_channels), ("time_embed.2", "linear", ted, ted)]
    if cfg.adm_in_channels:
        mods += [("label_emb.0.0", "linear", ted, cfg.adm_in_channels), ("label_emb.0.2", "linear", ted, ted)]
    proj = "linear" if cfg.linear_proj else "conv1"
    inputs, middle, outputs = unet_layout(cfg)
    for prefix, blocks in [("input_blocks", inputs), ("middle_block", [middle]), ("output_blocks", outputs)]:
        for n, layers in enumerate(blocks):
            for j, layer in enumerate(layers):
                key = f"{prefix}.{n}.{j}" if prefix != "middle_block" else f"middle_block.{j}"
                if layer[0] == "conv_in":
                    mods.append((key, "conv3", layer[2], layer[1]))
                elif layer[0] == "res":
                    cin, cout = layer[1], layer[2]
                    mods += [(key + ".in_layers.2", "conv3", cout, cin), (key + ".out_layers.3", "conv3", cout, cout),
                             (key + ".emb_layers.1", "linear", cout, ted)]
                    if cin != cout:
                        mods.append((key + ".skip_connection", "conv1", cout, cin))
                elif layer[0] == "attn":
                    c = layer[1]
                    mods += [(key + ".proj_in", proj, c, c), (key + ".proj_out", proj, c, c)]
                    for d in range(layer[2]):
                        t = f"{key}.transformer_blocks.{d}"
                        for a, ctx in (("attn1", c), ("attn2", cfg.context_dim)):
                            mods += [(f"{t}.{a}.to_q", "linear", c, c), (f"{t}.{a}.to_k", "linear", c, ctx),
                                     (f"{t}.{a}.to_v", "linear", c, ctx), (f"{t}.{a}.to_out.0", "linear", c, c)]
                        mods += [(f"{t}.ff.net.0.proj", "linear", 8 * c, c), (f"{t}.ff.net.2", "linear", c, 4 * c)]
                elif layer[0] == "down":
                    mods.append((key + ".op", "conv3", layer[1], layer[1]))
                elif layer[0] == "up":
                    mods.append((key + ".conv", "conv3", layer[1], layer[1]))
    mods.append(("out.2", "conv3", cfg.out_channels, cfg.model_channels))
    return mods


def _diffusers_name(path: str, blocks: Dict[str, str]) -> str:
    """kohya's diffusers-form module name of an ldm UNet module path (inverse of lora.to_compvis)"""
    flat = path.replace(".", "_")
    if flat == "input_blocks_0_0":
        return "lora_unet_conv_in"
    if flat == "out_2":
        return "lora_unet_conv_out"
    if flat.startswith("time_embed_"):
        return f"lora_unet_time_embedding_linear_{int(flat[len('time_embed_'):]) // 2 + 1}"
    inverse = {"in_layers_2": "conv1", "out_layers_3": "conv2", "emb_layers_1": "time_emb_proj",
               "skip_connection": "conv_shortcut"}
    for diff, ldm in sorted(blocks.items(), key=lambda kv: -len(kv[1])):
        if flat.startswith(ldm + "_"):
            suffix = flat[len(ldm) + 1:]
            if "_resnets_" in diff:
                suffix = inverse.get(suffix, suffix)
            elif "_downsamplers_" in diff and suffix == "op":
                suffix = "conv"
            return f"lora_unet_{diff}_{suffix}"
    return "lora_unet_" + flat   # no diffusers name (SDXL's label_emb): the compvis form


def make_lora_state_dict(unet: UNetConfig, clip: CLIPConfig, seed: int = 0, rank: int = 8, form: str = "diffusers",
                         unet_modules: bool = True, te_modules: bool = True) -> Dict[str, torch.Tensor]:
    """A seeded kohya-format LoRA (LoCon) for the model of (unet, clip): `<module>.lora_down.weight`,
    `.lora_up.weight`, `.alpha` (rank / 2) for every UNet linear / conv layer (3x3 convs as LoCon: down [r, Cin, 3, 3],
    up [Cout, r, 1, 1]) and every text-tower attention / MLP linear, under kohya's names: `lora_unet_` in the diffusers
    form (`down_blocks_0_resnets_1_conv1`, ...) or the compvis form (`input_blocks_1_0_in_layers_2`, ...; SDXL files use
    it), `lora_te_` (SD1.x, SD 2.x), `lora_te1_` / `lora_te2_` (SDXL) with HF CLIP layer names.  Each delta is about 15 %
    of its weight at multiplier 1."""
    from .lora import diffusers_blocks
    if form not in ("diffusers", "compvis"):
        raise ValueError(form)
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def add(name, kind, cout, cin):
        k = 3 if kind == "conv3" else 1
        conv = kind != "linear"
        down = torch.randn((rank, cin * k * k), generator=g) / math.sqrt(cin * k * k)
        up = torch.randn((cout, rank), generator=g) * (0.3 / math.sqrt(rank))
        sd[name + ".lora_down.weight"] = down.reshape(rank, cin, k, k) if conv else down
        sd[name + ".lora_up.weight"] = up.reshape(cout, rank, 1, 1) if conv else up
        sd[name + ".alpha"] = torch.tensor(rank / 2.0)

    if unet_modules:
        blocks = diffusers_blocks(unet)
        for path, kind, cout, cin in _lora_unet_modules(unet):
            add(_diffusers_name(path, blocks) if form == "diffusers" else "lora_unet_" + path.replace(".", "_"),
                kind, cout, cin)
    if te_modules:
        towers = [("lora_te1_", clip.width, clip.layers), ("lora_te2_", clip.xl_width, clip.xl_layers)] if clip.xl_width \
            else [("lora_te_", clip.width, clip.layers)]
        for prefix, w, layers in towers:
            for l in range(layers):
                p = f"{prefix}text_model_encoder_layers_{l}_"
                for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
                    add(p + "self_attn_" + n, "linear", w, w)
                add(p + "mlp_fc1", "linear", 4 * w, w)
                add(p + "mlp_fc2", "linear", w, 4 * w)
    return sd
