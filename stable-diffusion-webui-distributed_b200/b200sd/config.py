"""Model hyper-parameters and block topology (ldm UNetModel / kl-f8 AutoencoderKL / CLIP text tower).

Mirrors upstream ctor arguments (v1-inference.yaml); key names produced by `unet_layout` follow the ldm
state_dict so real checkpoints map 1:1.
"""
from dataclasses import dataclass
from typing import Optional, Tuple


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    model_channels: int = 320
    channel_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    attention_levels: Tuple[int, ...] = (0, 1, 2)
    num_heads: int = 8
    context_dim: int = 768
    transformer_depth: int = 1
    # SDXL (sgm UNetModel, sd_xl_base.yaml): transformer depth per level (0 = no attention there; overrides
    # attention_levels / transformer_depth), the middle block's depth, heads = channels / num_head_channels, Linear
    # proj_in / proj_out, and the vector conditioning (label_emb: Linear(adm, ted), SiLU, Linear(ted, ted), added to the
    # time embedding)
    transformer_depths: Optional[Tuple[int, ...]] = None
    middle_depth: Optional[int] = None
    num_head_channels: int = 0
    linear_proj: bool = False
    adm_in_channels: int = 0

    @property
    def time_embed_dim(self) -> int:
        return 4 * self.model_channels

    def depth(self, level: int) -> int:
        if self.transformer_depths is not None:
            return self.transformer_depths[level]
        return self.transformer_depth if level in self.attention_levels else 0

    def heads(self, channels: int) -> int:
        return channels // self.num_head_channels if self.num_head_channels else self.num_heads


@dataclass(frozen=True)
class VAEConfig:
    ch: int = 128
    ch_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 4
    out_ch: int = 3
    scale_factor: float = 0.18215


@dataclass(frozen=True)
class CLIPConfig:
    vocab: int = 49408
    width: int = 768
    layers: int = 12
    heads: int = 12
    ctx: int = 77
    # SDXL conditioner (sgm GeneralConditioner, sd_xl_base.yaml): embedder 0 = this CLIP-L tower read at hidden layer 11
    # (no final LayerNorm), embedder 1 = an OpenCLIP ViT-bigG text tower (penultimate layer + pooled/projected EOS token);
    # xl_width == 0: the SD1.x single-tower conditioner
    xl_width: int = 0
    xl_layers: int = 0
    xl_heads: int = 0
    xl_proj: int = 0          # text_projection output = pooled size (1280)
    size_embed_dim: int = 256  # ConcatTimestepEmbedderND outdim for the six size / crop scalars
    # SD 2.x (ldm FrozenOpenCLIPEmbedder, layer="penultimate"): the single tower (width / layers / heads above) is an
    # OpenCLIP text transformer under cond_stage_model.model., read as ln_final of the residual stream before its last block
    open_clip: bool = False
    # token after the first EOS of every 77-token chunk: None = EOS (CLIP); 0 for OpenCLIP (sdwui
    # FrozenOpenCLIPEmbedderWithCustomWords: id_pad = 0)
    pad_id: Optional[int] = None

    @property
    def context_dim(self) -> int:
        return self.width + self.xl_width


SD15_UNET = UNetConfig()
SD15_VAE = VAEConfig()
SD15_CLIP = CLIPConfig()
# SDXL-base (BASELINE config 4): 2.57 B parameter UNet, two text towers, vector conditioning 1280 + 6 * 256 = 2816
SDXL_UNET = UNetConfig(channel_mult=(1, 2, 4), transformer_depths=(0, 2, 10), middle_depth=10, num_head_channels=64,
                       context_dim=2048, linear_proj=True, adm_in_channels=2816)
SDXL_VAE = VAEConfig(scale_factor=0.13025)
SDXL_CLIP = CLIPConfig(xl_width=1280, xl_layers=32, xl_heads=20, xl_proj=1280)
# same topology, reduced width: fast tests (every channel count stays a multiple of 64)
TINY_UNET = UNetConfig(model_channels=64, num_heads=2, context_dim=64)
TINY_VAE = VAEConfig(ch=64, ch_mult=(1, 2), num_res_blocks=1)
TINY_CLIP = CLIPConfig(vocab=1000, width=64, layers=2, heads=2)
# SDXL topology at reduced width (d_head 64 as in SDXL: the attention kernel's unpadded-head path)
TINYXL_UNET = UNetConfig(model_channels=64, channel_mult=(1, 2, 4), transformer_depths=(0, 1, 2), middle_depth=2,
                         num_head_channels=64, context_dim=128, linear_proj=True, adm_in_channels=64 + 6 * 32)
TINYXL_VAE = VAEConfig(ch=64, ch_mult=(1, 2), num_res_blocks=1, scale_factor=0.13025)
TINYXL_CLIP = CLIPConfig(vocab=1000, width=64, layers=3, heads=2, xl_width=64, xl_layers=3, xl_heads=2, xl_proj=64,
                         size_embed_dim=32)
# SD 2.x (v2-inference-v.yaml): d_head 64, Linear proj_in / proj_out, 1024-wide OpenCLIP ViT-H/14 context; SD1's VAE
# (scale 0.18215) and noise schedule.  865 910 724 UNet parameters.  Served with v-prediction by default (768-v).
SD21_UNET = UNetConfig(num_head_channels=64, context_dim=1024, linear_proj=True)
SD21_VAE = VAEConfig()
SD21_CLIP = CLIPConfig(width=1024, layers=24, heads=16, open_clip=True, pad_id=0)
# SD 2.x topology at reduced width (d_head 64 in the UNet), for tests
TINY21_UNET = UNetConfig(model_channels=64, num_head_channels=64, context_dim=64, linear_proj=True)
TINY21_VAE = VAEConfig(ch=64, ch_mult=(1, 2), num_res_blocks=1)
TINY21_CLIP = CLIPConfig(vocab=1000, width=64, layers=3, heads=2, open_clip=True, pad_id=0)
XL_PREFIX0 = "conditioner.embedders.0.transformer.text_model."
XL_PREFIX1 = "conditioner.embedders.1.model."

UNET_PREFIX = "model.diffusion_model."
VAE_PREFIX = "first_stage_model."
CLIP_PREFIX = "cond_stage_model.transformer.text_model."
OPENCLIP_PREFIX = "cond_stage_model.model."


def unet_layout(cfg: UNetConfig):
    """(input_blocks, middle_block, output_blocks); a block is a list of layer tuples:
    ('conv_in', cin, cout) | ('res', cin, cout) | ('attn', c, depth) | ('down', c) | ('up', c)."""
    mc = cfg.model_channels
    inputs = [[("conv_in", cfg.in_channels, mc)]]
    skip_ch = [mc]
    ch = mc
    last = len(cfg.channel_mult) - 1
    for level, mult in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            layers = [("res", ch, mult * mc)]
            ch = mult * mc
            if cfg.depth(level):
                layers.append(("attn", ch, cfg.depth(level)))
            inputs.append(layers)
            skip_ch.append(ch)
        if level != last:
            inputs.append([("down", ch)])
            skip_ch.append(ch)
    mid_depth = cfg.middle_depth if cfg.middle_depth is not None else cfg.transformer_depth
    middle = [("res", ch, ch), ("attn", ch, mid_depth), ("res", ch, ch)]
    outputs = []
    for level in range(last, -1, -1):
        mult = cfg.channel_mult[level]
        for i in range(cfg.num_res_blocks + 1):
            layers = [("res", ch + skip_ch.pop(), mult * mc)]
            ch = mult * mc
            if cfg.depth(level):
                layers.append(("attn", ch, cfg.depth(level)))
            if level > 0 and i == cfg.num_res_blocks:
                layers.append(("up", ch))
            outputs.append(layers)
    return inputs, middle, outputs
