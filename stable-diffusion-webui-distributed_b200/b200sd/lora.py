"""LoRA networks named in prompts (sdwui's built-in Lora extension: extra_networks.parse_prompt, networks.load_network,
network_lora.NetworkModuleLora), merged into the engine's packed weights on the GPU.

  * parse_prompt: every `<type:arg:arg...>` tag is cut out of the prompt (re.sub, nothing else trimmed); `lora` and its
    alias `lyco` take name, te multiplier (positional 1 or te=, default 1), unet multiplier (positional 2 or unet=,
    default te) and dyn dim (positional 3 or dyn=: the first dyn ranks only).  Other tag types are dropped with a warning.
  * LoraFile: a kohya-format state dict (`<module>.lora_up.weight`, `.lora_down.weight`, `.alpha`).  Network types sdwui
    would apply but this executor does not serve (LoHa, LoKr, IA3, OFT, DoRA, CP / lora_mid, full diff, diffusers / PEFT
    lora_A / lora_B) are refused with ValueError when the file is read, before any weight changes.
  * Module names: sdwui's network_layer_mapping (every weight module of the model, dots -> underscores) and
    convert_diffusers_name_to_compvis, with the diffusers block indices derived from config.unet_layout.
  * plan: per packed tensor, the networks' factors scaled (alpha / rank x multiplier, folded into up), scattered
    through the packers' Placements (weights.py) and concatenated along the rank; ops.lora_merge applies them.
"""
import logging
import re
from collections import defaultdict
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from .config import UNetConfig, unet_layout

log = logging.getLogger("distributed")

_TAG = re.compile(r"<(\w+):([^>]+)>")      # sdwui extra_networks.re_extra_net
LORA_TYPES = ("lora", "lyco")
SERVED_PARTS = ("lora_up.weight", "lora_down.weight", "alpha")
# network-part markers of the module types sdwui applies and this executor refuses
REFUSED = (("hada_", "LoHa"), ("lokr_", "LoKr"), ("on_input", "IA3"), ("oft_", "OFT"), ("dora_scale", "DoRA"),
           ("lora_mid", "LoRA with a mid (CP / Tucker) factor"), ("diff", "full-weight diff"),
           ("lora_A", "diffusers / PEFT LoRA"), ("lora_B", "diffusers / PEFT LoRA"),
           ("lora.up", "diffusers LoRA"), ("lora.down", "diffusers LoRA"), ("lora_linear_layer", "diffusers LoRA"))


# ------------------------------------------------------------------------------------------------ prompt tags
@dataclass(frozen=True)
class LoraRef:
    """one `<lora:...>` tag: file name and sdwui's te / unet multipliers and dyn dim"""
    name: str
    te: float = 1.0
    unet: float = 1.0
    dyn: Optional[int] = None


def parse_prompt(text: str) -> Tuple[str, List[LoraRef]]:
    """(prompt without its tags, the lora / lyco tags in prompt order) — sdwui extra_networks.parse_prompt and
    ExtraNetworkLora.activate's argument rules.  Tags of other types are removed and ignored with a warning."""
    refs: List[LoraRef] = []
    other = []

    def found(m):
        kind, items = m.group(1), m.group(2).split(":")
        if kind not in LORA_TYPES:
            other.append(kind)
            return ""
        positional, named = [], {}
        for item in items:
            parts = item.split("=", 2)
            if len(parts) == 2:
                named[parts[0]] = parts[1]
            else:
                positional.append(item)
        if not positional:
            raise ValueError(f"extra network tag {m.group(0)!r} names no network")
        te = float(positional[1]) if len(positional) > 1 else 1.0
        te = float(named.get("te", te))
        unet = float(positional[2]) if len(positional) > 2 else te
        unet = float(named.get("unet", unet))
        dyn = int(positional[3]) if len(positional) > 3 else None
        dyn = int(named["dyn"]) if "dyn" in named else dyn
        refs.append(LoraRef(positional[0], te, unet, dyn))
        return ""

    out = _TAG.sub(found, text)
    for kind in sorted(set(other)):
        log.warning("extra network type %r is not served: its tags are removed from the prompt and ignored", kind)
    return out, refs


# ------------------------------------------------------------------------------------------------ files
@dataclass
class LoraModule:
    up: torch.Tensor                 # fp32 [out, r(, 1, 1)]
    down: torch.Tensor               # fp32 [r, in(, kh, kw)]
    alpha: Optional[float] = None


@dataclass
class LoraFile:
    """a parsed kohya LoRA file: module name (`lora_unet_...`, `lora_te_...`) -> factors; `key` identifies the file
    (name, size, mtime) in the engine's record of what is merged"""
    name: str
    modules: Dict[str, LoraModule]
    key: tuple = ()


def load_state_dict(name: str, sd: Dict[str, torch.Tensor], key: tuple = ()) -> LoraFile:
    """kohya state dict -> LoraFile; ValueError for a network type that is not served"""
    parts: Dict[str, Dict[str, torch.Tensor]] = defaultdict(dict)
    for k, v in sd.items():
        module, _, part = k.partition(".")
        for marker, what in REFUSED:
            if part.startswith(marker) or (marker in ("lora_A", "lora_B") and marker in k):
                raise ValueError(f"LoRA {name!r} holds {what} modules ({k}): only plain LoRA / LoCon networks are served")
        parts[module][part] = v
    modules = {}
    for module, p in parts.items():
        if module == "bundle_emb":
            continue
        unknown = set(p) - set(SERVED_PARTS)
        if unknown or "lora_up.weight" not in p or "lora_down.weight" not in p:
            raise ValueError(f"LoRA {name!r}: module {module} has parts {sorted(p)}: not a LoRA module this executor serves")
        alpha = p.get("alpha")
        modules[module] = LoraModule(p["lora_up.weight"].float(), p["lora_down.weight"].float(),
                                     None if alpha is None else float(alpha))
    return LoraFile(name, modules, key)


# ------------------------------------------------------------------------------------------------ module names
_RES_SUFFIX = {"conv1": "in_layers_2", "conv2": "out_layers_3", "norm1": "in_layers_0", "norm2": "out_layers_0",
               "time_emb_proj": "emb_layers_1", "conv_shortcut": "skip_connection"}


def diffusers_blocks(cfg: UNetConfig) -> Dict[str, str]:
    """diffusers UNet block prefix -> ldm block prefix (sdwui convert_diffusers_name_to_compvis), from the layout:
    `down_blocks_i_resnets_j` / `_attentions_j` -> `input_blocks_n_0` / `_1`, `down_blocks_i_downsamplers_0` ->
    `input_blocks_n_0`, `mid_block_resnets_j` / `_attentions_0`, `up_blocks_u_resnets_j` / `_attentions_j` /
    `_upsamplers_0` (up block u is level L-1-u)."""
    inputs, middle, outputs = unet_layout(cfg)
    out = {}
    n, levels = 1, len(cfg.channel_mult)
    for level in range(levels):
        for j in range(cfg.num_res_blocks):
            out[f"down_blocks_{level}_resnets_{j}"] = f"input_blocks_{n}_0"
            if len(inputs[n]) > 1:
                out[f"down_blocks_{level}_attentions_{j}"] = f"input_blocks_{n}_1"
            n += 1
        if n < len(inputs) and inputs[n][0][0] == "down":
            out[f"down_blocks_{level}_downsamplers_0"] = f"input_blocks_{n}_0"
            n += 1
    for j, layer in enumerate(middle):
        if layer[0] == "res":
            out[f"mid_block_resnets_{j // 2}"] = f"middle_block_{j}"
        else:
            out["mid_block_attentions_0"] = f"middle_block_{j}"
    n = 0
    for u in range(levels):
        for j in range(cfg.num_res_blocks + 1):
            layers = outputs[n]
            out[f"up_blocks_{u}_resnets_{j}"] = f"output_blocks_{n}_0"
            if len(layers) > 1 and layers[1][0] == "attn":
                out[f"up_blocks_{u}_attentions_{j}"] = f"output_blocks_{n}_1"
            if layers[-1][0] == "up":
                out[f"up_blocks_{u}_upsamplers_0"] = f"output_blocks_{n}_{len(layers) - 1}"
            n += 1
    return out


_DIFFUSERS = re.compile(r"lora_unet_((?:down_blocks|up_blocks)_\d+_(?:resnets|attentions|downsamplers|upsamplers)_\d+|"
                        r"mid_block_(?:resnets|attentions)_\d+)_(.+)")
_X_PROJ = re.compile(r"(.*)_([qkv]_proj)$")


def to_compvis(key: str, blocks: Dict[str, str], open_clip_te: bool) -> str:
    """sdwui convert_diffusers_name_to_compvis for a module name (blocks: diffusers_blocks of the model); a name it does
    not convert comes back unchanged"""
    if key.startswith("lora_unet_conv_in"):
        return "diffusion_model_input_blocks_0_0" + key[len("lora_unet_conv_in"):]
    if key.startswith("lora_unet_conv_out"):
        return "diffusion_model_out_2" + key[len("lora_unet_conv_out"):]
    m = re.match(r"lora_unet_time_embedding_linear_(\d+)(.*)", key)
    if m:
        return f"diffusion_model_time_embed_{int(m.group(1)) * 2 - 2}{m.group(2)}"
    m = _DIFFUSERS.match(key)
    if m and m.group(1) in blocks:
        block, suffix = m.group(1), m.group(2)
        if "_resnets_" in block:
            suffix = _RES_SUFFIX.get(suffix, suffix)
        elif "_downsamplers_" in block and suffix == "conv":
            suffix = "op"
        return f"diffusion_model_{blocks[block]}_{suffix}"

    def open_clip(prefix, rest):
        if "mlp_fc1" in rest:
            return f"{prefix}{rest.replace('mlp_fc1', 'mlp_c_fc')}"
        if "mlp_fc2" in rest:
            return f"{prefix}{rest.replace('mlp_fc2', 'mlp_c_proj')}"
        return f"{prefix}{rest.replace('self_attn', 'attn')}"

    m = re.match(r"lora_te_text_model_encoder_layers_(\d+)_(.+)", key)
    if m:
        if open_clip_te:
            return open_clip(f"model_transformer_resblocks_{m.group(1)}_", m.group(2))
        return f"transformer_text_model_encoder_layers_{m.group(1)}_{m.group(2)}"
    m = re.match(r"lora_te2_text_model_encoder_layers_(\d+)_(.+)", key)
    if m:
        return open_clip(f"1_model_transformer_resblocks_{m.group(1)}_", m.group(2))
    return key


@dataclass
class Target:
    """where a LoRA module lands: its owner ("unet", "t0", "t1"), the ldm weight key, the row block of a q / k / v
    projection inside OpenCLIP's attn.in_proj_weight (None: the whole weight) and whether the te multiplier applies"""
    owner: str
    ldm_key: str
    block: Optional[int] = None
    text: bool = False


class KeyTable:
    """sdwui's network_layer_mapping of one engine (every placed weight, module name with dots -> underscores, without
    the model's top-level prefix: `diffusion_model_...`, `transformer_text_model_...`, `model_transformer_...` (SD 2.x),
    `0_transformer_...` / `1_model_...` (SDXL)), and the lookup of LoRA module names in it"""

    def __init__(self, owners, unet_cfg: UNetConfig, open_clip_te: bool):
        """owners: [(owner name, placements {ldm key: Placement}, top-level prefix cut from module names, text?)]"""
        self.names: Dict[str, Target] = {}
        self.shapes: Dict[str, tuple] = {}
        for owner, place, cut, text in owners:
            for k in place:
                module = k[:-len(".in_proj_weight")] if k.endswith(".in_proj_weight") else k[:-len(".weight")]
                self.names[module[len(cut):].replace(".", "_")] = Target(owner, k, None, text)
                self.shapes[k] = place[k].shape
        self.blocks = diffusers_blocks(unet_cfg)
        self.open_clip_te = open_clip_te

    def find(self, module: str) -> Optional[Target]:
        """networks.load_network's lookup order for one module name"""
        key = to_compvis(module, self.blocks, self.open_clip_te)
        t = self.names.get(key)
        if t is None:
            m = _X_PROJ.match(key)
            if m and m.group(1) in self.names and self.names[m.group(1)].ldm_key.endswith(".in_proj_weight"):
                base = self.names[m.group(1)]
                return Target(base.owner, base.ldm_key, "qkv".index(m.group(2)[0]), base.text)
        if t is None and "lora_unet" in module:
            t = self.names.get(module.replace("lora_unet", "diffusion_model"))
        elif t is None and "lora_te1_text_model" in module:
            t = self.names.get(module.replace("lora_te1_text_model", "0_transformer_text_model"))
            if t is None:
                t = self.names.get(module.replace("lora_te1_text_model", "transformer_text_model"))
        if t is not None and t.ldm_key.endswith(".in_proj_weight"):
            return None   # the attention module itself takes no LoRA of its own name
        return t


def delta_factors(mod: LoraModule, dyn: Optional[int]):
    """(up [out, r'] , down [r', in_flat], scale): sdwui rebuild_conventional's factors (dyn: the first dyn ranks) and
    calc_scale (alpha / rank of the whole file module)"""
    up = mod.up.reshape(mod.up.shape[0], -1)
    down = mod.down.reshape(mod.down.shape[0], -1)
    rank = down.shape[0]
    if dyn is not None:
        up, down = up[:, :dyn], down[:dyn]
    scale = mod.alpha / rank if mod.alpha is not None else 1.0
    return up, down, scale


def resolve(table: KeyTable, nets):
    """nets: [(LoraFile, LoraRef)] -> per network [(Target, up [out, r], down [r, in], factor)] with factor = scale x
    multiplier, after sdwui's rules: unmatched modules are skipped (debug log), a module whose delta does not fit its
    weight is skipped with one warning per network, and OpenCLIP attention takes its q / k / v / out_proj modules only
    when a network has all four (network_apply_weights' MultiheadAttention case)."""
    out = []
    for f, ref in nets:
        entries, failed, bad = [], [], []
        attn: Dict[str, Dict[str, tuple]] = defaultdict(dict)
        for module, mod in f.modules.items():
            t = table.find(module)
            if t is None:
                failed.append(module)
                continue
            up, down, scale = delta_factors(mod, ref.dyn)
            shape = table.shapes[t.ldm_key]
            rows = shape[0] // 3 if t.block is not None else shape[0]
            numel = rows * (shape[1] if t.block is not None else int(torch.tensor(shape[1:]).prod()))
            if up.shape[0] != rows or up.shape[0] * down.shape[1] != numel or up.shape[1] != down.shape[0]:
                bad.append(module)
                continue
            e = (t, up, down, scale * (ref.te if t.text else ref.unet))
            open_clip_attn = t.ldm_key.endswith((".in_proj_weight", ".attn.out_proj.weight"))
            if open_clip_attn:
                base = t.ldm_key.rsplit(".", 2)[0] if t.block is None else t.ldm_key.rsplit(".", 1)[0]
                attn[base]["qkv"[t.block] if t.block is not None else "o"] = e
            else:
                entries.append(e)
        for base, parts in attn.items():
            if set(parts) == {"q", "k", "v", "o"}:
                entries.extend(parts[p] for p in "qkvo")
        if failed:
            log.debug("LoRA %s: %d keys matched no module of the model: %s", f.name, len(failed), failed[:8])
        if bad:
            log.warning("LoRA %s: %d modules do not fit the model's weights and are skipped (%s, ...)", f.name, len(bad),
                        bad[0])
        out.append(entries)
    return out


@dataclass
class Group:
    """rows [lo, hi) of one packed tensor with the ranks that touch them (U [hi - lo, R], D [R, cols]; R = 0: restore)"""
    lo: int
    hi: int
    U: Optional[torch.Tensor] = None
    D: Optional[torch.Tensor] = None


def plan(entries, placements: Dict[str, Dict[str, object]], packed: Dict[str, Dict[str, torch.Tensor]], device):
    """Per packed tensor (owner, name) touched by `entries` (resolve's output, all networks), its Groups covering every
    row: the networks' factors with the factor folded into up, scattered through the Placements — up rows to packed rows,
    down columns to packed columns — and concatenated along the rank in network order.  Factor preparation runs on
    `device` in fp32."""
    per: Dict[tuple, list] = defaultdict(list)   # (owner, tensor) -> [(packed rows, U [n, r], D [r, cols])]
    for net in entries:
        for t, up, down, factor in net:
            pl = placements[t.owner][t.ldm_key]
            w = packed[t.owner][pl.tensor]
            cols = w.shape[1]
            u = up.to(device=device, dtype=torch.float32) * factor
            d = down.to(device=device, dtype=torch.float32)
            src = torch.arange(u.shape[0])
            if t.block is not None:
                src = src + t.block * u.shape[0]
            rows = src if pl.rows is None else pl.rows[src]
            if pl.cols is not None:
                c = pl.cols.to(device)
                dp = torch.zeros((d.shape[0], cols), device=device, dtype=torch.float32)
                valid = c >= 0
                dp[:, valid] = d[:, c[valid]]
                d = dp
            assert d.shape[1] == cols, (t.ldm_key, tuple(d.shape), cols)
            per[(t.owner, pl.tensor)].append((rows, u, d))
    out: Dict[tuple, List[Group]] = {}
    for key, items in per.items():
        nrows = packed[key[0]][key[1]].shape[0]
        spans = sorted(((int(r.min()), int(r.max()) + 1, i) for i, (r, _, _) in enumerate(items)))
        groups: List[list] = []
        for lo, hi, i in spans:
            if groups and lo < groups[-1][1]:
                groups[-1][1] = max(groups[-1][1], hi)
                groups[-1][2].append(i)
            else:
                groups.append([lo, hi, [i]])
        res, at = [], 0
        for lo, hi, idx in groups:
            if lo > at:
                res.append(Group(at, lo))
            idx.sort()   # network order, then module order within a network
            rank = sum(items[i][1].shape[1] for i in idx)
            U = torch.zeros((hi - lo, rank), device=device, dtype=torch.float32)
            o = 0
            for i in idx:
                rows, u, _ = items[i]
                U[(rows - lo).to(device), o:o + u.shape[1]] = u
                o += u.shape[1]
            res.append(Group(lo, hi, U, torch.cat([items[i][2] for i in idx]).contiguous()))
            at = hi
        if at < nrows:
            res.append(Group(at, nrows))
        out[key] = res
    return out
