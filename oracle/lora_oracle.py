"""Oracle: sdwui's LoRA extension (extensions-builtin/Lora) restated on an fp32 ldm state dict.

  * parse_prompt: extra_networks.parse_prompt (re.sub of `<(\\w+):([^>]+)>`, ExtraNetworkParams) and
    ExtraNetworkLora.activate's te / unet / dyn rules.
  * network_layer_mapping + convert_diffusers_name_to_compvis with sdwui's own block arithmetic (SD1.5 topology:
    `1 + i * 3 + j`), networks.load_network's lookup order.
  * merge: NetworkModuleLora.calc_updown (rebuild_conventional, alpha / rank, te multiplier for text modules), added to
    the weights; OpenCLIP's MultiheadAttention takes q / k / v stacked into in_proj_weight and out_proj only when a
    network has all four (network_apply_weights).

The existing samplers (sd_oracle, prompt_oracle, the SDXL / v oracles) then run on the merged state dict unchanged.
"""
import re
from collections import defaultdict

import torch

re_extra_net = re.compile(r"<(\w+):([^>]+)>")
re_digits = re.compile(r"\d+")
re_x_proj = re.compile(r"(.*)_([qkv]_proj)$")

suffix_conversion = {
    "attentions": {},
    "resnets": {"conv1": "in_layers_2", "conv2": "out_layers_3", "norm1": "in_layers_0", "norm2": "out_layers_0",
                "time_emb_proj": "emb_layers_1", "conv_shortcut": "skip_connection"},
}


def parse_prompt(prompt):
    """-> (prompt without tags, {type: [items lists]})"""
    res = defaultdict(list)

    def found(m):
        res[m.group(1)].append(m.group(2).split(":"))
        return ""

    return re.sub(re_extra_net, found, prompt), res


def lora_args(items):
    """ExtraNetworkParams + ExtraNetworkLora.activate -> (name, te, unet, dyn)"""
    positional, named = [], {}
    for item in items:
        parts = item.split("=", 2)
        if len(parts) == 2:
            named[parts[0]] = parts[1]
        else:
            positional.append(item)
    te = float(positional[1]) if len(positional) > 1 else 1.0
    te = float(named.get("te", te))
    unet = float(positional[2]) if len(positional) > 2 else te
    unet = float(named.get("unet", unet))
    dyn = int(positional[3]) if len(positional) > 3 else None
    dyn = int(named["dyn"]) if "dyn" in named else dyn
    return positional[0], te, unet, dyn


def networks_of(prompt):
    """(prompt without tags, [(name, te, unet, dyn)] of its lora and lyco tags in sdwui's order: lora tags first)"""
    text, res = parse_prompt(prompt)
    return text, [lora_args(items) for kind in ("lora", "lyco") for items in res.get(kind, [])]


def convert_diffusers_name_to_compvis(key, is_sd2):
    def match(match_list, regex_text):
        r = re.match(regex_text, key)
        if not r:
            return False
        match_list.clear()
        match_list.extend([int(x) if re.match(re_digits, x) else x for x in r.groups()])
        return True

    m = []
    if match(m, r"lora_unet_conv_in(.*)"):
        return f"diffusion_model_input_blocks_0_0{m[0]}"
    if match(m, r"lora_unet_conv_out(.*)"):
        return f"diffusion_model_out_2{m[0]}"
    if match(m, r"lora_unet_time_embedding_linear_(\d+)(.*)"):
        return f"diffusion_model_time_embed_{m[0] * 2 - 2}{m[1]}"
    if match(m, r"lora_unet_down_blocks_(\d+)_(attentions|resnets)_(\d+)_(.+)"):
        suffix = suffix_conversion.get(m[1], {}).get(m[3], m[3])
        return f"diffusion_model_input_blocks_{1 + m[0] * 3 + m[2]}_{1 if m[1] == 'attentions' else 0}_{suffix}"
    if match(m, r"lora_unet_mid_block_(attentions|resnets)_(\d+)_(.+)"):
        suffix = suffix_conversion.get(m[0], {}).get(m[2], m[2])
        return f"diffusion_model_middle_block_{1 if m[0] == 'attentions' else m[1] * 2}_{suffix}"
    if match(m, r"lora_unet_up_blocks_(\d+)_(attentions|resnets)_(\d+)_(.+)"):
        suffix = suffix_conversion.get(m[1], {}).get(m[3], m[3])
        return f"diffusion_model_output_blocks_{m[0] * 3 + m[2]}_{1 if m[1] == 'attentions' else 0}_{suffix}"
    if match(m, r"lora_unet_down_blocks_(\d+)_downsamplers_0_conv"):
        return f"diffusion_model_input_blocks_{3 + m[0] * 3}_0_op"
    if match(m, r"lora_unet_up_blocks_(\d+)_upsamplers_0_conv"):
        return f"diffusion_model_output_blocks_{2 + m[0] * 3}_{2 if m[0] > 0 else 1}_conv"
    if match(m, r"lora_te_text_model_encoder_layers_(\d+)_(.+)"):
        if is_sd2:
            if "mlp_fc1" in m[1]:
                return f"model_transformer_resblocks_{m[0]}_{m[1].replace('mlp_fc1', 'mlp_c_fc')}"
            elif "mlp_fc2" in m[1]:
                return f"model_transformer_resblocks_{m[0]}_{m[1].replace('mlp_fc2', 'mlp_c_proj')}"
            else:
                return f"model_transformer_resblocks_{m[0]}_{m[1].replace('self_attn', 'attn')}"
        return f"transformer_text_model_encoder_layers_{m[0]}_{m[1]}"
    if match(m, r"lora_te2_text_model_encoder_layers_(\d+)_(.+)"):
        if "mlp_fc1" in m[1]:
            return f"1_model_transformer_resblocks_{m[0]}_{m[1].replace('mlp_fc1', 'mlp_c_fc')}"
        elif "mlp_fc2" in m[1]:
            return f"1_model_transformer_resblocks_{m[0]}_{m[1].replace('mlp_fc2', 'mlp_c_proj')}"
        else:
            return f"1_model_transformer_resblocks_{m[0]}_{m[1].replace('self_attn', 'attn')}"
    return key


def layer_mapping(sd):
    """network_layer_mapping of an ldm state dict: module name (top-level prefix cut, dots -> underscores) -> ldm weight
    key of every weight module (Linear / Conv2d `.weight`, MultiheadAttention `.in_proj_weight`)"""
    xl = any(k.startswith("conditioner.") for k in sd)
    out = {}
    for k, v in sd.items():
        if k.endswith(".in_proj_weight"):
            module = k[:-len(".in_proj_weight")]
        elif k.endswith(".weight") and v.dim() >= 2 and "embedding" not in k:
            module = k[:-len(".weight")]
        else:
            continue
        for cut in ("model.", "cond_stage_model.", "conditioner.embedders."):
            if module.startswith(cut) and (cut != "model." or module.startswith("model.diffusion_model.")):
                if cut == "cond_stage_model." and xl:
                    continue
                out[module[len(cut):].replace(".", "_")] = k
                break
    return out


def match_key(mapping, key_network_without_network_parts, is_sd2):
    """networks.load_network's lookup: -> (converted key, ldm weight key or None, q/k/v block of an in_proj or None)"""
    key = convert_diffusers_name_to_compvis(key_network_without_network_parts, is_sd2)
    sd_key = mapping.get(key)
    block = None
    if sd_key is not None and sd_key.endswith(".in_proj_weight"):
        sd_key = None
    if sd_key is None:
        m = re_x_proj.match(key)
        if m and m.group(1) in mapping and mapping[m.group(1)].endswith(".in_proj_weight"):
            return key, mapping[m.group(1)], "qkv".index(m.group(2)[0])
    if sd_key is None and "lora_unet" in key_network_without_network_parts:
        key = key_network_without_network_parts.replace("lora_unet", "diffusion_model")
        sd_key = mapping.get(key)
    elif sd_key is None and "lora_te1_text_model" in key_network_without_network_parts:
        key = key_network_without_network_parts.replace("lora_te1_text_model", "0_transformer_text_model")
        sd_key = mapping.get(key)
        if sd_key is None:
            key = key_network_without_network_parts.replace("lora_te1_text_model", "transformer_text_model")
            sd_key = mapping.get(key)
    return key, sd_key, block


def merge(sd, networks):
    """networks: [(kohya state dict, te, unet, dyn)] -> a copy of the fp32 ldm state dict `sd` with every network's
    deltas added (fp64 math, fp32 result)"""
    mapping = layer_mapping(sd)
    is_sd2 = "model_transformer_resblocks_0_attn" in mapping and not any(k.startswith("conditioner.") for k in sd)
    delta = defaultdict(lambda: None)
    for lsd, te, unet, dyn in networks:
        modules = defaultdict(dict)
        for k, v in lsd.items():
            base, _, part = k.partition(".")
            modules[base][part] = v
        attn = defaultdict(dict)
        for base, w in modules.items():
            _, sd_key, block = match_key(mapping, base, is_sd2)
            if sd_key is None:
                continue
            up = w["lora_up.weight"].double()
            down = w["lora_down.weight"].double()
            rank = down.shape[0]
            up2, down2 = up.reshape(up.shape[0], -1), down.reshape(rank, -1)
            if dyn is not None:
                up2, down2 = up2[:, :dyn], down2[:dyn]
            scale = float(w["alpha"]) / rank if "alpha" in w else 1.0
            text = not sd_key.startswith("model.diffusion_model.")
            ud = (up2 @ down2) * scale * (te if text else unet)
            if block is not None or sd_key.endswith(".attn.out_proj.weight"):
                a = sd_key.rsplit(".", 1)[0] if block is not None else sd_key.rsplit(".", 2)[0]
                attn[a]["qkv"[block] if block is not None else "o"] = (sd_key, ud)
                continue
            ref = sd[sd_key]
            if ud.numel() != ref.numel():
                continue
            d = ud.reshape(ref.shape)
            delta[sd_key] = d if delta[sd_key] is None else delta[sd_key] + d
        for a, parts in attn.items():
            if set(parts) != {"q", "k", "v", "o"}:
                continue
            qkv_key = parts["q"][0]
            d = torch.vstack([parts[p][1] for p in "qkv"])
            delta[qkv_key] = d if delta[qkv_key] is None else delta[qkv_key] + d
            ok, od = parts["o"]
            delta[ok] = od if delta[ok] is None else delta[ok] + od
    out = dict(sd)
    for k, d in delta.items():
        out[k] = (sd[k].double() + d.to(sd[k].device)).to(sd[k].dtype)
    return out
