"""Engine construction for the local-GPU workers: one SDEngine per CUDA device, built lazily and cached.

Weights: `SD_CKPT=/path/model.safetensors` (ldm key names; read for sd15 and sd21) when present, otherwise the seeded
synthetic weights of synth.py (no checkpoint exists offline — every benchmark / parity number in this repo uses those).
Model family: B200SD_MODEL = sd15 (default) | sdxl | sd21 | tiny | tinyxl | tiny21, each also as an inpainting model with
a 9-channel UNet (`sd15-inpainting`, ...).  A checkpoint's own conv_in decides between the two: SD_CKPT of an inpainting
checkpoint serves it as one.  Prediction type: each family's default (v for sd21 / tiny21, eps for the others and for
every inpainting model, as sdwui's v2-inpainting-inference.yaml), overridden by B200SD_PREDICTION = eps | v.
ControlNets (controlnet()): B200SD_CONTROLNET_DIR/<model>.safetensors, otherwise seeded synthetic weights.
LoRA networks (loras()): B200SD_LORA_DIR/<name>.safetensors (kohya format), otherwise a seeded synthetic LoRA.
"""
import dataclasses
import logging
import os
import threading
import zlib
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import torch

from . import config as C
from .engine import SDEngine
from . import lora as L
from .synth import make_controlnet_state_dict, make_lora_state_dict, make_state_dict
from .unet_exec import ControlNetWeights

log = logging.getLogger("distributed")
_LOCK = threading.Lock()
_ENGINES: Dict[str, SDEngine] = {}
_STATE: Dict[str, Dict[str, torch.Tensor]] = {}
CKPT_FAMILIES = ("sd15", "sd21")      # families whose weights SD_CKPT replaces (SDXL keeps its synthetic weights)
V_FAMILIES = ("sd21", "tiny21")       # families served as v-prediction unless B200SD_PREDICTION says otherwise
INPAINTING = "-inpainting"            # family suffix of the 9-channel inpainting UNets


def _load_safetensors(path: str) -> Dict[str, torch.Tensor]:
    from safetensors.torch import load_file  # optional dependency; only needed for a real checkpoint
    return load_file(path)


def state_dict(size: str = "sd15", seed: int = 0) -> Dict[str, torch.Tensor]:
    key = f"{size}:{seed}:{os.environ.get('SD_CKPT', '')}"
    with _LOCK:
        if key not in _STATE:
            ckpt = os.environ.get("SD_CKPT")
            if ckpt and _base(size) in CKPT_FAMILIES:
                _STATE[key] = _load_safetensors(ckpt)
            else:
                cfgs = configs(size)
                _STATE[key] = make_state_dict(*cfgs, seed=seed)
        return _STATE[key]


def _base(size: str) -> str:
    """the family without its inpainting suffix"""
    return size[:-len(INPAINTING)] if size.endswith(INPAINTING) else size


def configs(size: str = "sd15"):
    """(UNet, VAE, text encoder) configs of a family; `<family>-inpainting` is the family's 9-channel UNet"""
    if size.endswith(INPAINTING):
        unet, vae, clip = configs(_base(size))
        return dataclasses.replace(unet, in_channels=9), vae, clip
    if size == "sd15":
        return C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP
    if size == "tiny":
        return C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP
    if size == "sdxl":
        return C.SDXL_UNET, C.SDXL_VAE, C.SDXL_CLIP
    if size == "tinyxl":
        return C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP
    if size == "sd21":
        return C.SD21_UNET, C.SD21_VAE, C.SD21_CLIP
    if size == "tiny21":
        return C.TINY21_UNET, C.TINY21_VAE, C.TINY21_CLIP
    raise ValueError(size)


def checkpoint_in_channels(sd: Dict[str, torch.Tensor]) -> int:
    """input channels of a checkpoint's UNet conv_in: 4, 9 for an inpainting model (8 instruct-pix2pix, 5 depth2img)"""
    return int(sd[C.UNET_PREFIX + "input_blocks.0.0.weight"].shape[1])


def prediction(size: str, in_channels: int = 4) -> str:
    """what the family's UNet predicts: B200SD_PREDICTION (eps | v) when set, otherwise v for SD 2.x (768-v), eps for the
    rest.  SD 2.x-base is B200SD_PREDICTION=eps; v-prediction SD1.5 / SDXL finetunes are B200SD_PREDICTION=v.  A 9-channel
    (inpainting) UNet is eps in every family, as sdwui's v2-inpainting-inference.yaml configures 512-inpainting-ema."""
    env = os.environ.get("B200SD_PREDICTION", "").strip()
    if env:
        if env not in ("eps", "v"):
            raise ValueError(f"B200SD_PREDICTION={env!r}: expected 'eps' or 'v'")
        return env
    return "v" if size in V_FAMILIES and in_channels == 4 else "eps"


def default_engine_factory(device: str, size: str = None) -> SDEngine:
    size = size or os.environ.get("B200SD_MODEL", "sd15")
    sd = state_dict(size)
    unet_cfg, vae_cfg, clip_cfg = configs(size)
    if os.environ.get("SD_CKPT") and _base(size) in CKPT_FAMILIES:
        # the checkpoint's conv_in decides: an inpainting checkpoint under a plain family name is served as one, and
        # 8- / 5-channel models are refused by SDEngine instead of being padded to 64 channels
        unet_cfg = dataclasses.replace(unet_cfg, in_channels=checkpoint_in_channels(sd))
    pred = prediction(size, unet_cfg.in_channels)
    key = f"{device}:{size}:{pred}"
    with _LOCK:
        eng = _ENGINES.get(key)
    if eng is None:
        if size != "tiny" and not os.environ.get("SD_CKPT"):
            log.warning("b200sd: SD_CKPT is not set — serving SEEDED SYNTHETIC %s weights (images are noise); "
                        "set SD_CKPT=/path/model.safetensors for a real checkpoint", size)
        if size != "tiny" and not os.environ.get("SD_TOKENIZER"):
            log.warning("b200sd: SD_TOKENIZER is not set — prompts are hashed to token ids, not BPE-tokenised")
        # SDXL runs in bf16 (BASELINE config 4; its VAE overflows fp16 — sdwui upcasts it, SURVEY App. C)
        dtype = torch.bfloat16 if _base(size) in ("sdxl", "tinyxl") else torch.float16
        eng = SDEngine(sd, unet_cfg, vae_cfg, clip_cfg, device=device, dtype=dtype, prediction=pred)
        with _LOCK:
            _ENGINES[key] = eng
    return eng


def evict(device: str) -> int:
    """forget the cached engines and ControlNets of `device` (LocalGPUWorker.restart): their weights, plans and graphs
    are freed once the last reference goes"""
    with _LOCK:
        keys = [k for k in _ENGINES if k.startswith(f"{device}:")]
        for k in keys:
            _ENGINES.pop(k).release()
        for k in [k for k in _CONTROLNETS if k[0] == str(device)]:
            del _CONTROLNETS[k]
    return len(keys)


MAX_CONTROLNETS = 3   # packed ControlNet models kept per device; the least recently used one is dropped beyond that
_CONTROLNETS: "OrderedDict[tuple, ControlNetWeights]" = OrderedDict()


def _controlnet_state(name: str, size: str) -> Dict[str, torch.Tensor]:
    """B200SD_CONTROLNET_DIR/<name>.safetensors (ldm ControlNet keys, with or without `control_model.`), or seeded
    synthetic weights (crc32 of the name) when the variable is not set"""
    root = os.environ.get("B200SD_CONTROLNET_DIR")
    if not root:
        log.warning("b200sd: B200SD_CONTROLNET_DIR is not set — ControlNet %r uses SEEDED SYNTHETIC weights; set it to a "
                    "directory of <model>.safetensors files for real ControlNets", name)
        return make_controlnet_state_dict(configs(size)[0], seed=zlib.crc32(name.encode("utf-8")))
    path = os.path.join(root, name + ".safetensors")
    if not os.path.isfile(path):
        raise FileNotFoundError(f"ControlNet model {name!r} not found: no {path}")
    sd = _load_safetensors(path)
    if any(k.startswith(("controlnet_cond_embedding.", "controlnet_down_blocks.")) for k in sd):
        raise ValueError(f"{path} is a diffusers-layout ControlNet: only ldm ControlNet checkpoints are served")
    return {(k if k.startswith(C.CONTROL_PREFIX) else C.CONTROL_PREFIX + k): v for k, v in sd.items()}


def controlnet(name: str, size: str = None, device: str = "cuda:0", dtype=torch.float16) -> ControlNetWeights:
    """ControlNet `name` for the `size` family (default B200SD_MODEL), packed on `device` and cached there"""
    size = size or os.environ.get("B200SD_MODEL", "sd15")
    key = (str(device), size, name, os.environ.get("B200SD_CONTROLNET_DIR", ""), dtype)
    with _LOCK:
        cw = _CONTROLNETS.get(key)
        if cw is not None:
            _CONTROLNETS.move_to_end(key)
            return cw
    cw = ControlNetWeights(_controlnet_state(name, size), configs(size)[0], torch.device(device), dtype, name=name)
    with _LOCK:
        _CONTROLNETS[key] = cw
        mine = [k for k in _CONTROLNETS if k[0] == str(device)]
        for k in mine[:max(0, len(mine) - MAX_CONTROLNETS)]:
            del _CONTROLNETS[k]
    return cw


MAX_LORAS = 8   # parsed LoRA files kept per process; the least recently used one is dropped beyond that
_LORAS: "OrderedDict[tuple, L.LoraFile]" = OrderedDict()


def lora_file(name: str, unet_cfg: C.UNetConfig, clip_cfg: C.CLIPConfig) -> Optional[L.LoraFile]:
    """LoRA `name` parsed (lora.load_state_dict: ValueError for a network type that is not served) and cached under
    (path, size, mtime): B200SD_LORA_DIR/<name>.safetensors, None with a warning when the variable is set and the file is
    missing (sdwui's "Networks not found"), or a seeded synthetic LoRA for the model of (unet_cfg, clip_cfg) (crc32 of
    the name) when it is not set"""
    root = os.environ.get("B200SD_LORA_DIR")
    if not root:
        log.warning("b200sd: B200SD_LORA_DIR is not set — LoRA %r is a SEEDED SYNTHETIC network; set it to a directory "
                    "of <name>.safetensors files for real ones", name)
        key = ("synthetic", unet_cfg, clip_cfg, name)
    else:
        path = os.path.join(root, name + ".safetensors")
        if not os.path.isfile(path):
            log.warning("b200sd: Networks not found: %s (no %s)", name, path)
            return None
        st = os.stat(path)
        key = (path, st.st_size, st.st_mtime_ns)
    with _LOCK:
        f = _LORAS.get(key)
        if f is not None:
            _LORAS.move_to_end(key)
            return f
    if not root:
        sd = make_lora_state_dict(unet_cfg, clip_cfg, seed=zlib.crc32(name.encode("utf-8")),
                                  form="compvis" if clip_cfg.xl_width else "diffusers")
    else:
        sd = _load_safetensors(key[0])
    f = L.load_state_dict(name, sd, key)
    with _LOCK:
        _LORAS[key] = f
        while len(_LORAS) > MAX_LORAS:
            _LORAS.popitem(last=False)
    return f


def loras(refs, eng) -> List[tuple]:
    """prompt tags (lora.LoraRef) -> [(LoraFile, LoraRef)] for the SDEngine `eng`; missing files are skipped with a
    warning.  Every file is read (and refused if need be) before the engine changes any weight."""
    out = []
    for ref in refs:
        f = lora_file(ref.name, eng.unet_cfg, eng.clip_cfg)
        if f is not None:
            out.append((f, ref))
    return out


def refresh_loras():
    """forget the parsed LoRA files (refresh-loras): the next request reads them again"""
    with _LOCK:
        _LORAS.clear()


def model_identity(size: str = None) -> str:
    """what /sd-models and /options report as the loaded checkpoint"""
    size = size or os.environ.get("B200SD_MODEL", "sd15")
    ckpt = os.environ.get("SD_CKPT")
    return os.path.basename(ckpt) if ckpt and _base(size) in CKPT_FAMILIES else f"synthetic-{size}-seed0"


_TOKENIZER = {}


def _clip_tokenizer():
    """transformers.CLIPTokenizer over a LOCAL directory (SD_TOKENIZER=/path with vocab.json + merges.txt — the files of
    openai/clip-vit-large-patch14, which cannot be fetched offline), or None."""
    path = os.environ.get("SD_TOKENIZER")
    if not path:
        return None
    if path not in _TOKENIZER:
        from transformers import CLIPTokenizer
        _TOKENIZER[path] = CLIPTokenizer(os.path.join(path, "vocab.json"), os.path.join(path, "merges.txt"))
    return _TOKENIZER[path]


def synthetic_tokens(prompts: List[str], vocab: int, ctx: int = 77, pad: Optional[int] = None) -> torch.Tensor:
    """pad: the id after the first EOS (None: EOS; SD 2.x's OpenCLIP tower: 0)"""
    tok = _clip_tokenizer()
    if tok is not None:
        # the real BPE ids, padded with the end-of-text token like sdwui's FrozenCLIPEmbedderWithCustomWords (plain
        # prompts up to 75 tokens; emphasis syntax, BREAK and >75-token chunking are interpreted by tokenize_prompts)
        ids = tok(list(prompts), padding="max_length", max_length=ctx, truncation=True, return_tensors="pt").input_ids.long()
        eos = tok.eos_token_id
        first_eos = (ids == eos).float().argmax(dim=1)
        for i in range(ids.shape[0]):
            ids[i, int(first_eos[i]):] = eos
            if pad is not None:
                ids[i, int(first_eos[i]) + 1:] = pad
        if int(ids.max()) >= vocab:
            raise ValueError("the tokenizer's ids do not fit the text encoder's vocabulary")
        return ids
    return _hashed_tokens(prompts, vocab, ctx, pad)


def tokenize_prompts(prompts: List[str], vocab: int, pad: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Prompts with sdwui's syntax (b200sd.prompts: emphasis, BREAK, chunks of 75 tokens with comma backtracking) ->
    (ids int64 [n, 77 * k], multipliers fp32 [n, 77 * k]); a prompt with fewer chunks than the longest one is padded with
    empty chunks, as sdwui pads a batch.  Tokeniser: the CLIP BPE of SD_TOKENIZER (comma ",</w>"), otherwise the crc32
    word hash of synthetic_tokens per segment (no comma token, so no backtracking).  A prompt without brackets, BREAK or
    more than 75 tokens gets exactly synthetic_tokens' ids, all multipliers 1.  pad: the id after each chunk's first EOS
    (None: EOS, CLIP; 0 for SD 2.x's OpenCLIP tower, whose tokenizer has the same vocabulary and merges)."""
    from .prompts import tokenize_prompt
    tok = _clip_tokenizer()
    if tok is not None:
        bos, eos = tok.bos_token_id, tok.eos_token_id
        comma = tok.get_vocab().get(",</w>")

        def ids_of(text):
            return tok(text, truncation=False, add_special_tokens=False)["input_ids"] if text else []
    else:
        bos, eos, comma = vocab - 2, vocab - 1, None

        def ids_of(text):
            return [zlib.crc32(w.encode("utf-8")) % (vocab - 3) for w in text.split()]
    per = [tokenize_prompt(p or "", ids_of, bos, eos, comma, pad) for p in prompts]
    k = max(len(c) for c, _ in per)
    empty = [bos, eos] + [eos if pad is None else pad] * 75
    ids = torch.tensor([sum(c + [empty] * (k - len(c)), []) for c, _ in per], dtype=torch.long)
    mult = torch.tensor([sum(m + [[1.0] * 77] * (k - len(m)), []) for _, m in per], dtype=torch.float32)
    if int(ids.max()) >= vocab:
        raise ValueError("the tokenizer's ids do not fit the text encoder's vocabulary")
    return ids, mult


def _hashed_tokens(prompts: List[str], vocab: int, ctx: int = 77, pad: Optional[int] = None) -> torch.Tensor:
    """Deterministic stand-in for the CLIP BPE tokenizer (its vocabulary files are not available offline):
    [BOS] + one id per whitespace-separated word (crc32 mod vocab-3) + [EOS] padding, length 77 (with `pad`: one EOS,
    then `pad`)."""
    bos, eos = vocab - 2, vocab - 1
    out = torch.full((len(prompts), ctx), eos, dtype=torch.long)
    out[:, 0] = bos
    for i, text in enumerate(prompts):
        ids = [zlib.crc32(w.encode("utf-8")) % (vocab - 3) for w in (text or "").split()][: ctx - 2]
        if ids:
            out[i, 1:1 + len(ids)] = torch.tensor(ids)
        if pad is not None:
            out[i, 2 + len(ids):] = pad
    return out
