"""Engine construction for the local-GPU workers: one SDEngine per CUDA device, built lazily and cached.

Weights: `SD_CKPT=/path/model.safetensors` (ldm key names; read for sd15 and sd21) when present, otherwise the seeded
synthetic weights of synth.py (no checkpoint exists offline — every benchmark / parity number in this repo uses those).
Model family: B200SD_MODEL = sd15 (default) | sdxl | sd21 | tiny | tinyxl | tiny21.  Prediction type: each family's
default (v for sd21 / tiny21, eps for the others), overridden by B200SD_PREDICTION = eps | v.
"""
import logging
import os
import threading
import zlib
from typing import Dict, List, Optional, Tuple

import torch

from . import config as C
from .engine import SDEngine
from .synth import make_state_dict

log = logging.getLogger("distributed")
_LOCK = threading.Lock()
_ENGINES: Dict[str, SDEngine] = {}
_STATE: Dict[str, Dict[str, torch.Tensor]] = {}
CKPT_FAMILIES = ("sd15", "sd21")      # families whose weights SD_CKPT replaces (SDXL keeps its synthetic weights)
V_FAMILIES = ("sd21", "tiny21")       # families served as v-prediction unless B200SD_PREDICTION says otherwise


def _load_safetensors(path: str) -> Dict[str, torch.Tensor]:
    from safetensors.torch import load_file  # optional dependency; only needed for a real checkpoint
    return load_file(path)


def state_dict(size: str = "sd15", seed: int = 0) -> Dict[str, torch.Tensor]:
    key = f"{size}:{seed}:{os.environ.get('SD_CKPT', '')}"
    with _LOCK:
        if key not in _STATE:
            ckpt = os.environ.get("SD_CKPT")
            if ckpt and size in CKPT_FAMILIES:
                _STATE[key] = _load_safetensors(ckpt)
            else:
                cfgs = configs(size)
                _STATE[key] = make_state_dict(*cfgs, seed=seed)
        return _STATE[key]


def configs(size: str = "sd15"):
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


def prediction(size: str) -> str:
    """what the family's UNet predicts: B200SD_PREDICTION (eps | v) when set, otherwise v for SD 2.x (768-v), eps for the
    rest.  SD 2.x-base is B200SD_PREDICTION=eps; v-prediction SD1.5 / SDXL finetunes are B200SD_PREDICTION=v."""
    env = os.environ.get("B200SD_PREDICTION", "").strip()
    if env:
        if env not in ("eps", "v"):
            raise ValueError(f"B200SD_PREDICTION={env!r}: expected 'eps' or 'v'")
        return env
    return "v" if size in V_FAMILIES else "eps"


def default_engine_factory(device: str, size: str = None) -> SDEngine:
    size = size or os.environ.get("B200SD_MODEL", "sd15")
    pred = prediction(size)
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
        dtype = torch.bfloat16 if size in ("sdxl", "tinyxl") else torch.float16
        eng = SDEngine(state_dict(size), *configs(size), device=device, dtype=dtype, prediction=pred)
        with _LOCK:
            _ENGINES[key] = eng
    return eng


def evict(device: str) -> int:
    """forget the cached engines of `device` (LocalGPUWorker.restart): their weights, plans and graphs are freed once the
    last reference goes"""
    with _LOCK:
        keys = [k for k in _ENGINES if k.startswith(f"{device}:")]
        for k in keys:
            _ENGINES.pop(k).release()
    return len(keys)


def model_identity(size: str = None) -> str:
    """what /sd-models and /options report as the loaded checkpoint"""
    size = size or os.environ.get("B200SD_MODEL", "sd15")
    ckpt = os.environ.get("SD_CKPT")
    return os.path.basename(ckpt) if ckpt and size in CKPT_FAMILIES else f"synthetic-{size}-seed0"


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
