"""ControlNet units of a request: the sd-webui-controlnet API form (alwayson_scripts["controlnet"]["args"], one dict per
unit) -> what SDEngine's `controls` take.  Host logic only (decoding and resizing the control maps with cv2, as sdwui's
extension does); the refusals below are raised as ValueError and reach the dispatcher as InvalidWorkerResponse.

Served: preprocessor "none" (the image is the control map), Balanced control mode, "Just Resize" and "Crop and Resize",
no unit mask, at most 3 units.  Fields that only drive preprocessors (pixel_perfect, processor_res, threshold_a/b,
low_vram, save_detected_map) are accepted and ignored.
"""
import base64
import io
import re
from dataclasses import dataclass
from typing import List

import numpy as np
import torch

MAX_UNITS = 3
RESIZE_MODES = {"just resize": 0, "crop and resize": 1, "resize and fill": 2, 0: 0, 1: 1, 2: 2}
CONTROL_MODES = {"balanced": 0, "my prompt is more important": 1, "controlnet is more important": 2, 0: 0, 1: 1, 2: 2}


@dataclass
class Unit:
    model: str            # ControlNet model name, without a trailing " [hash]"
    image: torch.Tensor   # control map uint8 [H, W, 3] at the generation size
    weight: float
    start: float          # guidance_start / guidance_end: active at sampler step i of n when start <= i / n <= end
    end: float


def _enum(value, table, what):
    key = value.strip().lower() if isinstance(value, str) else value
    if key not in table:
        raise ValueError(f"ControlNet {what} {value!r} is not recognised")
    return table[key]


def _decode(img) -> np.ndarray:
    """a base64 PNG / data URL -> uint8 [H, W, 3] RGB"""
    from PIL import Image
    if not isinstance(img, str):
        raise ValueError(f"ControlNet image of type {type(img).__name__}: expected a base64 PNG or a data URL")
    data = img.split(",", 1)[1] if img.startswith("data:") else img
    return np.asarray(Image.open(io.BytesIO(base64.b64decode(data))).convert("RGB")).copy()


def _nonzero_mask(mask) -> bool:
    return mask is not None and mask != "" and bool(_decode(mask).any())


def resize_map(arr: np.ndarray, width: int, height: int, mode: int) -> np.ndarray:
    """"Just Resize" (0): straight to (width, height); "Crop and Resize" (1): scale by the larger ratio, then crop the
    centre.  cv2 INTER_AREA when shrinking, INTER_CUBIC when enlarging."""
    import cv2
    h0, w0 = arr.shape[:2]
    if (w0, h0) == (width, height):
        return arr
    if mode == 0:
        interp = cv2.INTER_AREA if width * height < w0 * h0 else cv2.INTER_CUBIC
        return cv2.resize(arr, (width, height), interpolation=interp)
    k = max(width / w0, height / h0)
    nw, nh = int(np.round(w0 * k)), int(np.round(h0 * k))
    big = cv2.resize(arr, (nw, nh), interpolation=cv2.INTER_AREA if k < 1 else cv2.INTER_CUBIC)
    y0, x0 = (nh - height) // 2, (nw - width) // 2
    return np.ascontiguousarray(big[y0:y0 + height, x0:x0 + width])


def parse_units(alwayson_scripts, width: int, height: int) -> List[Unit]:
    """the enabled ControlNet units of a payload's alwayson_scripts (key matched case-insensitively); [] when none"""
    args = None
    for name, entry in (alwayson_scripts or {}).items():
        if str(name).lower() == "controlnet":
            args = (entry or {}).get("args") or []
    units = []
    for u in args or []:
        if not isinstance(u, dict):
            raise ValueError(f"ControlNet unit of type {type(u).__name__}: expected the API's dict form")
        if not u.get("enabled", True):
            continue
        module = u.get("module") or "none"
        if str(module).lower() != "none":
            raise ValueError(f"ControlNet preprocessor {module!r} is not served: send the control map with module 'none'")
        if _enum(u.get("control_mode", 0), CONTROL_MODES, "control mode") != 0:
            raise ValueError(f"ControlNet control mode {u.get('control_mode')!r} is not served: only 'Balanced'")
        mode = _enum(u.get("resize_mode", 1), RESIZE_MODES, "resize mode")
        if mode == 2:
            raise ValueError("ControlNet resize mode 'Resize and Fill' is not served")
        img = u.get("image") if u.get("image") is not None else u.get("input_image")
        mask = u.get("mask") if u.get("mask") is not None else u.get("mask_image")
        if isinstance(img, dict):
            img, mask = img.get("image"), img.get("mask") if mask is None else mask
        if img is None:
            raise ValueError("ControlNet unit without an image")
        if _nonzero_mask(mask):
            raise ValueError("ControlNet unit masks are not served")
        model = re.sub(r"\s?\[[^]]*]$", "", str(u.get("model") or ""))
        if not model or model.lower() == "none":
            raise ValueError("ControlNet unit without a model")
        start, end = float(u.get("guidance_start", 0.0)), float(u.get("guidance_end", 1.0))
        if not 0.0 <= start <= end <= 1.0:
            raise ValueError(f"ControlNet guidance window ({start}, {end}) is not within 0 <= start <= end <= 1")
        arr = resize_map(_decode(img), width, height, mode)
        units.append(Unit(model, torch.from_numpy(arr), float(u.get("weight", 1.0)), start, end))
    if len(units) > MAX_UNITS:
        raise ValueError(f"{len(units)} ControlNet units: at most {MAX_UNITS} are served")
    return units
