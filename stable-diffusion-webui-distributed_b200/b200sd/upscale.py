"""The hires fix's upscalers (sdwui `hr_upscaler`) on the device.

Latent modes: `F.interpolate` of the first-pass latents (sdwui shared.latent_upscale_modes).  "Latent" keeps its own
kernel (b200sd_resize_latent_bilinear); the others run b200sd_resize_latent_table on tables built here.

Pixel upscalers: sdwui images.resize_image(0, img, w, h, upscaler) on the decoded uint8 images.
  - "None": one Pillow LANCZOS resize; "Lanczos" / "Nearest": sdwui's UpscalerLanczos / UpscalerNearest;
  - ESRGAN-family models (basicsr RRDBNet, 4x): upscaler_utils.upscale_with_model — split_grid tiles, the network in
    fp16 on the tensor-core convolutions, round-to-nearest quantisation, combine_grid's masked pastes.
Pillow's resampling and paste arithmetic are reproduced bit for bit: the host builds Pillow's fixed-point coefficient
tables, the kernels apply them.
"""
import logging
import math
import os
import threading
import zlib
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import ops

log = logging.getLogger("b200sd")

# sdwui shared.latent_upscale_modes: name -> (F.interpolate mode, antialias)
LATENT_MODES = {
    "Latent": ("bilinear", False),
    "Latent (antialiased)": ("bilinear", True),
    "Latent (bicubic)": ("bicubic", False),
    "Latent (bicubic antialiased)": ("bicubic", True),
    "Latent (nearest)": ("nearest", False),
    "Latent (nearest-exact)": ("nearest-exact", False),
}
PIL_UPSCALERS = ("None", "Lanczos", "Nearest")
# sdwui's built-in ESRGAN-family names -> model file stem (and the block count of the released model)
ESRGAN_BUILTINS = {"R-ESRGAN 4x+": "RealESRGAN_x4plus", "R-ESRGAN 4x+ Anime6B": "RealESRGAN_x4plus_anime_6B",
                   "ESRGAN_4x": "ESRGAN_4x"}
BUILTIN_BLOCKS = {"RealESRGAN_x4plus_anime_6B": 6}
# sdwui upscalers with other architectures (pixel-unshuffle RRDBNet, SRVGG, SwinIR, SCUNet, LDSR, DAT): not served
UNSERVED_PREFIXES = ("R-ESRGAN 2x+", "R-ESRGAN General", "R-ESRGAN AnimeVideo", "SwinIR", "ScuNET", "LDSR", "DAT")
DEFAULT_TILE, DEFAULT_OVERLAP = 192, 8   # sdwui opts.ESRGAN_tile / ESRGAN_tile_overlap
SCALE = 4


class UnsupportedUpscaler(ValueError):
    pass


def kind(name: str) -> Tuple[str, str]:
    """("latent", name) | ("pil", name) | ("esrgan", file stem); UnsupportedUpscaler for the architectures not served"""
    if name in LATENT_MODES:
        return "latent", name
    if name in PIL_UPSCALERS:
        return "pil", name
    if name in ESRGAN_BUILTINS:
        return "esrgan", ESRGAN_BUILTINS[name]
    if not name or name.startswith(UNSERVED_PREFIXES) or os.sep in name or name.startswith("."):
        raise UnsupportedUpscaler(f"hires upscaler {name!r} is not served")
    return "esrgan", name


# ------------------------------------------------------------------------------------------------ latent tables
def _torch_aa_filter(mode: str, x: float) -> float:
    x = abs(x)
    if mode == "bilinear":
        return 1.0 - x if x < 1.0 else 0.0
    a = -0.5   # torch's antialiased bicubic uses Keys' a = -0.5 (as Pillow), not the -0.75 of mode="bicubic"
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0
    if x < 2.0:
        return (((x - 5.0) * x + 8.0) * x - 4.0) * a
    return 0.0


def _latent_axis(mode: str, antialias: bool, n_in: int, n_out: int) -> Tuple[np.ndarray, np.ndarray]:
    """(indices int32 [n_out, k], weights fp32 [n_out, k]) of F.interpolate(mode, align_corners=False, antialias) along one
    axis; padding taps have weight 0 and index 0"""
    f32 = np.float32
    scale = f32(f32(n_in) / f32(n_out))
    o = np.arange(n_out)
    if mode in ("nearest", "nearest-exact"):
        pos = o.astype(f32) * scale if mode == "nearest" else (o.astype(f32) + f32(0.5)) * scale
        idx = np.minimum(np.floor(pos).astype(np.int64), n_in - 1)
        return idx.reshape(-1, 1).astype(np.int32), np.ones((n_out, 1), f32)
    if not antialias:
        if mode == "bilinear":
            raise ValueError("plain bilinear is b200sd_resize_latent_bilinear")
        # upsample_bicubic2d: real = scale * (o + 0.5) - 0.5, taps floor(real) - 1 .. + 2 clamped, A = -0.75
        real = scale * (o.astype(f32) + f32(0.5)) - f32(0.5)
        i0 = np.floor(real)
        t = (real - i0).astype(f32)
        A = f32(-0.75)

        def c1(x):  # |x| <= 1
            return ((A + 2) * x - (A + 3)) * x * x + 1

        def c2(x):  # 1 < |x| < 2
            return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A

        w = np.stack([c2(t + 1), c1(t), c1(1 - t), c2(2 - t)], axis=1).astype(f32)
        idx = np.clip(i0.astype(np.int64)[:, None] + np.arange(-1, 3)[None, :], 0, n_in - 1)
        return idx.astype(np.int32), w
    interp = 2 if mode == "bilinear" else 4
    support = (interp * 0.5) * float(scale) if scale >= 1.0 else interp * 0.5
    invscale = 1.0 / float(scale) if scale >= 1.0 else 1.0
    k = int(math.ceil(support)) * 2 + 1
    idx, wts = np.zeros((n_out, k), np.int32), np.zeros((n_out, k), f32)
    for i in range(n_out):
        center = float(scale) * (i + 0.5)
        xmin = max(int(center - support + 0.5), 0)
        xsize = min(int(center + support + 0.5), n_in) - xmin
        w = [_torch_aa_filter(mode, (j + xmin - center + 0.5) * invscale) for j in range(xsize)]
        total = sum(w)
        idx[i, :xsize] = np.arange(xmin, xmin + xsize)
        wts[i, :xsize] = [v / total if total != 0.0 else v for v in w]
    return idx, wts


def latent_tables(name: str, h: int, w: int, ho: int, wo: int, device) -> tuple:
    """device tables of b200sd_resize_latent_table for the latent mode `name`: ((ix, wx), (iy, wy))"""
    mode, aa = LATENT_MODES[name]
    out = []
    for n_in, n_out in ((w, wo), (h, ho)):
        i, wt = _latent_axis(mode, aa, n_in, n_out)
        out.append((torch.from_numpy(i).to(device), torch.from_numpy(wt).to(device)))
    return tuple(out)


def resize_latents(lat: torch.Tensor, name: str, h: int, w: int, ho: int, wo: int) -> torch.Tensor:
    """fp32 NHWC latents [b, h*w, 4] -> [b, ho*wo, 4] with the latent mode `name` (not "Latent")"""
    up = torch.empty((lat.shape[0], ho * wo, 4), device=lat.device, dtype=torch.float32)
    ops.resize_latent_table(lat.contiguous(), up, h, w, ho, wo, *latent_tables(name, h, w, ho, wo, lat.device))
    return up


# ------------------------------------------------------------------------------------------------ Pillow tables
PRECISION_BITS = 22   # Pillow Resample.c: 32 - 8 - 2


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x: float) -> float:
    return _sinc(x) * _sinc(x / 3.0) if -3.0 <= x < 3.0 else 0.0


def pil_lanczos_coeffs(n_in: int, n_out: int) -> Tuple[np.ndarray, np.ndarray]:
    """Pillow precompute_coeffs + normalize_coeffs_8bpc for a LANCZOS resize over the whole axis:
    bounds int32 [n_out, 2] = (first input, count), kk int32 [n_out, ksize]"""
    scale = filterscale = float(n_in) / n_out
    if filterscale < 1.0:
        filterscale = 1.0
    support = 3.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((n_out, 2), np.int32)
    kk = np.zeros((n_out, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in) - xmin
        k = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in k:
            ww += v
        if ww != 0.0:
            k = [v / ww for v in k]
        kk[xx, :xmax] = [int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
                         for v in k]
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def pil_nearest_index(n_in: int, n_out: int) -> np.ndarray:
    """Pillow's NEAREST resize (ImagingScaleAffine): source index of each output position, accumulated in doubles"""
    a = float(n_in) / n_out
    xo = a * 0.5
    out = np.zeros(n_out, np.int64)
    for x in range(n_out):
        out[x] = -1 if xo < 0.0 else int(xo)
        xo += a
    return out


def pil_tables(filt: str, n_in: int, n_out: int) -> Tuple[np.ndarray, np.ndarray]:
    """(bounds, kk) of b200sd_resample_u8 for Pillow's LANCZOS or NEAREST along one axis"""
    if filt == "lanczos":
        return pil_lanczos_coeffs(n_in, n_out)
    idx = pil_nearest_index(n_in, n_out)
    bounds = np.stack([idx, np.ones_like(idx)], axis=1).astype(np.int32)
    return bounds, np.full((n_out, 1), 1 << PRECISION_BITS, np.int32)


def pil_resize(img: torch.Tensor, w: int, h: int, filt: str = "lanczos") -> torch.Tensor:
    """PIL Image.resize((w, h), LANCZOS | NEAREST) of uint8 RGB images [b, H, W, 3] on the device, bitwise: the horizontal
    pass first, a pass whose size does not change is skipped (Pillow ImagingResample)"""
    b, hh, ww, _ = img.shape
    if (ww, hh) == (w, h):
        return img
    x = img.contiguous()
    for vertical, n_in, n_out in ((False, ww, w), (True, hh, h)):
        if n_in == n_out:
            continue
        bounds, kk = pil_tables(filt, n_in, n_out)
        shape = (b, n_out if vertical else x.shape[1], x.shape[2] if vertical else n_out, 3)
        out = torch.empty(shape, dtype=torch.uint8, device=img.device)
        ops.resample_u8(x, out, vertical, torch.from_numpy(bounds).to(img.device), torch.from_numpy(kk).to(img.device))
        x = out
    return x


# ------------------------------------------------------------------------------------------------ tile geometry
def split_grid(w: int, h: int, tile_w: int, tile_h: int, overlap: int) -> Tuple[List[int], List[int]]:
    """sdwui images.split_grid: (row y positions, column x positions) of the tiles of a w x h image; a position is
    negative when the image is smaller than a tile (the crop is black-padded there)"""
    cols = math.ceil((w - overlap) / (tile_w - overlap))
    rows = math.ceil((h - overlap) / (tile_h - overlap))
    dx = (w - tile_w) / (cols - 1) if cols > 1 else 0
    dy = (h - tile_h) / (rows - 1) if rows > 1 else 0
    ys, xs = [], []
    for row in range(rows):
        y = int(row * dy)
        if y + tile_h >= h:
            y = h - tile_h
        ys.append(y)
    for col in range(cols):
        x = int(col * dx)
        if x + tile_w >= w:
            x = w - tile_w
        xs.append(x)
    return ys, xs


def blend_mask(overlap: int) -> np.ndarray:
    """combine_grid's mask values: (arange(overlap, float32) * 255 / overlap).astype(uint8)"""
    return (np.arange(overlap, dtype=np.float32) * 255 / overlap).astype(np.uint8)


def crop_tiles(img: torch.Tensor, ys: List[int], xs: List[int], th: int, tw: int) -> torch.Tensor:
    """uint8 [b, H, W, 3] -> tiles [b * rows * cols, th, tw, 3] (PIL crop: black outside the image)"""
    b, hh, ww, _ = img.shape
    out = torch.zeros((b, len(ys), len(xs), th, tw, 3), dtype=torch.uint8, device=img.device)
    for r, y in enumerate(ys):
        for c, x in enumerate(xs):
            y0, x0 = max(y, 0), max(x, 0)
            y1, x1 = min(y + th, hh), min(x + tw, ww)
            out[:, r, c, y0 - y:y1 - y, x0 - x:x1 - x] = img[:, y0:y1, x0:x1]
    return out.reshape(-1, th, tw, 3)


# ------------------------------------------------------------------------------------------------ RRDBNet weights
def _rrdb_keys(num_block: int) -> List[str]:
    keys = ["conv_first"]
    for i in range(num_block):
        keys += [f"body.{i}.rdb{r}.conv{c}" for r in (1, 2, 3) for c in range(1, 6)]
    return keys + ["conv_body", "conv_up1", "conv_up2", "conv_hr", "conv_last"]


def to_basicsr(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """an RRDBNet state dict in basicsr's layout (`params_ema` / `params` unwrapped) or old ESRGAN's (`model.0`,
    `model.1.sub.i.RDBk.convj.0`, `model.3/6/8/10`) -> basicsr keys.  UnsupportedUpscaler for any other network."""
    for wrap in ("params_ema", "params"):
        if wrap in sd and isinstance(sd[wrap], dict):
            sd = sd[wrap]
            break
    if "model.0.weight" in sd:
        old = {"model.0": "conv_first", "model.3": "conv_up1", "model.6": "conv_up2", "model.8": "conv_hr",
               "model.10": "conv_last"}
        subs = [int(k.split(".")[3]) for k in sd if k.startswith("model.1.sub.") and k.endswith(".weight")]
        nb = max(subs) if subs else 0
        out = {}
        for k, v in sd.items():
            stem, _, leaf = k.rpartition(".")
            if stem in old:
                out[f"{old[stem]}.{leaf}"] = v
            elif stem == f"model.1.sub.{nb}":
                out[f"conv_body.{leaf}"] = v
            elif stem.startswith("model.1.sub.") and ".RDB" in stem:
                p = stem.split(".")   # model 1 sub i RDBk convj 0
                out[f"body.{p[3]}.rdb{p[4][3:]}.{p[5]}.{leaf}"] = v
            else:
                raise UnsupportedUpscaler(f"unexpected ESRGAN key {k!r}")
        sd = out
    blocks = {int(k.split(".")[1]) for k in sd if k.startswith("body.")}
    nb = len(blocks)
    want = {f"{s}.{leaf}" for s in _rrdb_keys(nb) for leaf in ("weight", "bias")}
    if nb == 0 or set(sd) != want or blocks != set(range(nb)):
        raise UnsupportedUpscaler("not a basicsr / ESRGAN RRDBNet state dict")
    if tuple(sd["conv_first.weight"].shape) != (64, 3, 3, 3) or tuple(sd["conv_last.weight"].shape) != (3, 64, 3, 3) or \
            tuple(sd["body.0.rdb1.conv1.weight"].shape) != (32, 64, 3, 3):
        raise UnsupportedUpscaler("only 4x RRDBNets with 3 input channels, 64 features and growth 32 are served")
    return sd


def num_blocks(sd: Dict[str, torch.Tensor]) -> int:
    return len({int(k.split(".")[1]) for k in sd if k.startswith("body.")})


def synthetic_state_dict(num_block: int = 23, seed: int = 0) -> Dict[str, torch.Tensor]:
    """basicsr RRDBNet init: PyTorch's default conv init, and in the dense blocks kaiming_normal x 0.1 with zero bias
    (basicsr default_init_weights(..., 0.1)), so activations stay O(1) through the 23 blocks"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key in _rrdb_keys(num_block):
        if key.startswith("body."):
            c = int(key[-1])
            cin, cout = 64 + 32 * (c - 1), (64 if c == 5 else 32)
            w = torch.randn((cout, cin, 3, 3), generator=g) * math.sqrt(2.0 / (cin * 9)) * 0.1
            b = torch.zeros(cout)
        else:
            cin, cout = (3, 64) if key == "conv_first" else (64, 3) if key == "conv_last" else (64, 64)
            bound = 1.0 / math.sqrt(cin * 9)
            w = (torch.rand((cout, cin, 3, 3), generator=g) * 2 - 1) * bound
            b = (torch.rand(cout, generator=g) * 2 - 1) * bound
        sd[f"{key}.weight"], sd[f"{key}.bias"] = w, b
    return sd


def load_state_dict(stem: str) -> Dict[str, torch.Tensor]:
    """B200SD_UPSCALER_DIR/<stem>.pth | .safetensors in basicsr keys, or seeded synthetic weights (crc32 of the stem)
    when the variable is not set"""
    root = os.environ.get("B200SD_UPSCALER_DIR")
    if not root:
        log.warning("b200sd: B200SD_UPSCALER_DIR is not set — upscaler %r uses SEEDED SYNTHETIC weights; set it to a "
                    "directory of <model>.pth / .safetensors files for real ESRGAN models", stem)
        return synthetic_state_dict(BUILTIN_BLOCKS.get(stem, 23), seed=zlib.crc32(stem.encode("utf-8")))
    for ext in (".pth", ".safetensors"):
        path = os.path.join(root, stem + ext)
        if os.path.isfile(path):
            try:
                if ext == ".pth":
                    sd = torch.load(path, map_location="cpu", weights_only=True)
                else:
                    from safetensors.torch import load_file
                    sd = load_file(path)
            except Exception as e:   # a pickle weights_only refuses, a corrupt file, safetensors not installed
                raise UnsupportedUpscaler(f"{path} cannot be read as a state dict: {type(e).__name__}: {e}") from e
            if not isinstance(sd, dict):
                raise UnsupportedUpscaler(f"{path} does not hold a state dict")
            try:
                return to_basicsr(sd)
            except UnsupportedUpscaler:
                raise
            except (KeyError, IndexError, ValueError, AttributeError, TypeError) as e:   # keys of another network
                raise UnsupportedUpscaler(f"{path} is not an RRDBNet state dict: {type(e).__name__}: {e}") from e
    raise UnsupportedUpscaler(f"upscaler model {stem!r} not found in {root}")


# ------------------------------------------------------------------------------------------------ packing
# One RDB works in a 224-channel NHWC buffer laid out [x4 | x | x1 | x2 | x3 | zeros] (32, 64, 32, 32, 32, 32 channels).
# Each conv reads a contiguous window of it, which the conv kernel needs in multiples of 64 channels: conv2's 96 inputs
# are read as the 128-channel window [x4, x, x1] and conv4's 160 as [x, x1, x2, x3, zeros], with zero weight columns
# for x4 / zeros.  The window never includes the slot the conv writes, so a conv never reads what it is writing, and
# x4 holds finite values from its allocation on (zeros, then earlier conv4 outputs).
CAT = 224
SLOT = {"x4": (0, 32), "x": (32, 64), "x1": (96, 32), "x2": (128, 32), "x3": (160, 32), "z": (192, 32)}
# conv j of an RDB: input window (first channel, width), the window's source channels in basicsr's concat order
# [x, x1, x2, x3, x4] (-1: zero column), output slot
_ORDER = {"x": range(0, 64), "x1": range(64, 96), "x2": range(96, 128), "x3": range(128, 160), "x4": range(160, 192)}


def _window(slots):
    return [i for s in slots for i in (_ORDER[s] if s in _ORDER else [-1] * 32)]


RDB_CONVS = [((32, 64), _window(["x"]), "x1"),
             ((0, 128), _window(["z", "x", "x1"]), "x2"),     # x4's slot read with zero weights
             ((32, 128), _window(["x", "x1", "x2"]), "x3"),
             ((32, 192), _window(["x", "x1", "x2", "x3", "z"]), "x4"),
             ((0, 192), _window(["x4", "x", "x1", "x2", "x3"]), "x")]


def _pack(w: torch.Tensor, src: List[int], rows: Optional[List[int]] = None, cout: Optional[int] = None) -> torch.Tensor:
    """basicsr conv weight [Cout, Cin, 3, 3] -> [cout, 9 * len(src)] with input channel j taken from src[j] (-1: zero)
    and output row i from rows[i] (-1 / beyond: zero), K ordered (ky, kx, c)"""
    rows = list(range(w.shape[0])) if rows is None else rows
    ri, ci = torch.tensor([max(r, 0) for r in rows]), torch.tensor([max(c, 0) for c in src])
    keep = torch.tensor([r >= 0 for r in rows])[:, None, None, None] & torch.tensor([c >= 0 for c in src])[None, :, None, None]
    sel = torch.where(keep, w.float()[ri][:, ci], 0.0)            # [rows, src, 3, 3]
    out = torch.zeros((cout or len(rows), 3, 3, len(src)), dtype=torch.float32)
    out[:len(rows)] = sel.permute(0, 2, 3, 1)
    return out.reshape(out.shape[0], -1)


class RRDBWeights:
    """A basicsr RRDBNet packed for the device in fp16.  RGB is folded in: conv_first's input channels and conv_last's
    output rows are reversed (the network was trained on BGR), and conv_first reads 64 channels of which 3 are image."""

    def __init__(self, sd: Dict[str, torch.Tensor], device, name: str = ""):
        sd = to_basicsr(sd)
        self.name, self.device, self.dtype = name, torch.device(device), torch.float16
        self.num_block = num_blocks(sd)

        def dev(t):
            return t.to(self.device, self.dtype).contiguous()

        def bias(key, n=None):
            b = sd[f"{key}.bias"].float()
            if n is not None:
                b = torch.cat([b, torch.zeros(n - b.numel())])
            return b.to(self.device).contiguous()

        self.first = (dev(_pack(sd["conv_first.weight"], [2, 1, 0] + [-1] * 61)), bias("conv_first"))
        self.blocks = []
        for i in range(self.num_block):
            rdbs = []
            for r in (1, 2, 3):
                rdbs.append([(dev(_pack(sd[f"body.{i}.rdb{r}.conv{c + 1}.weight"], src)),
                              bias(f"body.{i}.rdb{r}.conv{c + 1}")) for c, (_, src, _) in enumerate(RDB_CONVS)])
            self.blocks.append(rdbs)
        same = list(range(64))
        self.body = (dev(_pack(sd["conv_body.weight"], same)), bias("conv_body"))
        self.up1 = (dev(_pack(sd["conv_up1.weight"], same)), bias("conv_up1"))
        self.up2 = (dev(_pack(sd["conv_up2.weight"], same)), bias("conv_up2"))
        self.hr = (dev(_pack(sd["conv_hr.weight"], same)), bias("conv_hr"))
        b_last = sd["conv_last.bias"].float()
        self.last = (dev(_pack(sd["conv_last.weight"], same, rows=[2, 1, 0], cout=32)),
                     torch.cat([b_last.flip(0), torch.zeros(29)]).to(self.device).contiguous())

    def flops_per_tile(self, h: int, w: int) -> float:
        """tensor-core FLOPs of one h x w tile as the kernels run it (zero weight columns and padded channels counted)"""
        px = h * w
        rdb = sum(9 * width * (32 if slot != "x" else 64) for (_, width), _, slot in RDB_CONVS)
        macs = px * (9 * 64 * 64 + self.num_block * 3 * rdb + 9 * 64 * 64) + 4 * px * 9 * 64 * 64 + \
            16 * px * (2 * 9 * 64 * 64 + 9 * 64 * 32)
        return 2.0 * macs


class RRDBProgram:
    """Buffers for `n` tiles of h x w through one RRDBWeights; run(tiles_u8) -> uint8 [n, 4h, 4w, 3]"""

    def __init__(self, wts: RRDBWeights, n: int, h: int, w: int):
        d, dt = wts.device, wts.dtype
        self.wts, self.n, self.h, self.w = wts, n, h, w
        self.inp = torch.zeros((n, h, w, 64), device=d, dtype=dt)
        self.fea = torch.empty((n, h, w, 64), device=d, dtype=dt)
        self.cat = [torch.zeros((n, h, w, CAT), device=d, dtype=dt) for _ in range(3)]
        self.u1 = torch.empty((n, 2 * h, 2 * w, 64), device=d, dtype=dt)
        self.u1o = torch.empty((n, 2 * h, 2 * w, 64), device=d, dtype=dt)
        self.u2 = torch.empty((n, 4 * h, 4 * w, 64), device=d, dtype=dt)
        self.u2o = torch.empty((n, 4 * h, 4 * w, 64), device=d, dtype=dt)
        self.last = torch.empty((n, 4 * h, 4 * w, 32), device=d, dtype=dt)
        self.u8 = torch.empty((n, 16 * h * w, 3), device=d, dtype=torch.uint8)

    @staticmethod
    def _slot(buf, name):
        a, c = SLOT[name]
        return buf[..., a:a + c]

    def _rdb(self, src, dst, convs):
        for ((a, width), _, slot), (wt, b) in zip(RDB_CONVS, convs):
            x = src[..., a:a + width]
            if slot == "x":    # x5: D = x + 0.2 * conv5, into the next buffer's x slot
                ops.conv2d_scaled(x, wt, self._slot(dst, "x"), bias=b, residual=self._slot(src, "x"), res_scale=0.2)
            else:
                ops.conv2d_scaled(x, wt, self._slot(src, slot), bias=b, lrelu=True)

    def run(self, tiles_u8: torch.Tensor, n: int) -> torch.Tensor:
        """the first n of the program's tiles: tiles_u8 uint8 [n, h, w, 3] -> self.u8[:n] [n, 16 h w, 3]"""
        W = self.wts
        v = lambda t: t[:n]  # noqa: E731  (a short micro-batch runs on the leading tiles; the kernels are batch-invariant)
        inp, fea, (A, B, Cb) = v(self.inp), v(self.fea), [v(c) for c in self.cat]
        ops.hint_to_nhwc(tiles_u8.reshape(n, self.h * self.w, 3), inp.view(n, self.h * self.w, 64))
        ops.conv2d_scaled(inp, W.first[0], fea, bias=W.first[1])
        xa = self._slot(A, "x")
        xa.copy_(fea)
        for rdbs in W.blocks:   # RRDB: A.x -> rdb1 -> B.x -> rdb2 -> C.x -> rdb3 -> B.x; A.x += 0.2 * B.x
            self._rdb(A, B, rdbs[0])
            self._rdb(B, Cb, rdbs[1])
            self._rdb(Cb, B, rdbs[2])
            ops.scaled_add_(xa, self._slot(B, "x"), 0.2)
        ops.conv2d_scaled(xa, W.body[0], self._slot(B, "x"), bias=W.body[1], residual=fea)   # trunk: fea + conv_body
        u1, u1o, u2, u2o = v(self.u1), v(self.u1o), v(self.u2), v(self.u2o)
        ops.upsample2x(self._slot(B, "x"), u1)
        ops.conv2d_scaled(u1, W.up1[0], u1o, bias=W.up1[1], lrelu=True)
        ops.upsample2x(u1o, u2)
        ops.conv2d_scaled(u2, W.up2[0], u2o, bias=W.up2[1], lrelu=True)
        ops.conv2d_scaled(u2o, W.hr[0], u2, bias=W.hr[1], lrelu=True)
        last = v(self.last)
        ops.conv2d_scaled(u2, W.last[0], last, bias=W.last[1])
        ops.quantize_unit_u8(last.view(n, 16 * self.h * self.w, 32), v(self.u8))
        return v(self.u8)


# ------------------------------------------------------------------------------------------------ caches
MAX_MODELS = 2                  # packed upscaler models kept per device; the least recently used one is dropped
TILE_BUDGET_BYTES = 6 << 30     # activation memory of one micro-batch of tiles, at most (see _tiles_per_batch)
_LOCK = threading.Lock()
_MODELS: "OrderedDict[tuple, RRDBWeights]" = OrderedDict()


def model(stem: str, device) -> RRDBWeights:
    key = (str(device), stem, os.environ.get("B200SD_UPSCALER_DIR", ""))
    with _LOCK:
        m = _MODELS.get(key)
        if m is not None:
            _MODELS.move_to_end(key)
            return m
    m = RRDBWeights(load_state_dict(stem), device, name=stem)
    with _LOCK:
        _MODELS[key] = m
        mine = [k for k in _MODELS if k[0] == str(device)]
        for k in mine[:max(0, len(mine) - MAX_MODELS)]:
            del _MODELS[k]
    return m


def evict(device) -> None:
    """forget the packed upscaler models of `device`"""
    with _LOCK:
        for k in [k for k in _MODELS if k[0] == str(device)]:
            del _MODELS[k]


def tile_bytes(h: int, w: int) -> int:
    """device bytes one h x w tile occupies in an RRDBProgram (fp16 activations + the uint8 output)"""
    px = h * w
    return 2 * px * (64 + 64 + 3 * CAT + 4 * (64 + 64) + 16 * (64 + 64 + 32)) + 48 * px


def _tiles_per_batch(device, n_tiles: int, h: int, w: int) -> int:
    """tiles per micro-batch: activations of at most TILE_BUDGET_BYTES and at most half of the device memory that is
    free now (the driver's free memory plus what torch's allocator holds unused)"""
    dev = torch.device(device)
    free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    return max(1, min(n_tiles, min(TILE_BUDGET_BYTES, free // 2) // tile_bytes(h, w)))


# ------------------------------------------------------------------------------------------------ sdwui's resize path
def upscale_with_model(wts: RRDBWeights, img: torch.Tensor, tile: int = DEFAULT_TILE,
                       overlap: int = DEFAULT_OVERLAP) -> torch.Tensor:
    """sdwui upscaler_utils.upscale_with_model on uint8 [b, H, W, 3] -> [b, 4H, 4W, 3]: the tiles of every image form
    the network's batch, run in micro-batches (_tiles_per_batch).  The tile buffers live for this call only: nothing
    but the packed weights stays on the device afterwards."""
    b, hh, ww, _ = img.shape
    if tile <= 0:
        ys, xs, th, tw, overlap = [0], [0], hh, ww, 0
    else:
        ys, xs = split_grid(ww, hh, tile, tile, overlap)
        th = tw = tile
    tiles = crop_tiles(img, ys, xs, th, tw)
    prog = RRDBProgram(wts, _tiles_per_batch(img.device, tiles.shape[0], th, tw), th, tw)
    up = torch.empty((tiles.shape[0], SCALE * th, SCALE * tw, 3), dtype=torch.uint8, device=img.device)
    for i in range(0, tiles.shape[0], prog.n):
        n = min(prog.n, tiles.shape[0] - i)
        up[i:i + n].copy_(prog.run(tiles[i:i + n], n).view(n, SCALE * th, SCALE * tw, 3))
    out = torch.empty((b, SCALE * hh, SCALE * ww, 3), dtype=torch.uint8, device=img.device)
    dev = img.device
    ov = overlap * SCALE
    ops.combine_tiles_u8(up, out, torch.tensor([y * SCALE for y in ys], dtype=torch.int32, device=dev),
                         torch.tensor([x * SCALE for x in xs], dtype=torch.int32, device=dev),
                         torch.from_numpy(blend_mask(max(ov, 1))).to(dev), ov)
    return out


def _do_upscale(name: str, img: torch.Tensor, scale: float, tile: int, overlap: int) -> torch.Tensor:
    k, arg = kind(name)
    if k == "pil":   # UpscalerLanczos / UpscalerNearest.do_upscale
        h, w = img.shape[1], img.shape[2]
        return pil_resize(img, int(w * scale), int(h * scale), "lanczos" if name == "Lanczos" else "nearest")
    return upscale_with_model(model(arg, img.device), img, tile, overlap)


def resize_image(img: torch.Tensor, width: int, height: int, name: str, tile: int = DEFAULT_TILE,
                 overlap: int = DEFAULT_OVERLAP) -> torch.Tensor:
    """sdwui images.resize_image(0, img, width, height, upscaler_name=name) with Upscaler.upscale, on uint8 [b, H, W, 3]"""
    h, w = img.shape[1], img.shape[2]
    if name == "None":
        return pil_resize(img, width, height)
    scale = max(width / w, height / h)
    if scale > 1.0:
        dest_w, dest_h = int((w * scale) // 8 * 8), int((h * scale) // 8 * 8)
        for i in range(3):
            if img.shape[2] >= dest_w and img.shape[1] >= dest_h and (i > 0 or scale != 1):
                break
            shape = img.shape
            img = _do_upscale(name, img, scale, tile, overlap)
            if shape == img.shape:
                break
        img = pil_resize(img, dest_w, dest_h)
    return pil_resize(img, width, height)
