"""Weight packing for the sm_90a kernels (one-time, at model load).

Upstream (ldm) layouts -> kernel layouts:
  conv  [Cout, Cin, kh, kw]        -> [Cout, kh*kw*Cin]  (tap-major, channels innermost: matches NHWC im2col order)
  GEGLU proj [2*inner, C] (+bias)  -> rows interleaved per output tile: [value half | gate half] per block_n rows
  q/k/v projections [h*d, C]       -> [h*d_pad, C] with zero rows for the padded head columns

Every packer also records, per ldm weight key, a Placement: where each source row and column landed.  LoRA merging
(b200sd/lora.py) scatters its factors through these, so the layouts are known here only.  They are found by running the
packers themselves on index tensors (value = source index + 1, 0 = padding).
"""
from dataclasses import dataclass
from typing import Optional

import torch


@dataclass
class Placement:
    """an ldm weight of `shape` [out, in...] inside a packed tensor: tensor name in its owner's dict, the packed row of
    every source row (None: row i -> row i) and the source column (flattened [Cin, kh, kw]) of every packed column (-1:
    padding; None: identity)"""
    tensor: str
    shape: tuple
    rows: Optional[torch.Tensor] = None
    cols: Optional[torch.Tensor] = None


def index_column(n: int) -> torch.Tensor:
    """[n, 1] float64 with value i + 1 in row i: a weight whose packing shows where each row goes"""
    return (torch.arange(n, dtype=torch.float64) + 1)[:, None]


def source_rows(packed: torch.Tensor) -> torch.Tensor:
    """packed [R', 1] (an index_column through a packer) -> int64 [n]: the packed row of each source row"""
    v = packed[:, 0].long() - 1
    pos = torch.nonzero(v >= 0)[:, 0]
    out = torch.empty(int(v.max()) + 1, dtype=torch.long)
    out[v[pos]] = pos
    return out


def conv_columns(shape, cin_pad: int = 0) -> torch.Tensor:
    """source column of every packed column of pack_conv(w [Cout, Cin, kh, kw], cin_pad) (-1: padded channel)"""
    _, cin, kh, kw = shape
    idx = (torch.arange(cin * kh * kw, dtype=torch.float64) + 1).reshape(1, cin, kh, kw)
    return pack_conv(idx, cin_pad)[0].long() - 1


def pack_conv(w: torch.Tensor, cin_pad: int = 0, cout_pad: int = 0) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> [Cout', kh*kw*Cin'] with optional zero padding of Cin / Cout."""
    cout, cin, kh, kw = w.shape
    cin_p = max(cin, cin_pad)
    cout_p = max(cout, cout_pad)
    out = torch.zeros((cout_p, kh, kw, cin_p), dtype=w.dtype, device=w.device)
    out[:cout, :, :, :cin] = w.permute(0, 2, 3, 1)
    return out.reshape(cout_p, kh * kw * cin_p).contiguous()


def pack_geglu(w: torch.Tensor, b: torch.Tensor, block_n: int):
    """w [2*inner, C], b [2*inner] (value rows first, gate rows second) -> tile-interleaved copies."""
    two_inner, c = w.shape
    inner = two_inner // 2
    half = block_n // 2
    assert inner % half == 0
    t = inner // half
    wv = w[:inner].reshape(t, half, c)
    wg = w[inner:].reshape(t, half, c)
    wp = torch.cat([wv, wg], dim=1).reshape(two_inner, c).contiguous()
    bv = b[:inner].reshape(t, half)
    bg = b[inner:].reshape(t, half)
    bp = torch.cat([bv, bg], dim=1).reshape(two_inner).contiguous()
    return wp, bp


def pad_heads(w: torch.Tensor, heads: int, d: int, d_pad: int) -> torch.Tensor:
    """[heads*d, C] -> [heads*d_pad, C]; rows d..d_pad of every head are zero."""
    c = w.shape[1]
    out = torch.zeros((heads, d_pad, c), dtype=w.dtype, device=w.device)
    out[:, :d] = w.reshape(heads, d, c)
    return out.reshape(heads * d_pad, c).contiguous()
