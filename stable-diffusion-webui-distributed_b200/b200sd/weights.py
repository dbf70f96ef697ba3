"""Weight packing for the sm_90a kernels (one-time, at model load).

Upstream (ldm) layouts -> kernel layouts:
  conv  [Cout, Cin, kh, kw]        -> [Cout, kh*kw*Cin]  (tap-major, channels innermost: matches NHWC im2col order)
  GEGLU proj [2*inner, C] (+bias)  -> rows interleaved per output tile: [value half | gate half] per block_n rows
  q/k/v projections [h*d, C]       -> [h*d_pad, C] with zero rows for the padded head columns
"""
import torch


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
