"""Thin torch-tensor wrappers over the C ABI (include/b200sd.h).

torch is used for device memory and streams only; every op below launches hand-written sm_90a kernels
from libb200sd.so on torch's current stream.  Tensors are NHWC / row-major; `ld`-style pitches come from
`tensor.stride(-2)` so channel slices of wider buffers can be passed directly.
"""
import ctypes
from typing import Optional

import torch

from . import _lib
from ._lib import BF16, EPI_GEGLU, EPI_LRELU, EPI_SILU, F16, Epilogue, check

LAUNCHES = 0  # number of b200sd kernels launched through this module (bench.py's gpu_launches)


def _count(n: int = 1):
    global LAUNCHES
    LAUNCHES += n


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"b200sd ops take fp16/bf16 activations, got {t.dtype}")


def _stream() -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _rows2d(t: torch.Tensor):
    """(rows, cols, pitch) of a tensor whose last dim is contiguous and whose leading dims collapse to rows."""
    assert t.stride(-1) == 1, "last dim must be contiguous"
    cols = t.shape[-1]
    pitch = t.stride(-2) if t.dim() >= 2 else cols
    rows = t.numel() // cols
    # leading dims must be contiguous over the pitch
    exp = pitch
    for d in range(t.dim() - 2, -1, -1):
        if t.shape[d] != 1:
            assert t.stride(d) == exp, f"tensor is not row-collapsible: shape {tuple(t.shape)} stride {t.stride()}"
        exp *= t.shape[d]
    return rows, cols, pitch


def _epi(bias, bias_group_rows, residual, flags):
    e = Epilogue()
    e.bias = 0 if bias is None else bias.data_ptr()
    e.bias_group_rows = int(bias_group_rows)
    e.residual = 0 if residual is None else residual.data_ptr()
    e.ldr = 0 if residual is None else _rows2d(residual)[2]
    e.flags = int(flags)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    return e


NUM_SMS = 132  # H100 SXM


def pick_block_n(n: int, geglu: bool = False, m: Optional[int] = None) -> int:
    """Tile width of the persistent GEMM.  Without `m` (and always for GEGLU, whose weights are interleaved per tile at
    pack time) the widest divisor of N; with `m`, the divisor that wastes the fewest SM-slots in the last wave of
    ceil(M/128) * N/bn tiles over NUM_SMS SMs, with a mild preference for wide MMAs.  Tiles wider than 160 columns are
    never picked: their 64 x bn accumulator per warpgroup does not fit the register budget without spills."""
    cands = [bn for bn in (160, 128, 96, 64, 32) if n % bn == 0 and (not geglu or bn % 64 == 0)]
    if not cands:
        raise ValueError(f"N={n} has no supported tile width")
    if geglu or m is None:
        return cands[0]
    mt = (m + 127) // 128
    best = None
    for bn in cands:
        if bn < 128 <= cands[0]:
            continue
        tiles = mt * (n // bn)
        waves = -(-tiles // NUM_SMS)
        score = tiles / (waves * NUM_SMS) * (1.0 if bn >= 160 else 0.97 if bn >= 128 else 0.93)
        if best is None or score > best[0] + 1e-9:
            best = (score, bn)
    return best[1]


def linear(a: torch.Tensor, wt: torch.Tensor, out: torch.Tensor, bias: Optional[torch.Tensor] = None,
           bias_group_rows: int = 0, residual: Optional[torch.Tensor] = None, flags: int = 0,
           block_n: Optional[int] = None, max_ctas: int = 0):
    """out[M, N_out] = epilogue(a[M, K] @ wt[N, K]^T)"""
    m, k, lda = _rows2d(a)
    n, k2 = wt.shape
    assert k == k2 and wt.is_contiguous()
    mo, no, ldd = _rows2d(out)
    geglu = bool(flags & EPI_GEGLU)
    assert mo == m and no == (n // 2 if geglu else n), (mo, m, no, n)
    bn = block_n or pick_block_n(n, geglu, m)
    e = _epi(bias, bias_group_rows, residual, flags)
    rc = _lib.lib().b200sd_linear(_p(a), ctypes.c_longlong(lda), _p(wt), _p(out), ctypes.c_longlong(ldd), m, n, k, bn,
                                  ctypes.byref(e), _dt(a), max_ctas, _stream())
    check(rc, f"b200sd_linear M={m} N={n} K={k} bn={bn}")
    _count()
    return out


def conv2d(x: torch.Tensor, wt: torch.Tensor, out: torch.Tensor, ksize: int, stride: int = 1, pad: int = 1,
           pad_end: Optional[int] = None, bias: Optional[torch.Tensor] = None, bias_group_rows: int = 0,
           residual: Optional[torch.Tensor] = None, flags: int = 0, block_n: Optional[int] = None, max_ctas: int = 0):
    """x [NB, H, W, C] NHWC (channel pitch x.stride(2)), wt [Cout, k*k*C]; out rows = output pixels."""
    nb, h, w, c = x.shape
    assert x.stride(3) == 1 and x.stride(1) == w * x.stride(2) and x.stride(0) == h * x.stride(1)
    cout, kk = wt.shape
    assert kk == ksize * ksize * c and wt.is_contiguous()
    pe = pad if pad_end is None else pad_end
    mo, no, ldd = _rows2d(out)
    bn = block_n or pick_block_n(cout, False, mo)
    e = _epi(bias, bias_group_rows, residual, flags)
    rc = _lib.lib().b200sd_conv2d(_p(x), ctypes.c_longlong(x.stride(2)), nb, h, w, c, _p(wt), ksize, stride, pad, pe,
                                  _p(out), ctypes.c_longlong(ldd), cout, bn, ctypes.byref(e), _dt(x), max_ctas,
                                  _stream())
    check(rc, f"b200sd_conv2d NB={nb} H={h} W={w} C={c} Cout={cout} k={ksize} s={stride}")
    _count()
    return out


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, heads: int, d: int, d_pad: int,
              scale: float, v_ones_col: bool = False, kv_len: Optional[torch.Tensor] = None):
    """q [B, Sq, >=heads*d_pad], k/v [B, Skv, >=heads*d_pad] (pitch = stride(1)), out [B, Sq, heads*d].
    v_ones_col: v[..., h*d_pad + d] == 1 for every head (softmax denominators come out of the P.V MMA).
    kv_len: int32 [B] on the device — row b attends to keys [0, kv_len[b]) only (b200sd_attention_varlen; the kernel
    reads the lengths, so a captured graph follows later writes to the tensor).  None: every row attends to all Skv."""
    b, sq, _ = q.shape
    skv = k.shape[1]
    for t in (q, k, v, out):
        assert t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    if kv_len is None:
        rc = _lib.lib().b200sd_attention(_p(q), ctypes.c_longlong(q.stride(1)), _p(k), ctypes.c_longlong(k.stride(1)),
                                         _p(v), ctypes.c_longlong(v.stride(1)), _p(out), ctypes.c_longlong(out.stride(1)),
                                         b, heads, sq, skv, d, d_pad, ctypes.c_float(scale), int(bool(v_ones_col)),
                                         _dt(q), _stream())
        check(rc, f"b200sd_attention B={b} h={heads} Sq={sq} Skv={skv} d={d}")
    else:
        assert kv_len.dtype == torch.int32 and kv_len.is_contiguous() and kv_len.numel() == b
        assert kv_len.device == q.device, "kv_len must live on the device"
        rc = _lib.lib().b200sd_attention_varlen(_p(q), ctypes.c_longlong(q.stride(1)), _p(k),
                                                ctypes.c_longlong(k.stride(1)), _p(v), ctypes.c_longlong(v.stride(1)),
                                                _p(out), ctypes.c_longlong(out.stride(1)), b, heads, sq, skv,
                                                _p(kv_len), d, d_pad, ctypes.c_float(scale), int(bool(v_ones_col)),
                                                _dt(q), _stream())
        check(rc, f"b200sd_attention_varlen B={b} h={heads} Sq={sq} Skv={skv} d={d}")
    _count()
    return out


_GN_FLOATS = {}


def groupnorm_stats_floats(nb: int, hw: int, c: int, groups: int) -> int:
    """fp32 elements a `stats` buffer for groupnorm() must hold (results + the reduction's scratch)"""
    key = (nb, hw, c, groups)
    n = _GN_FLOATS.get(key)
    if n is None:
        n = int(_lib.lib().b200sd_groupnorm_stats_floats(nb, hw, c, groups))
        if n < 0:
            raise _lib.B200SDError(f"groupnorm: unsupported shape C={c}")
        _GN_FLOATS[key] = n
    return n


def groupnorm(x: torch.Tensor, out: torch.Tensor, stats: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor,
              groups: int, eps: float, silu: bool):
    """x, out [NB, HW, C] (pitch = stride(1)); stats: flat fp32 buffer of groupnorm_stats_floats(...) elements,
    zero-filled once at allocation (may be shared by successive calls on one stream); its first NB*groups*2 elements
    receive (sum, sumsq) per (image, group) — deterministically, run to run.  Two launches: statistics, then apply."""
    nb, hw, c = x.shape
    assert x.stride(2) == 1 and out.stride(2) == 1 and x.stride(0) == hw * x.stride(1)
    assert stats.dtype == torch.float32 and stats.is_contiguous()
    assert stats.numel() >= groupnorm_stats_floats(nb, hw, c, groups), "stats buffer too small"
    rc = _lib.lib().b200sd_groupnorm(_p(x), ctypes.c_longlong(x.stride(1)), _p(out), ctypes.c_longlong(out.stride(1)), nb,
                                     hw, c, groups, _p(stats), _p(gamma), _p(beta), ctypes.c_float(eps), int(silu),
                                     _dt(x), _stream())
    check(rc, "b200sd_groupnorm")
    _count(2)
    return out


def layernorm(x: torch.Tensor, out: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5):
    rows, c, ldx = _rows2d(x)
    _, _, ldy = _rows2d(out)
    rc = _lib.lib().b200sd_layernorm(_p(x), ctypes.c_longlong(ldx), _p(out), ctypes.c_longlong(ldy), rows, c, _p(gamma),
                                     _p(beta), ctypes.c_float(eps), _dt(x), _stream())
    check(rc, "b200sd_layernorm")
    _count()
    return out


def upsample2x(x: torch.Tensor, out: torch.Tensor):
    nb, h, w, c = x.shape
    rc = _lib.lib().b200sd_upsample2x(_p(x), ctypes.c_longlong(x.stride(2)), _p(out), ctypes.c_longlong(out.stride(2)),
                                      nb, h, w, c, _dt(x), _stream())
    check(rc, "b200sd_upsample2x")
    _count()
    return out


def softmax_rows_(s: torch.Tensor, scale: float):
    rows, cols, lds = _rows2d(s)
    rc = _lib.lib().b200sd_softmax_rows(_p(s), ctypes.c_longlong(lds), rows, cols, ctypes.c_float(scale), _dt(s),
                                        _stream())
    check(rc, "b200sd_softmax_rows")
    _count()
    return s


def silu(x: torch.Tensor, out: torch.Tensor):
    assert x.is_contiguous() and out.is_contiguous()
    rc = _lib.lib().b200sd_silu(_p(x), _p(out), ctypes.c_longlong(x.numel()), _dt(x), _stream())
    check(rc, "b200sd_silu")
    _count()
    return out


def timestep_embedding(t: torch.Tensor, out: torch.Tensor):
    assert t.dtype == torch.float32 and t.is_contiguous()
    rc = _lib.lib().b200sd_timestep_embedding(_p(t), t.numel(), out.shape[1], _p(out), ctypes.c_longlong(out.stride(0)),
                                              _dt(out), _stream())
    check(rc, "b200sd_timestep_embedding")
    _count()
    return out


def fold_bias(emb: torch.Tensor, bias: torch.Tensor, table: torch.Tensor):
    t, c = table.shape
    assert table.dtype == torch.float32 and table.is_contiguous() and bias.numel() == c
    rc = _lib.lib().b200sd_fold_bias(_p(emb), ctypes.c_longlong(emb.stride(0)), _p(bias), _p(table), t, c, _dt(emb),
                                     _stream())
    check(rc, "b200sd_fold_bias")
    _count()
    return table


def select_step(table: torch.Tensor, step_counter: torch.Tensor, cur: torch.Tensor):
    assert table.dtype == torch.float32 and cur.dtype == torch.float32 and step_counter.dtype == torch.int32
    rc = _lib.lib().b200sd_select_step(_p(table), ctypes.c_longlong(table.shape[1]), _p(step_counter), _p(cur), _stream())
    check(rc, "b200sd_select_step")
    _count()
    return cur


def pack_unet_input(x: torch.Tensor, xin: torch.Tensor, in_scale: float = 1.0):
    """x fp32 [B, HW, 4]; xin [2B, HW, pitch]"""
    b, hw, _ = x.shape
    rc = _lib.lib().b200sd_pack_unet_input(_p(x), _p(xin), ctypes.c_longlong(xin.stride(1)), b, hw,
                                           ctypes.c_float(in_scale), _dt(xin), _stream())
    check(rc, "b200sd_pack_unet_input")
    _count()
    return xin


def cfg_ddim_step(eps: torch.Tensor, x: torch.Tensor, xin: torch.Tensor, cfg_scale: float, coef: torch.Tensor,
                  step_counter: torch.Tensor):
    b, hw, _ = x.shape
    rc = _lib.lib().b200sd_cfg_ddim_step(_p(eps), ctypes.c_longlong(eps.stride(1)), _p(x), _p(xin),
                                         ctypes.c_longlong(xin.stride(1)), b, hw, ctypes.c_float(cfg_scale), _p(coef),
                                         _p(step_counter), _dt(xin), _stream())
    check(rc, "b200sd_cfg_ddim_step")
    _count(2)


def cfg_euler_a_step(eps: torch.Tensor, x: torch.Tensor, noise: Optional[torch.Tensor], xin: torch.Tensor,
                     cfg_scale: float, coef: torch.Tensor, step_counter: torch.Tensor):
    b, hw, _ = x.shape
    rc = _lib.lib().b200sd_cfg_euler_a_step(_p(eps), ctypes.c_longlong(eps.stride(1)), _p(x), _p(noise), _p(xin),
                                            ctypes.c_longlong(xin.stride(1)), b, hw, ctypes.c_float(cfg_scale),
                                            _p(coef), _p(step_counter), _dt(xin), _stream())
    check(rc, "b200sd_cfg_euler_a_step")
    _count(2)


def cfg_dpmpp_2m_step(eps: torch.Tensor, x: torch.Tensor, old_denoised: torch.Tensor, xin: torch.Tensor,
                      cfg_scale: float, coef8: torch.Tensor, step_counter: torch.Tensor):
    """coef8 [steps, 8] fp32: {sigma, sigma_next/sigma, c1, c2, in_scale_next, 0, 0, 0} per step"""
    b, hw, _ = x.shape
    assert coef8.shape[-1] == 8 and old_denoised.shape == x.shape
    rc = _lib.lib().b200sd_cfg_dpmpp_2m_step(_p(eps), ctypes.c_longlong(eps.stride(1)), _p(x), _p(old_denoised), _p(xin),
                                             ctypes.c_longlong(xin.stride(1)), b, hw, ctypes.c_float(cfg_scale),
                                             _p(coef8), _p(step_counter), _dt(xin), _stream())
    check(rc, "b200sd_cfg_dpmpp_2m_step")
    _count(2)



# v-prediction twins of the three fused steps (b200sd_cfg_*_step_v): `v` is the UNet output [2B, HW, pitch] of a
# v-prediction model; the kernel converts the CFG-combined v to eps with its own pre-update fp32 x, then steps as above
def cfg_ddim_step_v(v: torch.Tensor, x: torch.Tensor, xin: torch.Tensor, cfg_scale: float, coef: torch.Tensor,
                    step_counter: torch.Tensor):
    """coef [steps, 4]: the DDIM rows {sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev)}"""
    b, hw, _ = x.shape
    rc = _lib.lib().b200sd_cfg_ddim_step_v(_p(v), ctypes.c_longlong(v.stride(1)), _p(x), _p(xin),
                                           ctypes.c_longlong(xin.stride(1)), b, hw, ctypes.c_float(cfg_scale), _p(coef),
                                           _p(step_counter), _dt(xin), _stream())
    check(rc, "b200sd_cfg_ddim_step_v")
    _count(2)


def cfg_euler_a_step_v(v: torch.Tensor, x: torch.Tensor, noise: Optional[torch.Tensor], xin: torch.Tensor,
                       cfg_scale: float, coef8: torch.Tensor, step_counter: torch.Tensor):
    """coef8 [steps, 8]: {sigma, sigma_down, sigma_up, in_scale_next, kx, kv, 0, 0}"""
    b, hw, _ = x.shape
    assert coef8.shape[-1] == 8
    rc = _lib.lib().b200sd_cfg_euler_a_step_v(_p(v), ctypes.c_longlong(v.stride(1)), _p(x), _p(noise), _p(xin),
                                              ctypes.c_longlong(xin.stride(1)), b, hw, ctypes.c_float(cfg_scale),
                                              _p(coef8), _p(step_counter), _dt(xin), _stream())
    check(rc, "b200sd_cfg_euler_a_step_v")
    _count(2)


def cfg_dpmpp_2m_step_v(v: torch.Tensor, x: torch.Tensor, old_denoised: torch.Tensor, xin: torch.Tensor,
                        cfg_scale: float, coef8: torch.Tensor, step_counter: torch.Tensor):
    """coef8 [steps, 8]: {sigma, sigma_next/sigma, c1, c2, in_scale_next, kx, kv, 0}"""
    b, hw, _ = x.shape
    assert coef8.shape[-1] == 8 and old_denoised.shape == x.shape
    rc = _lib.lib().b200sd_cfg_dpmpp_2m_step_v(_p(v), ctypes.c_longlong(v.stride(1)), _p(x), _p(old_denoised), _p(xin),
                                               ctypes.c_longlong(xin.stride(1)), b, hw, ctypes.c_float(cfg_scale),
                                               _p(coef8), _p(step_counter), _dt(xin), _stream())
    check(rc, "b200sd_cfg_dpmpp_2m_step_v")
    _count(2)

def image_to_nhwc(img_u8: torch.Tensor, out: torch.Tensor):
    """img_u8 uint8 [B, HW, 3] -> out [B, HW, pitch] channels 0..2 = 2*x/255 - 1"""
    b, hw, _ = img_u8.shape
    assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous()
    rc = _lib.lib().b200sd_image_to_nhwc(_p(img_u8), _p(out), ctypes.c_longlong(out.stride(1)), b, hw, _dt(out), _stream())
    check(rc, "b200sd_image_to_nhwc")
    _count()
    return out


def hint_to_nhwc(img_u8: torch.Tensor, out: torch.Tensor):
    """img_u8 uint8 [B, HW, 3] -> out [B, HW, pitch]: channels 0..2 = x/255, the rest of the row 0 (ControlNet hint)"""
    b, hw, _ = img_u8.shape
    assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous()
    assert out.shape[:2] == (b, hw) and out.stride(2) == 1 and out.stride(0) == hw * out.stride(1)
    rc = _lib.lib().b200sd_hint_to_nhwc(_p(img_u8), _p(out), ctypes.c_longlong(out.stride(1)), b, hw, _dt(out), _stream())
    check(rc, "b200sd_hint_to_nhwc")
    _count()
    return out


def unpack_latent(moments: torch.Tensor, x: torch.Tensor, scale: float):
    """moments [B, HW, pitch] (first 4 channels = posterior mean) -> x fp32 [B, HW, 4] = mean * scale"""
    b, hw, _ = moments.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    rc = _lib.lib().b200sd_unpack_latent(_p(moments), ctypes.c_longlong(moments.stride(1)), _p(x), b, hw,
                                         ctypes.c_float(scale), _dt(moments), _stream())
    check(rc, "b200sd_unpack_latent")
    _count()
    return x


def quantize_u8(img: torch.Tensor, out: torch.Tensor):
    """img [B, HW, pitch>=3] -> out uint8 [B, HW, 3]"""
    b, hw, _ = img.shape
    assert out.dtype == torch.uint8 and out.is_contiguous()
    rc = _lib.lib().b200sd_quantize_u8(_p(img), ctypes.c_longlong(img.stride(1)), _p(out), b, hw, _dt(img), _stream())
    check(rc, "b200sd_quantize_u8")
    _count()
    return out


def blend_latent(x: torch.Tensor, init: torch.Tensor, latmask: torch.Tensor):
    """x, init fp32 [B, HW, 4]; latmask fp32 [HW]: x = x * latmask + init * (1 - latmask), in place"""
    b, hw, _ = x.shape
    assert x.dtype == init.dtype == latmask.dtype == torch.float32 and x.is_contiguous() and init.is_contiguous()
    assert init.shape == x.shape and latmask.shape == (hw,) and latmask.is_contiguous()
    rc = _lib.lib().b200sd_blend_latent(_p(x), _p(init), _p(latmask), b, hw, _stream())
    check(rc, "b200sd_blend_latent")
    _count()
    return x


def resize_latent_bilinear(x: torch.Tensor, y: torch.Tensor, h: int, w: int, ho: int, wo: int):
    """x fp32 [B, h*w, 4] -> y fp32 [B, ho*wo, 4] (F.interpolate bilinear, align_corners=False, no antialias)"""
    b = x.shape[0]
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous()
    assert x.shape == (b, h * w, 4) and y.shape == (b, ho * wo, 4)
    rc = _lib.lib().b200sd_resize_latent_bilinear(_p(x), _p(y), b, h, w, ho, wo, _stream())
    check(rc, "b200sd_resize_latent_bilinear")
    _count()
    return y


def cfg_eps(eps: torch.Tensor, e: torch.Tensor, cfg_scale: float):
    """eps [2B, HW, pitch] (cond | uncond) -> e fp32 [B, HW, 4] = eu + cfg * (ec - eu)"""
    b, hw, _ = e.shape
    assert e.dtype == torch.float32 and e.is_contiguous()
    rc = _lib.lib().b200sd_cfg_eps(_p(eps), ctypes.c_longlong(eps.stride(1)), _p(e), b, hw, ctypes.c_float(cfg_scale),
                                   _dt(eps), _stream())
    check(rc, "b200sd_cfg_eps")
    _count()
    return e


def latent_lincomb(dst: torch.Tensor, srcs, coef: torch.Tensor, col0: int, step_counter: torch.Tensor,
                   xin: Optional[torch.Tensor] = None, idx_col: int = -1):
    """dst fp32 [B, HW, 4] = sum_k coef[*step, col0 + k] * srcs[k]; a source of shape [R, B, HW, 4] is a stack indexed by
    (int)coef[*step, idx_col]; with `xin` the result * coef[*step, col0 + len(srcs)] is packed as the next UNet input."""
    b, hw, _ = dst.shape
    n = len(srcs)
    assert dst.dtype == torch.float32 and dst.is_contiguous() and coef.dtype == torch.float32 and coef.is_contiguous()
    ptrs = (ctypes.c_void_p * n)(*[s.data_ptr() for s in srcs])
    strides = (ctypes.c_longlong * n)(*[(s.stride(0) if s.dim() == 4 else 0) for s in srcs])
    for s in srcs:
        assert s.dtype == torch.float32 and s.is_contiguous() and s.shape[-3:] == dst.shape
    rc = _lib.lib().b200sd_latent_lincomb(_p(dst), ptrs, strides, n, _p(coef), coef.shape[1], col0, idx_col,
                                          _p(step_counter), _p(xin),
                                          ctypes.c_longlong(0 if xin is None else xin.stride(1)), b, hw,
                                          F16 if xin is None else _dt(xin), _stream())
    check(rc, "b200sd_latent_lincomb")
    _count()
    return dst


def bump_step(step_counter: torch.Tensor):
    rc = _lib.lib().b200sd_bump_step(_p(step_counter), _stream())
    check(rc, "b200sd_bump_step")
    _count()


# ---- hires fix upscalers (b200sd/upscale.py builds the tables these take)
def conv2d_scaled(x: torch.Tensor, wt: torch.Tensor, out: torch.Tensor, bias: Optional[torch.Tensor] = None,
                  residual: Optional[torch.Tensor] = None, res_scale: float = 1.0, lrelu: bool = False,
                  block_n: Optional[int] = None, max_ctas: int = 0):
    """3x3 / pad 1 conv with the RRDBNet epilogue: v = acc + bias, LeakyReLU(0.2) if `lrelu`, then
    out = residual + res_scale * v when a residual is given.  x [NB, H, W, C] NHWC (channel pitch x.stride(2))."""
    nb, h, w, c = x.shape
    assert x.stride(3) == 1 and x.stride(1) == w * x.stride(2) and x.stride(0) == h * x.stride(1)
    cout, kk = wt.shape
    assert kk == 9 * c and wt.is_contiguous()
    mo, no, ldd = _rows2d(out)
    bn = block_n or (64 if cout % 64 == 0 else 32)
    e = _epi(bias, 0, residual, EPI_LRELU if lrelu else 0)
    rc = _lib.lib().b200sd_conv2d_scaled(_p(x), ctypes.c_longlong(x.stride(2)), nb, h, w, c, _p(wt), 3, 1, 1, 1,
                                         _p(out), ctypes.c_longlong(ldd), cout, bn, ctypes.byref(e),
                                         ctypes.c_float(res_scale), _dt(x), max_ctas, _stream())
    check(rc, f"b200sd_conv2d_scaled NB={nb} H={h} W={w} C={c} Cout={cout}")
    _count()
    return out


def resample_u8(x: torch.Tensor, out: torch.Tensor, vertical: bool, bounds: torch.Tensor, kk: torch.Tensor):
    """one Pillow resampling pass, uint8 [B, H, W, 3] -> [B, Ho, Wo, 3]; bounds int32 [n, 2], kk int32 [n, ksize] on the
    device"""
    b, hi, wi, _ = x.shape
    _, ho, wo, _ = out.shape
    assert x.dtype == out.dtype == torch.uint8 and x.is_contiguous() and out.is_contiguous()
    assert bounds.dtype == kk.dtype == torch.int32 and bounds.is_contiguous() and kk.is_contiguous()
    assert bounds.shape == ((ho if vertical else wo), 2) and kk.shape[0] == bounds.shape[0]
    rc = _lib.lib().b200sd_resample_u8(_p(x), _p(out), b, hi, wi, ho, wo, int(vertical), _p(bounds), _p(kk),
                                       kk.shape[1], _stream())
    check(rc, "b200sd_resample_u8")
    _count()
    return out


def combine_tiles_u8(tiles: torch.Tensor, out: torch.Tensor, ys: torch.Tensor, xs: torch.Tensor, mask: torch.Tensor,
                     overlap: int):
    """tiles uint8 [B * rows * cols, th, tw, 3] -> out uint8 [B, H, W, 3] (sdwui combine_grid); ys/xs int32, mask uint8
    [overlap] on the device"""
    b, hh, ww, _ = out.shape
    _, th, tw, _ = tiles.shape
    rows, cols = ys.numel(), xs.numel()
    assert tiles.shape[0] == b * rows * cols and tiles.dtype == out.dtype == mask.dtype == torch.uint8
    assert tiles.is_contiguous() and out.is_contiguous() and ys.dtype == xs.dtype == torch.int32
    rc = _lib.lib().b200sd_combine_tiles_u8(_p(tiles), _p(out), b, hh, ww, th, tw, rows, cols, _p(ys), _p(xs), _p(mask),
                                            overlap, _stream())
    check(rc, "b200sd_combine_tiles_u8")
    _count()
    return out


def quantize_unit_u8(img: torch.Tensor, out: torch.Tensor):
    """img [B, HW, pitch>=3] -> out uint8 [B, HW, 3] = round(255 * clamp(v, 0, 1))"""
    b, hw, _ = img.shape
    assert out.dtype == torch.uint8 and out.is_contiguous() and img.stride(2) == 1 and img.stride(0) == hw * img.stride(1)
    rc = _lib.lib().b200sd_quantize_unit_u8(_p(img), ctypes.c_longlong(img.stride(1)), _p(out), b, hw, _dt(img),
                                            _stream())
    check(rc, "b200sd_quantize_unit_u8")
    _count()
    return out


def scaled_add_(y: torch.Tensor, x: torch.Tensor, alpha: float):
    """y += alpha * x over [rows, C] (row pitches from stride(-2)), in place"""
    rows, c, ldy = _rows2d(y)
    rx, cx, ldx = _rows2d(x)
    assert (rx, cx) == (rows, c) and x.dtype == y.dtype
    rc = _lib.lib().b200sd_scaled_add(_p(x), ctypes.c_longlong(ldx), _p(y), ctypes.c_longlong(ldy),
                                      ctypes.c_longlong(rows), c, ctypes.c_float(alpha), _dt(y), _stream())
    check(rc, "b200sd_scaled_add")
    _count()
    return y


def resize_latent_table(x: torch.Tensor, y: torch.Tensor, h: int, w: int, ho: int, wo: int, tx, ty):
    """x fp32 [B, h*w, 4] -> y fp32 [B, ho*wo, 4] by the separable tables tx = (ix int32 [wo, kx], wx fp32 [wo, kx]) and
    ty = (iy [ho, ky], wy [ho, ky]) on the device"""
    b = x.shape[0]
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous()
    assert x.shape == (b, h * w, 4) and y.shape == (b, ho * wo, 4)
    (ix, wx), (iy, wy) = tx, ty
    assert ix.shape == wx.shape and ix.shape[0] == wo and iy.shape == wy.shape and iy.shape[0] == ho
    rc = _lib.lib().b200sd_resize_latent_table(_p(x), _p(y), b, h, w, ho, wo, _p(ix), _p(wx), ix.shape[1], _p(iy),
                                               _p(wy), iy.shape[1], _stream())
    check(rc, "b200sd_resize_latent_table")
    _count()
    return y
