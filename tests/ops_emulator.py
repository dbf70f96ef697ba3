"""CPU emulation of b200sd.ops with identical signatures — TEST INFRASTRUCTURE.

Lets the host-side program construction (buffer plan, channel-slice views, weight packing, per-step bias table,
sampler bookkeeping) run on a machine without a GPU: tests monkeypatch `b200sd.ops.<name>` with these functions and
compare the programs' results with the oracle.  Never imported by the product.
"""
import math

import torch
import torch.nn.functional as F

EPI_GEGLU = 1
EPI_SILU = 2


def _rows(t):
    return t.reshape(-1, t.shape[-1]) if t.is_contiguous() else t.flatten(0, -2)


def _store(out, val):
    out.copy_(val.reshape(out.shape).to(out.dtype))


def linear(a, wt, out, bias=None, bias_group_rows=0, residual=None, flags=0, block_n=None, max_ctas=0):
    a2 = a.reshape(-1, a.shape[-1]).float()
    y = a2 @ wt.float().t()
    geglu = bool(flags & EPI_GEGLU)
    if bias is not None:
        if bias_group_rows > 0:
            y = y + bias.reshape(-1, y.shape[1]).repeat_interleave(bias_group_rows, dim=0)[: y.shape[0]]
        else:
            y = y + bias.reshape(1, -1)
    if geglu:
        bn = block_n or pick_block_n(wt.shape[0], True)
        t = y.reshape(y.shape[0], -1, 2, bn // 2)
        y = (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(y.shape[0], -1)
    if residual is not None:
        y = y + residual.reshape(-1, residual.shape[-1]).float()
    if flags & EPI_SILU:
        y = F.silu(y)
    _store(out, y)
    return out


def pick_block_n(n, geglu=False):
    for bn in (160, 128, 96, 64, 32):
        if n % bn == 0 and (not geglu or bn % 64 == 0):
            return bn
    raise ValueError(n)


def conv2d(x, wt, out, ksize, stride=1, pad=1, pad_end=None, bias=None, bias_group_rows=0, residual=None, flags=0,
           block_n=None, max_ctas=0):
    nb, h, w, c = x.shape
    cout = wt.shape[0]
    pe = pad if pad_end is None else pad_end
    wk = wt.float().reshape(cout, ksize, ksize, c).permute(0, 3, 1, 2)
    xi = F.pad(x.float().permute(0, 3, 1, 2), (pad, pe, pad, pe))
    y = F.conv2d(xi, wk, stride=stride).permute(0, 2, 3, 1).reshape(-1, cout)
    if bias is not None:
        if bias_group_rows > 0:
            y = y + bias.reshape(-1, cout).repeat_interleave(bias_group_rows, dim=0)[: y.shape[0]]
        else:
            y = y + bias.reshape(1, -1)
    if residual is not None:
        y = y + residual.reshape(-1, residual.shape[-1]).float()
    if flags & EPI_SILU:
        y = F.silu(y)
    _store(out, y)
    return out


def attention(q, k, v, out, heads, d, d_pad, scale, v_ones_col=False):
    b, sq, _ = q.shape
    skv = k.shape[1]
    qh = q.float().reshape(b, sq, heads, d_pad)[..., :d].permute(0, 2, 1, 3)
    kh = k.float().reshape(b, skv, heads, d_pad)[..., :d].permute(0, 2, 1, 3)
    if v_ones_col:
        assert bool((v.float().reshape(b, skv, heads, d_pad)[..., d] == 1).all()), "V lacks its ones column"
    vh = v.float().reshape(b, skv, heads, d_pad)[..., :d].permute(0, 2, 1, 3)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    _store(out, (p @ vh).permute(0, 2, 1, 3).reshape(b, sq, heads * d))
    return out


def groupnorm_stats_floats(nb, hw, c, groups):
    return nb * groups * 2


def groupnorm(x, out, stats, gamma, beta, groups, eps, silu, mode=0):
    y = F.group_norm(x.float().permute(0, 2, 1), groups, gamma, beta, eps).permute(0, 2, 1)
    if silu:
        y = F.silu(y)
    _store(out, y)
    return out


def layernorm(x, out, gamma, beta, eps=1e-5):
    _store(out, F.layer_norm(x.float(), (x.shape[-1],), gamma, beta, eps))
    return out


def upsample2x(x, out):
    _store(out, x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    return out


def softmax_rows_(s, scale):
    s.copy_(torch.softmax(s.float() * scale, dim=-1).to(s.dtype))
    return s


def silu(x, out):
    _store(out, F.silu(x.float()))
    return out


def timestep_embedding(t, out):
    half = out.shape[1] // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    _store(out, torch.cat([torch.cos(args), torch.sin(args)], dim=-1))
    return out


def fold_bias(emb, bias, table):
    table.copy_(emb.float() + bias[None])
    return table


def select_step(table, step_counter, cur):
    cur.copy_(table[int(step_counter.item())])
    return cur


def pack_unet_input(x, xin, in_scale=1.0):
    b = x.shape[0]
    v = (x * in_scale).to(xin.dtype)
    xin[:b, :, :4] = v
    xin[b:2 * b, :, :4] = v
    return xin


def cfg_ddim_step(eps, x, xin, cfg_scale, coef, step_counter):
    b = x.shape[0]
    s = int(step_counter.item())
    sa, s1a, sap, s1ap = (float(c) for c in coef[s])
    ec, eu = eps[:b, :, :4].float(), eps[b:, :, :4].float()
    e = eu + cfg_scale * (ec - eu)
    x0 = (x - s1a * e) / sa
    x.copy_(sap * x0 + s1ap * e)
    pack_unet_input(x, xin, 1.0)
    step_counter += 1


def cfg_euler_a_step(eps, x, noise, xin, cfg_scale, coef, step_counter):
    b = x.shape[0]
    s = int(step_counter.item())
    sigma, sdown, sup, in_next = (float(c) for c in coef[s])
    ec, eu = eps[:b, :, :4].float(), eps[b:, :, :4].float()
    e = eu + cfg_scale * (ec - eu)
    xn = x + e * (sdown - sigma)
    if noise is not None and sup > 0:
        xn = xn + noise[s] * sup
    x.copy_(xn)
    pack_unet_input(x, xin, in_next)
    step_counter += 1


def cfg_dpmpp_2m_step(eps, x, old_denoised, xin, cfg_scale, coef8, step_counter):
    b = x.shape[0]
    s = int(step_counter.item())
    sigma, a, c1, c2, in_next = (float(c) for c in coef8[s][:5])
    ec, eu = eps[:b, :, :4].float(), eps[b:, :, :4].float()
    e = eu + cfg_scale * (ec - eu)
    dn = x - sigma * e
    dd = c1 * dn - c2 * old_denoised if c2 != 0 else dn
    x.copy_(a * x + (1.0 - a) * dd)
    old_denoised.copy_(dn)
    pack_unet_input(x, xin, in_next)
    step_counter += 1


def quantize_u8(img, out):
    v = ((img[..., :3].float() + 1.0) * 0.5).clamp(0, 1)
    out.copy_((255.0 * v).to(torch.uint8))
    return out


def image_to_nhwc(img_u8, out):
    out[..., :3] = (img_u8.float() * (2.0 / 255.0) - 1.0).to(out.dtype)
    return out


def unpack_latent(moments, x, scale):
    x.copy_(moments[..., :4].float() * scale)
    return x


def blend_latent(x, init, latmask):
    m = latmask[None, :, None]
    x.copy_(x * m + init * (1.0 - m))
    return x


def resize_latent_bilinear(x, y, h, w, ho, wo):
    b = x.shape[0]
    t = F.interpolate(x.reshape(b, h, w, 4).permute(0, 3, 1, 2), size=(ho, wo), mode="bilinear", antialias=False)
    y.copy_(t.permute(0, 2, 3, 1).reshape(b, ho * wo, 4))
    return y


def cfg_eps(eps, e, cfg_scale):
    b = e.shape[0]
    ec, eu = eps[:b, :, :4].float(), eps[b:, :, :4].float()
    e.copy_(eu + cfg_scale * (ec - eu))
    return e


def latent_lincomb(dst, srcs, coef, col0, step_counter, xin=None, idx_col=-1):
    row = int(step_counter.item())
    idx = int(coef[row, idx_col]) if idx_col >= 0 else 0
    acc = torch.zeros_like(dst)
    for k, s in enumerate(srcs):
        w = float(coef[row, col0 + k])
        if w != 0.0:
            acc = acc + w * (s[idx] if s.dim() == 4 else s)
    dst.copy_(acc)
    if xin is not None:
        pack_unet_input(dst, xin, float(coef[row, col0 + len(srcs)]))
    return dst


def bump_step(step_counter):
    step_counter += 1


ALL = ["cfg_eps", "latent_lincomb", "bump_step", "resize_latent_bilinear", "blend_latent", "linear", "pick_block_n", "conv2d", "attention", "groupnorm", "groupnorm_stats_floats", "layernorm", "upsample2x", "softmax_rows_", "silu",
       "timestep_embedding", "fold_bias", "select_step", "pack_unet_input", "cfg_ddim_step", "cfg_euler_a_step", "cfg_dpmpp_2m_step",
       "quantize_u8", "image_to_nhwc", "unpack_latent"]


def install(monkeypatch, ops_module):
    import sys
    me = sys.modules[__name__]
    for name in ALL:
        monkeypatch.setattr(ops_module, name, getattr(me, name))
