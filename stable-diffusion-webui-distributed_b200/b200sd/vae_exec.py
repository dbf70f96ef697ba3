"""kl-f8 VAE decoder / encoder as static programs of libb200sd kernels (NHWC fp16).

Decoder: stands in for upstream `AutoencoderKL.decode` (ldm/modules/diffusionmodules/model.py::Decoder) + sdwui's
clamp/255/uint8 conversion — the "final VAE decode" of the north star (SURVEY.md §8 a-ext x11).
Encoder: `AutoencoderKL.encode(...).mean` (model.py::Encoder + quant_conv) for img2img (§8 a-ext x12) and for the
conditioning image of inpainting models (a masked program of its own); its Downsample
(pad (0,1,0,1), 3x3 stride 2, no padding) is the conv kernel with pad=0 / pad_end=1 and TMA elementStrides=2.

The single-head d=C mid-block attention is expressed with the GEMM kernel: per image S = q k^T, row softmax,
V^T = Wv h^T (so P.V needs no transpose), O = P V^T^T; the v bias is folded into proj_out's bias (softmax rows sum
to one, so P (V0 + 1 bv^T) = P V0 + bv exactly).
"""
from typing import Dict, List

import torch

from . import ops
from .config import VAE_PREFIX, VAEConfig
from .unet_exec import Pool, emit_conv3
from .weights import pack_conv


class _Packer:
    """ldm VAE state_dict -> kernel layouts on `device` (shared by decoder and encoder)."""

    def __init__(self, sd, device, dtype):
        self.sd, self.device, self.dtype = sd, device, dtype
        self.t: Dict[str, torch.Tensor] = {}
        self.p = VAE_PREFIX

    def dev(self, t, dt=None):
        return t.to(device=self.device, dtype=dt or self.dtype).contiguous()

    def conv(self, name, key, cin_pad=0, cout_pad=0):
        self.t[name + ".w"] = self.dev(pack_conv(self.sd[self.p + key + ".weight"], cin_pad, cout_pad))
        b = self.sd[self.p + key + ".bias"]
        if cout_pad > b.numel():
            b = torch.cat([b, b.new_zeros(cout_pad - b.numel())])
        self.t[name + ".b"] = self.dev(b, torch.float32)

    def norm(self, name, key):
        self.t[name + ".g"] = self.dev(self.sd[self.p + key + ".weight"], torch.float32)
        self.t[name + ".beta"] = self.dev(self.sd[self.p + key + ".bias"], torch.float32)

    def res(self, name, key, cin, cout):
        self.norm(name + ".gn1", key + ".norm1")
        self.conv(name + ".conv1", key + ".conv1")
        self.norm(name + ".gn2", key + ".norm2")
        self.conv(name + ".conv2", key + ".conv2")
        if cin != cout:
            self.conv(name + ".skip", key + ".nin_shortcut")

    def attn(self, key, c):
        self.norm("attn.norm", key + ".norm")
        for n in ("q", "k", "v", "proj_out"):
            self.conv("attn." + n, f"{key}.{n}")
        wp = self.sd[self.p + key + ".proj_out.weight"].reshape(c, c).double()
        bv = self.sd[self.p + key + ".v.bias"].double()
        self.t["attn.proj_out.b"] = self.dev((self.sd[self.p + key + ".proj_out.bias"].double() + wp @ bv).float(),
                                             torch.float32)


class VAEDecoderWeights:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: VAEConfig, device, dtype=torch.float16):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        pk = _Packer(sd, device, dtype)
        self.t = pk.t
        pk.conv("post_quant", "post_quant_conv", cin_pad=64, cout_pad=64)  # 1x1 z->z, both sides padded to 64
        nlev = len(cfg.ch_mult)
        cin = cfg.ch * cfg.ch_mult[-1]
        pk.conv("conv_in", "decoder.conv_in", cin_pad=64)
        pk.res("mid1", "decoder.mid.block_1", cin, cin)
        pk.attn("decoder.mid.attn_1", cin)
        pk.res("mid2", "decoder.mid.block_2", cin, cin)
        self.levels = []
        for lvl in reversed(range(nlev)):
            cout = cfg.ch * cfg.ch_mult[lvl]
            blocks = []
            for b in range(cfg.num_res_blocks + 1):
                pk.res(f"up{lvl}.{b}", f"decoder.up.{lvl}.block.{b}", cin, cout)
                blocks.append((cin, cout))
                cin = cout
            if lvl != 0:
                pk.conv(f"up{lvl}.upsample", f"decoder.up.{lvl}.upsample.conv")
            self.levels.append((lvl, blocks))
        pk.norm("norm_out", "decoder.norm_out")
        pk.conv("conv_out", "decoder.conv_out", cout_pad=32)
        self.mid_ch = cfg.ch * cfg.ch_mult[-1]
        self.out_ch = cin


class VAEEncoderWeights:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: VAEConfig, device, dtype=torch.float16):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        pk = _Packer(sd, device, dtype)
        self.t = pk.t
        pk.conv("conv_in", "encoder.conv_in", cin_pad=64)   # RGB padded to 64 input channels
        nlev = len(cfg.ch_mult)
        cin = cfg.ch
        self.levels = []
        for lvl in range(nlev):
            cout = cfg.ch * cfg.ch_mult[lvl]
            blocks = []
            for b in range(cfg.num_res_blocks):
                pk.res(f"down{lvl}.{b}", f"encoder.down.{lvl}.block.{b}", cin, cout)
                blocks.append((cin, cout))
                cin = cout
            if lvl != nlev - 1:
                pk.conv(f"down{lvl}.downsample", f"encoder.down.{lvl}.downsample.conv")
            self.levels.append((lvl, blocks))
        pk.res("mid1", "encoder.mid.block_1", cin, cin)
        pk.attn("encoder.mid.attn_1", cin)
        pk.res("mid2", "encoder.mid.block_2", cin, cin)
        pk.norm("norm_out", "encoder.norm_out")
        pk.conv("conv_out", "encoder.conv_out", cout_pad=64)      # 2z = 8 moment channels, padded to 64
        pk.conv("quant", "quant_conv", cin_pad=64, cout_pad=64)   # 1x1 on the moments
        self.mid_ch = cin


class _VAEProgram:
    """Shared layer emitters: every op is recorded once, run() replays them (allocation- and sync-free)."""

    def __init__(self, weights, b: int, tiling: bool = False):
        """tiling: every 3x3 conv with padding 1 pads circularly (sdwui's tiling option)"""
        self.w, self.b = weights, b
        self.circular = tiling
        self.dev, self.dt = weights.device, weights.dtype
        self.pool = Pool(self.dev, self.dt)
        self.ops: List = []
        self.gn_stats: List = []
        self.gn_need = 0

    def _finish(self):
        # one statistics buffer serves every GroupNorm (they run back to back on one stream); zeroed once, here
        self.stats_all = torch.zeros((max(1, self.gn_need),), device=self.dev, dtype=torch.float32)
        for holder in self.gn_stats:
            holder[0] = self.stats_all

    def _emit(self, fn, *a, **k):
        self.ops.append((fn, a, k))

    def _gn(self, x, out, name, silu):
        holder = [None]
        self.gn_stats.append(holder)
        self.gn_need = max(self.gn_need, ops.groupnorm_stats_floats(x.shape[0], x.shape[1], x.shape[2], 32))
        g, beta = self.w.t[name + ".g"], self.w.t[name + ".beta"]
        self._emit(lambda: ops.groupnorm(x, out, holder[0], g, beta, 32, 1e-6, silu))

    def _res(self, name, x, cin, cout, h, wd):
        b, hw, t = self.b, h * wd, self.w.t
        a = self.pool.get(b, hw, cin)
        self._gn(x, a, name + ".gn1", True)
        c1 = self.pool.get(b, hw, cout)
        emit_conv3(self, a, h, wd, t[name + ".conv1.w"], c1, bias=t[name + ".conv1.b"])
        self.pool.put(a)
        a2 = self.pool.get(b, hw, cout)
        self._gn(c1, a2, name + ".gn2", True)
        self.pool.put(c1)
        if cin != cout:
            s = self.pool.get(b, hw, cout)
            self._emit(ops.linear, x, t[name + ".skip.w"], s, bias=t[name + ".skip.b"])
        else:
            s = x
        out = self.pool.get(b, hw, cout)
        emit_conv3(self, a2, h, wd, t[name + ".conv2.w"], out, bias=t[name + ".conv2.b"], residual=s)
        self.pool.put(a2)
        if s is not x:
            self.pool.put(s)
        return out

    def _attn(self, x, c, h, wd):
        b, s, t = self.b, h * wd, self.w.t
        hn = self.pool.get(b, s, c)
        self._gn(x, hn, "attn.norm", False)
        q = self.pool.get(b, s, c)
        k = self.pool.get(b, s, c)
        self._emit(ops.linear, hn, t["attn.q.w"], q, bias=t["attn.q.b"])
        self._emit(ops.linear, hn, t["attn.k.w"], k, bias=t["attn.k.b"])
        o = self.pool.get(b, s, c)
        scores = self.pool.get(s, s)
        vt = self.pool.get(c, s)
        for i in range(b):
            self._emit(ops.linear, q[i], k[i], scores)                  # S = q k^T        [s, s]
            self._emit(ops.softmax_rows_, scores, float(c) ** -0.5)     # softmax(S * c^-1/2)
            self._emit(ops.linear, t["attn.v.w"], hn[i], vt)            # V^T = Wv h^T      [c, s]
            self._emit(ops.linear, scores, vt, o[i])                    # O = P V           [s, c]
        out = self.pool.get(b, s, c)
        self._emit(ops.linear, o, t["attn.proj_out.w"], out, bias=t["attn.proj_out.b"], residual=x)
        for tmp in (hn, q, k, o, scores, vt):
            self.pool.put(tmp)
        return out

    def _mid(self, x, c, h, wd):
        for stage in ("mid1", "attn", "mid2"):
            y = self._attn(x, c, h, wd) if stage == "attn" else self._res(stage, x, c, c, h, wd)
            self.pool.put(x)
            x = y
        return x

    def run(self):
        for fn, a, k in self.ops:
            fn(*a, **k)


class VAEDecoderProgram(_VAEProgram):
    """Decode `b` latents of size h x w -> uint8 [b, 8h*.., 3]."""

    def __init__(self, w: VAEDecoderWeights, b: int, h: int, wd: int, tiling: bool = False):
        super().__init__(w, b, tiling)
        self.h, self.wd = h, wd
        self.zin = torch.zeros((2 * b, h * wd, 64), device=self.dev, dtype=self.dt)  # pack_unet_input writes both halves
        self._build()
        self._finish()

    def _build(self):
        b, h, wd, t = self.b, self.h, self.wd, self.w.t
        c = self.w.mid_ch
        z = self.pool.get(b, h * wd, 64)
        self._emit(ops.linear, self.zin[:b], t["post_quant.w"], z, bias=t["post_quant.b"])
        x = self.pool.get(b, h * wd, c)
        emit_conv3(self, z, h, wd, t["conv_in.w"], x, bias=t["conv_in.b"])
        self.pool.put(z)
        x = self._mid(x, c, h, wd)
        for lvl, blocks in self.w.levels:
            for i, (cin, cout) in enumerate(blocks):
                y = self._res(f"up{lvl}.{i}", x, cin, cout, h, wd)
                self.pool.put(x)
                x = y
                c = cout
            if lvl != 0:
                up = self.pool.get(b, 4 * h * wd, c)
                self._emit(ops.upsample2x, x.unflatten(1, (h, wd)), up.unflatten(1, (2 * h, 2 * wd)))
                self.pool.put(x)
                h, wd = 2 * h, 2 * wd
                x = self.pool.get(b, h * wd, c)
                emit_conv3(self, up, h, wd, t[f"up{lvl}.upsample.w"], x, bias=t[f"up{lvl}.upsample.b"])
                self.pool.put(up)
        a = self.pool.get(b, h * wd, c)
        self._gn(x, a, "norm_out", True)
        self.pool.put(x)
        self.img = torch.empty((b, h * wd, 32), device=self.dev, dtype=self.dt)   # RGB in channels 0..2, in [-1, 1]
        emit_conv3(self, a, h, wd, t["conv_out.w"], self.img, bias=t["conv_out.b"])
        self.pool.put(a)
        self.out_h, self.out_w = h, wd
        self.u8 = torch.empty((b, h * wd, 3), device=self.dev, dtype=torch.uint8)
        self._emit(ops.quantize_u8, self.img, self.u8)

    def set_latents(self, x: torch.Tensor, scale_factor: float):
        """x fp32 [b, h*w, 4] (scaled latents): writes x / scale_factor into the padded fp16 input."""
        ops.pack_unet_input(x, self.zin, 1.0 / scale_factor)

    def run(self):
        super().run()
        return self.u8


class VAEEncoderProgram(_VAEProgram):
    """Encode `b` RGB images of size H x W (uint8) -> scaled latents fp32 [b, (H/f)*(W/f), 4] (posterior mean).
    masked: the encoded image is an inpainting model's conditioning image s * (1 - weight * [mask >= 128]) of the uint8
    images, with the mask and weight of set_condition."""

    def __init__(self, w: VAEEncoderWeights, b: int, height: int, width: int, tiling: bool = False, masked: bool = False):
        super().__init__(w, b, tiling)
        self.height, self.width = height, width
        self.img_u8 = torch.zeros((b, height * width, 3), device=self.dev, dtype=torch.uint8)
        self.xin = torch.zeros((b, height * width, 64), device=self.dev, dtype=self.dt)  # RGB in channels 0..2
        if masked:
            self.mask_u8 = torch.zeros((height * width,), device=self.dev, dtype=torch.uint8)
            self.set_condition(None, 1.0)
        self._build(masked)
        self._finish()

    def set_condition(self, mask_u8, weight: float):
        """the pixel mask uint8 [H, W] (None: all ones) and inpainting_mask_weight of the next run()s (masked programs)"""
        if mask_u8 is not None:
            self.mask_u8.copy_(mask_u8.reshape(-1))
        self.cond_mask = None if mask_u8 is None else self.mask_u8
        self.cond_weight = float(weight)

    def _condition_input(self):
        ops.masked_image_to_nhwc(self.img_u8, self.cond_mask, self.cond_weight, self.xin)

    def _build(self, masked: bool = False):
        b, h, wd, t = self.b, self.height, self.width, self.w.t
        if masked:
            self._emit(self._condition_input)
        else:
            self._emit(ops.image_to_nhwc, self.img_u8, self.xin)
        c = self.w.cfg.ch
        x = self.pool.get(b, h * wd, c)
        emit_conv3(self, self.xin, h, wd, t["conv_in.w"], x, bias=t["conv_in.b"])
        nlev = len(self.w.levels)
        for lvl, blocks in self.w.levels:
            for i, (cin, cout) in enumerate(blocks):
                y = self._res(f"down{lvl}.{i}", x, cin, cout, h, wd)
                self.pool.put(x)
                x = y
                c = cout
            if lvl != nlev - 1:
                ho, wo = h // 2, wd // 2
                y = self.pool.get(b, ho * wo, c)
                # F.pad((0, 1, 0, 1)) with zeros, then a conv with padding 0: tiling leaves it as it is
                self._emit(ops.conv2d, x.unflatten(1, (h, wd)), t[f"down{lvl}.downsample.w"], y, ksize=3, stride=2, pad=0,
                           pad_end=1, bias=t[f"down{lvl}.downsample.b"])
                self.pool.put(x)
                x, h, wd = y, ho, wo
        x = self._mid(x, c, h, wd)
        a = self.pool.get(b, h * wd, c)
        self._gn(x, a, "norm_out", True)
        self.pool.put(x)
        m = self.pool.get(b, h * wd, 64)
        emit_conv3(self, a, h, wd, t["conv_out.w"], m, bias=t["conv_out.b"])
        self.pool.put(a)
        moments = self.pool.get(b, h * wd, 64)
        self._emit(ops.linear, m, t["quant.w"], moments, bias=t["quant.b"])
        self.lat_h, self.lat_w = h, wd
        self.latents = torch.empty((b, h * wd, 4), device=self.dev, dtype=torch.float32)
        self._emit(ops.unpack_latent, moments, self.latents, self.w.cfg.scale_factor)

    def run(self):
        super().run()
        return self.latents
