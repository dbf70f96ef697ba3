"""UNet eps-prediction as a static program of libb200sd kernels (NHWC fp16, CUDA-graph friendly).

Stands in for upstream ldm `UNetModel.forward` as called once per sampler step by sdwui's CFGDenoiser (reached
from the reference at scripts/spartan/world.py:196 and, remotely, worker.py:432).  Differences in *how*, not *what*:

  * batch = [cond images | uncond images] (CFG), activations are [N, H*W, C] row-major, every op takes a pitch,
    so the up-path `torch.cat([h, skip])` never happens: producers write straight into channel slices of a
    pre-allocated concat buffer and consumers read the slice in place.
  * the timestep embedding depends only on t, never on x: `time_embed` + every ResBlock's `emb_layers` run ONCE
    per request for all sampler steps (as GEMM rows) and are folded into the conv1 biases; a tiny kernel selects
    the current step's bias rows on the device, so one captured graph replays for every step.
  * cross-attention K/V of the (constant) text context are projected once per request, into buffers of `ctx_len`
    (the context capacity, a multiple of 77) rows per image.  A longer prompt grows them (grow_context); a grown
    program attends row i to its own first kv_len[i] keys (b200sd_attention_varlen), so cond and uncond contexts of
    different lengths share one batched evaluation and each gets what sdwui's separate UNet calls would give.
  * q/k/v projection weights carry zero rows so each head is padded to a multiple of 64 columns — exactly one
    TMA SWIZZLE_128B box per head chunk in the attention kernel.
"""
import contextlib
from typing import Dict, List, Optional

import torch

from . import ops
from .config import CONTROL_PREFIX, UNET_PREFIX, UNetConfig, controlnet_layout, unet_layout
from .weights import Placement, conv_columns, index_column, pack_conv, pack_geglu, pad_heads, source_rows


MAX_CONTROLS = 3   # ControlNet units per request (sd-webui-controlnet's default unit count)


def _pad64(d: int) -> int:
    """head pitch of q / k / v: d itself when it is a multiple of 64 (SDXL), otherwise d + 1 (room for V's ones column)
    rounded up to the P.V MMA's N granularity of 16 — 40 -> 48, 80 -> 96, 160 -> 176 (round 1 padded to 64 / 128 / 192:
    a quarter more q/k/v projection FLOPs and bytes for d = 40)"""
    return d if d % 64 == 0 else (d + 1 + 15) // 16 * 16


class Pool:
    """Exact-shape free lists: deterministic buffer reuse inside a fixed program (safe under graph replay)."""

    def __init__(self, device, dtype):
        self.device, self.dtype = device, dtype
        self.free: Dict[tuple, List[torch.Tensor]] = {}
        self.bytes = 0

    def get(self, *shape, dtype=None, zero=False):
        dt = dtype or self.dtype
        key = (tuple(shape), dt)
        lst = self.free.get(key)
        if lst:
            t = lst.pop()
            if zero:
                t.zero_()
            return t
        t = (torch.zeros if zero else torch.empty)(shape, device=self.device, dtype=dt)
        self.bytes += t.numel() * t.element_size()
        return t

    def put(self, t: torch.Tensor):
        self.free.setdefault((tuple(t.shape), t.dtype), []).append(t)


class UNetWeights:
    """Packs an ldm state_dict (fp32, any device) into kernel layouts on `device`."""
    PREFIX = UNET_PREFIX
    ENCODER_ONLY = False   # time embedding, input blocks and middle block only (ControlNetWeights)

    def __init__(self, sd: Dict[str, torch.Tensor], cfg: UNetConfig, device, dtype=torch.float16):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        self.p = self.PREFIX
        self.sd = sd
        self.t: Dict[str, torch.Tensor] = {}
        self.layout = unet_layout(cfg)
        self.res_keys: List[str] = []     # every ResBlock in execution order
        self.res_off: Dict[str, int] = {}  # offset of its conv1 bias inside the per-step bias row
        self.place: Dict[str, Placement] = {}   # ldm weight key -> where it lies in self.t (b200sd/lora.py)
        self._pack()

    # -- helpers
    def _w(self, key):
        return self.sd[self.p + key]

    def _dev(self, t, dtype=None):
        return t.to(device=self.device, dtype=dtype or self.dtype).contiguous()

    def _f32(self, key):
        return self._dev(self._w(key), torch.float32)

    def _conv(self, name, key, cin_pad=0, cout_pad=0):
        w = self._w(key + ".weight")
        self.t[name + ".w"] = self._dev(pack_conv(w, cin_pad, cout_pad))
        self.place[self.p + key + ".weight"] = Placement(name + ".w", tuple(w.shape), None, conv_columns(w.shape, cin_pad))
        b = self._w(key + ".bias")
        if cout_pad > b.numel():
            b = torch.cat([b, b.new_zeros(cout_pad - b.numel())])
        self.t[name + ".b"] = self._dev(b, torch.float32)

    def _lin(self, name, key, bias=True):
        w = self._w(key + ".weight")
        self.t[name + ".w"] = self._dev(w.reshape(w.shape[0], -1))
        self.place[self.p + key + ".weight"] = Placement(name + ".w", tuple(w.shape))
        if bias:
            self.t[name + ".b"] = self._f32(key + ".bias")

    def _norm(self, name, key):
        self.t[name + ".g"] = self._f32(key + ".weight")
        self.t[name + ".beta"] = self._f32(key + ".bias")

    def _pack(self):
        cfg = self.cfg
        self._lin("time_embed.0", "time_embed.0")
        self._lin("time_embed.2", "time_embed.2")
        if cfg.adm_in_channels:   # SDXL vector conditioning
            self._lin("label_emb.0", "label_emb.0.0")
            self._lin("label_emb.2", "label_emb.0.2")
        inputs, middle, outputs = self.layout
        emb_w, emb_b, conv1_b = [], [], []
        off = 0

        def res(key, cin, cout):
            nonlocal off
            self._norm(key + ".gn1", key + ".in_layers.0")
            self._conv(key + ".conv1", key + ".in_layers.2")
            self._norm(key + ".gn2", key + ".out_layers.0")
            self._conv(key + ".conv2", key + ".out_layers.3")
            if cin != cout:
                self._lin(key + ".skip", key + ".skip_connection")
            emb_w.append(self._w(key + ".emb_layers.1.weight"))
            self.place[self.p + key + ".emb_layers.1.weight"] = Placement("emb_all.w", (cout, cfg.time_embed_dim),
                                                                          torch.arange(cout) + off)
            emb_b.append(self._w(key + ".emb_layers.1.bias"))
            conv1_b.append(self._w(key + ".in_layers.2.bias"))
            self.res_keys.append(key)
            self.res_off[key] = off
            off += cout

        def attn(key, c, depth):
            heads = cfg.heads(c)
            d = c // heads
            dp = _pad64(d)
            self._norm(key + ".norm", key + ".norm")
            self._lin(key + ".proj_in", key + ".proj_in")    # conv 1x1 (SD1.x) and Linear (SDXL) are the same GEMM in NHWC
            self._lin(key + ".proj_out", key + ".proj_out")
            head_rows = source_rows(pad_heads(index_column(c), heads, d, dp))
            for i in range(depth):
                t = f"{key}.transformer_blocks.{i}"
                for n in ("norm1", "norm2", "norm3"):
                    self._norm(f"{t}.{n}", f"{t}.{n}")
                qkv = torch.cat([pad_heads(self._w(f"{t}.attn1.to_{n}.weight"), heads, d, dp) for n in "qkv"])
                self.t[f"{t}.attn1.qkv.w"] = self._dev(qkv)
                for j, n in enumerate("qkv"):
                    self.place[f"{self.p}{t}.attn1.to_{n}.weight"] = Placement(f"{t}.attn1.qkv.w", (c, c),
                                                                                head_rows + j * heads * dp)
                # V's first pad column of every head is driven to exactly 1 through the bias: the P.V MMA then
                # returns the softmax denominators in accumulator column d (b200sd_attention v_ones_col)
                ones = torch.zeros((heads, dp))
                if dp > d:
                    ones[:, d] = 1.0
                self.t[f"{t}.attn1.qkv.b"] = self._dev(torch.cat([torch.zeros(2 * heads * dp), ones.reshape(-1)]),
                                                       torch.float32)
                self.t[f"{t}.attn2.kv.b"] = self._dev(torch.cat([torch.zeros(heads * dp), ones.reshape(-1)]),
                                                      torch.float32)
                self._lin(f"{t}.attn1.out", f"{t}.attn1.to_out.0")
                self.t[f"{t}.attn2.q.w"] = self._dev(pad_heads(self._w(f"{t}.attn2.to_q.weight"), heads, d, dp))
                self.place[f"{self.p}{t}.attn2.to_q.weight"] = Placement(f"{t}.attn2.q.w", (c, c), head_rows)
                kv = torch.cat([pad_heads(self._w(f"{t}.attn2.to_{n}.weight"), heads, d, dp) for n in "kv"])
                self.t[f"{t}.attn2.kv.w"] = self._dev(kv)
                for j, n in enumerate("kv"):
                    self.place[f"{self.p}{t}.attn2.to_{n}.weight"] = Placement(f"{t}.attn2.kv.w", (c, cfg.context_dim),
                                                                              head_rows + j * heads * dp)
                self._lin(f"{t}.attn2.out", f"{t}.attn2.to_out.0")
                w, b = self._w(f"{t}.ff.net.0.proj.weight"), self._w(f"{t}.ff.net.0.proj.bias")
                bn = ops.pick_block_n(w.shape[0], geglu=True)
                wp, bp = pack_geglu(w, b, bn)
                self.t[f"{t}.ff1.w"] = self._dev(wp)
                idx = index_column(w.shape[0])
                self.place[f"{self.p}{t}.ff.net.0.proj.weight"] = Placement(
                    f"{t}.ff1.w", tuple(w.shape), source_rows(pack_geglu(idx, idx[:, 0], bn)[0]))
                self.t[f"{t}.ff1.b"] = self._dev(bp, torch.float32)
                self._lin(f"{t}.ff2", f"{t}.ff.net.2")

        def block(prefix, layers):
            for j, layer in enumerate(layers):
                key = f"{prefix}.{j}"
                if layer[0] == "conv_in":
                    self._conv(key, key, cin_pad=64)
                elif layer[0] == "res":
                    res(key, layer[1], layer[2])
                elif layer[0] == "attn":
                    attn(key, layer[1], layer[2])
                elif layer[0] == "down":
                    self._conv(key, key + ".op")
                elif layer[0] == "up":
                    self._conv(key, key + ".conv")

        for n, layers in enumerate(inputs):
            block(f"input_blocks.{n}", layers)
        block("middle_block", middle)
        if not self.ENCODER_ONLY:
            for n, layers in enumerate(outputs):
                block(f"output_blocks.{n}", layers)
            self._norm("out.gn", "out.0")
            self._conv("out.conv", "out.2", cout_pad=32)
        self._pack_extra()
        self.t["emb_all.w"] = self._dev(torch.cat(emb_w))
        self.t["emb_all.b"] = self._dev(torch.cat(emb_b), torch.float32)
        self.t["conv1_bias_all"] = self._dev(torch.cat(conv1_b), torch.float32)
        self.emb_total = off
        self.sd = None  # drop the reference to the fp32 dict

    def _pack_extra(self):
        """layers a subclass adds to the UNet's (ControlNetWeights: hint block and zero convs)"""


def _pad_to(c: int, m: int) -> int:
    return -(-c // m) * m


def emit_conv3(prog, x: torch.Tensor, h: int, wd: int, *a, **k):
    """emit a 3x3 conv with padding 1 on x [n, h*wd, C] into `prog` (a UNet or VAE program: its `_emit`, `pool` and
    `circular`).  Zero padding is the conv kernel's own; with `prog.circular` (sdwui's tiling) it is circular: x is
    copied into pool scratch one pixel larger on each side with the halo wrapped around (ops.pad_circular), and the conv
    reads that with no padding.  Stride 2 then gives the same output size as zero padding 1."""
    if not prog.circular:
        prog._emit(ops.conv2d, x.unflatten(1, (h, wd)), *a, ksize=3, **k)
        return
    xp = prog.pool.get(x.shape[0], (h + 2) * (wd + 2), x.shape[-1])
    prog._emit(ops.pad_circular, x.unflatten(1, (h, wd)), xp.unflatten(1, (h + 2, wd + 2)), 1)
    prog._emit(ops.conv2d, xp.unflatten(1, (h + 2, wd + 2)), *a, ksize=3, pad=0, **k)
    prog.pool.put(xp)


class ControlNetWeights(UNetWeights):
    """An ldm ControlNet (keys `control_model.*`, factory.controlnet) packed for a UNet of config `cfg`: its time
    embedding, input blocks and middle block go through UNetWeights' packers under the same names (`input_blocks.1.0.
    conv1.w`, `emb_all.w`, ...), plus
      hint.j.w / .b   input_hint_block conv j (3x3; input channels padded to a multiple of 64, outputs to one of 32, as
                      conv_in and out.conv are padded: the padded weights are zero)
      zero.i.w / .b   zero conv i (1x1, a linear over channels); zero.mid the middle_block_out conv.
    `name` identifies the model in graph names and caches."""
    PREFIX = CONTROL_PREFIX
    ENCODER_ONLY = True

    def __init__(self, sd: Dict[str, torch.Tensor], cfg: UNetConfig, device, dtype=torch.float16, name: str = "control"):
        self.name = name
        self.hint_layout = controlnet_layout(cfg)[2]
        super().__init__(sd, cfg, device, dtype)

    def _pack_extra(self):
        _, _, hint, zero_ch = controlnet_layout(self.cfg)
        for j, (cin, cout, _) in enumerate(hint):
            self._conv(f"hint.{j}", f"input_hint_block.{2 * j}", cin_pad=_pad_to(cin, 64), cout_pad=_pad_to(cout, 32))
        for i in range(len(zero_ch)):
            self._lin(f"zero.{i}", f"zero_convs.{i}.0")
        self._lin("zero.mid", "middle_block_out.0")
        self.n_zero = len(zero_ch)


class UNetProgram:
    """One UNet evaluation for a fixed (N, H, W): `run()` launches ~700 kernels, no allocation, no sync."""

    def __init__(self, w: UNetWeights, n: int, h: int, wd: int, ctx_len: int = 77, tiling: bool = False,
                 token_merging: int = 0):
        """tiling: every 3x3 conv of the UNet pads circularly (sdwui's tiling option); ControlNet segments never do.
        token_merging: r > 0 merges r of the h*wd tokens before the self-attention of every transformer block at the full
        latent resolution (tomesd as sdwui's token_merging_ratio applies it); ControlNet segments never merge."""
        self.w, self.cfg = w, w.cfg
        self.tiling = self.circular = tiling
        self.token_merging = self.merging = token_merging
        # per merging transformer block: the matching of the last evaluation, int32 (slot [n, h*wd], members [n, h*wd],
        # seg [n, h*wd - r + 1]; include/b200sd.h b200sd_tome_match), persistent like kv_len
        self.tome: Dict[str, tuple] = {}
        self.tome_ws: Optional[torch.Tensor] = None   # b200sd_tome_match's workspace, shared by those blocks
        self.n, self.h, self.wd = n, h, wd
        self.dev, self.dt = w.device, w.dtype
        self.pool = Pool(self.dev, self.dt)
        self.ctx_len = ctx_len      # context capacity: rows of every cross-attention K/V buffer
        self.ctx_len0 = ctx_len     # ... as built: at this capacity the cross-attention calls take no lengths
        # keys each batch row attends to, read by the kernels (graph replays follow it); used once the capacity grew
        self.kv_len = torch.full((n,), ctx_len, device=self.dev, dtype=torch.int32)
        self._xattn: List[tuple] = []   # (op index, transformer block, q, out, heads, d, d_pad, scale) per attn2
        cfg = self.cfg
        # persistent I/O
        self.xin = torch.zeros((n, h * wd, 64), device=self.dev, dtype=self.dt)    # latent channels 0..3, rest zero
        self.eps = torch.zeros((n, h * wd, 32), device=self.dev, dtype=self.dt)    # eps channels 0..3
        # this step's conv1 biases (time embedding folded in): one row of Cout floats per ResBlock — or, with a vector
        # conditioning (SDXL: the embedding differs per sample), n rows per ResBlock, block r at offset n * res_off[r]
        self.per_sample = cfg.adm_in_channels > 0
        self.cur_bias = torch.zeros((w.emb_total * (n if self.per_sample else 1),), device=self.dev, dtype=torch.float32)
        self.gn_stats: List[torch.Tensor] = []
        self.gn_need = 0
        self.ctx_kv: Dict[str, torch.Tensor] = {}
        self.ops: List = []
        self.op_flops: List = []
        self.gn_elems = self.ln_elems = 0     # elements normalised per evaluation (bench.py's HBM roofline)
        self.segments: List[Optional["ControlSegment"]] = [None] * MAX_CONTROLS   # ControlNet unit slots
        self._build()
        # one statistics buffer serves every GroupNorm (they run back to back on one stream); zeroed once, here
        self.stats_all = torch.zeros((max(1, self.gn_need),), device=self.dev, dtype=torch.float32)
        for holder in self.gn_stats:
            holder[0] = self.stats_all

    # ---------------------------------------------------------------- per-request precompute
    def set_context(self, ctx: torch.Tensor, lengths=None):
        """ctx [N, L, context_dim] (cond rows first, uncond rows second), L <= ctx_len, rows of an image beyond its length
        zero; lengths: tokens per row (None: L for every row).  Projects K/V of every attn2 once."""
        n, l, c = ctx.shape
        assert n == self.n and l <= self.ctx_len, (ctx.shape, self.ctx_len)
        lengths = [l] * n if lengths is None else [int(v) for v in lengths]
        assert len(lengths) == n and all(1 <= v <= l for v in lengths), lengths
        if self.ctx_len == self.ctx_len0:
            assert all(v == self.ctx_len for v in lengths), "a context shorter than the capacity needs grow_context"
        if l < self.ctx_len:   # zero rows up to the capacity: their keys are masked, their values finite
            ctx = torch.cat([ctx, ctx.new_zeros((n, self.ctx_len - l, c))], dim=1)
        self.project_context(ctx, [s for s in self.segments if s is not None])
        if self.ctx_len != self.ctx_len0:
            self.kv_len.copy_(torch.tensor(lengths, dtype=torch.int32))

    def project_context(self, ctx: torch.Tensor, segments):
        """K/V of every attn2 of the UNet and of the ControlNet `segments` from ctx [N, ctx_len, context_dim]"""
        n, l = self.n, self.ctx_len
        ctx2 = ctx.reshape(n * l, ctx.shape[-1])
        for w, ctx_kv in [(self.w, self.ctx_kv)] + [(s.w, s.ctx_kv) for s in segments]:
            for key, buf in ctx_kv.items():
                ops.linear(ctx2, w.t[key + ".attn2.kv.w"], buf.reshape(n * l, -1), bias=w.t[key + ".attn2.kv.b"])

    def grow_context(self, cap: int):
        """Reallocate every cross-attention K/V buffer with `cap` rows per image (cap > ctx_len) and point the program's
        attn2 launches at them, now with per-row key counts.  Activation buffers are untouched.  Graphs captured before
        hold the old buffers' addresses: the caller drops them."""
        assert cap > self.ctx_len
        self.ctx_len = cap
        for ctx_kv, xattn, op_list in [(self.ctx_kv, self._xattn, self.ops)] + \
                [(s.ctx_kv, s.xattn, s.ops) for s in self.segments if s is not None]:
            for tb in list(ctx_kv):
                old = ctx_kv[tb]
                ctx_kv[tb] = torch.zeros((self.n, cap, old.shape[2]), device=self.dev, dtype=self.dt)
            self._varlen_xattn(ctx_kv, xattn, op_list)

    def _varlen_xattn(self, ctx_kv, xattn, op_list):
        """point the attn2 launches listed in `xattn` at the K/V buffers of `ctx_kv`, with per-row key counts"""
        for i, tb, q2, o, heads, d, dp, scale in xattn:
            kv = ctx_kv[tb]
            op_list[i] = (ops.attention, (q2, kv[..., :heads * dp], kv[..., heads * dp:], o, heads, d, dp, scale, dp > d),
                          {"kv_len": self.kv_len})

    # ---------------------------------------------------------------- ControlNet
    def set_control(self, slot: int, cw: "ControlNetWeights", table_rows: int, step: torch.Tensor) -> bool:
        """Make unit slot `slot` (0 .. MAX_CONTROLS-1) run ControlNet `cw`, its time-embedding rows selected by the
        device counter `step`: builds the slot's segment unless it already holds that model.  Returns True when it built
        one (graphs that ran the slot's old segment are then stale)."""
        if self.per_sample:
            raise ValueError("ControlNet is not served for SDXL")
        seg = self.segments[slot]
        if seg is not None and seg.w is cw:
            return False
        self.segments[slot] = None   # the old segment's buffers go before the new ones are allocated
        self.segments[slot] = ControlSegment(self, cw, table_rows, step)
        return True

    @contextlib.contextmanager
    def emitting_into(self, seg: "ControlSegment"):
        """the emitters (_run_layers, _res, _attn) build `seg`'s ops: its weights, biases, K/V buffers and op list stand in
        for the UNet's, and the element counters of the UNet's roofline stay as they are"""
        saved = (self.w, self.cur_bias, self.ctx_kv, self._xattn, self.ops, self.op_flops, self.gn_elems, self.ln_elems)
        self.w, self.cur_bias, self.ctx_kv, self._xattn, self.ops, self.op_flops = \
            seg.w, seg.cur_bias, seg.ctx_kv, seg.xattn, seg.ops, seg.op_flops
        # sd-webui-controlnet's model is not part of the sd model that sdwui's tiling makes circular and tomesd
        # patches: zero padding, no merging
        self.circular = False
        self.merging = 0
        try:
            yield
        finally:
            (self.w, self.cur_bias, self.ctx_kv, self._xattn, self.ops, self.op_flops, self.gn_elems,
             self.ln_elems) = saved
            self.circular = self.tiling
            self.merging = self.token_merging

    def _run_layers(self, prefix, layers, x, h, wd, final_dest, conv_in_residual=None):
        """x: input view; the LAST layer writes into final_dest (a view with the right channel count).  conv_in reads the
        program's input xin; `conv_in_residual` (a ControlNet's hint features) is added in its epilogue."""
        cfg, n, t = self.cfg, self.n, self.w.t
        prev_tmp = None
        for li, layer in enumerate(layers):
            key = f"{prefix}.{li}"
            last = li == len(layers) - 1
            kind = layer[0]
            tmp = None
            if kind == "conv_in":
                dest = final_dest
                emit_conv3(self, self.xin, h, wd, t[key + ".w"], dest, bias=t[key + ".b"], residual=conv_in_residual,
                           algo_flops=2.0 * n * h * wd * 9 * cfg.in_channels * layer[2])
            elif kind == "res":
                dest = final_dest if last else self.pool.get(n, h * wd, layer[2])
                tmp = None if last else dest
                self._res(key, x, layer[1], layer[2], h, wd, dest)
            elif kind == "attn":
                dest = final_dest if last else self.pool.get(n, h * wd, layer[1])
                tmp = None if last else dest
                self._attn(key, x, layer[1], layer[2], h, wd, dest)
            elif kind == "down":
                dest = final_dest
                emit_conv3(self, x, h, wd, t[key + ".w"], dest, stride=2, bias=t[key + ".b"])
                h, wd = (h + 1) // 2, (wd + 1) // 2
            elif kind == "up":
                up = self.pool.get(n, 4 * h * wd, layer[1])
                self._emit(ops.upsample2x, x.unflatten(1, (h, wd)), up.unflatten(1, (2 * h, 2 * wd)))
                h, wd = 2 * h, 2 * wd
                dest = final_dest
                emit_conv3(self, up, h, wd, t[key + ".w"], dest, bias=t[key + ".b"])
                self.pool.put(up)
            if prev_tmp is not None:  # the previous layer's scratch output has now been consumed
                self.pool.put(prev_tmp)
            prev_tmp = tmp
            x = dest
        return x, h, wd

    # ---------------------------------------------------------------- program construction
    def _emit(self, fn, *a, algo_flops=None, **k):
        """algo_flops: the launch's ALGORITHMIC FLOPs when they differ from 2*M*N*K of the packed operands (zero-padded
        head columns / latent channels are layout, not work) — read by bench.py's roofline, never by the kernels"""
        self.ops.append((fn, a, k))
        self.op_flops.append(algo_flops)

    def _gn(self, x, out, name, eps, silu):
        holder = [None]
        self.gn_stats.append(holder)
        self.gn_need = max(self.gn_need, ops.groupnorm_stats_floats(x.shape[0], x.shape[1], x.shape[2], 32))
        g, b = self.w.t[name + ".g"], self.w.t[name + ".beta"]
        self.gn_elems += x.shape[0] * x.shape[1] * x.shape[2]
        self._emit(lambda: ops.groupnorm(x, out, holder[0], g, b, 32, eps, silu))

    def _res(self, key, x, cin, cout, h, wd, dest):
        n, hw, t = self.n, h * wd, self.w.t
        a = self.pool.get(n, hw, cin)
        self._gn(x, a, key + ".gn1", 1e-5, True)
        off = self.w.res_off[key]
        b = self.pool.get(n, hw, cout)
        if self.per_sample:   # a bias row per image: rows [i * hw, (i + 1) * hw) of the GEMM take row i
            bsl = self.cur_bias[n * off: n * (off + cout)]
            emit_conv3(self, a, h, wd, t[key + ".conv1.w"], b.reshape(n * hw, cout), bias=bsl, bias_group_rows=hw)
        else:
            bsl = self.cur_bias[off: off + cout]
            emit_conv3(self, a, h, wd, t[key + ".conv1.w"], b.reshape(n * hw, cout), bias=bsl)
        self.pool.put(a)
        c = self.pool.get(n, hw, cout)
        self._gn(b, c, key + ".gn2", 1e-5, True)
        self.pool.put(b)
        if cin != cout:
            s = self.pool.get(n, hw, cout)
            self._emit(ops.linear, x, t[key + ".skip.w"], s, bias=t[key + ".skip.b"])
            skip = s
        else:
            s, skip = None, x
        emit_conv3(self, c, h, wd, t[key + ".conv2.w"], dest, bias=t[key + ".conv2.b"], residual=skip)
        self.pool.put(c)
        if s is not None:
            self.pool.put(s)

    def _attn(self, key, x, c, depth, h, wd, dest):
        n, hw, t, heads = self.n, h * wd, self.w.t, self.cfg.heads(c)
        d = c // heads
        dp = _pad64(d)
        scale = d ** -0.5
        a = self.pool.get(n, hw, c)
        self._gn(x, a, key + ".norm", 1e-6, False)
        hcur = self.pool.get(n, hw, c)
        self._emit(ops.linear, a, t[key + ".proj_in.w"], hcur, bias=t[key + ".proj_in.b"])
        for i in range(depth):
            tb = f"{key}.transformer_blocks.{i}"
            self.ln_elems += 3 * n * hw * c
            # --- self attention
            self._emit(ops.layernorm, hcur, a, t[tb + ".norm1.g"], t[tb + ".norm1.beta"], 1e-5)
            if self.merging and (h, wd) == (self.h, self.wd):
                h1 = self._merged_self_attention(tb, hcur, a, h, wd, c, heads, d, dp, scale)
                o = self.pool.get(n, hw, c)
            else:
                qkv = self.pool.get(n, hw, 3 * heads * dp)
                self._emit(ops.linear, a, t[tb + ".attn1.qkv.w"], qkv, bias=t[tb + ".attn1.qkv.b"],
                           algo_flops=2.0 * n * hw * 3 * c * c)
                q, k, v = (qkv[..., j * heads * dp:(j + 1) * heads * dp] for j in range(3))
                o = self.pool.get(n, hw, c)
                self._emit(ops.attention, q, k, v, o, heads, d, dp, scale, dp > d)
                self.pool.put(qkv)
                h1 = self.pool.get(n, hw, c)
                self._emit(ops.linear, o, t[tb + ".attn1.out.w"], h1, bias=t[tb + ".attn1.out.b"], residual=hcur)
            self.pool.put(hcur)
            # --- cross attention (K/V of the context are precomputed per request)
            self._emit(ops.layernorm, h1, a, t[tb + ".norm2.g"], t[tb + ".norm2.beta"], 1e-5)
            q2 = self.pool.get(n, hw, heads * dp)
            self._emit(ops.linear, a, t[tb + ".attn2.q.w"], q2, algo_flops=2.0 * n * hw * c * c)
            kv = torch.zeros((n, self.ctx_len, 2 * heads * dp), device=self.dev, dtype=self.dt)
            self.ctx_kv[tb] = kv
            self._xattn.append((len(self.ops), tb, q2, o, heads, d, dp, scale))
            self._emit(ops.attention, q2, kv[..., :heads * dp], kv[..., heads * dp:], o, heads, d, dp, scale, dp > d)
            self.pool.put(q2)
            h2 = self.pool.get(n, hw, c)
            self._emit(ops.linear, o, t[tb + ".attn2.out.w"], h2, bias=t[tb + ".attn2.out.b"], residual=h1)
            self.pool.put(h1)
            self.pool.put(o)
            # --- GEGLU feed-forward
            self._emit(ops.layernorm, h2, a, t[tb + ".norm3.g"], t[tb + ".norm3.beta"], 1e-5)
            g = self.pool.get(n, hw, 4 * c)
            self._emit(ops.linear, a, t[tb + ".ff1.w"], g, bias=t[tb + ".ff1.b"], flags=ops.EPI_GEGLU)
            hcur = self.pool.get(n, hw, c)
            self._emit(ops.linear, g, t[tb + ".ff2.w"], hcur, bias=t[tb + ".ff2.b"], residual=h2)
            self.pool.put(g)
            self.pool.put(h2)
        self._emit(ops.linear, hcur, t[key + ".proj_out.w"], dest, bias=t[key + ".proj_out.b"], residual=x)
        self.pool.put(hcur)
        self.pool.put(a)

    def _merged_self_attention(self, tb, hcur, a, h, wd, c, heads, d, dp, scale):
        """tomesd's ToMeBlock self-attention, u(attn1(m(norm1(x)))) + x: match on the block input hcur, merge the
        LayerNorm output `a` into h*wd - r rows, q/k/v projection, attention and out-projection on those rows, then
        give every token its slot's row plus its residual.  Returns h1 [n, h*wd, c] (pool)."""
        n, hw, t, r = self.n, h * wd, self.w.t, self.merging
        nm = hw - r
        if self.tome_ws is None:
            self.tome_ws = torch.zeros((ops.tome_workspace_bytes(n, h, wd, c),), device=self.dev, dtype=torch.uint8)
        slot, members, seg = self.tome[tb] = tuple(torch.zeros((n, cols), device=self.dev, dtype=torch.int32)
                                                   for cols in (hw, hw, nm + 1))
        self._emit(ops.tome_match, hcur, h, wd, r, slot, members, seg, self.tome_ws)
        am = self.pool.get(n, nm, c)
        self._emit(ops.tome_merge, a, members, seg, am)
        qkv = self.pool.get(n, nm, 3 * heads * dp)
        self._emit(ops.linear, am, t[tb + ".attn1.qkv.w"], qkv, bias=t[tb + ".attn1.qkv.b"],
                   algo_flops=2.0 * n * nm * 3 * c * c)
        self.pool.put(am)
        q, k, v = (qkv[..., j * heads * dp:(j + 1) * heads * dp] for j in range(3))
        om = self.pool.get(n, nm, c)
        self._emit(ops.attention, q, k, v, om, heads, d, dp, scale, dp > d)
        self.pool.put(qkv)
        y = self.pool.get(n, nm, c)
        self._emit(ops.linear, om, t[tb + ".attn1.out.w"], y, bias=t[tb + ".attn1.out.b"])
        self.pool.put(om)
        h1 = self.pool.get(n, hw, c)
        self._emit(ops.tome_unmerge_add, hcur, y, slot, h1)
        self.pool.put(y)
        return h1

    def _build(self):
        cfg, n, t = self.cfg, self.n, self.w.t
        inputs, middle, outputs = self.w.layout
        # ---- plan: channel count / resolution of every input-block output, and the concat buffer it lands in
        in_out_ch, in_res = [], []
        h, wd = self.h, self.wd
        for layers in inputs:
            for layer in layers:
                if layer[0] == "down":
                    h, wd = (h + 1) // 2, (wd + 1) // 2
            last = layers[0]
            in_out_ch.append(last[2] if last[0] in ("conv_in", "res") else last[1])
            in_res.append((h, wd))
        n_in = len(inputs)
        # output block i consumes cat([h_prev, skip_{n_in-1-i}])
        cats = []
        ch_prev = in_out_ch[-1]  # middle block keeps the channel count
        for i, layers in enumerate(outputs):
            j = n_in - 1 - i
            hh, ww = in_res[j]
            cats.append(torch.empty((n, hh * ww, ch_prev + in_out_ch[j]), device=self.dev, dtype=self.dt))
            ch_prev = layers[0][2]
        self.pool.bytes += sum(c.numel() * 2 for c in cats)

        def skip_slot(j):  # where input block j must write its output
            i = n_in - 1 - j
            c = cats[i]
            return c[..., c.shape[-1] - in_out_ch[j]:]

        # ---- input blocks
        h, wd = self.h, self.wd
        x = None
        for j, layers in enumerate(inputs):
            x, h, wd = self._run_layers(f"input_blocks.{j}", layers, x, h, wd, skip_slot(j))
        # ---- middle block -> first concat buffer's h slot
        c0 = cats[0]
        x, h, wd = self._run_layers("middle_block", middle, x, h, wd, c0[..., :c0.shape[-1] - in_out_ch[n_in - 1]])
        # ControlNet segments run here, between the middle block and the decoder: every pool buffer is free at this point,
        # so a segment shares the pool; their outputs are added in place into these views, the skips and the middle result
        self.mid_op = len(self.ops)
        self.control_dest = [skip_slot(j) for j in range(n_in)] + [c0[..., :c0.shape[-1] - in_out_ch[n_in - 1]]]
        self.in_res = in_res
        # ---- output blocks
        final = torch.empty((n, self.h * self.wd, cfg.model_channels), device=self.dev, dtype=self.dt)
        for i, layers in enumerate(outputs):
            cat = cats[i]
            hh, ww = in_res[n_in - 1 - i]
            if i + 1 < len(outputs):
                nxt = cats[i + 1]
                dest = nxt[..., :nxt.shape[-1] - in_out_ch[n_in - 2 - i]]
            else:
                dest = final
            x, h, wd = self._run_layers(f"output_blocks.{i}", layers, cat, hh, ww, dest)
        # ---- out: GN + SiLU + conv3x3 -> eps (4 channels padded to 32)
        a = self.pool.get(n, self.h * self.wd, cfg.model_channels)
        self._gn(final, a, "out.gn", 1e-5, True)
        emit_conv3(self, a, self.h, self.wd, t["out.conv.w"], self.eps.reshape(-1, 32), bias=t["out.conv.b"],
                   algo_flops=2.0 * n * self.h * self.wd * 9 * cfg.model_channels * cfg.out_channels)
        self.pool.put(a)

    # ---------------------------------------------------------------- execution
    def run(self, active=()):
        """one evaluation; `active`: the ControlNet slots whose segments run (between the middle block and the decoder)"""
        if not active:
            for fn, a, k in self.ops:
                fn(*a, **k)
            return
        for fn, a, k in self.ops[:self.mid_op]:
            fn(*a, **k)
        for slot in active:
            for fn, a, k in self.segments[slot].ops:
                fn(*a, **k)
        for fn, a, k in self.ops[self.mid_op:]:
            fn(*a, **k)


class ControlSegment:
    """ControlNet unit slot of a UNetProgram (ldm ControlNet as sd-webui-controlnet drives it, Balanced mode).

    `ops` is one evaluation of the ControlNet on the UNet's own input xin, timestep and contexts, run between the UNet's
    middle block and its decoder (UNetProgram.run(active)): select this step's conv1 biases from `table`; conv_in with the
    hint features as its epilogue residual; the input blocks and the middle block through the UNet's own emitters and
    pool; after each block its zero conv, as a linear whose output and residual are the UNet's skip slice (or middle
    result) — an in-place add into the concat buffer (b200sd_epilogue: residual == D).  The zero-conv weights are this
    slot's copies, scaled by the unit's weight in set_hint, so a new weight needs no new graph.

    `hint_ops` is the hint block on one image at the generation size (8h x 8w), run once per request by set_hint; its
    [1, h*w, model_channels] output is broadcast to the [n, h*w, model_channels] features every batch row reads."""

    def __init__(self, prog: UNetProgram, cw: "ControlNetWeights", table_rows: int, step: torch.Tensor):
        self.w = cw
        n, dev, dt = prog.n, prog.dev, prog.dt
        self.n = n
        self.cur_bias = torch.zeros((cw.emb_total,), device=dev, dtype=torch.float32)
        self.table = torch.zeros((table_rows, cw.emb_total), device=dev, dtype=torch.float32)   # TimeEmbedding(cw) rows
        self.hint_feat = torch.zeros((n, prog.h * prog.wd, cw.cfg.model_channels), device=dev, dtype=dt)
        names = [f"zero.{i}" for i in range(cw.n_zero)] + ["zero.mid"]
        self.zero = [(torch.zeros_like(cw.t[k + ".w"]), torch.zeros_like(cw.t[k + ".b"]), k) for k in names]
        self.ctx_kv: Dict[str, torch.Tensor] = {}
        self.xattn: List[tuple] = []
        self.ops: List = []
        self.op_flops: List = []
        self._build(prog, step)
        self._build_hint(prog)

    def _build(self, prog: UNetProgram, step: torch.Tensor):
        inputs, middle, _ = self.w.layout
        n, zc = self.n, self.zero
        holders = len(prog.gn_stats)
        with prog.emitting_into(self):
            prog._emit(ops.select_step, self.table, step, self.cur_bias)
            h, wd = prog.h, prog.wd
            x = prev = None
            for j, layers in enumerate(inputs):
                hh, ww = prog.in_res[j]
                dest = prog.pool.get(n, hh * ww, prog.control_dest[j].shape[-1])
                x, h, wd = prog._run_layers(f"input_blocks.{j}", layers, x, h, wd, dest,
                                            conv_in_residual=self.hint_feat if j == 0 else None)
                skip = prog.control_dest[j]
                prog._emit(ops.linear, dest, zc[j][0], skip, bias=zc[j][1], residual=skip)
                if prev is not None:
                    prog.pool.put(prev)
                prev = dest
            mid = prog.pool.get(n, h * wd, prog.control_dest[-1].shape[-1])
            x, h, wd = prog._run_layers("middle_block", middle, x, h, wd, mid)
            prog.pool.put(prev)
            out = prog.control_dest[-1]
            prog._emit(ops.linear, mid, zc[-1][0], out, bias=zc[-1][1], residual=out)
            prog.pool.put(mid)
        assert prog.gn_need <= prog.stats_all.numel(), "a ControlNet GroupNorm needs more statistics than the UNet's"
        for holder in prog.gn_stats[holders:]:
            holder[0] = prog.stats_all
        if prog.ctx_len != prog.ctx_len0:
            prog._varlen_xattn(self.ctx_kv, self.xattn, self.ops)

    def _build_hint(self, prog: UNetProgram):
        cw, dev, dt = self.w, prog.dev, prog.dt
        hh, ww = 8 * prog.h, 8 * prog.wd
        cin_pads = [_pad_to(cin, 64) for cin, _, _ in cw.hint_layout]
        self.hint_u8 = torch.zeros((1, hh * ww, 3), device=dev, dtype=torch.uint8)
        cur = torch.zeros((1, hh * ww, cin_pads[0]), device=dev, dtype=dt)
        self.hint_ops = [(ops.hint_to_nhwc, (self.hint_u8, cur), {})]
        last = len(cw.hint_layout) - 1
        for j, (_, cout, stride) in enumerate(cw.hint_layout):
            cp = _pad_to(cout, 32)
            ho, wo = (hh + 1) // 2 if stride == 2 else hh, (ww + 1) // 2 if stride == 2 else ww
            # zero from allocation beyond the cp written channels: the next conv's padded input channels
            out = torch.zeros((1, ho * wo, cp if j == last else max(cp, cin_pads[j + 1])), device=dev, dtype=dt)
            self.hint_ops.append((ops.conv2d, (cur[..., :cin_pads[j]].unflatten(1, (hh, ww)), cw.t[f"hint.{j}.w"],
                                               out[..., :cp]),
                                  dict(ksize=3, stride=stride, bias=cw.t[f"hint.{j}.b"],
                                       flags=0 if j == last else ops.EPI_SILU)))
            cur, hh, ww = out, ho, wo
        assert (hh, ww) == (prog.h, prog.wd) and cur.shape[-1] == cw.cfg.model_channels
        self.hint_out = cur

    def set_hint(self, hint_u8: torch.Tensor, weight: float):
        """per request: the control map uint8 [8h, 8w, 3] (RGB, at the generation size) and the unit's weight"""
        self.hint_u8.copy_(hint_u8.reshape(1, -1, 3))
        for fn, a, k in self.hint_ops:
            fn(*a, **k)
        self.hint_feat.copy_(self.hint_out.expand(self.n, -1, -1))
        for wt, b, key in self.zero:
            wt.copy_(self.w.t[key + ".w"].float() * weight)
            b.copy_(self.w.t[key + ".b"] * weight)


class TimeEmbedding:
    """time_embed MLP + all ResBlock emb_layers for every sampler timestep at once -> fp32 bias table
    table[step] = conv1_bias_all + Linear(SiLU(time_embed(t_step)))  (ldm ResBlock: h + emb_out[..., None, None]).
    With a vector conditioning y [n, adm] (SDXL: emb = time_embed(t) + label_emb(y), sgm UNetModel.forward) the embedding
    differs per sample: table[step] holds, per ResBlock, n rows of Cout floats (UNetProgram.per_sample)."""

    def __init__(self, w: UNetWeights):
        self.w = w

    def table(self, timesteps: torch.Tensor, y: torch.Tensor = None) -> torch.Tensor:
        w, t = self.w, self.w.t
        dev, dt = w.device, w.dtype
        steps = timesteps.numel()
        mc, ted = w.cfg.model_channels, w.cfg.time_embed_dim
        ns = 1 if y is None else y.shape[0]
        n = steps * ns
        ts = timesteps.to(device=dev, dtype=torch.float32)
        if y is not None:
            ts = ts.repeat_interleave(ns)          # row = step * ns + sample
        sin = torch.empty((n, mc), device=dev, dtype=dt)
        ops.timestep_embedding(ts.contiguous(), sin)
        h1 = torch.empty((n, ted), device=dev, dtype=dt)
        ops.linear(sin, t["time_embed.0.w"], h1, bias=t["time_embed.0.b"], flags=ops.EPI_SILU)
        h2 = torch.empty((n, ted), device=dev, dtype=dt)
        if y is None:
            ops.linear(h1, t["time_embed.2.w"], h2, bias=t["time_embed.2.b"], flags=ops.EPI_SILU)  # SiLU of emb_layers.0
        else:
            l1 = torch.empty((ns, ted), device=dev, dtype=dt)
            ops.linear(y.to(device=dev, dtype=dt).contiguous(), t["label_emb.0.w"], l1, bias=t["label_emb.0.b"], flags=ops.EPI_SILU)
            le = torch.empty((ns, ted), device=dev, dtype=dt)
            ops.linear(l1, t["label_emb.2.w"], le, bias=t["label_emb.2.b"])
            # emb = time_embed(t) + label_emb(y), then emb_layers' SiLU: the label part rides in as the GEMM's residual
            ops.linear(h1, t["time_embed.2.w"], h2, bias=t["time_embed.2.b"], residual=le.repeat(steps, 1).contiguous(),
                       flags=ops.EPI_SILU)
        emb = torch.empty((n, w.emb_total), device=dev, dtype=dt)
        ops.linear(h2, t["emb_all.w"], emb, bias=t["emb_all.b"])
        table = torch.empty((n, w.emb_total), device=dev, dtype=torch.float32)
        ops.fold_bias(emb, t["conv1_bias_all"], table)
        if y is None:
            return table
        # [steps, ns, sum Cout] -> per step, ResBlock after ResBlock, ns rows of its Cout floats
        tv = table.reshape(steps, ns, w.emb_total)
        parts = []
        offs = sorted(w.res_off.values()) + [w.emb_total]
        for a, b in zip(offs[:-1], offs[1:]):
            parts.append(tv[:, :, a:b].reshape(steps, ns * (b - a)))
        return torch.cat(parts, dim=1).contiguous()
