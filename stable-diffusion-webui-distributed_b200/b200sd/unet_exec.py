"""UNet eps-prediction as a static program of libb200sd kernels (NHWC fp16, CUDA-graph friendly).

Stands in for upstream ldm `UNetModel.forward` as called once per sampler step by sdwui's CFGDenoiser (reached
from the reference at scripts/spartan/world.py:196 and, remotely, worker.py:432).  Differences in *how*, not *what*:

  * batch = [cond images | uncond images] (CFG), activations are [N, H*W, C] row-major, every op takes a pitch,
    so the up-path `torch.cat([h, skip])` never happens: producers write straight into channel slices of a
    pre-allocated concat buffer and consumers read the slice in place.
  * the timestep embedding depends only on t, never on x: `time_embed` + every ResBlock's `emb_layers` run ONCE
    per request for all sampler steps (as GEMM rows) and are folded into the conv1 biases; a tiny kernel selects
    the current step's bias rows on the device, so one captured graph replays for every step.
  * cross-attention K/V of the (constant) text context are projected once per request.
  * q/k/v projection weights carry zero rows so each head is padded to a multiple of 64 columns — exactly one
    TMA SWIZZLE_128B box per head chunk in the attention kernel.
"""
from typing import Dict, List

import torch

from . import ops
from .config import UNET_PREFIX, UNetConfig, unet_layout
from .weights import pack_conv, pack_geglu, pad_heads


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

    def __init__(self, sd: Dict[str, torch.Tensor], cfg: UNetConfig, device, dtype=torch.float16):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        self.p = UNET_PREFIX
        self.sd = sd
        self.t: Dict[str, torch.Tensor] = {}
        self.layout = unet_layout(cfg)
        self.res_keys: List[str] = []     # every ResBlock in execution order
        self.res_off: Dict[str, int] = {}  # offset of its conv1 bias inside the per-step bias row
        self._pack()

    # -- helpers
    def _w(self, key):
        return self.sd[self.p + key]

    def _dev(self, t, dtype=None):
        return t.to(device=self.device, dtype=dtype or self.dtype).contiguous()

    def _f32(self, key):
        return self._dev(self._w(key), torch.float32)

    def _conv(self, name, key, cin_pad=0, cout_pad=0):
        self.t[name + ".w"] = self._dev(pack_conv(self._w(key + ".weight"), cin_pad, cout_pad))
        b = self._w(key + ".bias")
        if cout_pad > b.numel():
            b = torch.cat([b, b.new_zeros(cout_pad - b.numel())])
        self.t[name + ".b"] = self._dev(b, torch.float32)

    def _lin(self, name, key, bias=True):
        w = self._w(key + ".weight")
        self.t[name + ".w"] = self._dev(w.reshape(w.shape[0], -1))
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
            for i in range(depth):
                t = f"{key}.transformer_blocks.{i}"
                for n in ("norm1", "norm2", "norm3"):
                    self._norm(f"{t}.{n}", f"{t}.{n}")
                qkv = torch.cat([pad_heads(self._w(f"{t}.attn1.to_{n}.weight"), heads, d, dp) for n in "qkv"])
                self.t[f"{t}.attn1.qkv.w"] = self._dev(qkv)
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
                kv = torch.cat([pad_heads(self._w(f"{t}.attn2.to_{n}.weight"), heads, d, dp) for n in "kv"])
                self.t[f"{t}.attn2.kv.w"] = self._dev(kv)
                self._lin(f"{t}.attn2.out", f"{t}.attn2.to_out.0")
                w, b = self._w(f"{t}.ff.net.0.proj.weight"), self._w(f"{t}.ff.net.0.proj.bias")
                bn = ops.pick_block_n(w.shape[0], geglu=True)
                wp, bp = pack_geglu(w, b, bn)
                self.t[f"{t}.ff1.w"] = self._dev(wp)
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
        for n, layers in enumerate(outputs):
            block(f"output_blocks.{n}", layers)
        self._norm("out.gn", "out.0")
        self._conv("out.conv", "out.2", cout_pad=32)
        self.t["emb_all.w"] = self._dev(torch.cat(emb_w))
        self.t["emb_all.b"] = self._dev(torch.cat(emb_b), torch.float32)
        self.t["conv1_bias_all"] = self._dev(torch.cat(conv1_b), torch.float32)
        self.emb_total = off
        self.sd = None  # drop the reference to the fp32 dict


class UNetProgram:
    """One UNet evaluation for a fixed (N, H, W): `run()` launches ~700 kernels, no allocation, no sync."""

    def __init__(self, w: UNetWeights, n: int, h: int, wd: int, ctx_len: int = 77):
        self.w, self.cfg = w, w.cfg
        self.n, self.h, self.wd = n, h, wd
        self.dev, self.dt = w.device, w.dtype
        self.pool = Pool(self.dev, self.dt)
        self.ctx_len = ctx_len
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
        self._build()
        # one statistics buffer serves every GroupNorm (they run back to back on one stream); zeroed once, here
        self.stats_all = torch.zeros((max(1, self.gn_need),), device=self.dev, dtype=torch.float32)
        for holder in self.gn_stats:
            holder[0] = self.stats_all

    # ---------------------------------------------------------------- per-request precompute
    def set_context(self, ctx: torch.Tensor):
        """ctx [N, ctx_len, context_dim] (cond rows first, uncond rows second): project K/V of every attn2 once."""
        n, l, c = ctx.shape
        assert n == self.n and l == self.ctx_len
        ctx2 = ctx.reshape(n * l, c)
        for key, buf in self.ctx_kv.items():
            ops.linear(ctx2, self.w.t[key + ".attn2.kv.w"], buf.reshape(n * l, -1), bias=self.w.t[key + ".attn2.kv.b"])

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
            self._emit(ops.conv2d, a.unflatten(1, (h, wd)), t[key + ".conv1.w"], b.reshape(n * hw, cout), ksize=3, bias=bsl,
                       bias_group_rows=hw)
        else:
            bsl = self.cur_bias[off: off + cout]
            self._emit(ops.conv2d, a.unflatten(1, (h, wd)), t[key + ".conv1.w"], b.reshape(n * hw, cout), ksize=3, bias=bsl)
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
        self._emit(ops.conv2d, c.unflatten(1, (h, wd)), t[key + ".conv2.w"], dest, ksize=3, bias=t[key + ".conv2.b"],
                   residual=skip)
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

        def run_layers(prefix, layers, x, h, wd, final_dest):
            """x: input view; the LAST layer writes into final_dest (a view with the right channel count)."""
            prev_tmp = None
            for li, layer in enumerate(layers):
                key = f"{prefix}.{li}"
                last = li == len(layers) - 1
                kind = layer[0]
                tmp = None
                if kind == "conv_in":
                    dest = final_dest
                    self._emit(ops.conv2d, self.xin.unflatten(1, (h, wd)), t[key + ".w"], dest, ksize=3, bias=t[key + ".b"],
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
                    self._emit(ops.conv2d, x.unflatten(1, (h, wd)), t[key + ".w"], dest, ksize=3, stride=2, bias=t[key + ".b"])
                    h, wd = (h + 1) // 2, (wd + 1) // 2
                elif kind == "up":
                    up = self.pool.get(n, 4 * h * wd, layer[1])
                    self._emit(ops.upsample2x, x.unflatten(1, (h, wd)), up.unflatten(1, (2 * h, 2 * wd)))
                    h, wd = 2 * h, 2 * wd
                    dest = final_dest
                    self._emit(ops.conv2d, up.unflatten(1, (h, wd)), t[key + ".w"], dest, ksize=3, bias=t[key + ".b"])
                    self.pool.put(up)
                if prev_tmp is not None:  # the previous layer's scratch output has now been consumed
                    self.pool.put(prev_tmp)
                prev_tmp = tmp
                x = dest
            return x, h, wd

        # ---- input blocks
        h, wd = self.h, self.wd
        x = None
        for j, layers in enumerate(inputs):
            x, h, wd = run_layers(f"input_blocks.{j}", layers, x, h, wd, skip_slot(j))
        # ---- middle block -> first concat buffer's h slot
        c0 = cats[0]
        x, h, wd = run_layers("middle_block", middle, x, h, wd, c0[..., :c0.shape[-1] - in_out_ch[n_in - 1]])
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
            x, h, wd = run_layers(f"output_blocks.{i}", layers, cat, hh, ww, dest)
        # ---- out: GN + SiLU + conv3x3 -> eps (4 channels padded to 32)
        a = self.pool.get(n, self.h * self.wd, cfg.model_channels)
        self._gn(final, a, "out.gn", 1e-5, True)
        self._emit(ops.conv2d, a.unflatten(1, (self.h, self.wd)), t["out.conv.w"], self.eps.reshape(-1, 32), ksize=3,
                   bias=t["out.conv.b"], algo_flops=2.0 * n * self.h * self.wd * 9 * cfg.model_channels * cfg.out_channels)
        self.pool.put(a)

    # ---------------------------------------------------------------- execution
    def run(self):
        for fn, a, k in self.ops:
            fn(*a, **k)


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
