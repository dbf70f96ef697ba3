"""Text conditioning in plain torch (fp16 / bf16 on the GPU).

Runs once per request (cond + uncond prompts), 0.04 % of an image's FLOPs — SURVEY.md §8 a-ext x13 keeps it out of
kernel scope ("run in torch").
  * SD1.x: CLIP ViT-L/14 text tower, same math as transformers' CLIPTextModel — causal mask, quick-gelu MLP, final LN,
    last hidden state (sdwui CLIP_stop_at_last_layers = 1).
  * SDXL (sgm GeneralConditioner, sd_xl_base.yaml): the CLIP-L tower read at hidden layer 11 (no final LN) next to an
    OpenCLIP ViT-bigG tower (penultimate layer; pooled = ln_final(last)[EOS] @ text_projection), and the vector
    conditioning cat(pooled, Fourier features of original size, crop, target size) that feeds the UNet's label_emb.
  * SD 2.x (ldm FrozenOpenCLIPEmbedder, layer="penultimate"): the OpenCLIP ViT-H/14 tower run through all but its last
    block, then ln_final.
  * Prompts longer than one chunk (sdwui FrozenCLIPEmbedderWithCustomWordsBase): tokens [B, 77 * k] are k separate
    77-token sequences through the tower, concatenated along the tokens; emphasis multipliers scale each chunk's output
    as sdwui's EmphasisOriginal does.
"""
import math
import threading
from typing import Dict, NamedTuple, Optional

import torch
import torch.nn.functional as F

from .config import CLIP_PREFIX, OPENCLIP_PREFIX, XL_PREFIX0, XL_PREFIX1, CLIPConfig
from .weights import Placement


CAPTURE_LOCK = threading.Lock()   # CUDA graph captures are serialised across the per-device worker threads (engine.py too)


class Cond(NamedTuple):
    ctx: torch.Tensor                 # [B, 77 * k, context_dim] cross-attention context
    y: Optional[torch.Tensor] = None  # [B, adm_in_channels] vector conditioning (SDXL), or None


def emphasis(z: torch.Tensor, mult: torch.Tensor) -> torch.Tensor:
    """sdwui EmphasisOriginal on one chunk of one prompt: z [77, W] tower output, mult [77]: z * m, rescaled so that the
    mean over the chunk's 77 x W values is what it was; fp32 math.  One sequence per call, so the reductions have the
    same shape whatever the batch (a batched mean may sum in another order)."""
    zf = z.float()
    before = zf.mean()
    zf = zf * mult.to(device=z.device, dtype=torch.float32)[:, None]
    zf = zf * (before / zf.mean())
    return zf.to(z.dtype)


def _placements(w: Dict[str, torch.Tensor], prefix: str) -> Dict[str, Placement]:
    """ldm key -> Placement of every linear weight of a tower's `w` (stored as in the checkpoint: identity placements;
    OpenCLIP's attn.in_proj_weight holds q, k and v as its three row blocks)"""
    return {prefix + k: Placement(k, tuple(v.shape)) for k, v in w.items()
            if (k.endswith(".weight") and v.dim() == 2 and "embedding" not in k) or k.endswith(".in_proj_weight")}


def _attend(q, k, v, mask):
    d = q.shape[-1]
    return torch.softmax((q @ k.transpose(-1, -2)).float() * d ** -0.5 + mask, dim=-1).to(q.dtype) @ v


class ClipText:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: CLIPConfig, device, dtype=torch.float16, prefix: str = CLIP_PREFIX):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        n = len(prefix)
        self.prefix = prefix
        self.w = {k[n:]: v.to(device=device, dtype=dtype) for k, v in sd.items() if k.startswith(prefix)}
        self.place = _placements(self.w, prefix)

    @torch.no_grad()
    def hidden(self, tokens: torch.Tensor, layers: int) -> torch.Tensor:
        """residual stream after `layers` encoder layers (transformers hidden_states[layers]), no final LayerNorm"""
        w, cfg = self.w, self.cfg
        tokens = tokens.to(self.device)
        b, n = tokens.shape
        x = w["embeddings.token_embedding.weight"][tokens] + w["embeddings.position_embedding.weight"][None, :n]
        mask = torch.full((n, n), float("-inf"), device=self.device, dtype=torch.float32).triu(1)
        d = cfg.width // cfg.heads
        for i in range(layers):
            p = f"encoder.layers.{i}"
            h = F.layer_norm(x, (cfg.width,), w[p + ".layer_norm1.weight"], w[p + ".layer_norm1.bias"], 1e-5)
            q, k, v = (F.linear(h, w[f"{p}.self_attn.{m}_proj.weight"], w[f"{p}.self_attn.{m}_proj.bias"])
                       .reshape(b, n, cfg.heads, d).permute(0, 2, 1, 3) for m in "qkv")
            att = _attend(q, k, v, mask).permute(0, 2, 1, 3).reshape(b, n, cfg.width)
            x = x + F.linear(att, w[p + ".self_attn.out_proj.weight"], w[p + ".self_attn.out_proj.bias"])
            h = F.layer_norm(x, (cfg.width,), w[p + ".layer_norm2.weight"], w[p + ".layer_norm2.bias"], 1e-5)
            h = F.linear(h, w[p + ".mlp.fc1.weight"], w[p + ".mlp.fc1.bias"])
            h = h * torch.sigmoid(1.702 * h)
            x = x + F.linear(h, w[p + ".mlp.fc2.weight"], w[p + ".mlp.fc2.bias"])
        return x

    @torch.no_grad()
    def __call__(self, tokens: torch.Tensor) -> torch.Tensor:
        """tokens int64 [B, 77] -> [B, 77, width]: last hidden state after the final LayerNorm"""
        w, cfg = self.w, self.cfg
        return F.layer_norm(self.hidden(tokens, cfg.layers), (cfg.width,), w["final_layer_norm.weight"],
                            w["final_layer_norm.bias"], 1e-5)


class OpenClipText:
    """OpenCLIP text transformer (ViT-bigG-14 for SDXL, ViT-H-14 for SD 2.x): pre-LN resblocks with a packed in_proj,
    GELU MLP, causal mask.  Its size is the config's xl_* fields for SDXL's second tower, width / layers / heads for SD 2.x."""

    def __init__(self, sd: Dict[str, torch.Tensor], cfg: CLIPConfig, device, dtype, prefix: str = XL_PREFIX1):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        self.width, self.layers, self.heads = ((cfg.xl_width, cfg.xl_layers, cfg.xl_heads) if cfg.xl_width else
                                               (cfg.width, cfg.layers, cfg.heads))
        n = len(prefix)
        self.prefix = prefix
        self.w = {k[n:]: v.to(device=device, dtype=dtype) for k, v in sd.items() if k.startswith(prefix)}
        self.place = _placements(self.w, prefix)

    def _blocks(self, x: torch.Tensor, start: int, stop: int, mask: torch.Tensor) -> torch.Tensor:
        """resblocks [start, stop) on the residual stream x [B, n, W]"""
        w, wd, heads = self.w, self.width, self.heads
        b, n, _ = x.shape
        d = wd // heads
        for i in range(start, stop):
            p = f"transformer.resblocks.{i}"
            h = F.layer_norm(x, (wd,), w[p + ".ln_1.weight"], w[p + ".ln_1.bias"], 1e-5)
            q, k, v = (t.reshape(b, n, heads, d).permute(0, 2, 1, 3)
                       for t in F.linear(h, w[p + ".attn.in_proj_weight"], w[p + ".attn.in_proj_bias"]).chunk(3, dim=-1))
            att = _attend(q, k, v, mask).permute(0, 2, 1, 3).reshape(b, n, wd)
            x = x + F.linear(att, w[p + ".attn.out_proj.weight"], w[p + ".attn.out_proj.bias"])
            h = F.layer_norm(x, (wd,), w[p + ".ln_2.weight"], w[p + ".ln_2.bias"], 1e-5)
            x = x + F.linear(F.gelu(F.linear(h, w[p + ".mlp.c_fc.weight"], w[p + ".mlp.c_fc.bias"])),
                             w[p + ".mlp.c_proj.weight"], w[p + ".mlp.c_proj.bias"])
        return x

    def _penultimate(self, tokens: torch.Tensor):
        """(residual stream before the last resblock [B, n, W], causal mask)"""
        w = self.w
        n = tokens.shape[1]
        x = w["token_embedding.weight"][tokens] + w["positional_embedding"][None, :n]
        mask = torch.full((n, n), float("-inf"), device=self.device, dtype=torch.float32).triu(1)
        return self._blocks(x, 0, self.layers - 1, mask), mask

    @torch.no_grad()
    def __call__(self, tokens: torch.Tensor):
        """SDXL's second tower -> (penultimate residual stream [B, 77, W], pooled [B, proj])"""
        w, wd = self.w, self.width
        tokens = tokens.to(self.device)
        b = tokens.shape[0]
        penultimate, mask = self._penultimate(tokens)
        x = self._blocks(penultimate, self.layers - 1, self.layers, mask)
        last = F.layer_norm(x, (wd,), w["ln_final.weight"], w["ln_final.bias"], 1e-5)
        pooled = last[torch.arange(b, device=self.device), tokens.argmax(dim=-1)] @ w["text_projection"]
        return penultimate, pooled

    @torch.no_grad()
    def encode(self, tokens: torch.Tensor) -> torch.Tensor:
        """SD 2.x: tokens [B, 77] -> ln_final of the penultimate residual stream [B, 77, W] (ldm FrozenOpenCLIPEmbedder
        with layer="penultimate": all but the last resblock run, then ln_final)"""
        w, wd = self.w, self.width
        x, _ = self._penultimate(tokens.to(self.device))
        return F.layer_norm(x, (wd,), w["ln_final.weight"], w["ln_final.bias"], 1e-5)


def fourier(scalars: torch.Tensor, dim: int) -> torch.Tensor:
    """sgm ConcatTimestepEmbedderND's timestep_embedding(x, dim): cat(cos, sin)(x * 10000^(-k / (dim / 2)))"""
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=scalars.device) / half)
    args = scalars[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


class Conditioner:
    """tokens -> Cond for either model family"""

    def __init__(self, sd: Dict[str, torch.Tensor], cfg: CLIPConfig, device, dtype, use_graphs: bool = False):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        self.device = torch.device(device)
        self.use_graphs = use_graphs and self.device.type == "cuda"
        self._graphs = {}     # tower name -> (graph, static token buffer, static outputs)
        self._stream = None
        self.xl = cfg.xl_width > 0
        if self.xl:
            self.t0 = ClipText(sd, cfg, device, dtype, XL_PREFIX0)
            self.t1 = OpenClipText(sd, cfg, device, dtype, XL_PREFIX1)
        elif cfg.open_clip:
            self.t0 = OpenClipText(sd, cfg, device, dtype, OPENCLIP_PREFIX)
        else:
            self.t0 = ClipText(sd, cfg, device, dtype)

    CHUNK = 8   # sequences per text-tower call, always exactly this many

    def _chunked(self, name: str, fn, tokens: torch.Tensor):
        """Run a text tower batch-invariantly: the towers are library GEMMs (cuBLAS picks kernels — split-K included — by
        the M = sequences x 77 of the call, so the same prompt encoded inside a batch of 17 or of 2 differed in the last
        bit, which broke "a sharded batch equals the whole batch" at 8 GPUs).  Unique token rows only (a request normally
        carries ONE prompt for all its images), always in calls of exactly CHUNK sequences (the tail padded by repetition):
        every sequence then goes through the same kernels whatever the batch it arrived in."""
        uniq, inverse = torch.unique(tokens.cpu(), dim=0, return_inverse=True)
        outs = None
        for i in range(0, uniq.shape[0], self.CHUNK):
            part = uniq[i:i + self.CHUNK]
            n = part.shape[0]
            if n < self.CHUNK:
                part = torch.cat([part, part[-1:].expand(self.CHUNK - n, -1)])
            res = self._run(name, fn, part)
            outs = [[] for _ in res] if outs is None else outs
            for o, r in zip(outs, res):
                o.append(r[:n])
        inverse = inverse.to(self.device)
        return tuple(torch.cat(o)[inverse] for o in outs)

    def _run(self, name: str, fn, part: torch.Tensor):
        """one fixed-shape tower call.  With graphs on it is ONE replay instead of ~150 eager launches per tower: the towers
        are 0.04 % of an image's FLOPs but were most of a request's HOST time, which is what serialises the per-device job
        threads of an in-process World (8 GPUs, 4 images each: 384 ms per request against 221 ms of device work)."""
        if not self.use_graphs:
            res = fn(part)
            return res if isinstance(res, tuple) else (res,)
        if name not in self._graphs:
            with torch.cuda.device(self.device):
                if self._stream is None:
                    self._stream = torch.cuda.Stream(device=self.device)
                static_tok = part.to(self.device).clone()
                side = torch.cuda.Stream(device=self.device)
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    fn(static_tok)               # warm-up outside capture (cuBLAS handles / workspaces)
                torch.cuda.current_stream().wait_stream(side)
                g = torch.cuda.CUDAGraph()
                with CAPTURE_LOCK:
                    with torch.cuda.graph(g, stream=self._stream, capture_error_mode="thread_local"):
                        res = fn(static_tok)
                res = res if isinstance(res, tuple) else (res,)
                self._graphs[name] = (g, static_tok, res)
        g, static_tok, res = self._graphs[name]
        with torch.cuda.device(self.device):
            static_tok.copy_(part, non_blocking=True)
            g.replay()
            return tuple(r.clone() for r in res)

    @torch.no_grad()
    def __call__(self, tokens: torch.Tensor, width: int = 512, height: int = 512, zero_txt: bool = False,
                 multipliers: Optional[torch.Tensor] = None) -> Cond:
        """tokens [B, 77 * k]; multipliers [B, 77 * k] emphasis weights (None or all 1: none applied).
        zero_txt (SDXL): sdwui's force_zero_embeddings=['txt'] for an all-empty negative prompt"""
        b, n = tokens.shape
        if n % 77:
            raise ValueError(f"prompt tokens must come in chunks of 77, got {n}")
        k = n // 77
        if multipliers is not None:
            if tuple(multipliers.shape) != (b, n):
                raise ValueError(f"multipliers {tuple(multipliers.shape)} do not match tokens {(b, n)}")
            if bool((multipliers == 1.0).all()):
                multipliers = None
        seqs = tokens.reshape(b * k, 77)   # sequence i * k + j = chunk j of prompt i
        first = None
        if multipliers is not None:   # each distinct (tokens, multipliers) sequence is weighted once
            mult = multipliers.reshape(b * k, 77).cpu().float()
            keys = [(tuple(t), tuple(m)) for t, m in zip(seqs.cpu().tolist(), mult.tolist())]
            seen = {}
            first = [seen.setdefault(key, i) for i, key in enumerate(keys)]

        def ctx_of(z):   # [b * k, 77, W] tower output -> emphasis -> [b, 77 * k, W]
            if first is not None:
                done = {i: emphasis(z[i], mult[i]) for i in sorted(set(first))}
                z = torch.stack([done[i] for i in first])
            return z.reshape(b, n, z.shape[-1])

        if not self.xl:
            tower = self.t0.encode if self.cfg.open_clip else self.t0
            return Cond(ctx_of(self._chunked("t0", tower, seqs)[0]))
        cfg = self.cfg
        (h0,) = self._chunked("t0_hidden", lambda t: self.t0.hidden(t, cfg.layers - 1), seqs)
        h1, pooled = self._chunked("t1", self.t1, seqs)
        pooled = pooled.reshape(b, k, -1)[:, 0]   # sdwui: the pooled vector of the first chunk, unweighted
        ctx = torch.cat([ctx_of(h0), ctx_of(h1)], dim=-1)
        if zero_txt:
            ctx, pooled = torch.zeros_like(ctx), torch.zeros_like(pooled)
        scal = torch.tensor([height, width, 0, 0, height, width], dtype=torch.float32, device=self.device)
        size = fourier(scal, cfg.size_embed_dim).reshape(1, -1).expand(b, -1).to(ctx.dtype)
        return Cond(ctx, torch.cat([pooled, size], dim=-1))
