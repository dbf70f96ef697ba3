"""fp32 oracle of sdwui's token merging, built from the unchanged sd_oracle, v_oracle and controlnet_oracle functions.

sdwui (>= 1.6, `sd_models.apply_token_merging`) calls `tomesd.apply_patch(sd_model, ratio, use_rand=False,
merge_attn=True, merge_crossattn=False, merge_mlp=False)` with sx = sy = 2 and max_downsample = 1 (tomesd 0.1.3).  Every
BasicTransformerBlock of the UNet then computes `x = u(attn1(m(norm1(x)))) + x` before its unchanged cross-attention and
feed-forward, where m / u come from `bipartite_soft_matching_random2d` on the block's input x, and only blocks whose token
count is the latent's h*w merge (`downsample <= max_downsample`).  This restates it (the sdwui / tomesd sources are
restated, not pinned, like the other sdwui restatements), with the decisions tomesd leaves to unstable sorts fixed:

  * dst tokens: the top-left token of every 2x2 block; src tokens: the others, in ascending token order;
  * metric = x / ||x||; node_max / node_idx = max / argmax over dst of the metric dot products, ties to the lowest dst;
  * the r = min(num_src, int(N * ratio)) src tokens with the largest (node_max desc, src index asc) keys are merged;
  * merged sequence: unmerged src tokens in ascending token order, then the dst tokens; a dst slot holds the mean of
    itself and its merged src tokens; unmerge gives every token its slot's row.

A matching is `slot` int64 [B, N]: the merged-sequence slot of every token.  The oracle runs under a shim: `unet_forward`
records the latent size, `transformer_block` merges where N = h*w (its self-attention call goes through merge / unmerge),
and `controlnet_forward` runs outside the shim (sd-webui-controlnet's model is not part of the patched sd model).
"""
import contextlib

import torch

from oracle import controlnet_oracle as CN
from oracle import sd_oracle as O


def merged_tokens(h: int, w: int, ratio: float) -> int:
    """r of a level-0 block of an h x w latent: tomesd's int(N * ratio) (Python double) capped at the src count; a
    ratio <= 0 does not merge (sdwui patches nothing)"""
    if not ratio > 0:
        return 0
    n = h * w
    return max(0, min(n - (h // 2) * (w // 2), int(n * ratio)))


def grid(h: int, w: int, device=None):
    """(src token indices, dst token indices) in ascending token order"""
    t = torch.arange(h * w, device=device)
    dst = ((t // w) % 2 == 0) & ((t % w) % 2 == 0)
    return t[~dst], t[dst]


def match(x: torch.Tensor, h: int, w: int, r: int) -> torch.Tensor:
    """x [B, N, C] (the block input) -> slot int64 [B, N], computed in fp32"""
    src, dst = grid(h, w, x.device)
    ns = src.numel()
    metric = x.float() / x.float().norm(dim=-1, keepdim=True)
    scores = metric[:, src] @ metric[:, dst].transpose(-1, -2)
    node_idx = scores.argmax(dim=-1)                       # the first maximum: the lowest dst index
    node_max = scores.gather(-1, node_idx[..., None])[..., 0]
    order = torch.sort(node_max, dim=-1, descending=True, stable=True).indices   # ties: lower src index first
    merged = torch.zeros_like(node_max, dtype=torch.bool).scatter(-1, order[:, :r], True)
    unm_rank = torch.cumsum((~merged).long(), dim=-1) - 1
    slot = torch.empty((x.shape[0], h * w), dtype=torch.long, device=x.device)
    slot[:, src] = torch.where(merged, ns - r + node_idx, unm_rank)
    slot[:, dst] = ns - r + torch.arange(dst.numel(), device=x.device)
    return slot


def merge(x: torch.Tensor, slot: torch.Tensor, nm: int) -> torch.Tensor:
    """[B, N, C] -> [B, nm, C]: the mean of every slot's tokens"""
    b, _, c = x.shape
    acc = torch.zeros((b, nm, c), dtype=x.dtype, device=x.device).scatter_add(1, slot[..., None].expand(-1, -1, c), x)
    cnt = torch.zeros((b, nm), dtype=x.dtype, device=x.device).scatter_add(1, slot, torch.ones_like(slot, dtype=x.dtype))
    return acc / cnt[..., None]


def unmerge(y: torch.Tensor, slot: torch.Tensor) -> torch.Tensor:
    """[B, nm, C] -> [B, N, C]: every token gets its slot's row"""
    return y.gather(1, slot[..., None].expand(-1, -1, y.shape[-1]))


def partition(slot: torch.Tensor, nm: int):
    """slot [B, N] -> (members [B, N]: tokens by slot, ascending within a slot; seg [B, nm + 1]: slot starts)"""
    members = torch.sort(slot * slot.shape[1] + torch.arange(slot.shape[1]), dim=-1).indices
    cnt = torch.zeros((slot.shape[0], nm), dtype=torch.long).scatter_add(1, slot, torch.ones_like(slot))
    seg = torch.cat([torch.zeros((slot.shape[0], 1), dtype=torch.long), torch.cumsum(cnt, dim=-1)], dim=-1)
    return members, seg


class _State:
    ratio = 0.0
    hw = None          # (h, w) of the latent of the current unet_forward
    active = True      # False inside controlnet_forward
    matchings = None   # {block prefix: slot} to use instead of computing them
    used = None        # {block prefix: slot} of the last evaluation


_S = _State()


def _record(fn):
    def unet_forward(sd, cfg, x, *a, **k):
        saved = _S.hw
        _S.hw = (x.shape[2], x.shape[3])
        try:
            return fn(sd, cfg, x, *a, **k)
        finally:
            _S.hw = saved
    return unet_forward


def _unmerged(fn):
    def controlnet_forward(*a, **k):
        saved = _S.active
        _S.active = False
        try:
            return fn(*a, **k)
        finally:
            _S.active = saved
    return controlnet_forward


def _block(fn):
    def transformer_block(sd, p, x, context, heads):
        h, w = _S.hw if _S.hw is not None else (0, 0)
        r = merged_tokens(h, w, _S.ratio)
        if not _S.active or r == 0 or x.shape[1] != h * w:
            return fn(sd, p, x, context, heads)
        slot = _S.matchings[p] if _S.matchings is not None else match(x, h, w, r)
        slot = slot.to(device=x.device, dtype=torch.long)
        _S.used[p] = slot
        nm = h * w - r
        attend = O.cross_attention

        def cross_attention(sd_, p_, x_, context_, heads_):
            if context_ is not None:
                return attend(sd_, p_, x_, context_, heads_)
            return unmerge(attend(sd_, p_, merge(x_, slot, nm), None, heads_), slot)

        O.cross_attention = cross_attention
        try:
            return fn(sd, p, x, context, heads)
        finally:
            O.cross_attention = attend
    return transformer_block


@contextlib.contextmanager
def merging(ratio: float, matchings=None):
    """inside: the oracle's UNet merges tokens at `ratio` (sdwui's token_merging_ratio); `matchings` {transformer block
    prefix, e.g. "input_blocks.1.1.transformer_blocks.0": slot [B, N]} replaces the computed ones"""
    saved = (O.unet_forward, CN.unet_forward, CN.controlnet_forward, O.transformer_block, _S.ratio, _S.matchings, _S.used)
    O.unet_forward, CN.unet_forward = _record(saved[0]), _record(saved[1])
    CN.controlnet_forward = _unmerged(saved[2])
    O.transformer_block = _block(saved[3])
    _S.ratio, _S.matchings, _S.used = ratio, matchings, {}
    try:
        yield _S.used
    finally:
        (O.unet_forward, CN.unet_forward, CN.controlnet_forward, O.transformer_block, _S.ratio, _S.matchings,
         _S.used) = saved


def run(fn, *a, ratio: float, matchings=None, **k):
    """fn(*a, **k) — any sd_oracle / v_oracle / controlnet_oracle sampling entry point — with token merging at `ratio`"""
    with merging(ratio, matchings):
        return fn(*a, **k)

