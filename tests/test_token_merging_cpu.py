"""Token merging (sdwui's token_merging_ratio, tomesd) on the CPU: the token-merging oracle pinned against a literal
restatement of tomesd's bipartite_soft_matching_random2d, the engine with merging on (b200sd.ops emulated:
tests/ops_emulator.py plus the tome ops below) against the oracle on tiny and tiny21, which blocks the programs merge,
the worker's resolution of the ratios and the REST passthrough."""
import json
import types

import pytest
import torch

import ops_emulator
from test_controlnet_cpu import _hint, hint_to_nhwc
from test_tiling_cpu import pad_circular
from test_vpred_cpu import cfg_ddim_step_v, cfg_dpmpp_2m_step_v, cfg_euler_a_step_v


# ------------------------------------------------------------------------------------------------ emulated tome ops
def tome_workspace_bytes(nb, h, w, c):
    return 0


def tome_match(x, h, w, r, slot, members, seg, workspace):
    """b200sd_tome_match: the oracle's matching (fp32) in the kernel's output form"""
    from oracle import tome_oracle as TO
    s = TO.match(x, h, w, r)
    m, sg = TO.partition(s, h * w - r)
    slot.copy_(s)
    members.copy_(m)
    seg.copy_(sg)


def _slots(members, seg):
    """slot [B, N] from members / seg"""
    n = members.shape[1]
    owner = torch.searchsorted(seg.long().contiguous(), torch.arange(n).expand(members.shape[0], -1).contiguous(),
                               right=True) - 1
    return torch.empty_like(owner).scatter_(1, members.long(), owner)


def tome_merge(x, members, seg, out):
    from oracle import tome_oracle as TO
    out.copy_(TO.merge(x.float(), _slots(members, seg), out.shape[1]).to(out.dtype))
    return out


def tome_unmerge_add(residual, y, slot, out):
    from oracle import tome_oracle as TO
    out.copy_((residual.float() + TO.unmerge(y.float(), slot.long())).to(out.dtype))
    return out


def _install(monkeypatch):
    from b200sd import engine as E, ops
    ops_emulator.install(monkeypatch, ops)
    for fn in (pad_circular, hint_to_nhwc, cfg_ddim_step_v, cfg_euler_a_step_v, cfg_dpmpp_2m_step_v,
               tome_workspace_bytes, tome_match, tome_merge, tome_unmerge_add):
        monkeypatch.setattr(ops, fn.__name__, fn)
    monkeypatch.setattr(E.SDEngine, "_require_cuda", False)


def _rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


# ------------------------------------------------------------------------------------------------ oracle pins
def tomesd_bipartite(metric, w, h, r):
    """tomesd 0.1.3 merge.bipartite_soft_matching_random2d(metric, w, h, sx=2, sy=2, r, no_rand=True), restated with
    gather / scatter_reduce / argsort; the argsorts are made stable (tomesd leaves their tie order to the backend)"""
    B, N, _ = metric.shape
    sx = sy = 2
    hsy, wsx = h // sy, w // sx
    rand_idx = torch.zeros(hsy, wsx, 1, dtype=torch.int64)
    idx_buffer_view = torch.zeros(hsy, wsx, sy * sx, dtype=torch.int64)
    idx_buffer_view.scatter_(dim=2, index=rand_idx, src=-torch.ones_like(rand_idx))
    idx_buffer_view = idx_buffer_view.view(hsy, wsx, sy, sx).transpose(1, 2).reshape(hsy * sy, wsx * sx)
    idx_buffer = idx_buffer_view
    rand_idx = idx_buffer.reshape(1, -1, 1).argsort(dim=1, stable=True)
    num_dst = hsy * wsx
    a_idx = rand_idx[:, num_dst:, :]
    b_idx = rand_idx[:, :num_dst, :]

    def split(x):
        C = x.shape[-1]
        src = x.gather(dim=1, index=a_idx.expand(B, N - num_dst, C))
        dst = x.gather(dim=1, index=b_idx.expand(B, num_dst, C))
        return src, dst

    metric = metric / metric.norm(dim=-1, keepdim=True)
    a, b = split(metric)
    scores = a @ b.transpose(-1, -2)
    r = min(a.shape[1], r)
    node_max, node_idx = scores.max(dim=-1)
    edge_idx = node_max.argsort(dim=-1, descending=True, stable=True)[..., None]
    unm_idx = edge_idx[..., r:, :]
    src_idx = edge_idx[..., :r, :]
    dst_idx = node_idx[..., None].gather(dim=-2, index=src_idx)

    def merge(x):
        src, dst = split(x)
        n, t1, c = src.shape
        unm = src.gather(dim=-2, index=unm_idx.expand(n, t1 - r, c))
        src = src.gather(dim=-2, index=src_idx.expand(n, r, c))
        dst = dst.scatter_reduce(-2, dst_idx.expand(n, r, c), src, reduce="mean")
        return torch.cat([unm, dst], dim=1)

    def unmerge(x):
        unm_len = unm_idx.shape[1]
        unm, dst = x[..., :unm_len, :], x[..., unm_len:, :]
        _, _, c = unm.shape
        src = dst.gather(dim=-2, index=dst_idx.expand(B, r, c))
        out = torch.zeros(B, N, c, dtype=x.dtype)
        out.scatter_(dim=-2, index=b_idx.expand(B, num_dst, c), src=dst)
        out.scatter_(dim=-2, index=torch.gather(a_idx.expand(B, a_idx.shape[1], 1), dim=1, index=unm_idx).expand(B, unm_len, c), src=unm)
        out.scatter_(dim=-2, index=torch.gather(a_idx.expand(B, a_idx.shape[1], 1), dim=1, index=src_idx).expand(B, r, c), src=src)
        return out

    return merge, unmerge, unm_idx[..., 0]


@pytest.mark.parametrize("h,w,ratio", [(4, 4, 0.5), (8, 8, 0.3), (8, 12, 0.5), (16, 8, 0.75), (6, 10, 0.9), (8, 8, 0.01)])
def test_oracle_is_tomesd_bipartite_matching(h, w, ratio):
    from oracle import tome_oracle as TO
    g = torch.Generator().manual_seed(h * 100 + w)
    x = torch.randn((3, h * w, 16), generator=g, dtype=torch.float64)
    y = torch.randn((3, h * w, 16), generator=g, dtype=torch.float64)
    r = TO.merged_tokens(h, w, ratio)
    assert r == min(h * w * 3 // 4, int(h * w * ratio))
    merge, unmerge, unm_src = tomesd_bipartite(x, w, h, r)
    slot = TO.match(x, h, w, r)
    nm = h * w - r
    assert slot.shape == (3, h * w) and int(slot.max()) == nm - 1 and len(torch.unique(slot)) == nm
    got, ref = TO.merge(y, slot, nm), merge(y)
    # tomesd lists the unmerged src tokens by descending node_max, the oracle by ascending token: the same rows
    order = torch.argsort(unm_src, dim=-1)
    ref_unm = ref[:, :nm - h * w // 4].gather(1, order[..., None].expand(-1, -1, 16))
    assert torch.allclose(got[:, :nm - h * w // 4], ref_unm, rtol=0, atol=1e-12)
    assert torch.allclose(got[:, nm - h * w // 4:], ref[:, nm - h * w // 4:], rtol=0, atol=1e-12)
    z = torch.randn((3, nm, 16), generator=g, dtype=torch.float64)
    z_tomesd = torch.cat([z[:, :nm - h * w // 4].gather(
        1, torch.argsort(order, dim=-1)[..., None].expand(-1, -1, 16)), z[:, nm - h * w // 4:]], dim=1)
    assert torch.equal(TO.unmerge(z, slot), unmerge(z_tomesd))


def test_dst_tokens_are_the_2x2_top_lefts_and_ties_follow_the_rule():
    from oracle import tome_oracle as TO
    h, w = 4, 6
    src, dst = TO.grid(h, w)
    assert dst.tolist() == [0, 2, 4, 12, 14, 16] and src.numel() == 18
    # every src token equals dst 1 and dst 4 exactly (argmax ties: dst 1); src tokens 3 and 5 are twins of 0
    x = torch.randn((1, h * w, 8), generator=torch.Generator().manual_seed(3))
    x[0, dst[4]] = x[0, dst[1]]
    x[0, src] = x[0, dst[1]] + 0.05 * torch.randn((18, 8), generator=torch.Generator().manual_seed(4))
    x[0, src[3]] = x[0, src[5]] = x[0, src[0]]
    r = 2
    slot = TO.match(x, h, w, r)
    ns = 18
    metric = x / x.norm(dim=-1, keepdim=True)
    nmax = (metric[0, src] @ metric[0, dst].T).max(-1).values
    # all node_idx go to dst 1 (lowest of the tied dsts); the r merged are the largest node_max, lower index first
    merged = [int(a) for a in range(ns) if int(slot[0, src[a]]) >= ns - r]
    assert all(int(slot[0, src[a]]) == ns - r + 1 for a in merged)
    keys = sorted(range(ns), key=lambda a: (-float(nmax[a]), a))[:r]
    assert merged == sorted(keys)
    # src 0, 3 and 5 tie: selecting 2 of them takes 0 and 3
    x2 = x.clone()
    x2[0, src] = x2[0, src[0]] * torch.linspace(0.5, 1.5, ns)[:, None] + 0.3 * torch.randn(
        (ns, 8), generator=torch.Generator().manual_seed(5))
    x2[0, src[3]] = x2[0, src[5]] = x2[0, src[0]]
    nmax2 = ((x2 / x2.norm(dim=-1, keepdim=True))[0, src] @ (x2 / x2.norm(dim=-1, keepdim=True))[0, dst].T).max(-1).values
    top = sorted(range(ns), key=lambda a: (-float(nmax2[a]), a))
    k = top.index(0) + 2   # r up to two of the three tied tokens
    s2 = TO.match(x2, h, w, k)
    got = [a for a in (0, 3, 5) if int(s2[0, src[a]]) >= ns - k]
    assert got == [0, 3]


@pytest.fixture(scope="module")
def tiny():
    from b200sd import config as C, synth
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    return cfgs, synth.make_state_dict(*cfgs, seed=0)


def test_ratio_0_is_the_sd_oracle_and_0_5_is_not(tiny):
    from oracle import sd_oracle as O, tome_oracle as TO
    cfgs, sd = tiny
    tok, neg = O.random_prompt_tokens(2, vocab_hi=997), O.empty_prompt_tokens(2, vocab_hi=997)
    kw = dict(seed=5, steps=4, height=64, width=64)
    with torch.no_grad():
        ref = O.txt2img(sd, *cfgs, tok, neg, **kw)
        off = TO.run(O.txt2img, sd, *cfgs, tok, neg, ratio=0.0, **kw)
        with TO.merging(0.5) as used:
            on = O.txt2img(sd, *cfgs, tok, neg, **kw)
            blocks = sorted(used)
    assert all(torch.equal(a, b) for a, b in zip(off, ref))
    assert _rel(on[1], ref[1]) > 1e-3
    # the level-0 blocks: input_blocks 1, 2 and output_blocks 9, 10, 11
    assert blocks == sorted(f"{k}.1.transformer_blocks.0" for k in
                            ("input_blocks.1", "input_blocks.2", "output_blocks.9", "output_blocks.10", "output_blocks.11"))


# ------------------------------------------------------------------------------------------------ engine vs oracle
@pytest.fixture(params=["tiny", "tiny21"])
def env(request, monkeypatch):
    from b200sd import config as C, engine as E, synth
    from b200sd.unet_exec import ControlNetWeights
    from oracle import sd_oracle as O, v_oracle as V
    _install(monkeypatch)
    if request.param == "tiny":
        cfgs, pred = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP), "eps"
    else:
        cfgs, pred = (C.TINY21_UNET, C.TINY21_VAE, C.TINY21_CLIP), "v"
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2, prediction=pred)
    csd = synth.make_controlnet_state_dict(cfgs[0], seed=11)
    cw = ControlNetWeights(csd, cfgs[0], "cpu", torch.float32, name="cn0")
    b = 2
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    enc = O.clip_text_encode if pred == "eps" else V.sd21_text_encode
    return types.SimpleNamespace(E=E, eng=eng, sd=sd, cfgs=cfgs, csd=csd, cw=cw, b=b, tok=tok, neg=neg, pred=pred,
                                 cond=enc(sd, cfgs[2], tok), unc=enc(sd, cfgs[2], neg))


def _oracle(env, name, steps, nz, ratio, init=None, d=None, nmask=None, units=(), tiling=False):
    from oracle import controlnet_oracle as CN, tiling_oracle as T, tome_oracle as TO
    unet = CN.ControlledUNet(env.sd, env.cfgs[0], list(units))
    mask = None if nmask is None else (init, nmask[None, None])
    with torch.no_grad(), T.circular(tiling), TO.merging(ratio):
        z = CN.run_sampler(name, unet, env.cond, env.unc, 7.0, steps, nz[0], list(nz[1:]), init=init,
                           denoising_strength=d, mask=mask, prediction=env.pred)
    return z if nmask is None else z * nmask + init * (1 - nmask)


def _key(env, hw, ratio, tiling=False):
    r = env.eng.merged_tokens(hw, hw, ratio)
    return (env.b, hw, hw) + (("tiling",) if tiling else ()) + ("tome", r)


def _check(env, z, ref_z, hw):
    lat = z.reshape(env.b, hw, hw, 4).permute(0, 3, 1, 2)
    assert _rel(lat, ref_z) <= 1e-4, _rel(lat, ref_z)


@pytest.mark.parametrize("name", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_txt2img_matches_the_token_merging_oracle(env, name):
    hw, steps, ratio = 8, 6, 0.5
    pr = env.eng.program(name, None, steps)
    nz = env.E.per_image_noise(4100, env.b, (4, hw, hw), 1 + pr.draws)
    got = env.eng.txt2img(env.tok, env.neg, 4100, steps=steps, height=8 * hw, width=8 * hw, sampler=name,
                          token_merging_ratio=ratio)
    ref = _oracle(env, name, steps, nz, ratio)
    _check(env, env.eng.plans[_key(env, hw, ratio)].x, ref, hw)
    plain = env.eng.txt2img(env.tok, env.neg, 4100, steps=steps, height=8 * hw, width=8 * hw, sampler=name)
    assert (env.b, hw, hw) in env.eng.plans and not torch.equal(plain, got)


def _init_u8(b, px):
    return torch.randint(0, 256, (b, px, px, 3), generator=torch.Generator().manual_seed(9), dtype=torch.uint8)


@pytest.mark.parametrize("name,masked", [("DDIM", False), ("Euler a", True)])
def test_img2img_matches_the_token_merging_oracle(env, name, masked):
    from oracle import sd_oracle as O
    hw, steps, d, ratio = 8, 8, 0.75, 0.3
    init_u8 = _init_u8(env.b, hw * 2 ** (len(env.cfgs[1].ch_mult) - 1))
    nmask = (torch.rand((hw, hw), generator=torch.Generator().manual_seed(5)) > 0.5).float() if masked else None
    pr = env.eng.program(name, None, steps, denoise=d, masked=masked)
    nz = env.E.per_image_noise(31, env.b, (4, hw, hw), 1 + pr.draws)
    kw = {} if nmask is None else {"latmask": nmask.reshape(-1)}
    env.eng.img2img(env.tok, env.neg, 31, init_u8, denoising_strength=d, steps=steps, sampler=name,
                    token_merging_ratio=ratio, **kw)
    with torch.no_grad():
        init = O.vae_encode_mean(env.sd, env.cfgs[1], O.image_to_model_input(init_u8)) * env.cfgs[1].scale_factor
    ref = _oracle(env, name, steps, nz, ratio, init=init, d=d, nmask=nmask)
    _check(env, env.eng.plans[_key(env, hw, ratio)].x, ref, hw)


def test_hires_fix_merges_each_pass_at_its_own_ratio(env):
    from oracle import upscale_oracle as UO
    hw, steps, hr_steps, d = 8, 5, 6, 0.6
    env.eng.txt2img_hires(env.tok, env.neg, 77, steps=steps, height=8 * hw, width=8 * hw, hr_scale=2.0,
                          hr_steps=hr_steps, denoising_strength=d, token_merging_ratio=0.3, token_merging_ratio_hr=0.5)
    nz1 = env.E.per_image_noise(77, env.b, (4, hw, hw), 1)
    nz2 = env.E.per_image_noise(77, env.b, (4, 2 * hw, 2 * hw), 1)
    z1 = _oracle(env, "DDIM", steps, nz1, 0.3)
    _check(env, env.eng.plans[_key(env, hw, 0.3)].x, z1, hw)
    with torch.no_grad():
        up = UO.hires_upscale(env.sd, env.cfgs[1], z1, 2 * hw, 2 * hw, "Latent")
    ref = _oracle(env, "DDIM", hr_steps, nz2, 0.5, init=up, d=d)
    _check(env, env.eng.plans[_key(env, 2 * hw, 0.5)].x, ref, 2 * hw)


def test_tiling_and_a_controlnet_unit_compose_with_merging(env):
    hw, steps, name, ratio = 8, 6, "Euler a", 0.5
    hint = _hint(20, 8 * hw, 8 * hw)
    pr = env.eng.program(name, None, steps)
    nz = env.E.per_image_noise(12, env.b, (4, hw, hw), 1 + pr.draws)
    env.eng.txt2img(env.tok, env.neg, 12, steps=steps, height=8 * hw, width=8 * hw, sampler=name, tiling=True,
                    token_merging_ratio=ratio)
    ref = _oracle(env, name, steps, nz, ratio, tiling=True)
    _check(env, env.eng.plans[_key(env, hw, ratio, tiling=True)].x, ref, hw)
    env.eng.txt2img(env.tok, env.neg, 12, steps=steps, height=8 * hw, width=8 * hw, sampler=name,
                    controls=[(env.cw, hint, 0.8, 0.0, 1.0)], token_merging_ratio=ratio)
    ref = _oracle(env, name, steps, nz, ratio, units=[(env.csd, hint, 0.8, 0.0, 1.0)])
    _check(env, env.eng.plans[_key(env, hw, ratio)].x, ref, hw)


def test_inpainting_model_merges_like_the_oracle(monkeypatch):
    from b200sd import engine as E, factory, ops, synth
    from oracle import controlnet_oracle as CN, inpaint_model_oracle as IO, sd_oracle as O, tome_oracle as TO
    from test_inpaint_model_cpu import masked_image_to_nhwc, pack_image_cond
    _install(monkeypatch)
    for fn in (masked_image_to_nhwc, pack_image_cond):
        monkeypatch.setattr(ops, fn.__name__, fn)
    cfgs = factory.configs("tiny-inpainting")
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2)
    b, hw, steps, ratio = 2, 8, 5, 0.5
    f = 2 ** (len(cfgs[1].ch_mult) - 1)
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    eng.txt2img(tok, neg, 8, steps=steps, height=8 * hw, width=8 * hw, sampler="DDIM", token_merging_ratio=ratio)
    nz = E.per_image_noise(8, b, (4, hw, hw), 1)
    unet = CN.ControlledUNet(sd, cfgs[0], [])
    with torch.no_grad():
        c_concat = IO.txt2img_image_conditioning(sd, cfgs[1], b, f * hw, f * hw)
        with IO.concat(c_concat), TO.merging(ratio):
            ref = CN.run_sampler("DDIM", unet, O.clip_text_encode(sd, cfgs[2], tok),
                                 O.clip_text_encode(sd, cfgs[2], neg), 7.0, steps, nz[0], [])
    lat = eng.plans[(b, hw, hw, "tome", eng.merged_tokens(hw, hw, ratio))].x.reshape(b, hw, hw, 4).permute(0, 3, 1, 2)
    assert _rel(lat, ref) <= 1e-4


def test_sdxl_has_no_full_resolution_attention_so_merging_is_a_no_op(monkeypatch):
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O
    _install(monkeypatch)
    cfgs = (C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cpu", dtype=torch.float32, use_graphs=False,
                     vae_chunk=2)
    tok, neg = O.random_prompt_tokens(2, vocab_hi=997), O.empty_prompt_tokens(2, vocab_hi=997)
    kw = dict(steps=3, height=64, width=64, sampler="Euler a")
    assert eng.merged_tokens(8, 8, 0.5) == 0
    a = eng.txt2img(tok, neg, 7, **kw)
    b = eng.txt2img(tok, neg, 7, token_merging_ratio=0.5, **kw)
    assert torch.equal(a, b) and set(eng.plans) == {(2, 8, 8)}


# ------------------------------------------------------------------------------------------------ programs
def _signature(op_list):
    from test_tiling_cpu import _signature as sig
    return sig(op_list)


def test_only_full_resolution_unet_blocks_merge(monkeypatch):
    from b200sd import config as C, ops, synth
    from b200sd.unet_exec import ControlNetWeights, UNetProgram, UNetWeights
    _install(monkeypatch)
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    uw = UNetWeights(synth.make_state_dict(*cfgs, seed=0), cfgs[0], "cpu", torch.float32)
    plain, zero = UNetProgram(uw, 2, 16, 16), UNetProgram(uw, 2, 16, 16, token_merging=0)
    merged = UNetProgram(uw, 2, 16, 16, token_merging=100)
    assert _signature(plain.ops) == _signature(zero.ops) and not zero.tome
    names = [fn for fn, _, _ in merged.ops]
    want = ["input_blocks.1.1", "input_blocks.2.1", "output_blocks.9.1", "output_blocks.10.1", "output_blocks.11.1"]
    assert sorted(merged.tome) == sorted(f"{k}.transformer_blocks.0" for k in want)
    assert names.count(ops.tome_match) == names.count(ops.tome_merge) == names.count(ops.tome_unmerge_add) == 5
    for tb, (slot, members, seg) in merged.tome.items():
        assert slot.shape == members.shape == (2, 256) and seg.shape == (2, 157) and slot.dtype == torch.int32
    # the full-resolution self-attention runs on N - r rows, the other levels' and the cross-attention on all of them
    att = [a for fn, a, _ in merged.ops if fn is ops.attention]
    assert sorted({a[0].shape[1] for a in att if a[1].shape[1] == a[0].shape[1]}) == [4, 16, 64, 156]
    assert {a[0].shape[1] for a in att if a[1].shape[1] != a[0].shape[1]} == {4, 16, 64, 256}
    # ControlNet segments do not merge
    cw = ControlNetWeights(synth.make_controlnet_state_dict(cfgs[0], seed=1), cfgs[0], "cpu", torch.float32)
    step = torch.zeros((1,), dtype=torch.int32)
    plain.set_control(0, cw, 4, step)
    merged.set_control(0, cw, 4, step)
    assert _signature(plain.segments[0].ops) == _signature(merged.segments[0].ops)
    assert merged.merging == 100


def test_merged_plans_live_beside_the_plain_ones(env):
    eng = env.eng
    for ratio in (0.0, 0.5, 0.0, 0.3, -1.0):
        eng.txt2img(env.tok, env.neg, 3, steps=3, height=64, width=64, sampler="DDIM", token_merging_ratio=ratio)
    assert set(eng.plans) == {(env.b, 8, 8), (env.b, 8, 8, "tome", 32), (env.b, 8, 8, "tome", 19)}
    a = eng.txt2img(env.tok, env.neg, 3, steps=3, height=64, width=64, sampler="DDIM", token_merging_ratio=0.0)
    b = eng.txt2img(env.tok, env.neg, 3, steps=3, height=64, width=64, sampler="DDIM")
    assert torch.equal(a, b)
    assert eng.merged_tokens(8, 8, 5.0) == 48 and eng.merged_tokens(8, 8, 0.5) == int(64 * 0.5)


# ------------------------------------------------------------------------------------------------ worker / REST
@pytest.fixture()
def worker(monkeypatch):
    import logging
    from b200sd import config as C, engine as E, synth
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker
    logging.getLogger("distributed").setLevel(logging.ERROR)
    _install(monkeypatch)
    monkeypatch.setenv("B200SD_MODEL", "tiny")
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cpu", dtype=torch.float32, use_graphs=False,
                     vae_chunk=2)
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    calls = []
    for name in ("txt2img", "img2img", "txt2img_hires"):
        real = getattr(eng, name)
        monkeypatch.setattr(eng, name, (lambda real, name: lambda *a, **k: calls.append((name, k)) or real(*a, **k))(
            real, name))
    return LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0), calls


def _payload(**kw):
    p = {"prompt": "a b", "negative_prompt": "", "seed": 30, "subseed": 4, "subseed_strength": 0, "batch_size": 2,
         "n_iter": 1, "steps": 3, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0}
    p.update(kw)
    return p


def _png(px=64):
    import base64
    import io
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(_init_u8(1, px)[0].numpy()).save(buf, format="PNG")
    return base64.b64encode(buf.getvalue()).decode()


@pytest.mark.parametrize("fields,opts,want", [
    ({}, {}, 0), (dict(token_merging_ratio=0.5), {}, 0.5), (dict(token_merging_ratio=None), {"token_merging_ratio": 0.3}, 0.3),
    (dict(override_settings={"token_merging_ratio": 0.4}), {"token_merging_ratio": 0.3}, 0.4),
    (dict(token_merging_ratio=0.2, override_settings={"token_merging_ratio": 0.4}), {}, 0.2),
    (dict(token_merging_ratio=0), {"token_merging_ratio_img2img": 0.6}, 0),
    (dict(token_merging_ratio=-0.5), {}, -0.5)])
def test_worker_resolves_the_txt2img_ratio(worker, monkeypatch, fields, opts, want):
    import modules.shared as shared
    wk, calls = worker
    for k in ("token_merging_ratio", "token_merging_ratio_hr", "token_merging_ratio_img2img"):
        monkeypatch.setattr(shared.opts, k, opts.get(k, 0), raising=False)
    wk.request(_payload(**fields), None, False)
    name, kw = calls[-1]
    assert name == "txt2img"
    assert kw.get("token_merging_ratio", 0) == (want if want > 0 else 0) and (want > 0 or "token_merging_ratio" not in kw)
    info = json.loads(wk.response["info"])
    tail = f", Token merging ratio: {want}" if want != 0 else ""
    assert all(t.endswith(tail) and ("Token merging" in t) == (want != 0) for t in info["infotexts"])


@pytest.mark.parametrize("fields,opts,want", [
    (dict(token_merging_ratio=0.5), {}, (0.5, 0.5)),
    (dict(token_merging_ratio=0.5, token_merging_ratio_hr=0.2), {}, (0.5, 0.2)),
    (dict(token_merging_ratio=0.5), {"token_merging_ratio_hr": 0.3}, (0.5, 0.3)),
    (dict(override_settings={"token_merging_ratio_hr": 0.4}), {"token_merging_ratio": 0.1}, (0.1, 0.4)),
    ({}, {"token_merging_ratio_hr": 0.4}, (0, 0.4))])
def test_worker_resolves_the_hires_ratio(worker, monkeypatch, fields, opts, want):
    import modules.shared as shared
    wk, calls = worker
    for k in ("token_merging_ratio", "token_merging_ratio_hr", "token_merging_ratio_img2img"):
        monkeypatch.setattr(shared.opts, k, opts.get(k, 0), raising=False)
    wk.request(_payload(enable_hr=True, hr_scale=2.0, **fields), None, False)
    name, kw = calls[-1]
    assert name == "txt2img_hires"
    assert kw.get("token_merging_ratio", 0) == want[0] and kw.get("token_merging_ratio_hr", 0) == want[1]
    t = json.loads(wk.response["info"])["infotexts"][0]
    assert (f", Token merging ratio: {want[0]}" in t) == (want[0] != 0)
    assert (f", Token merging ratio hr: {want[1]}" in t) == (want[1] != 0)


@pytest.mark.parametrize("fields,opts,want", [
    (dict(token_merging_ratio=0.5), {"token_merging_ratio_img2img": 0.2}, 0.5),
    ({}, {"token_merging_ratio_img2img": 0.2, "token_merging_ratio": 0.6}, 0.2),
    ({}, {"token_merging_ratio": 0.6}, 0.6),
    (dict(override_settings={"token_merging_ratio": 0.1}), {"token_merging_ratio_img2img": 0.2}, 0.1),
    (dict(override_settings={"token_merging_ratio": 0}), {"token_merging_ratio_img2img": 0.2}, 0.2)])
def test_worker_resolves_the_img2img_ratio(worker, monkeypatch, fields, opts, want):
    import modules.shared as shared
    wk, calls = worker
    for k in ("token_merging_ratio", "token_merging_ratio_hr", "token_merging_ratio_img2img"):
        monkeypatch.setattr(shared.opts, k, opts.get(k, 0), raising=False)
    wk.request(_payload(init_images=[_png()], **fields), None, False)
    name, kw = calls[-1]
    assert name == "img2img" and kw.get("token_merging_ratio") == want
    t = json.loads(wk.response["info"])["infotexts"][0]
    assert t.endswith(f", Token merging ratio: {want}") and "hr:" not in t


def test_worker_refuses_a_non_numeric_ratio_and_keeps_the_plain_call(worker):
    from scripts.spartan.worker import InvalidWorkerResponse
    wk, calls = worker
    wk.request(_payload(), None, False)
    assert not any(k.startswith("token_merging") for k in calls[-1][1])
    n = len(calls)
    with pytest.raises((ValueError, InvalidWorkerResponse)):
        wk.request(_payload(token_merging_ratio="half"), None, False)
        raise AssertionError(wk.response)   # pragma: no cover - request() reports instead of raising
    assert len(calls) == n


def test_infotext_order_puts_the_ratios_before_tiling(worker):
    wk, _ = worker
    wk.request(_payload(tiling=True, token_merging_ratio=0.5, enable_hr=True, hr_scale=2.0, token_merging_ratio_hr=0.25),
               None, False)
    t = json.loads(wk.response["info"])["infotexts"][0]
    assert t.endswith(", Token merging ratio: 0.5, Token merging ratio hr: 0.25, Tiling: True")


class _RecordingEngine:
    def __init__(self):
        self.interrupted = False
        self.clip_cfg = types.SimpleNamespace(vocab=1000)
        self.calls = []

    def txt2img(self, tok, neg, seed, **kw):
        self.calls.append(kw)
        return torch.zeros((tok.shape[0], kw["height"], kw["width"], 3), dtype=torch.uint8)


def test_rest_server_forwards_the_ratio_fields():
    from fastapi.testclient import TestClient
    from server.sdapi import create_app
    eng = _RecordingEngine()
    client = TestClient(create_app(lambda device: eng, [0]))
    body = {"prompt": "a", "steps": 2, "width": 64, "height": 64, "sampler_name": "DDIM"}
    r = client.post("/sdapi/v1/txt2img", json=dict(body, token_merging_ratio=0.5))
    assert r.status_code == 200 and eng.calls[-1]["token_merging_ratio"] == 0.5
    assert json.loads(r.json()["info"])["infotexts"][0].endswith(", Token merging ratio: 0.5")
    r = client.post("/sdapi/v1/txt2img", json=dict(body, override_settings={"token_merging_ratio": 0.3}))
    assert r.status_code == 200 and eng.calls[-1]["token_merging_ratio"] == 0.3
    r = client.post("/sdapi/v1/txt2img", json=body)
    assert r.status_code == 200 and not any(k.startswith("token_merging") for k in eng.calls[-1])
