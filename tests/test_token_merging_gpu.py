"""Token merging on the GPU: b200sd_tome_match against an fp64 computation on the same normalised metric (node_max,
chosen dst, selection boundary, partition) at the SD1.5, tiny and large-latent shapes, exact ties bitwise; tome_merge and
tome_unmerge_add bitwise against a torch restatement; one full-size SD1.5 UNet evaluation at ratio 0.5 against the
oracle driven by the executor's own matchings; tiny requests against the token-merging oracle (oracle/tome_oracle.py)
with graphs on and off, batch invariance and ratio 0 against no keyword.  Measured values are appended to
tome_parity.jsonl in kutil.OUT_DIR."""
import json
import os

import pytest
import torch

from kutil import OUT_DIR

pytestmark = pytest.mark.gpu


def _record(name, **kw):
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "tome_parity.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **kw)) + "\n")


def _rel_rms(a, b):
    return float((a.float() - b.float()).pow(2).mean().sqrt() / b.float().pow(2).mean().sqrt())


def _run_match(x, h, w, r):
    from b200sd import ops
    nb, n, c = x.shape
    slot, members = (torch.full((nb, n), -1, dtype=torch.int32, device="cuda") for _ in range(2))
    seg = torch.full((nb, n - r + 1), -1, dtype=torch.int32, device="cuda")
    ws = torch.empty((ops.tome_workspace_bytes(nb, h, w, c),), dtype=torch.uint8, device="cuda")
    ops.tome_match(x, h, w, r, slot, members, seg, ws)
    torch.cuda.synchronize()
    _run_match.ws = ws
    return slot.long().cpu(), members.long().cpu(), seg.long().cpu()


def _kernel_metric(ws, nb, ns, nd, c):
    """the normalised src / dst metric b200sd_tome_match left in its workspace (tome_kernels.cu TomeWorkspace: fp16
    [nb][ns][c], then fp16 [nb][nd][c] at the next 256-byte boundary)"""
    a = nb * ns * c * 2
    b0 = (a + 255) // 256 * 256
    return (ws[:a].view(torch.float16).reshape(nb, ns, c).cpu(),
            ws[b0:b0 + nb * nd * c * 2].view(torch.float16).reshape(nb, nd, c).cpu())


def _metric16(x):
    """tomesd's normalisation in fp16: x / ||x|| with the norm rounded to fp16"""
    n = x.float().norm(dim=-1, keepdim=True).half().float()
    return (x.float() / n).half()


def _check_partition(slot, members, seg, h, w, r):
    from oracle import tome_oracle as TO
    nb, n = slot.shape
    nm = n - r
    src, dst = TO.grid(h, w)
    ns = src.numel()
    assert seg[:, 0].eq(0).all() and seg[:, -1].eq(n).all() and (seg[:, 1:] > seg[:, :-1]).all()
    ref_members, ref_seg = TO.partition(slot, nm)
    assert torch.equal(members, ref_members) and torch.equal(seg, ref_seg)
    assert (slot[:, src] < ns - r).sum(-1).eq(ns - r).all()              # exactly ns - r unmerged src tokens
    assert torch.equal(slot[:, dst], (ns - r + torch.arange(dst.numel())).expand(nb, -1))
    unm = slot[:, src] < ns - r
    for i in range(nb):   # unmerged src tokens take slots 0.. in ascending token order
        assert torch.equal(slot[i, src][unm[i]], torch.arange(ns - r))


@pytest.mark.parametrize("nb,h,w,c,ratio", [(4, 64, 64, 320, 0.5), (3, 64, 96, 320, 0.3), (4, 16, 16, 64, 0.5),
                                            (2, 128, 128, 320, 0.5), (1, 256, 256, 64, 0.6), (2, 8, 8, 64, 0.75)])
def test_match_against_fp64(nb, h, w, c, ratio):
    from oracle import tome_oracle as TO
    g = torch.Generator().manual_seed(h * w + c)
    x = (torch.randn((nb, h * w, c), generator=g) + 0.5 * torch.randn((nb, 1, c), generator=g)).half()
    r = TO.merged_tokens(h, w, ratio)
    slot, members, seg = _run_match(x.cuda(), h, w, r)
    _check_partition(slot, members, seg, h, w, r)
    src, dst = TO.grid(h, w)
    ns = src.numel()
    ms, md = _kernel_metric(_run_match.ws, nb, ns, dst.numel(), c)
    m = _metric16(x)   # the normalisation: within one fp16 rounding of x / ||x|| (the norm's own rounding may differ)
    assert (ms.float() - m[:, src].float()).abs().max() <= 2.0 ** -9 and (md.float() - m[:, dst].float()).abs().max() <= 2.0 ** -9
    scores = ms.cuda().double() @ md.cuda().double().transpose(-1, -2)
    best = scores.max(-1).values.cpu()
    tol = 2.0 ** -22 * c + 1e-6    # fp32 accumulation of c products of unit-norm fp16 vectors
    merged = slot[:, src] >= ns - r
    chosen = scores.gather(-1, (slot[:, src] - (ns - r)).clamp(min=0).cuda()[..., None])[..., 0].cpu()
    assert ((best - chosen).abs()[merged] <= tol).all()             # every merged src went to a best dst
    lo = torch.where(merged, best, torch.full_like(best, float("inf"))).min(-1).values
    hi = torch.where(~merged, best, torch.full_like(best, -float("inf"))).max(-1).values
    assert (lo >= hi - tol).all(), (lo, hi)                           # the r largest were merged
    flips = int(((best - chosen).abs() > 0)[merged].sum())
    _record(f"match {nb}x{h}x{w}x{c} r={r}", boundary_gap=float((lo - hi).min()), argmax_non_exact=flips)


def test_match_ties_follow_the_rule_bitwise():
    h, w, c = 16, 16, 64
    from oracle import tome_oracle as TO
    src, dst = TO.grid(h, w)
    ns = src.numel()
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, h * w, c), generator=g)
    x[:, dst[5]] = x[:, dst[2]] = x[:, dst[9]]                   # three identical dst tokens
    x[:, src] = x[:, dst[9]][:, None] + 0.2 * torch.randn((2, ns, c), generator=g)
    for a in (7, 30, 31, 100):                                  # five identical src tokens: 3, 7, 30, 31, 100
        x[:, src[a]] = x[:, src[3]]
    x = x.half()
    _run_match(x.cuda(), h, w, 1)
    ms, md = (m.double() for m in _kernel_metric(_run_match.ws, 2, ns, dst.numel(), c))
    scores = ms[0] @ md[0].T
    nmax = scores.max(-1).values
    top = sorted(range(ns), key=lambda a: (-float(nmax[a]), a))
    k = top.index(3) + 3      # r takes three of the five tied src tokens
    slot, members, seg = _run_match(x.cuda(), h, w, k)
    assert [a for a in (3, 7, 30, 31, 100) if int(slot[0, src[a]]) >= ns - k] == [3, 7, 30]
    # a merged src token whose best dst is one of the identical three goes to the lowest of them (dst 2)
    close = [a for a in range(ns) if int(slot[0, src[a]]) >= ns - k and int(torch.argmax(scores[a])) in (2, 5, 9)]
    assert close and all(int(slot[0, src[a]]) == ns - k + 2 for a in close)


def test_merge_and_unmerge_add_are_bitwise_their_restatement():
    from b200sd import ops
    from oracle import tome_oracle as TO
    nb, h, w, c = 3, 64, 64, 320
    g = torch.Generator().manual_seed(2)
    x = torch.randn((nb, h * w, c), generator=g).half()
    r = TO.merged_tokens(h, w, 0.5)
    slot, members, seg = _run_match(x.cuda(), h, w, r)
    nm = h * w - r
    a = torch.randn((nb, h * w, c), generator=g).half()
    out = torch.empty((nb, nm, c), dtype=torch.float16, device="cuda")
    ops.tome_merge(a.cuda(), members.int().cuda(), seg.int().cuda(), out)
    ref = torch.empty((nb, nm, c))
    af = a.float()
    for i in range(nb):   # fp32 sums in ascending token order, rounded once
        for s in range(nm):
            mem = members[i, seg[i, s]:seg[i, s + 1]]
            acc = torch.zeros(c)
            for t in mem.tolist():
                acc = acc + af[i, t]
            ref[i, s] = acc / len(mem)
    assert torch.equal(out.cpu(), ref.half())
    y = torch.randn((nb, nm, c), generator=g).half()
    res = torch.randn((nb, h * w, c), generator=g).half()
    o = torch.empty((nb, h * w, c), dtype=torch.float16, device="cuda")
    ops.tome_unmerge_add(res.cuda(), y.cuda(), slot.int().cuda(), o)
    torch.cuda.synchronize()
    assert torch.equal(o.cpu(), (res.float() + TO.unmerge(y.float(), slot)).half())


def test_bf16_is_refused():
    from b200sd import _lib, ops
    x = torch.zeros((1, 64, 64), dtype=torch.bfloat16, device="cuda")
    z = torch.zeros((1, 64), dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.B200SDError):
        ops.tome_match(x, 8, 8, 8, z, z.clone(), torch.zeros((1, 57), dtype=torch.int32, device="cuda"),
                       torch.zeros((1 << 20,), dtype=torch.uint8, device="cuda"))


# ------------------------------------------------------------------------------------------------ full-size SD1.5
def test_sd15_unet_evaluation_with_the_executors_matchings():
    from b200sd import config as C, engine as E, ops, synth
    from oracle import sd_oracle as O, tome_oracle as TO
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=False)
    b, h, w, ratio = 1, 64, 64, 0.5
    x = O.per_image_noise(5, b, (4, h, w))
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    outs = {}
    for rt in (0.0, ratio):
        plan = eng.plan(b, h, w, token_merging_ratio=rt)
        plan.set_context(eng.encode_prompts(tok), eng.encode_prompts(neg))
        plan.table[:1].copy_(eng.temb.table(torch.tensor([651.0])))
        plan.step.zero_()
        plan.x.copy_(x.cuda().permute(0, 2, 3, 1).reshape(b, h * w, 4))
        ops.pack_unet_input(plan.x, plan.unet.xin, 1.0)
        ops.select_step(plan.table, plan.step, plan.unet.cur_bias)
        plan.unet.run()
        torch.cuda.synchronize()
        outs[rt] = plan.unet.eps[..., :4].float().reshape(2 * b, h, w, 4).permute(0, 3, 1, 2).clone()
        if rt:
            given = {tb: m[0].long() for tb, m in plan.unet.tome.items()}
    dsd = {k: v.cuda() for k, v in sd.items()}
    ctx = torch.cat([O.clip_text_encode(dsd, cfgs[2], tok.cuda()), O.clip_text_encode(dsd, cfgs[2], neg.cuda())])
    t = torch.tensor([651.0, 651.0], device="cuda")
    xx = torch.cat([x, x]).cuda()
    with torch.no_grad():
        ref0 = O.unet_forward(dsd, cfgs[0], xx, t, ctx)
        with TO.merging(ratio, given):
            ref = O.unet_forward(dsd, cfgs[0], xx, t, ctx)
        with TO.merging(ratio) as own:
            O.unet_forward(dsd, cfgs[0], xx, t, ctx)
    flips = {tb: int((own[tb] != given[tb]).any(-1).sum()) for tb in given}
    flipped_tokens = sum(int((own[tb] != given[tb]).sum()) for tb in given)
    rel, rel0 = _rel_rms(outs[ratio], ref), _rel_rms(outs[0.0], ref0)
    _record("sd15 unet eval ratio 0.5", rel_rms=rel, rel_rms_ratio0=rel0, rel_rms_vs_unmerged=_rel_rms(outs[ratio], ref0),
            oracle_own_matching_rows_differing=flips, oracle_own_matching_tokens_differing=flipped_tokens)
    assert len(given) == 5 and all(m.shape == (2 * b, h * w) for m in given.values())
    assert rel <= 5e-3, (rel, rel0)
    eng.release()


# ------------------------------------------------------------------------------------------------ tiny requests
@pytest.fixture(scope="module")
def tiny():
    from b200sd import config as C, engine as E, synth
    from b200sd.unet_exec import ControlNetWeights
    from oracle import sd_oracle as O
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    csd = synth.make_controlnet_state_dict(C.TINY_UNET, seed=11)
    cw = ControlNetWeights(csd, C.TINY_UNET, torch.device("cuda:0"), name="cn0")
    engs = {g: E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=g) for g in (True, False)}
    dsd = {k: v.cuda() for k, v in sd.items()}
    return E, O, cfgs, engs, dsd, {k: v.cuda() for k, v in csd.items()}, cw


def _u8_check(name, got, ref, mean=2.0, within=(4, 0.95)):
    du8 = (got.cpu().int() - ref.cpu().int()).abs().float()
    rec = dict(u8_mean=float(du8.mean()), u8_max=float(du8.max()), u8_within=float((du8 <= within[0]).float().mean()))
    _record(name, **rec)
    assert got.shape == ref.shape
    assert rec["u8_mean"] <= mean and rec["u8_within"] >= within[1], rec


def _oracle(env, tok, neg, seed, sampler, steps, hw, ratio, init=None, d=None, nmask=None, units=()):
    from oracle import controlnet_oracle as CN, tome_oracle as TO
    E, O, cfgs, engs, dsd, dcsd, cw = env
    b = tok.shape[0]
    cond, unc = O.clip_text_encode(dsd, cfgs[2], tok.cuda()), O.clip_text_encode(dsd, cfgs[2], neg.cuda())
    pr = engs[False].program(sampler, None, steps, denoise=d, masked=nmask is not None)
    nz = E.per_image_noise(seed, b, (4, hw, hw), 1 + pr.draws).cuda()
    unet = CN.ControlledUNet(dsd, cfgs[0], [(dcsd, h.cuda(), w, 0.0, 1.0) for h, w in units])
    mask = None if nmask is None else (init, nmask[None, None].cuda())
    with torch.no_grad(), TO.merging(ratio):
        z = CN.run_sampler(sampler, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d,
                           mask=mask)
        if mask is not None:
            z = z * mask[1] + init * (1 - mask[1])
        return O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))


def _both(env, fn):
    got = {g: fn(env[3][g]).cpu() for g in (True, False)}
    assert torch.equal(got[True], got[False])
    return got[True]


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_tiny_txt2img_matches_the_token_merging_oracle(tiny, sampler):
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    b, hw, steps = 2, 16, 8
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    got = _both(tiny, lambda e: e.txt2img(tok, neg, 300, steps=steps, height=8 * hw, width=8 * hw, sampler=sampler,
                                          token_merging_ratio=0.5))
    _u8_check(f"tiny txt2img {sampler} ratio 0.5", got, _oracle(tiny, tok, neg, 300, sampler, steps, hw, 0.5))


def test_tiny_img2img_masked_and_controlnet_match_the_oracle(tiny):
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    b, hw, steps, d = 2, 16, 10, 0.75
    f = 2 ** (len(cfgs[1].ch_mult) - 1)
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    init_u8 = torch.randint(0, 256, (b, f * hw, f * hw, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    nmask = (torch.rand((hw, hw), generator=torch.Generator().manual_seed(5)) > 0.5).float()
    got = _both(tiny, lambda e: e.img2img(tok, neg, 41, init_u8, denoising_strength=d, steps=steps, sampler="DDIM",
                                          latmask=nmask.reshape(-1).cuda(), token_merging_ratio=0.5))
    with torch.no_grad():
        init = O.vae_encode_mean(dsd, cfgs[1], O.image_to_model_input(init_u8.cuda())) * cfgs[1].scale_factor
    _u8_check("tiny img2img masked ratio 0.5", got,
              _oracle(tiny, tok, neg, 41, "DDIM", steps, hw, 0.5, init=init, d=d, nmask=nmask))
    hint = torch.randint(0, 256, (8 * hw, 8 * hw, 3), generator=torch.Generator().manual_seed(6), dtype=torch.uint8)
    got = _both(tiny, lambda e: e.txt2img(tok, neg, 300, steps=8, height=8 * hw, width=8 * hw, sampler="Euler a",
                                          controls=[(cw, hint, 0.9, 0.0, 1.0)], token_merging_ratio=0.5))
    _u8_check("tiny txt2img ControlNet ratio 0.5", got,
              _oracle(tiny, tok, neg, 300, "Euler a", 8, hw, 0.5, units=[(hint, 0.9)]))


def test_tiny_batch_invariance_and_ratio_0_is_no_keyword(tiny):
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    eng = engs[True]
    tok, neg = O.random_prompt_tokens(1, vocab_hi=997), O.empty_prompt_tokens(1, vocab_hi=997)
    kw = dict(steps=6, height=128, width=128, sampler="Euler a")
    five = eng.txt2img(tok.expand(5, -1), neg.expand(5, -1), 300, token_merging_ratio=0.5, **kw).clone()
    two = eng.txt2img(tok.expand(2, -1), neg.expand(2, -1), 303, token_merging_ratio=0.5, **kw).clone()
    torch.cuda.synchronize()
    assert torch.equal(five[3:], two)
    off = eng.txt2img(tok.expand(2, -1), neg.expand(2, -1), 303, token_merging_ratio=0.0, **kw).clone()
    plain = eng.txt2img(tok.expand(2, -1), neg.expand(2, -1), 303, **kw).clone()
    assert torch.equal(off, plain) and not torch.equal(off, two)
