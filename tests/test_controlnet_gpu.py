"""ControlNet on the GPU: b200sd_hint_to_nhwc, the in-place residual contract of b200sd_linear / b200sd_conv2d, whole
tiny requests with 1 and 2 units against the ControlNet oracle (oracle/controlnet_oracle.py) with graphs on and off, the
bitwise identities (weight 0, an empty window, batch invariance), long prompts, one full-size SD1.5 evaluation and one
512^2 request.  uint8 tolerances as tests/test_engine_gpu.py: mean |d| <= 1.5 LSB and >= 97 % of the pixels within
2 LSB (fp16)."""
import json
import os

import pytest
import torch

from kutil import OUT_DIR

pytestmark = pytest.mark.gpu


def _record(name, **kw):
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "controlnet_parity.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **kw)) + "\n")


def _u8_check(name, got, ref, mean=1.5, within2=0.97):
    du8 = (got.cpu().int() - ref.cpu().int()).abs().float()
    rec = dict(u8_mean=float(du8.mean()), u8_max=float(du8.max()), u8_within2=float((du8 <= 2).float().mean()))
    _record(name, **rec)
    assert got.shape == ref.shape
    assert rec["u8_mean"] <= mean and rec["u8_within2"] >= within2, rec


def _hint(seed, hh, ww):
    return torch.randint(0, 256, (hh, ww, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_hint_to_nhwc_exact(dt):
    from b200sd import ops
    img = torch.randint(0, 256, (3, 1037, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
    out = torch.full((3, 1037, 64), 7.0, dtype=dt, device="cuda")
    ops.hint_to_nhwc(img.cuda(), out)
    torch.cuda.synchronize()
    ref = torch.zeros((3, 1037, 64), dtype=dt)
    ref[..., :3] = (img.float() / 255.0).to(dt)
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_linear_residual_in_place_on_a_channel_slice(dt):
    """out = residual = a strided channel slice of a concat buffer: bitwise the out-of-place call on a copy; the other
    channels untouched.  M spans 32 row tiles, N = 320 several column chunks."""
    from b200sd import ops
    g = torch.Generator().manual_seed(2)
    m, k, n = 4096, 320, 320
    a = torch.randn((m, k), generator=g).to(dt).cuda()
    w = (torch.randn((n, k), generator=g) / k ** 0.5).to(dt).cuda()
    bias = torch.randn((n,), generator=g).cuda()
    cat = torch.randn((m, 640), generator=g).to(dt).cuda()
    before = cat.clone()
    sl = cat[:, 320:]
    ref = torch.empty((m, n), dtype=dt, device="cuda")
    ops.linear(a, w, ref, bias=bias, residual=sl.clone())
    ops.linear(a, w, sl, bias=bias, residual=sl)
    torch.cuda.synchronize()
    assert torch.equal(sl, ref) and torch.equal(cat[:, :320], before[:, :320])


def test_conv2d_residual_in_place_on_a_channel_slice():
    from b200sd import ops
    g = torch.Generator().manual_seed(3)
    nb, h, w, c, cout = 2, 32, 32, 128, 192
    x = torch.randn((nb, h, w, c), generator=g).half().cuda()
    wt = (torch.randn((cout, 9 * c), generator=g) / (9 * c) ** 0.5).half().cuda()
    bias = torch.randn((cout,), generator=g).cuda()
    cat = torch.randn((nb * h * w, 320), generator=g).half().cuda()
    before = cat.clone()
    sl = cat[:, 128:]
    ref = torch.empty((nb * h * w, cout), dtype=torch.float16, device="cuda")
    ops.conv2d(x, wt, ref, ksize=3, bias=bias, residual=sl.clone())
    ops.conv2d(x, wt, sl, ksize=3, bias=bias, residual=sl)
    torch.cuda.synchronize()
    assert torch.equal(sl, ref) and torch.equal(cat[:, :128], before[:, :128])


# ------------------------------------------------------------------------------------------------ tiny requests
@pytest.fixture(scope="module")
def tiny():
    from b200sd import config as C, engine as E, synth
    from b200sd.unet_exec import ControlNetWeights
    from oracle import sd_oracle as O
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    csds = [synth.make_controlnet_state_dict(C.TINY_UNET, seed=s) for s in (11, 12)]
    cws = [ControlNetWeights(c, C.TINY_UNET, torch.device("cuda:0"), name=f"cn{k}") for k, c in enumerate(csds)]
    engs = {g: E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=g) for g in (True, False)}
    dsd = {k: v.cuda() for k, v in sd.items()}
    dcsds = [{k: v.cuda() for k, v in c.items()} for c in csds]
    return E, O, cfgs, engs, dsd, dcsds, cws


def _oracle(env, tok, neg, seed, sampler, steps, units, hw):
    from oracle import controlnet_oracle as CN
    E, O, cfgs, engs, dsd, dcsds, cws = env
    b = tok.shape[0]
    cond, unc = O.clip_text_encode(dsd, cfgs[2], tok.cuda()), O.clip_text_encode(dsd, cfgs[2], neg.cuda())
    pr = engs[False].program(sampler, None, steps)
    nz = E.per_image_noise(seed, b, (4, hw, hw), 1 + pr.draws).cuda()
    unet = CN.ControlledUNet(dsd, cfgs[0], [(dcsds[k], h.cuda(), w, a, e) for k, h, w, a, e in units])
    with torch.no_grad():
        z = CN.run_sampler(sampler, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]))
        return O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
@pytest.mark.parametrize("n_units", [1, 2])
def test_tiny_request_matches_the_oracle_graphs_on_and_off(tiny, sampler, n_units):
    from oracle import sd_oracle as O
    E, _, cfgs, engs, dsd, dcsds, cws = tiny
    b, hw, steps = 2, 16, 8
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    units = [(0, _hint(5, 8 * hw, 8 * hw), 0.9, 0.0, 1.0), (1, _hint(6, 8 * hw, 8 * hw), 0.6, 0.25, 0.75)][:n_units]
    controls = [(cws[k], h, w, a, e) for k, h, w, a, e in units]
    got = {g: engs[g].txt2img(tok, neg, 300, steps=steps, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler=sampler,
                              controls=controls).cpu() for g in (True, False)}
    assert torch.equal(got[True], got[False])
    ref = _oracle(tiny, tok, neg, 300, sampler, steps, units, hw)
    _u8_check(f"tiny {sampler} units={n_units}", got[True], ref)
    plain = engs[True].txt2img(tok, neg, 300, steps=steps, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler=sampler)
    assert not torch.equal(plain.cpu(), got[True])


def test_weight_zero_and_an_empty_window_are_bitwise_no_controlnet(tiny):
    from oracle import sd_oracle as O
    E, _, cfgs, engs, dsd, dcsds, cws = tiny
    eng = engs[True]
    b, hw = 2, 16
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    kw = dict(steps=8, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler="Euler a")
    plain = eng.txt2img(tok, neg, 301, **kw).cpu()
    zero = eng.txt2img(tok, neg, 301, controls=[(cws[0], _hint(7, 8 * hw, 8 * hw), 0.0, 0.0, 1.0)], **kw).cpu()
    # 8 steps: i / n takes 0, 0.125, ..., 0.875 — no step lies in [0.95, 1.0]
    empty = eng.txt2img(tok, neg, 301, controls=[(cws[0], _hint(7, 8 * hw, 8 * hw), 1.0, 0.95, 1.0)], **kw).cpu()
    assert torch.equal(plain, zero) and torch.equal(plain, empty)


def test_batch_invariance(tiny):
    from oracle import sd_oracle as O
    E, _, cfgs, engs, dsd, dcsds, cws = tiny
    eng = engs[True]
    hw = 16
    tok, neg = O.random_prompt_tokens(4, vocab_hi=997), O.empty_prompt_tokens(4, vocab_hi=997)
    controls = [(cws[0], _hint(8, 8 * hw, 8 * hw), 1.0, 0.0, 1.0)]
    kw = dict(steps=6, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler="DDIM", controls=controls)
    four = eng.txt2img(tok, neg, 500, **kw).cpu()
    for k in range(4):
        one = eng.txt2img(tok[k:k + 1], neg[k:k + 1], 500 + k, **kw).cpu()
        assert torch.equal(one[0], four[k]), k


def test_long_prompt_grows_the_segment_context(tiny):
    """a 150-token prompt (two chunks) against a one-chunk negative: the segment's cross-attention K/V grow with the
    plan's and attend to each row's own length"""
    from b200sd import factory
    from oracle import controlnet_oracle as CN, prompt_oracle as P, sd_oracle as O
    E, _, cfgs, engs, dsd, dcsds, cws = tiny
    eng = engs[True]
    b, hw, steps = 2, 16, 6
    prompt = " ".join(f"w{i}" for i in range(150))
    ids, mult = factory.tokenize_prompts([prompt] * b, cfgs[2].vocab)
    nids, _ = factory.tokenize_prompts([""] * b, cfgs[2].vocab)
    assert ids.shape[1] == 154 and nids.shape[1] == 77
    hint = _hint(9, 8 * hw, 8 * hw)
    got = eng.txt2img(ids, nids, 77, steps=steps, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler="DDIM",
                      controls=[(cws[0], hint, 1.0, 0.0, 1.0)]).cpu()
    cond = P.encode_sd1(dsd, cfgs[2], ids.cuda())
    unc = P.encode_sd1(dsd, cfgs[2], nids.cuda())
    nz = E.per_image_noise(77, b, (4, hw, hw), 1).cuda()
    ctl = CN.ControlledUNet(dsd, cfgs[0], [(dcsds[0], hint.cuda(), 1.0, 0.0, 1.0)])
    ctl.active = (0,)
    with torch.no_grad():
        x = nz[0]
        for (t, sa, s1a, sap, s1ap) in O.ddim_coefficients(steps):
            tt = torch.full((b,), float(t), device="cuda")
            ec, eu = ctl(x, tt, cond), ctl(x, tt, unc)   # sdwui's two UNet calls for contexts of different lengths
            e = eu + 7.0 * (ec - eu)
            x = sap * ((x - s1a * e) / sa) + s1ap * e
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], x / cfgs[1].scale_factor))
    _u8_check("tiny long prompt", got, ref)


# ------------------------------------------------------------------------------------------------ full size
@pytest.fixture(scope="module")
def sd15():
    from b200sd import config as C, engine as E, synth
    from b200sd.unet_exec import ControlNetWeights
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    csd = synth.make_controlnet_state_dict(C.SD15_UNET, seed=21)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    cw = ControlNetWeights(csd, C.SD15_UNET, torch.device("cuda:0"), name="synthetic")
    return E, cfgs, sd, csd, eng, cw


def test_sd15_evaluation_matches_the_oracle(sd15):
    """one controlled UNet evaluation at 512^2 (batch 1 + its uncond) against the fp32 oracle, rel-rms"""
    from oracle import controlnet_oracle as CN, sd_oracle as O
    E, cfgs, sd, csd, eng, cw = sd15
    hw = 64
    g = torch.Generator().manual_seed(4)
    x = torch.randn((1, 4, hw, hw), generator=g)
    ctx = torch.randn((2, 77, 768), generator=g) * 0.5
    hint = _hint(10, 512, 512)
    plan = eng.plan(1, hw, hw)
    with torch.no_grad():
        eng._windows = eng._set_controls(plan, [(cw, hint, 1.0, 0.0, 1.0)])
        eng._control_tables(plan, torch.tensor([500.0]))
        plan.unet.set_context(ctx.cuda().half())
        plan.table[:1].copy_(eng.temb.table(torch.tensor([500.0])))
        plan.step.zero_()
        plan.x.copy_(x.permute(0, 2, 3, 1).reshape(1, hw * hw, 4).cuda())
        from b200sd import ops
        ops.pack_unet_input(plan.x, plan.unet.xin, 1.0)
        ops.select_step(plan.table, plan.step, plan.unet.cur_bias)
        plan.unet.run((0,))
        got = plan.unet.eps[:, :, :4].float().reshape(2, hw, hw, 4).permute(0, 3, 1, 2).cpu()
        dsd = {k: v.cuda() for k, v in sd.items()}
        dcsd = {k: v.cuda() for k, v in csd.items()}
        ref = CN.unet_forward(dsd, cfgs[0], torch.cat([x, x]).cuda(), torch.full((2,), 500.0, device="cuda"), ctx.cuda(),
                              [(dcsd, CN.hint_input(hint[None]).cuda(), 1.0)]).cpu()
    rel = float((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
    _record("sd15 evaluation", rel_rms=rel)
    assert rel <= 5e-3, rel


def test_sd15_512_ddim_request(sd15):
    from oracle import controlnet_oracle as CN, sd_oracle as O
    E, cfgs, sd, csd, eng, cw = sd15
    tok, neg = O.random_prompt_tokens(1), O.empty_prompt_tokens(1)
    hint = _hint(11, 512, 512)
    steps = 6
    got = eng.txt2img(tok, neg, 900, steps=steps, cfg_scale=7.0, height=512, width=512, sampler="DDIM",
                      controls=[(cw, hint, 1.0, 0.0, 1.0)]).cpu()
    dsd = {k: v.cuda() for k, v in sd.items()}
    dcsd = {k: v.cuda() for k, v in csd.items()}
    with torch.no_grad():
        cond, unc = O.clip_text_encode(dsd, cfgs[2], tok.cuda()), O.clip_text_encode(dsd, cfgs[2], neg.cuda())
        nz = E.per_image_noise(900, 1, (4, 64, 64), 1).cuda()
        unet = CN.ControlledUNet(dsd, cfgs[0], [(dcsd, hint.cuda(), 1.0, 0.0, 1.0)])
        z = CN.run_sampler("DDIM", unet, cond, unc, 7.0, steps, nz[0])
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8_check("sd15 512 DDIM", got, ref)
