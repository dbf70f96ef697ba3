"""Prompt editing on the H100: b200sd_select_context against a torch gather + zero fill, and the engine's scheduled
requests on the tiny model (equal entries give the plain request bitwise, graphs on and off agree, [a:b:0] is b)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_select_context_is_a_gather_and_zero_fill(dtype):
    from b200sd import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    e, cap, c, rows = 5, 154, 768, 6
    bank = torch.randn((e, cap, c), device="cuda", generator=g).to(dtype)
    lens = torch.tensor([77, 154, 77, 154, 1], device="cuda", dtype=torch.int32)
    sched = torch.tensor([[0, 1, 2, 3, 4, 0], [4, 3, 2, 1, 0, 1]], device="cuda", dtype=torch.int32)
    ctx = torch.full((rows, cap, c), 7.0, device="cuda", dtype=dtype)
    kv = torch.zeros((rows,), device="cuda", dtype=torch.int32)
    for s in range(2):
        step = torch.tensor([s], device="cuda", dtype=torch.int32)
        ops.select_context(bank, lens, sched, step, ctx, kv)
        torch.cuda.synchronize()
        idx = sched[s].long()
        want = bank[idx].clone()
        n = lens[idx]
        want[torch.arange(cap, device="cuda")[None, :] >= n[:, None].long()] = 0
        assert torch.equal(ctx, want) and torch.equal(kv, n)


def test_select_context_refuses_bad_arguments():
    from b200sd import _lib, ops
    bank = torch.zeros((2, 77, 12), device="cuda", dtype=torch.float16)   # ctx_dim % 8 != 0
    z = torch.zeros((2,), device="cuda", dtype=torch.int32)
    with pytest.raises(_lib.B200SDError):
        ops.select_context(bank, z, torch.zeros((1, 2), device="cuda", dtype=torch.int32), z[:1],
                           torch.zeros((2, 77, 12), device="cuda", dtype=torch.float16), z)


def _engine(graphs):
    from b200sd import config as C, engine as E, synth
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    return E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=graphs)


def _sched(texts, ends):
    from b200sd.engine import PromptSchedule
    from b200sd.factory import tokenize_prompts
    return PromptSchedule(list(ends), tokenize_prompts(texts, 1000)[0])


def _tok(text, b=2):
    from b200sd.factory import tokenize_prompts
    return tokenize_prompts([text] * b, 1000)[0]


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_scheduled_requests_on_the_tiny_model(sampler):
    from b200sd.engine import total_steps
    kw = dict(seed=3, steps=6, height=128, width=128, sampler=sampler)
    end = total_steps(sampler, 6)
    on, off = _engine(True), _engine(False)
    plain = on.txt2img(_tok("a cat"), _tok(""), **kw)
    same = on.txt2img(_tok("x"), _tok(""), schedule=(_sched(["a cat", "a cat"], [2, end]), _sched([""], [end])), **kw)
    assert torch.equal(same, plain)
    sch = (_sched(["a cat", "a dog", "a cow"], [2, 4, end]), _sched(["ugly", ""], [3, end]))
    g = on.txt2img(_tok("x"), _tok(""), schedule=sch, **kw)
    e = off.txt2img(_tok("x"), _tok(""), schedule=sch, **kw)
    assert torch.equal(g, e) and not torch.equal(g, plain)
    one = on.txt2img(_tok("x", 1), _tok("", 1), schedule=sch, **kw)
    assert torch.equal(one[0], g[0])


def test_edit_at_zero_is_the_second_prompt():
    from b200sd.prompts import prompt_schedule
    eng = _engine(True)
    kw = dict(seed=3, steps=6, height=128, width=128, sampler="DDIM")
    (end, text), = prompt_schedule("a [cat:dog:0]", 6)
    got = eng.txt2img(_tok("x"), _tok(""), schedule=(_sched([text], [end]), _sched([""], [end])), **kw)
    assert torch.equal(got, eng.txt2img(_tok("a dog"), _tok(""), **kw))


# ------------------------------------------------------------------------------------------------ against the oracle
def _u8(name, got, ref, mean=1.5, within2=0.97, within4=0.0):
    """the LSB bounds of the existing GPU request tests: fp16 as tests/test_controlnet_gpu.py, bf16 (SDXL) as
    tests/test_sdxl_gpu.py (mean <= 2, >= 95 % within 4)"""
    d = (got.cpu().int() - ref.cpu().int()).abs().float()
    rec = dict(u8_mean=float(d.mean()), u8_max=float(d.max()), u8_within2=float((d <= 2).float().mean()),
               u8_within4=float((d <= 4).float().mean()))
    print(name, rec)
    assert got.shape == ref.shape and rec["u8_mean"] <= mean, (name, rec)
    assert rec["u8_within2"] >= within2 and rec["u8_within4"] >= within4, (name, rec)


def _of(text, steps, hires=None, base=None):
    from b200sd.prompts import prompt_schedule
    sch = prompt_schedule(text, base if hires else steps, hires)
    return _sched([t for _, t in sch], [e for e, _ in sch])


def _oracle_z(dsd, cfgs, name, steps, sched, nz, init=None, d=None, mask=None, units=()):
    from oracle import controlnet_oracle as CN, prompt_oracle as P, prompt_schedule_oracle as PSO
    cs, us = sched
    inner = CN.ControlledUNet(dsd, cfgs[0], list(units))
    unet = PSO.Scheduled(lambda x, t, c, y: inner(x, t, c), P.encode_sd1(dsd, cfgs[2], cs.tokens.cuda()),
                         P.encode_sd1(dsd, cfgs[2], us.tokens.cuda()), cs.ends, us.ends, inner=inner)
    c, u = unet.placeholders(nz.shape[1])
    z = CN.run_sampler(name, unet, c, u, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d, mask=mask)
    assert len(set(unet.entries)) >= 2
    return z if mask is None else z * mask[1] + init * (1 - mask[1])


@pytest.fixture(scope="module")
def tiny():
    from b200sd import config as C, engine as E, synth
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    return E, cfgs, sd, {k: v.cuda() for k, v in sd.items()}, E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)


LONG = "a dog " + " ".join(f"w{i}" for i in range(80))


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_tiny_txt2img_matches_the_oracle(tiny, sampler):
    from oracle import sd_oracle as O
    E, cfgs, sd, dsd, eng = tiny
    b, hw, steps = 2, 16, 6
    total = E.total_steps(sampler, steps)
    sched = (_of(f"a [cat:{LONG}:0.5]", total), _of("[:ugly:2]", total))
    pr = eng.program(sampler, None, steps)
    nz = E.per_image_noise(41, b, (4, hw, hw), 1 + pr.draws)
    got = eng.txt2img(_tok("x"), _tok(""), 41, steps=steps, height=8 * hw, width=8 * hw, sampler=sampler,
                      schedule=sched)
    plan = eng.plan(b, hw, hw)
    assert any(n.startswith("ctx") for n in plan.graphs) and plan.kv_len.tolist() == [154, 154, 77, 77]
    with torch.no_grad():
        z = _oracle_z(dsd, cfgs, sampler, steps, sched, nz.cuda())
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8(f"tiny {sampler}", got, ref)


def test_tiny_masked_img2img_hires_and_controlnet_match_the_oracle(tiny):
    from b200sd import synth
    from b200sd.unet_exec import ControlNetWeights
    from oracle import sd_oracle as O, upscale_oracle as UO
    E, cfgs, sd, dsd, eng = tiny
    b, hw, steps = 2, 16, 8
    sched = (_of("a [cat:dog:0.5]", steps), _of("[ugly:3]", steps))
    f = 2 ** (len(cfgs[1].ch_mult) - 1)
    init_u8 = torch.randint(0, 256, (b, f * hw, f * hw, 3), generator=torch.Generator().manual_seed(9),
                            dtype=torch.uint8)
    nmask = (torch.rand((hw, hw), generator=torch.Generator().manual_seed(5)) > 0.5).float()
    pr = eng.program("Euler a", None, steps, denoise=0.75, masked=True)
    nz = E.per_image_noise(31, b, (4, hw, hw), 1 + pr.draws).cuda()
    got = eng.img2img(_tok("x"), _tok(""), 31, init_u8, denoising_strength=0.75, steps=steps, sampler="Euler a",
                      latmask=nmask.reshape(-1), schedule=sched)
    with torch.no_grad():
        init = O.vae_encode_mean(dsd, cfgs[1], O.image_to_model_input(init_u8.cuda())) * cfgs[1].scale_factor
        z = _oracle_z(dsd, cfgs, "Euler a", steps, sched, nz, init=init, d=0.75, mask=(init, nmask.cuda()[None, None]))
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8("tiny masked img2img", got, ref)

    hr_steps, d = 8, 0.9
    second = (_of("b [c:1.5]", steps, hr_steps, steps), _of("", steps, hr_steps, steps))
    got = eng.txt2img_hires(_tok("x"), _tok(""), 77, steps=steps, height=8 * hw, width=8 * hw, hr_scale=2.0,
                            hr_steps=hr_steps, denoising_strength=d, schedule=sched, hr_schedule=second)
    with torch.no_grad():
        z1 = _oracle_z(dsd, cfgs, "DDIM", steps, sched, E.per_image_noise(77, b, (4, hw, hw), 1).cuda())
        up = UO.hires_upscale(dsd, cfgs[1], z1, 2 * hw, 2 * hw, "Latent")
        z = _oracle_z(dsd, cfgs, "DDIM", hr_steps, second, E.per_image_noise(77, b, (4, 2 * hw, 2 * hw), 1).cuda(),
                      init=up, d=d)
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8("tiny hires hr_prompt", got, ref)

    csd = synth.make_controlnet_state_dict(cfgs[0], seed=11)
    cw = ControlNetWeights(csd, cfgs[0], torch.device("cuda:0"), name="cn-tiny")
    hint = torch.randint(0, 256, (8 * hw, 8 * hw, 3), generator=torch.Generator().manual_seed(20), dtype=torch.uint8)
    pr = eng.program("Euler a", None, steps)
    nz = E.per_image_noise(12, b, (4, hw, hw), 1 + pr.draws).cuda()
    got = eng.txt2img(_tok("x"), _tok(""), 12, steps=steps, height=8 * hw, width=8 * hw, sampler="Euler a",
                      controls=[(cw, hint, 0.8, 0.0, 0.6)], schedule=sched)
    assert any(n.startswith("ctx|cn0=cn-tiny") for n in eng.plan(b, hw, hw).graphs)
    with torch.no_grad():
        dcsd = {k: v.cuda() for k, v in csd.items()}
        z = _oracle_z(dsd, cfgs, "Euler a", steps, sched, nz, units=[(dcsd, hint.cuda(), 0.8, 0.0, 0.6)])
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8("tiny ControlNet", got, ref)


def test_unscheduled_request_builds_no_ctx_graph(tiny):
    E, cfgs, sd, dsd, eng = tiny
    fresh = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    fresh.txt2img(_tok("a cat"), _tok(""), 5, steps=4, height=64, width=64, sampler="DDIM")
    assert set(fresh.plan(2, 8, 8).graphs) == {"DDIM:7.0", "vae"}


def test_tinyxl_matches_the_oracle():
    from b200sd import config as C, engine as E, synth
    from oracle import prompt_schedule_oracle as PSO, sd_oracle as O
    cfgs = (C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP)
    ocfgs = (O.TINYXL_UNET, O.TINYXL_VAE, O.TINYXL_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    dsd = {k: v.cuda() for k, v in sd.items()}
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True, dtype=torch.bfloat16)
    b, hw, steps = 2, 16, 5
    sched = (_of("a [cat:dog:1]", steps), _of("[:ugly:2]", steps))
    got = eng.txt2img(_tok("x"), _tok(""), 77, steps=steps, height=8 * hw, width=8 * hw, sampler="Euler a",
                      schedule=sched)
    with torch.no_grad():
        cc, yc = O.sdxl_conditioner(dsd, ocfgs[2], sched[0].tokens.cuda(), 8 * hw, 8 * hw)
        cu, yu = O.sdxl_conditioner(dsd, ocfgs[2], sched[1].tokens.cuda(), 8 * hw, 8 * hw)
        unet = PSO.Scheduled(lambda x, t, c, y: O.unet_forward(dsd, ocfgs[0], x, t, c, y=y), cc, cu, sched[0].ends,
                             sched[1].ends, yc, yu)
        nz = E.per_image_noise(77, b, (4, hw, hw), 1 + steps).cuda()
        c, u = unet.placeholders(b)
        z = O.run_sampler("Euler a", unet, c, u, 7.0, steps, nz[0], list(nz[1:]))
        ref = O.to_uint8(O.vae_decode(dsd, ocfgs[1], z / ocfgs[1].scale_factor))
    assert len(set(unet.entries)) == 3
    _u8("tinyxl Euler a", got, ref, mean=2.0, within2=0.0, within4=0.95)


# ------------------------------------------------------------------------------------------------ full size
@pytest.fixture(scope="module")
def sd15():
    from b200sd import config as C, engine as E, synth
    from b200sd.unet_exec import ControlNetWeights
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    csd = synth.make_controlnet_state_dict(C.SD15_UNET, seed=21)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    return E, cfgs, sd, csd, eng, ControlNetWeights(csd, C.SD15_UNET, torch.device("cuda:0"), name="synthetic")


def _evaluate(eng, plan, x, active):
    from b200sd import ops
    plan.step.zero_()
    plan.x.copy_(x)
    ops.pack_unet_input(plan.x, plan.unet.xin, 1.0)
    ops.select_step(plan.table, plan.step, plan.unet.cur_bias)
    plan.unet.run(active) if active else plan.unet.run()
    torch.cuda.synchronize()
    return plan.unet.eps.clone()


@pytest.mark.parametrize("control", [False, True])
def test_sd15_switch_is_set_context(sd15, control):
    """one full-size SD1.5 evaluation (512^2, batch 2): the ctx switch (select_context, then the K/V projections over
    the staging context) at a grown 154-token capacity, cond and uncond of different lengths, is bitwise the
    evaluation after set_context of the same entries"""
    E, cfgs, sd, csd, eng, cw = sd15
    b, hw = 2, 64
    g = torch.Generator().manual_seed(4)
    cond = (torch.randn((3, 154, 768), generator=g) * 0.5).cuda().half()
    unc = (torch.randn((2, 77, 768), generator=g) * 0.5).cuda().half()
    x = torch.randn((b, hw * hw, 4), generator=g).cuda()
    plan = eng.plan(b, hw, hw)
    active = ()
    with torch.no_grad():
        if control:
            hint = torch.randint(0, 256, (512, 512, 3), generator=g, dtype=torch.uint8)
            eng._windows = eng._set_controls(plan, [(cw, hint, 1.0, 0.0, 1.0)])
            eng._control_tables(plan, torch.tensor([500.0]))
            active = (0,)
        plan.table[:1].copy_(eng.temb.table(torch.tensor([500.0])))
        plan.set_context(cond[1:2].expand(b, -1, -1), unc[1:2, :77].expand(b, -1, -1))
        want = _evaluate(eng, plan, x, active)
        kv_want = plan.kv_len.clone()
        plan.set_context(cond[0:1].expand(b, -1, -1), cond[2:3].expand(b, -1, -1))   # other K/V in the buffers
        plan.set_bank(cond, unc)
        plan.set_sched(0, [(1, 4)])   # bank: cond entries 0..2, uncond entries 3, 4
        plan.step.zero_()
        plan.switch_context(active)
        got = _evaluate(eng, plan, x, active)
    assert plan.ctx_cap == 154 and plan.kv_len.tolist() == kv_want.tolist() == [154, 154, 77, 77]
    assert torch.equal(got, want)


def test_sd15_512_ddim_edit_matches_the_oracle(sd15):
    from oracle import sd_oracle as O
    E, cfgs, sd, csd, eng, cw = sd15
    steps = 6
    sched = (_of("a [cat:dog:0.5]", steps), _of("", steps))
    got = eng.txt2img(_tok("x", 1), _tok("", 1), 900, steps=steps, cfg_scale=7.0, height=512, width=512,
                      sampler="DDIM", schedule=sched)
    dsd = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        z = _oracle_z(dsd, cfgs, "DDIM", steps, sched, E.per_image_noise(900, 1, (4, 64, 64), 1).cuda())
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8("sd15 512 DDIM [cat:dog:0.5]", got, ref)
