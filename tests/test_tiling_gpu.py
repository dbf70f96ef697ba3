"""Seamless tiling on the GPU: b200sd_pad_circular bitwise against a torch.cat wrap, pad-then-conv against fp32
circular convolutions, shift equivariance of a full-size SD1.5 UNet evaluation and VAE decode (tiling off: it does not
hold), tiny requests against the tiling oracle (oracle/tiling_oracle.py) with graphs on and off, batch invariance,
tiling=False against no keyword, and one SD1.5 512^2 DDIM request, whose 2x2 mosaic is saved for inspection.
uint8 tolerances as tests/test_engine_gpu.py (fp16: mean |d| <= 1.5 LSB, >= 97 % within 2 LSB) and tests/test_sdxl_gpu.py
(bf16: mean <= 2 LSB, >= 95 % within 4 LSB)."""
import json
import os

import pytest
import torch

from kutil import OUT_DIR

pytestmark = pytest.mark.gpu
# rolled against unrolled evaluations: rel-rms of fp16 rounding in reordered GroupNorm / attention sums (the parity bound
# of one UNet evaluation against the fp32 oracle is 5e-3); zero-padded convs do not meet it
ROLL_REL_RMS = 5e-3


def _record(name, **kw):
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "tiling_parity.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **kw)) + "\n")


def _u8_check(name, got, ref, mean=1.5, within=(2, 0.97)):
    du8 = (got.cpu().int() - ref.cpu().int()).abs().float()
    rec = dict(u8_mean=float(du8.mean()), u8_max=float(du8.max()), u8_within=float((du8 <= within[0]).float().mean()))
    _record(name, **rec)
    assert got.shape == ref.shape
    assert rec["u8_mean"] <= mean and rec["u8_within"] >= within[1], rec


def _rel_rms(a, b):
    return float((a.float() - b.float()).pow(2).mean().sqrt() / b.float().pow(2).mean().sqrt())


# ------------------------------------------------------------------------------------------------ kernel
def _wrap(x, p):
    """x [NB, H, W, C] -> circularly padded by p, by concatenation"""
    x = torch.cat([x[:, -p:], x, x[:, :p]], dim=1)
    return torch.cat([x[:, :, -p:], x, x[:, :, :p]], dim=2)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (2, 64), (7, 2), (7, 7), (64, 64)])
@pytest.mark.parametrize("sliced", [False, True])
def test_pad_circular_is_a_wrap(dt, h, w, sliced):
    from b200sd import ops
    g = torch.Generator().manual_seed(h * 100 + w)
    c = 72
    full = torch.randn((3, h, w, 256 if sliced else c), generator=g).to(dt).cuda()
    x = full[..., 64:64 + c] if sliced else full
    for p in sorted({1, min(h, w)}):
        out = torch.full((3, h + 2 * p, w + 2 * p, c), 7.0, dtype=dt, device="cuda")
        ops.pad_circular(x, out, p)
        torch.cuda.synchronize()
        assert torch.equal(out, _wrap(x, p)), p


def test_pad_circular_refuses_a_halo_wider_than_the_image():
    from b200sd import _lib, ops
    x = torch.zeros((1, 1, 4, 8), dtype=torch.float16, device="cuda")
    out = torch.zeros((1, 5, 8, 8), dtype=torch.float16, device="cuda")
    with pytest.raises(_lib.B200SDError):
        ops.pad_circular(x, out, 2)


@pytest.mark.parametrize("name,nb,hw,c,cout,stride", [("unet 64x64x320", 2, 64, 320, 320, 1),
                                                       ("unet Downsample", 2, 64, 320, 320, 2),
                                                       ("unet 8x8x1280", 4, 8, 1280, 1280, 2),
                                                       ("vae 256x256x128", 1, 256, 128, 128, 1),
                                                       ("vae 128x128x512", 1, 128, 512, 256, 1)])
def test_pad_then_conv_is_a_circular_conv(name, nb, hw, c, cout, stride):
    from b200sd import ops
    from b200sd.weights import pack_conv
    g = torch.Generator().manual_seed(nb * hw + c)
    x = torch.randn((nb, hw, hw, c), generator=g).half().cuda()
    w = (torch.randn((cout, c, 3, 3), generator=g) / (9 * c) ** 0.5)
    bias = torch.randn((cout,), generator=g).cuda()
    xp = torch.empty((nb, hw + 2, hw + 2, c), dtype=torch.float16, device="cuda")
    ho = (hw + 1) // 2 if stride == 2 else hw
    out = torch.empty((nb * ho * ho, cout), dtype=torch.float16, device="cuda")
    ops.pad_circular(x, xp, 1)
    ops.conv2d(xp, pack_conv(w).half().cuda(), out, ksize=3, stride=stride, pad=0, bias=bias)
    torch.cuda.synchronize()
    conv = torch.nn.Conv2d(c, cout, 3, stride=stride, padding=1, padding_mode="circular").cuda()
    with torch.no_grad():
        conv.weight.copy_(w.half().float())
        conv.bias.copy_(bias)
        ref = conv(x.float().permute(0, 3, 1, 2)).permute(0, 2, 3, 1).reshape(-1, cout)
    rel = _rel_rms(out, ref)
    _record(f"pad+conv {name} s{stride}", rel_rms=rel, rel_max=float((out.float() - ref).abs().max() / ref.abs().max()))
    assert out.shape == ref.shape and rel <= 2e-3, rel


# ------------------------------------------------------------------------------------------------ full-size SD1.5
@pytest.fixture(scope="module")
def sd15():
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    yield E, O, cfgs, sd, eng
    eng.release()


def _unet_eval(eng, O, cfgs, x, tiling):
    """eps of one UNet evaluation on latents x [1, 4, h, w] (cond and uncond rows), fp32 [2, 4, h, w]"""
    from b200sd import ops
    b, _, h, w = x.shape
    plan = eng.plan(b, h, w, tiling)
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    plan.set_context(eng.encode_prompts(tok), eng.encode_prompts(neg))
    plan.table[:1].copy_(eng.temb.table(torch.tensor([651.0])))
    plan.step.zero_()
    plan.x.copy_(x.cuda().permute(0, 2, 3, 1).reshape(b, h * w, 4))
    ops.pack_unet_input(plan.x, plan.unet.xin, 1.0)
    ops.select_step(plan.table, plan.step, plan.unet.cur_bias)
    plan.unet.run()
    torch.cuda.synchronize()
    return plan.unet.eps[..., :4].float().reshape(2 * b, h, w, 4).permute(0, 3, 1, 2).clone()


@pytest.mark.parametrize("tiling", [True, False])
def test_sd15_unet_and_vae_are_shift_equivariant(sd15, tiling):
    """rolling the latents by 8 (a multiple of 2^(levels - 1) = 8) rolls the circular UNet's output and the decoded image
    by 64 pixels, to fp16 rounding; with zero padding it does not"""
    E, O, cfgs, sd, eng = sd15
    x = O.per_image_noise(5, 1, (4, 64, 64))
    roll = lambda a, k: torch.roll(a, (k, -k), dims=(2, 3))  # noqa: E731
    e, er = _unet_eval(eng, O, cfgs, x, tiling), _unet_eval(eng, O, cfgs, roll(x, 8), tiling)
    unet_rel = _rel_rms(er, roll(e, 8))

    def decoded(z):   # the decoder's fp16 output before quantisation, [1, 3, 512, 512]
        eng.decode(z.permute(0, 2, 3, 1).reshape(1, 64 * 64, 4).cuda().contiguous(), 64, 64, tiling=tiling)
        img = eng.plan(1, 64, 64, tiling).vae.img[..., :3]
        return img.float().reshape(1, 512, 512, 3).permute(0, 3, 1, 2).clone()

    img, img_r = decoded(x * 0.8), decoded(roll(x * 0.8, 8))
    vae_rel = _rel_rms(img_r, roll(img, 64))
    _record(f"sd15 roll equivariance tiling={tiling}", unet_rel_rms=unet_rel, vae_rel_rms=vae_rel)
    if tiling:
        assert unet_rel <= ROLL_REL_RMS and vae_rel <= ROLL_REL_RMS, (unet_rel, vae_rel)
    else:
        assert unet_rel > ROLL_REL_RMS and vae_rel > ROLL_REL_RMS, (unet_rel, vae_rel)


def test_sd15_512_ddim_request_matches_the_tiling_oracle(sd15):
    from PIL import Image
    from oracle import tiling_oracle as T
    E, O, cfgs, sd, eng = sd15
    b, steps = 1, 20
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    got = eng.txt2img(tok, neg, 1000, steps=steps, cfg_scale=7.0, height=512, width=512, sampler="DDIM", tiling=True)
    torch.cuda.synchronize()
    dsd = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        ref, _, _ = T.run(O.txt2img, dsd, *cfgs, tok, neg, seed=1000, steps=steps, cfg_scale=7.0, height=512, width=512,
                          device="cuda")
    del dsd
    _u8_check("sd15 512 DDIM tiled", got, ref)
    img = got[0].cpu()
    # across the wrap seam the image continues: its row / column steps there are like the interior ones
    seam = float(((img[0].float() - img[-1].float()).abs().mean() + (img[:, 0].float() - img[:, -1].float()).abs().mean()) / 2)
    interior = float((img[1:].float() - img[:-1].float()).abs().mean())
    _record("sd15 512 DDIM tiled seam", seam_step_mean=seam, interior_step_mean=interior)
    os.makedirs(OUT_DIR, exist_ok=True)
    Image.fromarray(torch.cat([torch.cat([img, img], 1)] * 2, 0).numpy()).save(os.path.join(OUT_DIR, "tiling_mosaic.png"))
    assert seam <= 2.0 * interior, (seam, interior)


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


def _oracle(env, tok, neg, seed, sampler, steps, hw, init=None, d=None, nmask=None, units=()):
    """uint8 images of the tiling oracle: the ControlNet oracle's sampler with `units` [(hint, weight)] under the shim"""
    from oracle import controlnet_oracle as CN, tiling_oracle as T
    E, O, cfgs, engs, dsd, dcsd, cw = env
    b = tok.shape[0]
    cond, unc = O.clip_text_encode(dsd, cfgs[2], tok.cuda()), O.clip_text_encode(dsd, cfgs[2], neg.cuda())
    pr = engs[False].program(sampler, None, steps, denoise=d, masked=nmask is not None)
    nz = E.per_image_noise(seed, b, (4, hw, hw), 1 + pr.draws).cuda()
    unet = CN.ControlledUNet(dsd, cfgs[0], [(dcsd, h.cuda(), w, 0.0, 1.0) for h, w in units])
    mask = None if nmask is None else (init, nmask[None, None].cuda())
    with torch.no_grad(), T.circular():
        z = CN.run_sampler(sampler, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d,
                           mask=mask)
        if mask is not None:
            z = z * mask[1] + init * (1 - mask[1])
        return O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))


def _both(env, fn):
    """fn(engine) with graphs on and off: bitwise equal; returns the images"""
    got = {g: fn(env[3][g]).cpu() for g in (True, False)}
    assert torch.equal(got[True], got[False])
    return got[True]


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_tiny_txt2img_matches_the_tiling_oracle(tiny, sampler):
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    b, hw, steps = 2, 16, 8
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    got = _both(tiny, lambda e: e.txt2img(tok, neg, 300, steps=steps, height=8 * hw, width=8 * hw, sampler=sampler,
                                          tiling=True))
    _u8_check(f"tiny txt2img {sampler}", got, _oracle(tiny, tok, neg, 300, sampler, steps, hw))


@pytest.mark.parametrize("sampler,masked", [("DDIM", False), ("Euler a", False), ("DDIM", True), ("Heun", True)])
def test_tiny_img2img_and_inpaint_match_the_tiling_oracle(tiny, sampler, masked):
    from oracle import tiling_oracle as T
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    b, hw, steps, d = 2, 16, 10, 0.75
    f = 2 ** (len(cfgs[1].ch_mult) - 1)
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    init_u8 = torch.randint(0, 256, (b, f * hw, f * hw, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    nmask = (torch.rand((hw, hw), generator=torch.Generator().manual_seed(5)) > 0.5).float() if masked else None
    kw = {} if nmask is None else {"latmask": nmask.reshape(-1).cuda()}
    got = _both(tiny, lambda e: e.img2img(tok, neg, 41, init_u8, denoising_strength=d, steps=steps, sampler=sampler,
                                          tiling=True, **kw))
    with torch.no_grad():
        init = T.run(O.vae_encode_mean, dsd, cfgs[1], O.image_to_model_input(init_u8.cuda())) * cfgs[1].scale_factor
    ref = _oracle(tiny, tok, neg, 41, sampler, steps, hw, init=init, d=d, nmask=nmask)
    _u8_check(f"tiny img2img {sampler} masked={masked}", got, ref)


def test_tiny_hires_fix_matches_the_tiling_oracle(tiny):
    from oracle import tiling_oracle as T
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    b, hw = 2, 16
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    got = _both(tiny, lambda e: e.txt2img_hires(tok, neg, 77, steps=6, height=8 * hw, width=8 * hw, hr_scale=2.0,
                                                hr_steps=8, denoising_strength=0.6, tiling=True))
    with torch.no_grad():
        ref, _ = T.run(O.txt2img_hires, dsd, *cfgs, tok, neg, seed=77, steps=6, height=8 * hw, width=8 * hw,
                       hr_scale=2.0, hr_steps=8, denoising_strength=0.6, device="cuda")
    _u8_check("tiny hires Latent", got, ref)


def test_tiny_controlnet_unit_on_a_circular_unet(tiny):
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    b, hw, steps = 2, 16, 8
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    hint = torch.randint(0, 256, (8 * hw, 8 * hw, 3), generator=torch.Generator().manual_seed(6), dtype=torch.uint8)
    got = _both(tiny, lambda e: e.txt2img(tok, neg, 300, steps=steps, height=8 * hw, width=8 * hw, sampler="Euler a",
                                          controls=[(cw, hint, 0.9, 0.0, 1.0)], tiling=True))
    _u8_check("tiny txt2img ControlNet", got, _oracle(tiny, tok, neg, 300, "Euler a", steps, hw, units=[(hint, 0.9)]))


def test_tiny_batch_invariance_and_tiling_false_is_no_keyword(tiny):
    E, O, cfgs, engs, dsd, dcsd, cw = tiny
    eng = engs[True]
    tok, neg = O.random_prompt_tokens(1, vocab_hi=997), O.empty_prompt_tokens(1, vocab_hi=997)
    kw = dict(steps=6, height=128, width=128, sampler="Euler a")
    five = eng.txt2img(tok.expand(5, -1), neg.expand(5, -1), 300, tiling=True, **kw).clone()
    two = eng.txt2img(tok.expand(2, -1), neg.expand(2, -1), 303, tiling=True, **kw).clone()
    torch.cuda.synchronize()
    assert torch.equal(five[3:], two)
    off = eng.txt2img(tok.expand(2, -1), neg.expand(2, -1), 303, tiling=False, **kw).clone()
    plain = eng.txt2img(tok.expand(2, -1), neg.expand(2, -1), 303, **kw).clone()
    assert torch.equal(off, plain) and not torch.equal(off, two)


def test_tiny_sdxl_topology_matches_the_tiling_oracle():
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O, tiling_oracle as T
    cfgs, ocfgs = (C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP), (O.TINYXL_UNET, O.TINYXL_VAE, O.TINYXL_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    dsd = {k: v.cuda() for k, v in sd.items()}
    b, hw, steps = 2, 16, 8
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    got = {}
    for g in (True, False):
        eng = E.SDEngine(sd, *cfgs, device="cuda:0", dtype=torch.bfloat16, use_graphs=g)
        got[g] = eng.txt2img(tok, neg, 77, steps=steps, height=8 * hw, width=8 * hw, sampler="Euler a", tiling=True).cpu()
        eng.release()
    assert torch.equal(got[True], got[False])
    ctx_c, y_c = O.sdxl_conditioner(dsd, ocfgs[2], tok.cuda(), 8 * hw, 8 * hw)
    ctx_u, y_u = O.sdxl_conditioner(dsd, ocfgs[2], neg.cuda(), 8 * hw, 8 * hw, zero_txt=True)
    y = torch.cat([y_c, y_u])
    nz = E.per_image_noise(77, b, (4, hw, hw), 1 + steps).cuda()
    with torch.no_grad(), T.circular():
        unet = lambda x, t, c: O.unet_forward(dsd, ocfgs[0], x, t, c, y=y)  # noqa: E731
        z = O.run_sampler("Euler a", unet, ctx_c, ctx_u, 7.0, steps, nz[0], list(nz[1:]))
        ref = O.to_uint8(O.vae_decode(dsd, ocfgs[1], z / ocfgs[1].scale_factor))
    _u8_check("tinyxl txt2img Euler a bf16", got[True], ref, mean=2.0, within=(4, 0.95))
