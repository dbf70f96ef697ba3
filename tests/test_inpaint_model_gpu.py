"""Inpainting checkpoints (9-channel UNets) on the GPU: b200sd_masked_image_to_nhwc and b200sd_pack_image_cond bitwise
against their torch formulas, tiny-inpainting requests against oracle/inpaint_model_oracle.py with graphs on and off, batch
invariance, a mask that moves the repainted region, a full-size SD1.5-inpainting UNet evaluation and one 512^2 masked DDIM
request.  uint8 tolerances as tests/test_engine_gpu.py (fp16: mean |d| <= 1.5 LSB, >= 97 % within 2 LSB)."""
import json
import os

import numpy as np
import pytest
import torch

from kutil import OUT_DIR

pytestmark = pytest.mark.gpu
UNET_REL_RMS = 5e-3   # one fp16 UNet evaluation against the fp32 oracle (tests/test_tiling_gpu.py, test_controlnet_gpu.py)


def _record(name, **kw):
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "inpaint_model_parity.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **kw)) + "\n")


def _u8_check(name, got, ref, mean=1.5, within=(2, 0.97)):
    du8 = (got.cpu().int() - ref.cpu().int()).abs().float()
    rec = dict(u8_mean=float(du8.mean()), u8_max=float(du8.max()), u8_within=float((du8 <= within[0]).float().mean()))
    _record(name, **rec)
    assert got.shape == ref.shape
    assert rec["u8_mean"] <= mean and rec["u8_within"] >= within[1], rec
    return rec


def _rel_rms(a, b):
    return float((a.float() - b.float()).pow(2).mean().sqrt() / b.float().pow(2).mean().sqrt())


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("w", [1.0, 0.5, 0.3, 0.0])
def test_masked_image_to_nhwc_is_its_formula(dt, w):
    from b200sd import ops
    g = torch.Generator().manual_seed(1)
    b, hw = 3, 1000
    img = torch.randint(0, 256, (b, hw, 3), generator=g, dtype=torch.uint8)
    img[0, :256] = torch.arange(256, dtype=torch.uint8)[:, None]   # every value
    mask = torch.randint(0, 256, (hw,), generator=g, dtype=torch.uint8)
    mask[:4] = torch.tensor([127, 128, 0, 255], dtype=torch.uint8)
    s = (img.double() * float(np.float32(2.0 / 255.0)) - 1.0).float()   # the FMA's single rounding
    for m in (mask, None):
        mm = torch.ones(hw, dtype=torch.bool) if m is None else m >= 128
        want = s * torch.where(mm, torch.tensor(1.0 - w, dtype=torch.float32), torch.tensor(1.0))[None, :, None]
        out = torch.full((b, hw, 64), 3.0, dtype=dt, device="cuda")
        ops.masked_image_to_nhwc(img.cuda(), None if m is None else m.cuda(), w, out)
        torch.cuda.synchronize()
        assert torch.equal(out[..., :3].cpu(), want.to(dt)) and bool((out[..., 3:] == 3.0).all())
    zero, plain = torch.zeros((b, hw, 64), dtype=dt, device="cuda"), torch.zeros((b, hw, 64), dtype=dt, device="cuda")
    ops.masked_image_to_nhwc(img.cuda(), torch.zeros(hw, dtype=torch.uint8, device="cuda"), w, zero)
    ops.image_to_nhwc(img.cuda(), plain)
    torch.cuda.synchronize()
    assert torch.equal(zero, plain)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("f,masked", [(8, True), (2, True), (8, False)])
def test_pack_image_cond_writes_channels_4_to_8_only(dt, f, masked):
    from b200sd import ops
    g = torch.Generator().manual_seed(f)
    b, h, w = 3, 6, 10
    z = torch.randn((b, h * w, 4), generator=g)
    mask = torch.randint(100, 156, (f * h, f * w), generator=g, dtype=torch.uint8) if masked else None
    xin0 = torch.randn((2 * b, h * w, 64), generator=g).to(dt)
    xin = xin0.cuda()
    ops.pack_image_cond(z.cuda(), None if mask is None else mask.cuda(), xin, h, w)
    torch.cuda.synchronize()
    xin = xin.cpu()
    m = torch.ones(h * w) if mask is None else (mask[::f, ::f] >= 128).float().reshape(-1)
    for half in (xin[:b], xin[b:]):
        assert torch.equal(half[..., 4], m.to(dt).expand(b, -1)) and torch.equal(half[..., 5:9], z.to(dt))
    assert torch.equal(xin[..., :4], xin0[..., :4]) and torch.equal(xin[..., 9:], xin0[..., 9:])


def test_pack_image_cond_refuses_narrow_or_misaligned_inputs():
    import ctypes
    from b200sd import _lib
    z = torch.zeros((1, 4, 4), device="cuda")
    xin = torch.zeros((2, 4, 64), dtype=torch.float16, device="cuda")
    call = lambda zp, xp, pitch: _lib.lib().b200sd_pack_image_cond(  # noqa: E731
        ctypes.c_void_p(zp), None, ctypes.c_void_p(xp), ctypes.c_longlong(pitch), 1, 2, 2, 1, 0, None)
    assert call(z.data_ptr(), xin.data_ptr(), 8) == -1
    assert call(z.data_ptr() + 4, xin.data_ptr(), 64) == -1
    assert call(z.data_ptr(), xin.data_ptr() + 2, 64) == -1
    assert call(z.data_ptr(), xin.data_ptr(), 64) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ tiny requests
@pytest.fixture(scope="module")
def tiny():
    from b200sd import engine as E, factory, synth
    from oracle import sd_oracle as O
    cfgs = factory.configs("tiny-inpainting")
    sd = synth.make_state_dict(*cfgs, seed=0)
    engs = {g: E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=g) for g in (True, False)}
    dsd = {k: v.cuda() for k, v in sd.items()}
    return E, O, cfgs, engs, dsd


def _oracle(env, tok, neg, seed, sampler, steps, hw, cc, init=None, d=None, nmask=None):
    from oracle import controlnet_oracle as CN, inpaint_model_oracle as IO
    E, O, cfgs, engs, dsd = env
    b = tok.shape[0]
    cond, unc = O.clip_text_encode(dsd, cfgs[2], tok.cuda()), O.clip_text_encode(dsd, cfgs[2], neg.cuda())
    pr = engs[False].program(sampler, None, steps, denoise=d, masked=nmask is not None)
    nz = E.per_image_noise(seed, b, (4, hw, hw), 1 + pr.draws).cuda()
    mask = None if nmask is None else (init, nmask[None, None].cuda())
    with torch.no_grad(), IO.concat(cc):
        z = CN.run_sampler(sampler, CN.ControlledUNet(dsd, cfgs[0], []), cond, unc, 7.0, steps, nz[0], list(nz[1:]),
                           init=init, denoising_strength=d, mask=mask)
        if mask is not None:
            z = z * mask[1] + init * (1 - mask[1])
        return O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor)), z


def _both(env, fn):
    got = {g: fn(env[3][g]).cpu() for g in (True, False)}
    assert torch.equal(got[True], got[False])
    return got[True]


def _prompts(O, b):
    return O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_tiny_txt2img_matches_the_oracle(tiny, sampler):
    from oracle import inpaint_model_oracle as IO
    E, O, cfgs, engs, dsd = tiny
    b, hw, steps = 2, 16, 8
    tok, neg = _prompts(O, b)
    got = _both(tiny, lambda e: e.txt2img(tok, neg, 300, steps=steps, height=8 * hw, width=8 * hw, sampler=sampler))
    with torch.no_grad():
        cc = IO.txt2img_image_conditioning(dsd, cfgs[1], b, 2 * hw, 2 * hw)
    _u8_check(f"tiny-inpainting txt2img {sampler}", got, _oracle(tiny, tok, neg, 300, sampler, steps, hw, cc)[0])


def _mask(px, x0, y0):
    m = torch.zeros((px, px), dtype=torch.uint8)
    m[y0:y0 + px // 2, x0:x0 + px // 2] = 255
    m[y0 + px // 2, x0:x0 + px // 2] = 128   # the rounding edge
    return m


@pytest.mark.parametrize("sampler,masked,fill,w", [("DDIM", False, 1, 0.5), ("Euler a", False, 1, 1.0),
                                                   ("DDIM", True, 1, 1.0), ("DDIM", True, 2, 0.5),
                                                   ("Heun", True, 3, 0.0), ("Euler a", True, 1, 0.5)])
def test_tiny_img2img_matches_the_oracle(tiny, sampler, masked, fill, w):
    from oracle import inpaint_model_oracle as IO
    E, O, cfgs, engs, dsd = tiny
    b, hw, steps, d = 2, 16, 10, 0.75
    px = 2 * hw   # the tiny VAE's factor is 2
    tok, neg = _prompts(O, b)
    init_u8 = torch.randint(0, 256, (b, px, px, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    image_mask = _mask(px, 5, 3) if masked else None
    latmask = (image_mask[::2, ::2] >= 128).float().reshape(-1) if masked else None
    kw = {} if not masked else {"latmask": latmask.cuda(), "image_mask": image_mask, "inpainting_fill": fill}
    got = _both(tiny, lambda e: e.img2img(tok, neg, 41, init_u8, denoising_strength=d, steps=steps, sampler=sampler,
                                          inpainting_mask_weight=w, **kw))
    with torch.no_grad():
        init = O.vae_encode_mean(dsd, cfgs[1], O.image_to_model_input(init_u8.cuda())) * cfgs[1].scale_factor
        cc = IO.img2img_image_conditioning(dsd, cfgs[1], init_u8.cuda(), None if image_mask is None else image_mask.cuda(), w)
    nmask = None
    if masked:
        nmask = latmask.reshape(hw, hw)
        if fill in (2, 3):
            nm = nmask.cuda()
            nz0 = E.per_image_noise(41, b, (4, hw, hw), 1)[0].cuda()
            init = init * (1 - nm) + (nz0 * nm if fill == 2 else 0)
    ref, _ = _oracle(tiny, tok, neg, 41, sampler, steps, hw, cc, init=init, d=d, nmask=nmask)
    _u8_check(f"tiny-inpainting img2img {sampler} masked={masked} fill={fill} w={w}", got, ref)


@pytest.mark.parametrize("upscaler", ["Latent", "Lanczos"])
def test_tiny_hires_fix_matches_the_oracle(tiny, upscaler):
    from PIL import Image
    from oracle import inpaint_model_oracle as IO, upscale_oracle as UO
    E, O, cfgs, engs, dsd = tiny
    b, hw, w = 2, 16, 1.0 if upscaler == "Latent" else 0.5
    tok, neg = _prompts(O, b)
    got = _both(tiny, lambda e: e.txt2img_hires(tok, neg, 77, steps=6, height=8 * hw, width=8 * hw, hr_scale=2.0,
                                                hr_steps=8, denoising_strength=0.6, upscaler=upscaler,
                                                inpainting_mask_weight=w))
    with torch.no_grad():
        cc1 = IO.txt2img_image_conditioning(dsd, cfgs[1], b, 2 * hw, 2 * hw)
        first, z1 = _oracle(tiny, tok, neg, 77, "DDIM", 6, hw, cc1)
        up = UO.hires_upscale(dsd, cfgs[1], z1, 2 * hw, 2 * hw, upscaler, device="cuda")
        upscaled = None if upscaler == "Latent" else torch.stack([torch.from_numpy(np.array(
            UO.resize_image(Image.fromarray(im.numpy()), 4 * hw, 4 * hw, upscaler))) for im in first.cpu()]).cuda()
        cc2 = IO.hires_image_conditioning(dsd, cfgs[1], upscaler, b, 4 * hw, 4 * hw, upscaled, w)
    ref, _ = _oracle(tiny, tok, neg, 77, "DDIM", 8, 2 * hw, cc2, init=up, d=0.6)
    _u8_check(f"tiny-inpainting hires {upscaler}", got, ref)


def test_tiny_batch_invariance_and_the_mask_moves_the_repainted_region(tiny):
    E, O, cfgs, engs, dsd = tiny
    eng = engs[True]
    tok, neg = _prompts(O, 1)
    px = 64
    init_u8 = torch.randint(0, 256, (5, px, px, 3), generator=torch.Generator().manual_seed(8), dtype=torch.uint8)
    mask = _mask(px, 4, 4)
    kw = dict(steps=8, sampler="DDIM", denoising_strength=0.9, inpainting_mask_weight=1.0)

    def run(images, seed, m):
        lat = (m[::2, ::2] >= 128).float().reshape(-1).cuda()
        return eng.img2img(tok.expand(images.shape[0], -1), neg.expand(images.shape[0], -1), seed, images,
                           latmask=lat, image_mask=m, **kw).cpu()

    five = run(init_u8, 300, mask)
    two = run(init_u8[3:].contiguous(), 303, mask)
    assert torch.equal(five[3:], two)
    moved = run(init_u8[3:].contiguous(), 303, _mask(px, 28, 28))
    d = (moved.int() - two.int()).abs().sum(-1)   # [2, px, px]
    inside_old, inside_new = mask >= 128, _mask(px, 28, 28) >= 128
    both_out = ~(inside_old | inside_new)
    assert float(d[:, inside_new].float().mean()) > 4 * float(d[:, both_out].float().mean() + 0.5)
    _record("tiny-inpainting moved mask", changed_inside=float(d[:, inside_new].float().mean()),
            changed_outside=float(d[:, both_out].float().mean()))


# ------------------------------------------------------------------------------------------------ full-size SD1.5
@pytest.fixture(scope="module")
def sd15():
    from b200sd import engine as E, factory, synth
    from oracle import sd_oracle as O
    cfgs = factory.configs("sd15-inpainting")
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    yield E, O, cfgs, sd, eng
    eng.release()


def test_sd15_inpainting_unet_evaluation_matches_the_oracle(sd15):
    from b200sd import ops
    from oracle import inpaint_model_oracle as IO
    E, O, cfgs, sd, eng = sd15
    b, h, w = 1, 64, 64
    x = O.per_image_noise(5, b, (4, h, w))
    g = torch.Generator().manual_seed(6)
    z = torch.randn((b, 4, h, w), generator=g)
    mask = torch.randint(0, 256, (8 * h, 8 * w), generator=g, dtype=torch.uint8)
    plan = eng.plan(b, h, w)
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    cond, unc = eng.encode_prompts(tok), eng.encode_prompts(neg)
    plan.set_context(cond, unc)
    plan.table[:1].copy_(eng.temb.table(torch.tensor([651.0])))
    plan.step.zero_()
    plan.x.copy_(x.cuda().permute(0, 2, 3, 1).reshape(b, h * w, 4))
    ops.pack_unet_input(plan.x, plan.unet.xin, 1.0)
    ops.pack_image_cond(z.cuda().permute(0, 2, 3, 1).reshape(b, h * w, 4).contiguous(), mask.cuda(), plan.unet.xin, h, w)
    ops.select_step(plan.table, plan.step, plan.unet.cur_bias)
    plan.unet.run()
    torch.cuda.synchronize()
    eps = plan.unet.eps[..., :4].float().reshape(2 * b, h, w, 4).permute(0, 3, 1, 2).cpu()
    cc = torch.cat([(mask[::8, ::8] >= 128).float()[None, None], z], dim=1)
    dsd = {k: v.cuda() for k, v in sd.items() if k.startswith("model.diffusion_model.")}
    with torch.no_grad(), IO.concat(cc.cuda()):
        ref = O.unet_forward(dsd, cfgs[0], torch.cat([x, x]).cuda(), torch.full((2,), 651.0, device="cuda"),
                             torch.cat([cond, unc]).float()).cpu()
    with torch.no_grad():
        zero = O.unet_forward(dsd, cfgs[0], torch.cat([torch.cat([x, x]), torch.zeros((2, 5, h, w))], 1).cuda(),
                              torch.full((2,), 651.0, device="cuda"), torch.cat([cond, unc]).float()).cpu()
    del dsd
    rel, rel0 = _rel_rms(eps, ref), _rel_rms(eps, zero)
    _record("sd15-inpainting UNet evaluation", rel_rms=rel, rel_rms_vs_zero_conditioning=rel0)
    assert rel <= UNET_REL_RMS < rel0, (rel, rel0)


def test_sd15_512_masked_ddim_request_matches_the_oracle(sd15):
    from oracle import controlnet_oracle as CN, inpaint_model_oracle as IO
    E, O, cfgs, sd, eng = sd15
    b, steps, d, hw = 1, 20, 0.75, 64
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    init_u8 = torch.randint(0, 256, (b, 512, 512, 3), generator=torch.Generator().manual_seed(2), dtype=torch.uint8)
    image_mask = _mask(512, 100, 140)
    latmask = (image_mask[::8, ::8] >= 128).float().reshape(-1)
    got = eng.img2img(tok, neg, 1000, init_u8, denoising_strength=d, steps=steps, sampler="DDIM",
                      latmask=latmask.cuda(), image_mask=image_mask, inpainting_mask_weight=1.0).cpu()
    dsd = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        cond, unc = O.clip_text_encode(dsd, cfgs[2], tok.cuda()), O.clip_text_encode(dsd, cfgs[2], neg.cuda())
        init = O.vae_encode_mean(dsd, cfgs[1], O.image_to_model_input(init_u8.cuda())) * cfgs[1].scale_factor
        cc = IO.img2img_image_conditioning(dsd, cfgs[1], init_u8.cuda(), image_mask.cuda(), 1.0)
        nz = E.per_image_noise(1000, b, (4, hw, hw), 1).cuda()
        nmask = latmask.reshape(1, 1, hw, hw).cuda()
        with IO.concat(cc):
            z = CN.run_sampler("DDIM", CN.ControlledUNet(dsd, cfgs[0], []), cond, unc, 7.0, steps, nz[0], [], init=init,
                               denoising_strength=d, mask=(init, nmask))
        z = z * nmask + init * (1 - nmask)
        ref = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor)).cpu()
    del dsd
    _u8_check("sd15-inpainting 512 masked DDIM", got, ref)
