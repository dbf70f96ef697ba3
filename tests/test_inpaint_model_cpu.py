"""Inpainting checkpoints (9-channel UNets) on the CPU: the oracle's conditioning against a direct restatement, the engine
(b200sd.ops emulated: tests/ops_emulator.py plus the two conditioning ops below) against the oracle on tiny-, tiny21- and
tinyxl-inpainting, 4-channel engines unchanged, the loader's channel detection, and the worker / REST plumbing of
inpainting_mask_weight.

Before inpainting models were served, channels 4..8 of the UNet input stayed zero: the tiny-inpainting comparisons below
then miss the oracle by far more than their bounds (test_zero_conditioning_is_far_from_the_oracle shows by how much)."""
import base64
import dataclasses
import io
import json
import types

import numpy as np
import pytest
import torch

from test_tiling_cpu import _install as _install_tiling


def masked_image_to_nhwc(img_u8, mask_u8, weight, out):
    """b200sd_masked_image_to_nhwc: (2x/255 - 1) with the kernel's single rounding (an FMA), times 1 - w [m >= 128]"""
    c = float(np.float32(2.0 / 255.0))
    s = (img_u8.double() * c - 1.0).float()
    m = torch.ones(img_u8.shape[1], dtype=torch.bool) if mask_u8 is None else mask_u8.reshape(-1) >= 128
    k = torch.where(m, torch.tensor(1.0 - weight, dtype=torch.float32), torch.tensor(1.0))
    out[..., :3] = (s * k[None, :, None]).to(out.dtype)
    return out


def pack_image_cond(z, mask_u8, xin, h, w):
    """b200sd_pack_image_cond"""
    b = z.shape[0]
    if mask_u8 is None:
        m = torch.ones(h * w)
    else:
        f = mask_u8.shape[0] // h
        m = (mask_u8[::f, ::f] >= 128).float().reshape(-1)
    for rows in (slice(0, b), slice(b, 2 * b)):
        xin[rows, :, 4] = m.to(xin.dtype)
        xin[rows, :, 5:9] = z.to(xin.dtype)
    return xin


def _install(monkeypatch):
    from b200sd import ops
    _install_tiling(monkeypatch)
    for fn in (masked_image_to_nhwc, pack_image_cond):
        monkeypatch.setattr(ops, fn.__name__, fn)


def _rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


# ------------------------------------------------------------------------------------------------ oracle pins
def test_conditioning_mask_rounds_at_128_and_goes_nearest_to_the_latent_size():
    from oracle import inpaint_model_oracle as IO
    m = torch.tensor([[0, 127, 128, 255], [126, 129, 64, 200], [1, 2, 3, 4], [250, 5, 130, 127]], dtype=torch.uint8)
    M = IO.conditioning_mask(m, 4, 4)
    assert torch.equal(M[0, 0], (m >= 128).float())
    big = torch.randint(0, 256, (32, 48), generator=torch.Generator().manual_seed(3), dtype=torch.uint8)
    small = torch.nn.functional.interpolate(IO.conditioning_mask(big, 32, 48), size=(4, 6))
    assert torch.equal(small[0, 0], (big[::8, ::8] >= 128).float())   # pixel (8i, 8j)
    assert torch.equal(IO.conditioning_mask(None, 3, 5), torch.ones((1, 1, 3, 5)))


@pytest.fixture(scope="module")
def tiny9():
    from b200sd import factory, synth
    cfgs = factory.configs("tiny-inpainting")
    return cfgs, synth.make_state_dict(*cfgs, seed=0)


def test_oracle_conditioning_is_the_direct_restatement(tiny9):
    from oracle import inpaint_model_oracle as IO, sd_oracle as O
    (ucfg, vcfg, _), sd = tiny9
    g = torch.Generator().manual_seed(4)
    init_u8 = torch.randint(0, 256, (2, 16, 16, 3), generator=g, dtype=torch.uint8)
    mask = torch.randint(120, 136, (16, 16), generator=g, dtype=torch.uint8)
    s = init_u8.permute(0, 3, 1, 2).float() * (2.0 / 255.0) - 1.0
    enc = lambda img: O.vae_encode_mean(sd, vcfg, img) * vcfg.scale_factor  # noqa: E731
    with torch.no_grad():
        for w in (1.0, 0.5, 0.0):
            got = IO.img2img_image_conditioning(sd, vcfg, init_u8, mask, w)
            M = (mask >= 128).float()
            assert torch.equal(got[:, 0], M[::2, ::2].expand(2, -1, -1))   # the tiny VAE's factor is 2
            assert _rel(got[:, 1:], enc(s * (1 - w * M))) < 1e-5
            plain = IO.img2img_image_conditioning(sd, vcfg, init_u8, None, w)
            assert bool((plain[:, 0] == 1).all()) and _rel(plain[:, 1:], enc(s * (1 - w))) < 1e-5
        gray = IO.txt2img_image_conditioning(sd, vcfg, 2, 16, 16)
        assert bool((gray[:, 0] == 1).all()) and torch.equal(gray[:, 1:], enc(torch.zeros((2, 3, 16, 16))))
        assert torch.equal(IO.hires_image_conditioning(sd, vcfg, "Latent (bicubic)", 2, 16, 16), gray)
        with pytest.raises(NotImplementedError):
            IO.hires_image_conditioning(sd, vcfg, "Latent", 2, 16, 16, weight=0.5)


def test_unet_shim_concatenates_and_restores(tiny9):
    from oracle import controlnet_oracle as CN, inpaint_model_oracle as IO, sd_oracle as O
    (ucfg, _, _), sd = tiny9
    g = torch.Generator().manual_seed(5)
    x, cc = torch.randn((4, 4, 8, 8), generator=g), torch.randn((2, 5, 8, 8), generator=g)
    ctx, t = torch.randn((4, 77, ucfg.context_dim), generator=g), torch.full((4,), 300.0)
    plain = (O.unet_forward, CN.unet_forward)
    with torch.no_grad():
        want = O.unet_forward(sd, ucfg, torch.cat([x, torch.cat([cc, cc])], dim=1), t, ctx)
        with IO.concat(cc):
            assert torch.equal(O.unet_forward(sd, ucfg, x, t, ctx), want)
            assert torch.equal(CN.unet_forward(sd, ucfg, x, t, ctx), want)
    assert (O.unet_forward, CN.unet_forward) == plain


def test_masked_image_emulation_is_image_to_nhwc_where_the_mask_is_zero():
    import ops_emulator
    img = torch.arange(256, dtype=torch.uint8).reshape(1, 256, 1).expand(1, 256, 3).contiguous()
    a, b = torch.zeros((1, 256, 8)), torch.zeros((1, 256, 8))
    masked_image_to_nhwc(img, torch.zeros(256, dtype=torch.uint8), 0.7, a)
    ops_emulator.image_to_nhwc(img, b)
    assert float((a - b).abs().max()) <= 1.2e-7   # ops_emulator rounds twice, the kernel once


# ------------------------------------------------------------------------------------------------ engine vs oracle
class _XLUNet:
    """unet(x, t, c) of the SDXL oracle with the request's vector conditioning, in ControlledUNet's shape"""
    units = ()

    def __init__(self, sd, cfg, y):
        self.sd, self.cfg, self.y = sd, cfg, y

    def __call__(self, x, t, c):
        from oracle import sd_oracle as O
        return O.unet_forward(self.sd, self.cfg, x, t, c, y=self.y)


@pytest.fixture(params=["tiny", "tiny21", "tinyxl"])
def env(request, monkeypatch):
    from b200sd import engine as E, factory, synth
    from oracle import sd_oracle as O, v_oracle as V
    _install(monkeypatch)
    fam = request.param
    cfgs = factory.configs(fam + "-inpainting")
    assert cfgs[0].in_channels == 9 and factory.prediction(fam + "-inpainting") == "eps"
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2)
    b = 2
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    ns = types.SimpleNamespace(E=E, eng=eng, sd=sd, cfgs=cfgs, b=b, tok=tok, neg=neg, fam=fam, xl=fam == "tinyxl")
    if ns.xl:
        ns.ocfgs = (dataclasses.replace(O.TINYXL_UNET, in_channels=9), O.TINYXL_VAE, O.TINYXL_CLIP)
    else:
        enc = O.clip_text_encode if fam == "tiny" else V.sd21_text_encode
        ns.cond, ns.unc = enc(sd, cfgs[2], tok), enc(sd, cfgs[2], neg)
    return ns


def _factor(env):
    return 2 ** (len(env.cfgs[1].ch_mult) - 1)


def _unet(env, width, height):
    """(oracle unet, cond, uncond) for a request whose conditioner sees width x height pixels"""
    from oracle import controlnet_oracle as CN, sd_oracle as O
    if not env.xl:
        return CN.ControlledUNet(env.sd, env.cfgs[0], []), env.cond, env.unc
    ctx_c, y_c = O.sdxl_conditioner(env.sd, env.ocfgs[2], env.tok, width, height)
    ctx_u, y_u = O.sdxl_conditioner(env.sd, env.ocfgs[2], env.neg, width, height, zero_txt=True)
    return _XLUNet(env.sd, env.ocfgs[0], torch.cat([y_c, y_u])), ctx_c, ctx_u


def _oracle(env, name, steps, nz, cc, size, init=None, d=None, nmask=None):
    from oracle import controlnet_oracle as CN, inpaint_model_oracle as IO
    unet, cond, unc = _unet(env, *size)
    mask = None if nmask is None else (init, nmask[None, None])
    with torch.no_grad(), IO.concat(cc):
        z = CN.run_sampler(name, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d,
                           mask=mask)
    return z if nmask is None else z * nmask + init * (1 - nmask)


def _check(env, got_u8, hw, ref_z):
    from oracle import sd_oracle as O
    lat = env.eng.plans[(env.b, hw, hw)].x.reshape(env.b, hw, hw, 4).permute(0, 3, 1, 2)
    assert _rel(lat, ref_z) <= (1e-3 if env.xl else 1e-4), _rel(lat, ref_z)
    vcfg = env.cfgs[1]
    with torch.no_grad():
        ref_u8 = O.to_uint8(O.vae_decode(env.sd, vcfg, ref_z / vcfg.scale_factor))
    d = (got_u8.int() - ref_u8.int()).abs()
    assert float((d <= 1).float().mean()) == 1.0 and float((d == 0).float().mean()) > 0.99


def _txt2img_case(env, name, hw=8, steps=6, seed=4100):
    from oracle import inpaint_model_oracle as IO
    f = _factor(env)
    pr = env.eng.program(name, None, steps)
    nz = env.E.per_image_noise(seed, env.b, (4, hw, hw), 1 + pr.draws)
    got = env.eng.txt2img(env.tok, env.neg, seed, steps=steps, height=8 * hw, width=8 * hw, sampler=name)
    with torch.no_grad():
        cc = IO.txt2img_image_conditioning(env.sd, env.cfgs[1], env.b, f * hw, f * hw)
    return got, nz, cc


@pytest.mark.parametrize("name", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_txt2img_matches_the_oracle(env, name):
    if env.xl and name in ("DPM++ 2M", "Heun"):
        pytest.skip("SDXL: DDIM and Euler a cover the conditioning; the samplers are the 4-channel engine's")
    hw, steps = 8, 6
    got, nz, cc = _txt2img_case(env, name, hw, steps)
    _check(env, got, hw, _oracle(env, name, steps, nz, cc, (8 * hw, 8 * hw)))


def test_zero_conditioning_is_far_from_the_oracle(env):
    """what serving the model with channels 4..8 left at zero (the 64-channel pad of conv_in) gives: far off"""
    if env.xl:
        pytest.skip("one family shows it")
    hw, steps = 8, 6
    _, nz, cc = _txt2img_case(env, "DDIM", hw, steps)
    ref = _oracle(env, "DDIM", steps, nz, cc, (8 * hw, 8 * hw))
    zero = _oracle(env, "DDIM", steps, nz, torch.zeros_like(cc), (8 * hw, 8 * hw))
    lat = env.eng.plans[(env.b, hw, hw)].x.reshape(env.b, hw, hw, 4).permute(0, 3, 1, 2)
    assert _rel(lat, ref) <= 1e-4 and _rel(zero, ref) > 1e-2


def _mask_image(px, seed=5):
    """a hand-drawn-like mask: a filled ellipse, mode 'L', px x px"""
    from PIL import Image, ImageDraw
    im = Image.new("L", (px, px), 0)
    r = np.random.default_rng(seed)
    x0, y0 = int(r.integers(0, px // 3)), int(r.integers(0, px // 3))
    ImageDraw.Draw(im).ellipse((x0, y0, x0 + px // 2, y0 + px // 2 + 1), fill=255)
    return im


def _init_u8(b, px, seed=9):
    return torch.randint(0, 256, (b, px, px, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def _img2img_case(env, name, init_u8, seed, w, latmask=None, image_mask=None, fill=1, steps=8, d=0.75):
    from oracle import inpaint_model_oracle as IO, sd_oracle as O
    hw = init_u8.shape[1] // _factor(env)
    kw = {} if latmask is None else {"latmask": latmask, "image_mask": image_mask, "inpainting_fill": fill}
    got = env.eng.img2img(env.tok, env.neg, seed, init_u8, denoising_strength=d, steps=steps, sampler=name,
                          inpainting_mask_weight=w, **kw)
    pr = env.eng.program(name, None, steps, denoise=d, masked=latmask is not None)
    nz = env.E.per_image_noise(seed, env.b, (4, hw, hw), 1 + pr.draws)
    vcfg = env.cfgs[1]
    with torch.no_grad():
        init = O.vae_encode_mean(env.sd, vcfg, O.image_to_model_input(init_u8)) * vcfg.scale_factor
        cc = IO.img2img_image_conditioning(env.sd, vcfg, init_u8, image_mask, w)
    nmask = None
    if latmask is not None:
        nmask = latmask.reshape(hw, hw)
        if fill in (2, 3):
            init = init * (1 - nmask) + (nz[0] * nmask if fill == 2 else 0)
    px = init_u8.shape[1]
    _check(env, got, hw, _oracle(env, name, steps, nz, cc, (px, px), init=init, d=d, nmask=nmask))


@pytest.mark.parametrize("w", [1.0, 0.5, 0.0])
def test_img2img_without_a_mask_matches_the_oracle(env, w):
    f = _factor(env)
    _img2img_case(env, "DDIM" if w != 0.5 else "Euler a", _init_u8(env.b, 8 * f), 31, w)


@pytest.mark.parametrize("fill,w,name", [(0, 1.0, "DDIM"), (1, 0.5, "DDIM"), (2, 1.0, "Euler a"), (3, 0.0, "Heun"),
                                         (1, 1.0, "DPM++ 2M")])
def test_masked_img2img_matches_the_oracle(env, fill, w, name):
    from b200sd import inpaint as inp
    from oracle import inpaint_model_oracle as IO
    f = _factor(env)
    px, hw = 8 * f, 8
    init_u8 = _init_u8(env.b, px)
    m = inp.prepare_mask(_mask_image(px), px, px, hw, hw, mask_blur=1)
    image_mask = torch.from_numpy(np.array(m.fill_mask.convert("L")))
    assert torch.equal(image_mask, IO.processed_mask(_mask_image(px), px, px, mask_blur=1))
    if fill == 0:
        init_u8 = inp.fill_masked(init_u8, m)
    _img2img_case(env, name, init_u8, 44, w, m.latmask, image_mask, fill)


def test_only_masked_matches_the_oracle(env):
    """"Only masked": the crop at the processing size is both the init image and the conditioning image, its resized
    mask the conditioning mask"""
    from PIL import Image
    from b200sd import inpaint as inp
    from oracle import inpaint_model_oracle as IO
    f = _factor(env)
    px, hw, full = 8 * f, 8, 40
    mask = _mask_image(full, seed=8)
    m = inp.prepare_mask_only_masked(mask, px, px, hw, hw, mask_blur=1, padding=4)
    image_mask = torch.from_numpy(np.array(m.fill_mask.convert("L")))
    assert torch.equal(image_mask, IO.processed_mask(mask, px, px, mask_blur=1, only_masked_padding=4))
    pics = [Image.fromarray(a.numpy()) for a in _init_u8(env.b, full, seed=12)]
    init_u8 = inp.crop_init_images(pics, m)
    _img2img_case(env, "DDIM", init_u8, 45, 0.5, m.latmask, image_mask)
    assert IO.processed_mask(Image.new("L", (full, full), 0), px, px, only_masked_padding=4) is None
    assert inp.prepare_mask_only_masked(Image.new("L", (full, full), 0), px, px, hw, hw) is None


@pytest.mark.parametrize("upscaler,w", [("Latent", 1.0), ("Lanczos", 0.5), ("Lanczos", 1.0)])
def test_hires_fix_matches_the_oracle(env, upscaler, w, monkeypatch):
    from PIL import Image
    from b200sd import upscale
    from oracle import inpaint_model_oracle as IO, upscale_oracle as UO
    if env.xl:
        pytest.skip("SDXL re-conditions the second pass on its size: covered by the engine's SDXL hires tests")

    def pil_resize(images, w_, h_, name, tile, overlap):
        return torch.stack([torch.from_numpy(np.array(UO.resize_image(Image.fromarray(im.numpy()), w_, h_, name)))
                            for im in images.cpu()])

    monkeypatch.setattr(upscale, "resize_image", pil_resize)
    f = _factor(env)
    hw, steps, hr_steps, d = 8, 5, 6, 0.6
    got = env.eng.txt2img_hires(env.tok, env.neg, 77, steps=steps, height=8 * hw, width=8 * hw, hr_scale=2.0,
                                hr_steps=hr_steps, denoising_strength=d, upscaler=upscaler, inpainting_mask_weight=w)
    nz1 = env.E.per_image_noise(77, env.b, (4, hw, hw), 1)
    nz2 = env.E.per_image_noise(77, env.b, (4, 2 * hw, 2 * hw), 1)
    vcfg = env.cfgs[1]
    with torch.no_grad():
        cc1 = IO.txt2img_image_conditioning(env.sd, vcfg, env.b, f * hw, f * hw)
    z1 = _oracle(env, "DDIM", steps, nz1, cc1, (8 * hw, 8 * hw))
    with torch.no_grad():
        up = UO.hires_upscale(env.sd, vcfg, z1, 2 * hw, 2 * hw, upscaler)
        upscaled = None
        if upscaler != "Latent":
            from oracle import sd_oracle as O
            first = O.to_uint8(O.vae_decode(env.sd, vcfg, z1 / vcfg.scale_factor))
            upscaled = pil_resize(first, 2 * hw * f, 2 * hw * f, upscaler, 0, 0)
        cc2 = IO.hires_image_conditioning(env.sd, vcfg, upscaler, env.b, 2 * hw * f, 2 * hw * f, upscaled, w)
    ref = _oracle(env, "DDIM", hr_steps, nz2, cc2, (16 * hw, 16 * hw), init=up, d=d)
    _check(env, got, 2 * hw, ref)


def test_latent_hires_with_a_weight_below_one_is_refused(env):
    with pytest.raises(ValueError, match="inpainting_mask_weight"):
        env.eng.txt2img_hires(env.tok, env.neg, 1, steps=3, height=64, width=64, upscaler="Latent (nearest)",
                              inpainting_mask_weight=0.9)
    assert not env.eng.plans   # refused before any work


def test_tiling_applies_to_the_conditioning_encode(env):
    from oracle import inpaint_model_oracle as IO, tiling_oracle as T
    if env.xl:
        pytest.skip("one family shows it")
    f = _factor(env)
    init_u8, mask = _init_u8(env.b, 8 * f), torch.randint(0, 256, (8 * f, 8 * f), dtype=torch.uint8)
    got = env.eng.encode_conditioning(init_u8, mask, 0.5, tiling=True)
    with torch.no_grad():
        ref = T.run(IO.img2img_image_conditioning, env.sd, env.cfgs[1], init_u8, mask, 0.5)
        flat = IO.img2img_image_conditioning(env.sd, env.cfgs[1], init_u8, mask, 0.5)
    assert _rel(got, ref[:, 1:]) <= 1e-4 and _rel(flat[:, 1:], ref[:, 1:]) > 1e-3


def test_an_inpainting_engine_needs_its_conditioning(env):
    hw = 8
    pr = env.eng.program("DDIM", None, 4)
    x = torch.zeros((env.b, 4, hw, hw))
    ctx = torch.zeros((env.b, 77, env.cfgs[0].context_dim))
    with pytest.raises(ValueError, match="image conditioning"):
        env.eng.run_program(ctx, ctx, x, pr, 7.0)
    with pytest.raises(ValueError, match="image_mask"):
        env.eng.img2img(env.tok, env.neg, 1, _init_u8(env.b, 8 * _factor(env)), steps=4,
                        latmask=torch.ones(hw * hw))


# ------------------------------------------------------------------------------------------------ 4-channel engines
@pytest.fixture()
def plain(monkeypatch):
    from b200sd import config as C, engine as E, ops, synth
    _install(monkeypatch)

    def never(*a, **k):
        raise AssertionError("a 4-channel engine built inpainting conditioning")

    monkeypatch.setattr(ops, "masked_image_to_nhwc", never)
    monkeypatch.setattr(ops, "pack_image_cond", never)
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    return E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cpu", dtype=torch.float32,
                      use_graphs=False, vae_chunk=2), cfgs


def test_four_channel_engines_build_no_conditioning(plain, monkeypatch):
    from b200sd import ops, upscale
    from b200sd.vae_exec import VAEEncoderProgram
    from oracle import sd_oracle as O
    eng, cfgs = plain
    assert not eng.inpainting
    tok, neg = O.random_prompt_tokens(2, vocab_hi=997), O.empty_prompt_tokens(2, vocab_hi=997)
    eng.txt2img(tok, neg, 3, steps=3, height=64, width=64, sampler="DDIM")
    eng.img2img(tok, neg, 3, _init_u8(2, 16), steps=4, latmask=torch.ones(64))
    monkeypatch.setattr(upscale, "resize_image", lambda im, w, h, *a: torch.nn.functional.interpolate(
        im.permute(0, 3, 1, 2).float(), size=(h, w)).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous())
    eng.txt2img_hires(tok, neg, 3, steps=3, height=64, width=64, upscaler="Lanczos")
    assert not any("masked" in k for k in eng.encoders)
    enc = VAEEncoderProgram(eng.vae_enc_w, 2, 32, 32)
    assert enc.ops[0][0] is ops.image_to_nhwc and not hasattr(enc, "mask_u8")
    ctx = torch.zeros((2, 77, cfgs[0].context_dim))
    with pytest.raises(ValueError, match="9-channel"):
        eng.run_program(ctx, ctx, torch.zeros((2, 4, 8, 8)), eng.program("DDIM", None, 4), 7.0,
                        image_cond=(torch.zeros((2, 4, 8, 8)), None))


def test_masked_encoder_is_a_program_of_its_own(tiny9, monkeypatch):
    from b200sd import ops
    from b200sd.vae_exec import VAEEncoderProgram, VAEEncoderWeights
    from test_tiling_cpu import _signature
    _install(monkeypatch)
    (_, vcfg, _), sd = tiny9
    ew = VAEEncoderWeights(sd, vcfg, "cpu", torch.float32)
    plain, masked = VAEEncoderProgram(ew, 2, 32, 32), VAEEncoderProgram(ew, 2, 32, 32, masked=True)
    assert plain.ops[0][0] is ops.image_to_nhwc and masked.ops[0][0] == masked._condition_input
    assert _signature(plain.ops[1:]) == _signature(masked.ops[1:])


# ------------------------------------------------------------------------------------------------ loading
def test_families_and_identity():
    from b200sd import config as C, factory
    for fam, base in (("sd15", C.SD15_UNET), ("sd21", C.SD21_UNET), ("sdxl", C.SDXL_UNET), ("tiny", C.TINY_UNET),
                      ("tiny21", C.TINY21_UNET), ("tinyxl", C.TINYXL_UNET)):
        u, v, c = factory.configs(fam + "-inpainting")
        assert u == dataclasses.replace(base, in_channels=9) and (v, c) == factory.configs(fam)[1:]
        assert factory.prediction(fam + "-inpainting") == "eps"
        assert factory.model_identity(fam + "-inpainting") == f"synthetic-{fam}-inpainting-seed0"


@pytest.mark.parametrize("channels,family,want", [(4, "sd15", (4, "eps")), (9, "sd15", (9, "eps")),
                                                   (4, "sd21", (4, "v")), (9, "sd21", (9, "eps")),
                                                   (8, "sd15", None), (5, "sd21", None)])
def test_checkpoint_conv_in_decides_the_model(monkeypatch, tmp_path, channels, family, want):
    from b200sd import factory
    built = []
    monkeypatch.setattr(factory, "_load_safetensors", lambda p: {
        "model.diffusion_model.input_blocks.0.0.weight": torch.zeros((320, channels, 3, 3))})
    monkeypatch.setattr(factory, "_STATE", {})
    monkeypatch.setattr(factory, "_ENGINES", {})
    monkeypatch.setenv("SD_CKPT", str(tmp_path / "model.safetensors"))
    monkeypatch.delenv("B200SD_PREDICTION", raising=False)
    real = factory.SDEngine

    def engine(sd, ucfg, vcfg, ccfg, **kw):
        if ucfg.in_channels not in (4, 9):
            return real(sd, ucfg, vcfg, ccfg, **kw)   # refuses before it reads a weight
        built.append((ucfg.in_channels, kw["prediction"]))
        return types.SimpleNamespace()

    monkeypatch.setattr(factory, "SDEngine", engine)
    if want is None:
        with pytest.raises(ValueError, match=f"{channels} input channels"):
            factory.default_engine_factory("cuda:0", family)
        return
    factory.default_engine_factory("cuda:0", family)
    assert built == [want]
    monkeypatch.setenv("B200SD_PREDICTION", "v")
    factory.default_engine_factory("cuda:0", family)
    assert built[-1] == (channels, "v")


def test_engine_refuses_a_conv_in_that_does_not_match_its_config(tiny9):
    from b200sd import config as C, engine as E
    (ucfg, vcfg, ccfg), sd = tiny9
    sd4 = dict(sd, **{"model.diffusion_model.input_blocks.0.0.weight":
                      sd["model.diffusion_model.input_blocks.0.0.weight"][:, :4].contiguous()})
    E.SDEngine._require_cuda = False
    try:
        with pytest.raises(ValueError, match="conv_in takes 4"):
            E.SDEngine(sd4, ucfg, vcfg, ccfg, device="cpu", dtype=torch.float32)
        with pytest.raises(ValueError, match="conv_in takes 9"):
            E.SDEngine(sd, C.TINY_UNET, vcfg, ccfg, device="cpu", dtype=torch.float32)
        with pytest.raises(ValueError, match="8 input channels"):
            E.SDEngine(sd, dataclasses.replace(ucfg, in_channels=8), vcfg, ccfg, device="cpu", dtype=torch.float32)
    finally:
        E.SDEngine._require_cuda = True


# ------------------------------------------------------------------------------------------------ worker / REST
def _worker(monkeypatch, family):
    import logging
    from b200sd import engine as E, factory, synth
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker
    logging.getLogger("distributed").setLevel(logging.ERROR)
    _install(monkeypatch)
    monkeypatch.setenv("B200SD_MODEL", family)
    cfgs = factory.configs(family)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cpu", dtype=torch.float32, use_graphs=False,
                     vae_chunk=2)
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    calls = []
    for name in ("txt2img", "img2img", "txt2img_hires"):
        real = getattr(eng, name)
        monkeypatch.setattr(eng, name, (lambda real, name: lambda *a, **k: calls.append((name, k)) or real(*a, **k))(
            real, name))
    return LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0), calls


@pytest.fixture()
def worker9(monkeypatch):
    return _worker(monkeypatch, "tiny-inpainting")


def _payload(**kw):
    p = {"prompt": "a b", "negative_prompt": "", "seed": 30, "subseed": 4, "subseed_strength": 0, "batch_size": 2,
         "n_iter": 1, "steps": 3, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0}
    p.update(kw)
    return p


def _b64(im):
    buf = io.BytesIO()
    im.save(buf, format="PNG")
    return base64.b64encode(buf.getvalue()).decode()


def _init_b64(px=64):
    from PIL import Image
    return _b64(Image.fromarray(_init_u8(1, px)[0].numpy()))


@pytest.mark.parametrize("override,opts,want", [({"inpainting_mask_weight": 0.25}, 0.75, 0.25), ({}, 0.75, 0.75),
                                                ({}, None, 1.0), ({"inpainting_mask_weight": 0}, None, 0.0),
                                                ({"inpainting_mask_weight": None}, 0.5, 0.5)])
def test_worker_resolves_the_weight_as_sdwui(worker9, monkeypatch, override, opts, want):
    import modules.shared as shared
    wk, calls = worker9
    if opts is not None:
        monkeypatch.setattr(shared.opts, "inpainting_mask_weight", opts, raising=False)
    else:
        monkeypatch.delattr(shared.opts, "inpainting_mask_weight", raising=False)
    wk.request(_payload(override_settings=override, init_images=[_init_b64()]), None, False)
    name, kw = calls[-1]
    assert name == "img2img" and kw["inpainting_mask_weight"] == want and "image_mask" not in kw
    info = json.loads(wk.response["info"])
    assert all(t.endswith(f", Conditional mask weight: {want}") for t in info["infotexts"])
    wk.request(_payload(override_settings=override), None, False)   # txt2img: the weight is passed, not reported
    assert calls[-1][0] == "txt2img" and calls[-1][1]["inpainting_mask_weight"] == want
    assert "Conditional mask weight" not in json.loads(wk.response["info"])["infotexts"][0]


def test_worker_passes_the_processed_mask(worker9):
    wk, calls = worker9
    mask = _b64(_mask_image(64))
    wk.request(_payload(init_images=[_init_b64()], mask=mask, mask_blur=2, inpainting_fill=1), None, False)
    name, kw = calls[-1]
    from oracle import inpaint_model_oracle as IO
    assert name == "img2img" and torch.equal(kw["image_mask"], IO.processed_mask(_mask_image(64), 64, 64, mask_blur=2))
    from PIL import Image
    blank = _b64(Image.new("L", (64, 64), 0))   # "Only masked" with a blank mask: plain img2img, all-ones mask
    wk.request(_payload(init_images=[_init_b64()], mask=blank, inpaint_full_res=True), None, False)
    assert "image_mask" not in calls[-1][1] and "latmask" not in calls[-1][1]
    wk.request(_payload(init_images=[_init_b64()], mask=mask, inpaint_full_res=True, inpaint_full_res_padding=8), None,
               False)
    assert torch.equal(calls[-1][1]["image_mask"],
                       IO.processed_mask(_mask_image(64), 64, 64, mask_blur=4, only_masked_padding=8))


@pytest.mark.parametrize("payload,match", [
    (dict(override_settings={"inpainting_mask_weight": 1.5}), "outside"),
    (dict(override_settings={"inpainting_mask_weight": -0.1}), "outside"),
    (dict(enable_hr=True, hr_scale=2.0, override_settings={"inpainting_mask_weight": 0.5}), "inpainting_mask_weight"),
    (dict(enable_hr=True, hr_scale=2.0, hr_upscaler="Latent (bicubic)", override_settings={"inpainting_mask_weight": 0.5}),
     "inpainting_mask_weight"),
    (dict(alwayson_scripts={"controlnet": {"args": [{"enabled": True, "model": "control_canny", "module": "none",
                                                     "image": None}]}}), "inpainting checkpoint")])
def test_worker_refusals(worker9, payload, match):
    from scripts.spartan.worker import InvalidWorkerResponse
    wk, calls = worker9
    if "alwayson_scripts" in payload:
        from PIL import Image
        payload["alwayson_scripts"]["controlnet"]["args"][0]["image"] = _b64(Image.new("RGB", (64, 64), (9, 9, 9)))
    with pytest.raises(InvalidWorkerResponse, match=match):
        wk.request(_payload(**payload), None, False)


def test_worker_serves_pixel_hires_with_a_weight_below_one(worker9, monkeypatch):
    from b200sd import upscale
    monkeypatch.setattr(upscale, "resize_image", lambda im, w, h, *a: torch.nn.functional.interpolate(
        im.permute(0, 3, 1, 2).float(), size=(h, w)).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous())
    wk, calls = worker9
    wk.request(_payload(enable_hr=True, hr_scale=2.0, hr_upscaler="Nearest",
                        override_settings={"inpainting_mask_weight": 0.5}), None, False)
    assert calls[-1][0] == "txt2img_hires" and calls[-1][1]["inpainting_mask_weight"] == 0.5
    assert wk.response["tensors"].shape[1] == 2 * 16   # 2x of 8 latent rows, at the tiny VAE's factor 2


def test_worker_leaves_four_channel_requests_as_they_were(monkeypatch):
    import modules.shared as shared
    wk, calls = _worker(monkeypatch, "tiny")
    monkeypatch.setattr(shared.opts, "inpainting_mask_weight", 0.5, raising=False)
    mask = _b64(_mask_image(64))
    for p in (_payload(), _payload(init_images=[_init_b64()], mask=mask, override_settings={"inpainting_mask_weight": 2}),
              _payload(enable_hr=True, hr_scale=2.0)):
        wk.request(p, None, False)
        kw = calls[-1][1]
        assert "inpainting_mask_weight" not in kw and "image_mask" not in kw
        assert "Conditional mask weight" not in json.loads(wk.response["info"])["infotexts"][0]


class _RecordingEngine:
    """the engine surface the worker's img2img path uses; records the keyword arguments"""

    def __init__(self):
        from b200sd import factory
        self.interrupted = False
        self.unet_cfg, self.vae_cfg, self.clip_cfg = factory.configs("sd15-inpainting")
        self.inpainting = True
        self.calls = []

    def img2img(self, tok, neg, seed, init_u8, **kw):
        self.calls.append(kw)
        return torch.zeros(init_u8.shape, dtype=torch.uint8)


def test_rest_server_passes_override_settings_through():
    from fastapi.testclient import TestClient
    from server.sdapi import create_app
    eng = _RecordingEngine()
    client = TestClient(create_app(lambda device: eng, [0]))
    body = {"prompt": "a", "steps": 2, "width": 64, "height": 64, "sampler_name": "DDIM", "init_images": [_init_b64()]}
    r = client.post("/sdapi/v1/img2img", json=dict(body, override_settings={"inpainting_mask_weight": 0.3}))
    assert r.status_code == 200 and eng.calls[-1]["inpainting_mask_weight"] == 0.3
    assert json.loads(r.json()["info"])["infotexts"][0].endswith(", Conditional mask weight: 0.3")
    r = client.post("/sdapi/v1/img2img", json=dict(body, override_settings={"inpainting_mask_weight": 3}))
    assert r.status_code != 200 and len(eng.calls) == 1
