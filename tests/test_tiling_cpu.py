"""Seamless tiling (sdwui's `tiling`) on the CPU: the tiling oracle's pins, the engine with tiling on (b200sd.ops emulated:
tests/ops_emulator.py plus the circular pad below) against the oracle on tiny, tiny21 and tiny SDXL, which convs the
programs make circular, the worker's resolution of the setting and the REST passthrough."""
import json
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ops_emulator
from test_controlnet_cpu import _hint, hint_to_nhwc
from test_vpred_cpu import cfg_ddim_step_v, cfg_dpmpp_2m_step_v, cfg_euler_a_step_v


def pad_circular(x, out, p):
    """b200sd_pad_circular"""
    out.copy_(F.pad(x.permute(0, 3, 1, 2), (p, p, p, p), mode="circular").permute(0, 2, 3, 1))
    return out


def _install(monkeypatch):
    from b200sd import engine as E, ops
    ops_emulator.install(monkeypatch, ops)
    for fn in (pad_circular, hint_to_nhwc, cfg_ddim_step_v, cfg_euler_a_step_v, cfg_dpmpp_2m_step_v):
        monkeypatch.setattr(ops, fn.__name__, fn)
    monkeypatch.setattr(E.SDEngine, "_require_cuda", False)


def _rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


# ------------------------------------------------------------------------------------------------ oracle pins
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("hw", [(1, 1), (2, 7), (7, 2), (8, 8), (9, 5)])
def test_shim_is_a_circular_conv2d(stride, hw):
    from oracle import controlnet_oracle as CN, sd_oracle as O, tiling_oracle as T
    g = torch.Generator().manual_seed(hw[0] * 10 + hw[1])
    conv = torch.nn.Conv2d(6, 5, 3, stride=stride, padding=1, padding_mode="circular")
    x = torch.randn((2, 6, *hw), generator=g)
    w1 = torch.randn((5, 6, 1, 1), generator=g)
    with torch.no_grad(), T.circular():
        assert torch.equal(O.F.conv2d(x, conv.weight, conv.bias, stride=stride, padding=1), conv(x))
        assert torch.equal(CN.F.conv2d(x, conv.weight, conv.bias, stride=stride, padding=1), conv(x))
        assert torch.equal(O.F.conv2d(x, w1), F.conv2d(x, w1))   # padding 0: the mode is irrelevant
    assert O.F is F and CN.F is F


@pytest.fixture(scope="module")
def tiny():
    from b200sd import config as C, synth
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    return cfgs, synth.make_state_dict(*cfgs, seed=0)


def test_tiling_off_is_the_sd_oracle_and_on_is_not(tiny):
    from oracle import sd_oracle as O, tiling_oracle as T
    cfgs, sd = tiny
    tok, neg = O.random_prompt_tokens(2, vocab_hi=997), O.empty_prompt_tokens(2, vocab_hi=997)
    kw = dict(seed=5, steps=4, height=64, width=64)
    with torch.no_grad():
        ref = O.txt2img(sd, *cfgs, tok, neg, **kw)
        off = T.run(O.txt2img, sd, *cfgs, tok, neg, tiling=False, **kw)
        on = T.run(O.txt2img, sd, *cfgs, tok, neg, **kw)
    assert all(torch.equal(a, b) for a, b in zip(off, ref))
    assert _rel(on[1], ref[1]) > 1e-2


def test_circular_oracle_unet_and_vae_are_shift_equivariant(tiny):
    """rolling the latents by a multiple of the UNet's total downsampling rolls its output, and the decoder's output by
    the autoencoder's factor times as much"""
    from oracle import sd_oracle as O, tiling_oracle as T
    (ucfg, vcfg, _), sd = tiny
    g = torch.Generator().manual_seed(1)
    x, ctx = torch.randn((2, 4, 16, 16), generator=g), torch.randn((2, 77, ucfg.context_dim), generator=g)
    t = torch.tensor([400.0, 400.0])
    roll = lambda a, k: torch.roll(a, (k, -k), dims=(2, 3))  # noqa: E731
    with torch.no_grad():
        for tiling, holds in ((True, True), (False, False)):
            e, er = (T.run(O.unet_forward, sd, ucfg, z, t, ctx, tiling=tiling) for z in (x, roll(x, 8)))
            d, dr = (T.run(O.vae_decode, sd, vcfg, z, tiling=tiling) for z in (x, roll(x, 3)))
            f = 2 ** (len(vcfg.ch_mult) - 1)
            assert (_rel(er, roll(e, 8)) < 1e-5) == holds and (_rel(dr, roll(d, 3 * f)) < 1e-5) == holds


def test_controlnet_runs_zero_padded_under_the_shim(tiny):
    from b200sd import synth
    from oracle import controlnet_oracle as CN, tiling_oracle as T
    (ucfg, _, _), sd = tiny
    csd = synth.make_controlnet_state_dict(ucfg, seed=7)
    g = torch.Generator().manual_seed(2)
    x, ctx = torch.randn((2, 4, 8, 8), generator=g), torch.randn((2, 77, ucfg.context_dim), generator=g)
    hint = CN.hint_input(_hint(1, 64, 64)[None])
    t = torch.tensor([500.0, 500.0])
    with torch.no_grad():
        ref = CN.controlnet_forward(csd, ucfg, x, hint, t, ctx)
        got = T.run(lambda: CN.controlnet_forward(csd, ucfg, x, hint, t, ctx))   # looked up as unet_forward does
    assert all(torch.equal(a, b) for a, b in zip(got, ref))


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


def _oracle(env, name, steps, nz, init=None, d=None, nmask=None, units=()):
    """final latents of the tiling oracle (the ControlNet oracle's sampler with its units, under the conv shim)"""
    from oracle import controlnet_oracle as CN, tiling_oracle as T
    unet = CN.ControlledUNet(env.sd, env.cfgs[0], list(units))
    mask = None if nmask is None else (init, nmask[None, None])
    with torch.no_grad(), T.circular():
        z = CN.run_sampler(name, unet, env.cond, env.unc, 7.0, steps, nz[0], list(nz[1:]), init=init,
                           denoising_strength=d, mask=mask, prediction=env.pred)
    return z if nmask is None else z * nmask + init * (1 - nmask)


def _decoded(env, z):
    from oracle import sd_oracle as O, tiling_oracle as T
    vcfg = env.cfgs[1]
    with torch.no_grad():
        return T.run(lambda: O.to_uint8(O.vae_decode(env.sd, vcfg, z / vcfg.scale_factor)))


def _check(env, got_u8, z, ref_z, hw):
    lat = z.reshape(env.b, hw, hw, 4).permute(0, 3, 1, 2)
    assert _rel(lat, ref_z) <= 1e-4, _rel(lat, ref_z)
    d = (got_u8.int() - _decoded(env, ref_z).int()).abs()
    assert float((d <= 1).float().mean()) == 1.0 and float((d == 0).float().mean()) > 0.99


@pytest.mark.parametrize("name", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
def test_txt2img_matches_the_tiling_oracle(env, name):
    hw, steps = 8, 6
    pr = env.eng.program(name, None, steps)
    nz = env.E.per_image_noise(4100, env.b, (4, hw, hw), 1 + pr.draws)
    got = env.eng.txt2img(env.tok, env.neg, 4100, steps=steps, height=8 * hw, width=8 * hw, sampler=name, tiling=True)
    ref = _oracle(env, name, steps, nz)
    _check(env, got, env.eng.plans[(env.b, hw, hw, "tiling")].x, ref, hw)
    plain = env.eng.txt2img(env.tok, env.neg, 4100, steps=steps, height=8 * hw, width=8 * hw, sampler=name)
    assert (env.b, hw, hw) in env.eng.plans and not torch.equal(plain, got)


def _init_u8(b, px):
    return torch.randint(0, 256, (b, px, px, 3), generator=torch.Generator().manual_seed(9), dtype=torch.uint8)


@pytest.mark.parametrize("name,masked", [("DDIM", False), ("Euler a", False), ("DDIM", True), ("Heun", True)])
def test_img2img_matches_the_tiling_oracle(env, name, masked):
    from oracle import sd_oracle as O, tiling_oracle as T
    hw, steps, d = 8, 8, 0.75
    init_u8 = _init_u8(env.b, hw * 2 ** (len(env.cfgs[1].ch_mult) - 1))   # the autoencoder's factor
    nmask = (torch.rand((hw, hw), generator=torch.Generator().manual_seed(5)) > 0.5).float() if masked else None
    pr = env.eng.program(name, None, steps, denoise=d, masked=masked)
    nz = env.E.per_image_noise(31, env.b, (4, hw, hw), 1 + pr.draws)
    kw = {} if nmask is None else {"latmask": nmask.reshape(-1)}
    got = env.eng.img2img(env.tok, env.neg, 31, init_u8, denoising_strength=d, steps=steps, sampler=name, tiling=True,
                          **kw)
    with torch.no_grad():
        init = T.run(O.vae_encode_mean, env.sd, env.cfgs[1], O.image_to_model_input(init_u8)) * env.cfgs[1].scale_factor
    assert _rel(env.eng.encode(init_u8, tiling=True), init) <= 1e-4
    ref = _oracle(env, name, steps, nz, init=init, d=d, nmask=nmask)
    _check(env, got, env.eng.plans[(env.b, hw, hw, "tiling")].x, ref, hw)


@pytest.mark.parametrize("upscaler", ["Latent", "Lanczos"])
def test_hires_fix_matches_the_tiling_oracle(env, upscaler, monkeypatch):
    """both passes, the latent or pixel upscale and the VAE decode / encode between them are tiled; Lanczos itself is
    Pillow's (the device resampler is tested on its own)"""
    from PIL import Image
    from b200sd import upscale
    from oracle import tiling_oracle as T, upscale_oracle as UO

    def pil_resize(images, w, h, name, tile, overlap):
        return torch.stack([torch.from_numpy(np.array(UO.resize_image(Image.fromarray(im.numpy()), w, h, name)))
                            for im in images.cpu()])

    monkeypatch.setattr(upscale, "resize_image", pil_resize)
    hw, steps, hr_steps, d = 8, 5, 6, 0.6
    got = env.eng.txt2img_hires(env.tok, env.neg, 77, steps=steps, height=8 * hw, width=8 * hw, hr_scale=2.0,
                                hr_steps=hr_steps, denoising_strength=d, upscaler=upscaler, tiling=True)
    nz1 = env.E.per_image_noise(77, env.b, (4, hw, hw), 1)
    nz2 = env.E.per_image_noise(77, env.b, (4, 2 * hw, 2 * hw), 1)
    z1 = _oracle(env, "DDIM", steps, nz1)
    with torch.no_grad():
        up = T.run(UO.hires_upscale, env.sd, env.cfgs[1], z1, 2 * hw, 2 * hw, upscaler)
    ref = _oracle(env, "DDIM", hr_steps, nz2, init=up, d=d)
    _check(env, got, env.eng.plans[(env.b, 2 * hw, 2 * hw, "tiling")].x, ref, 2 * hw)


def test_controlnet_unit_keeps_zero_padding_under_a_circular_unet(env):
    """the UNet is circular and the ControlNet is not: the engine matches that oracle and not one where both are"""
    from oracle import controlnet_oracle as CN, tiling_oracle as T
    hw, steps, name = 8, 6, "Euler a"
    hint = _hint(20, 8 * hw, 8 * hw)
    unit = (env.csd, hint, 0.8, 0.0, 1.0)
    pr = env.eng.program(name, None, steps)
    nz = env.E.per_image_noise(12, env.b, (4, hw, hw), 1 + pr.draws)
    got = env.eng.txt2img(env.tok, env.neg, 12, steps=steps, height=8 * hw, width=8 * hw, sampler=name, tiling=True,
                          controls=[(env.cw, hint, 0.8, 0.0, 1.0)])
    ref = _oracle(env, name, steps, nz, units=[unit])
    _check(env, got, env.eng.plans[(env.b, hw, hw, "tiling")].x, ref, hw)
    unet = CN.ControlledUNet(env.sd, env.cfgs[0], [unit])
    with torch.no_grad(), T._functional(T.CIRCULAR_F):   # the ControlNet circular too: not what sdwui does
        both = CN.run_sampler(name, unet, env.cond, env.unc, 7.0, steps, nz[0], list(nz[1:]), prediction=env.pred)
    lat = env.eng.plans[(env.b, hw, hw, "tiling")].x.reshape(env.b, hw, hw, 4).permute(0, 3, 1, 2)
    assert _rel(lat, both) > 1e-3


def test_sdxl_txt2img_matches_the_tiling_oracle(monkeypatch):
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O, tiling_oracle as T
    _install(monkeypatch)
    cfgs, ocfgs = (C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP), (O.TINYXL_UNET, O.TINYXL_VAE, O.TINYXL_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2)
    b, hw, steps = 2, 8, 5
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    ctx_c, y_c = O.sdxl_conditioner(sd, ocfgs[2], tok, hw * 8, hw * 8)
    ctx_u, y_u = O.sdxl_conditioner(sd, ocfgs[2], neg, hw * 8, hw * 8, zero_txt=True)
    y = torch.cat([y_c, y_u])
    nz = E.per_image_noise(77, b, (4, hw, hw), 1 + steps)
    with torch.no_grad(), T.circular():
        unet = lambda x, t, c: O.unet_forward(sd, ocfgs[0], x, t, c, y=y)  # noqa: E731
        z = O.run_sampler("Euler a", unet, ctx_c, ctx_u, 7.0, steps, nz[0], list(nz[1:]))
        ref_u8 = O.to_uint8(O.vae_decode(sd, ocfgs[1], z / ocfgs[1].scale_factor))
    got = eng.txt2img(tok, neg, seed=77, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, sampler="Euler a",
                      tiling=True)
    lat = eng.plans[(b, hw, hw, "tiling")].x.reshape(b, hw, hw, 4).permute(0, 3, 1, 2)
    assert _rel(lat, z) <= 1e-3
    d = (got.int() - ref_u8.int()).abs()
    assert float((d <= 1).float().mean()) == 1.0 and float((d == 0).float().mean()) > 0.99


# ------------------------------------------------------------------------------------------------ op lists
def _convs(op_list):
    """(kind, conv kwargs) per op: 'pad' for a circular pad, 'conv' for a conv, 'other' for the rest"""
    from b200sd import ops
    out = []
    for fn, a, k in op_list:
        out.append(("pad", a[1]) if fn is ops.pad_circular else ("conv", k) if fn is ops.conv2d else ("other", None))
    return out


def _shapes(args):
    """tensors by shape, everything else by value"""
    if isinstance(args, dict):
        return {key: _shapes(v) for key, v in args.items()}
    if isinstance(args, (list, tuple)):
        return [_shapes(v) for v in args]
    return tuple(args.shape) if torch.is_tensor(args) else args


def _signature(op_list):
    return [(getattr(fn, "__name__", None), _shapes(list(a)), _shapes(k)) for fn, a, k in op_list]


def _circularised(plain, tiled):
    """every 3x3 conv of `plain` with the kernel's padding 1 is a pad + pad-0 conv on the padded buffer in `tiled`, every
    other op is unchanged; returns how many convs became circular"""
    p, t = _convs(plain), _convs(tiled)
    i = n = 0
    for kind, k in p:
        if kind == "conv" and k["ksize"] == 3 and "pad" not in k:
            assert t[i][0] == "pad" and t[i + 1][0] == "conv" and t[i + 1][1]["pad"] == 0
            assert _shapes(t[i + 1][1]) == _shapes(dict(k, pad=0))
            i, n = i + 2, n + 1
        else:
            assert t[i][0] == kind and (kind != "conv" or _shapes(t[i][1]) == _shapes(k))
            i += 1
    assert i == len(t)
    return n


def test_programs_make_exactly_the_listed_convs_circular(monkeypatch):
    from b200sd import config as C, synth
    from b200sd.unet_exec import ControlNetWeights, UNetProgram, UNetWeights
    from b200sd.vae_exec import VAEDecoderProgram, VAEDecoderWeights, VAEEncoderProgram, VAEEncoderWeights
    _install(monkeypatch)
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    uw = UNetWeights(sd, cfgs[0], "cpu", torch.float32)
    progs = {t: UNetProgram(uw, 2, 16, 16, tiling=t) for t in (False, True)}
    default = UNetProgram(uw, 2, 16, 16)
    assert _signature(default.ops) == _signature(progs[False].ops)
    assert not any(k == "pad" for k, _ in _convs(progs[False].ops))
    # conv_in, two convs per ResBlock, the Downsample and Upsample convs, out.2
    inputs, middle, outputs = uw.layout
    layers = [layer[0] for blk in inputs + [middle] + outputs for layer in blk]
    want = 1 + 2 * layers.count("res") + layers.count("down") + layers.count("up") + 1
    assert _circularised(progs[False].ops, progs[True].ops) == want
    # ControlNet segments and hint blocks stay zero padded
    cw = ControlNetWeights(synth.make_controlnet_state_dict(cfgs[0], seed=1), cfgs[0], "cpu", torch.float32)
    step = torch.zeros((1,), dtype=torch.int32)
    for t in (False, True):
        progs[t].set_control(0, cw, 4, step)
    seg = [progs[t].segments[0] for t in (False, True)]
    assert _signature(seg[0].ops) == _signature(seg[1].ops) and _signature(seg[0].hint_ops) == _signature(seg[1].hint_ops)
    assert not any(k == "pad" for k, _ in _convs(seg[1].ops + seg[1].hint_ops))
    assert progs[True].circular   # restored after the segment was emitted
    # VAE decoder: conv_in, ResBlock convs, upsample convs, conv_out; encoder: conv_in, ResBlock convs, conv_out — its
    # downsample (F.pad (0, 1, 0, 1) with zeros, conv padding 0) stays pad=0 / pad_end=1
    vcfg = cfgs[1]
    nlev = len(vcfg.ch_mult)
    dw, ew = VAEDecoderWeights(sd, vcfg, "cpu", torch.float32), VAEEncoderWeights(sd, vcfg, "cpu", torch.float32)
    dec = {t: VAEDecoderProgram(dw, 2, 8, 8, tiling=t) for t in (False, True)}
    enc = {t: VAEEncoderProgram(ew, 2, 32, 32, tiling=t) for t in (False, True)}
    assert _signature(VAEDecoderProgram(dw, 2, 8, 8).ops) == _signature(dec[False].ops)
    assert _signature(VAEEncoderProgram(ew, 2, 32, 32).ops) == _signature(enc[False].ops)
    assert _circularised(dec[False].ops, dec[True].ops) == 1 + 2 * (2 + nlev * (vcfg.num_res_blocks + 1)) + (nlev - 1) + 1
    assert _circularised(enc[False].ops, enc[True].ops) == 1 + 2 * (nlev * vcfg.num_res_blocks + 2) + 1
    downs = [k for kind, k in _convs(enc[True].ops) if kind == "conv" and k.get("pad_end") == 1]
    assert len(downs) == nlev - 1 and all(k["pad"] == 0 and k["stride"] == 2 for k in downs)


def test_plans_of_both_modes_live_side_by_side(env):
    eng = env.eng
    for t in (False, True, False, True):
        eng.txt2img(env.tok, env.neg, 3, steps=3, height=64, width=64, sampler="DDIM", **({"tiling": True} if t else {}))
    assert set(eng.plans) == {(env.b, 8, 8), (env.b, 8, 8, "tiling")}
    assert len(eng.plans) <= env.E.MAX_PLANS
    a = eng.txt2img(env.tok, env.neg, 3, steps=3, height=64, width=64, sampler="DDIM", tiling=False)
    b = eng.txt2img(env.tok, env.neg, 3, steps=3, height=64, width=64, sampler="DDIM")
    assert torch.equal(a, b)


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


@pytest.mark.parametrize("fields,opts,want", [
    (dict(tiling=True), None, True), (dict(tiling=False), None, False), (dict(tiling=None), None, False), ({}, None, False),
    (dict(tiling=None, override_settings={"tiling": True}), None, True),
    (dict(override_settings={"tiling": False}), True, False), (dict(tiling=None), True, True),
    (dict(tiling=False), True, False), (dict(tiling=None, override_settings={}), False, False)])
def test_worker_resolves_tiling_as_sdwui(worker, monkeypatch, fields, opts, want):
    import modules.shared as shared
    wk, calls = worker
    if opts is not None:
        monkeypatch.setattr(shared.opts, "tiling", opts, raising=False)
    wk.request(_payload(**fields), None, False)
    name, kw = calls[-1]
    assert name == "txt2img" and kw.get("tiling", False) is want and (want or "tiling" not in kw)
    info = json.loads(wk.response["info"])
    assert all(t.endswith(", Tiling: True") == want for t in info["infotexts"])


def test_worker_untiled_payload_reaches_the_engine_as_before(worker):
    wk, calls = worker
    wk.request(_payload(), None, False)
    plain = wk.response["tensors"].clone()
    assert "tiling" not in calls[-1][1]
    wk.request(_payload(tiling=True), None, False)
    assert calls[-1][1]["tiling"] is True and not torch.equal(wk.response["tensors"], plain)


def test_worker_passes_tiling_to_img2img_and_the_hires_fix(worker):
    import base64
    import io
    from PIL import Image
    wk, calls = worker
    buf = io.BytesIO()
    Image.fromarray(_init_u8(1, 64)[0].numpy()).save(buf, format="PNG")
    wk.request(_payload(tiling=True, init_images=[base64.b64encode(buf.getvalue()).decode()]), None, False)
    assert calls[-1][0] == "img2img" and calls[-1][1]["tiling"] is True
    wk.request(_payload(enable_hr=True, hr_scale=2.0, override_settings={"tiling": True}), None, False)
    assert calls[-1][0] == "txt2img_hires" and calls[-1][1]["tiling"] is True


class _RecordingEngine:
    """the engine surface the worker's txt2img path uses; records the keyword arguments"""

    def __init__(self):
        self.interrupted = False
        self.clip_cfg = types.SimpleNamespace(vocab=1000)
        self.calls = []

    def txt2img(self, tok, neg, seed, **kw):
        self.calls.append(kw)
        return torch.zeros((tok.shape[0], kw["height"], kw["width"], 3), dtype=torch.uint8)


def test_rest_server_forwards_the_tiling_field():
    from fastapi.testclient import TestClient
    from server.sdapi import create_app
    eng = _RecordingEngine()
    client = TestClient(create_app(lambda device: eng, [0]))
    body = {"prompt": "a", "steps": 2, "width": 64, "height": 64, "sampler_name": "DDIM"}
    r = client.post("/sdapi/v1/txt2img", json=dict(body, tiling=True))
    assert r.status_code == 200 and eng.calls[-1]["tiling"] is True
    assert json.loads(r.json()["info"])["infotexts"][0].endswith(", Tiling: True")
    r = client.post("/sdapi/v1/txt2img", json=dict(body, tiling=None, override_settings={"tiling": True}))
    assert r.status_code == 200 and eng.calls[-1]["tiling"] is True
    r = client.post("/sdapi/v1/txt2img", json=body)
    assert r.status_code == 200 and "tiling" not in eng.calls[-1]
