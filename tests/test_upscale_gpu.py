"""Hires-fix upscalers on the H100: the RRDBNet conv epilogues, Pillow-exact resampling and tile blending, the latent
modes, the whole fp16 RRDBNet against the fp32 oracle, and whole hires requests against oracle/upscale_oracle.py."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from kutil import OUT_DIR

pytestmark = pytest.mark.gpu


def _record(name, **kw):
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "upscale_parity.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **kw)) + "\n")


# whole requests: the bounds of the existing hires parity tests — fp16 (test_engine_gpu.py U8_MAX / U8_MEAN / U8_EXACT)
# and bf16 SDXL (test_sdxl_gpu.py U8_MEAN_BF16 / U8_WITHIN4_BF16)
U8_MAX, U8_MEAN, U8_EXACT = 2, 0.3, 0.80
U8_MEAN_BF16, U8_WITHIN4_BF16 = 2.0, 0.95


def _u8_check(name, got, ref, bf16=False):
    du8 = (got.cpu().int() - ref.cpu().int()).abs().float()
    rec = dict(u8_mean=float(du8.mean()), u8_max=float(du8.max()), u8_exact=float((du8 == 0).float().mean()),
               u8_within4=float((du8 <= 4).float().mean()))
    _record(name, **rec)
    assert got.shape == ref.shape
    if bf16:
        assert rec["u8_mean"] <= U8_MEAN_BF16 and rec["u8_within4"] >= U8_WITHIN4_BF16, rec
    else:
        assert rec["u8_max"] <= U8_MAX and rec["u8_mean"] <= U8_MEAN and rec["u8_exact"] >= U8_EXACT, rec


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("cout,lrelu,res", [(32, True, False), (64, False, True), (32, False, True), (64, True, False)])
def test_conv2d_scaled_epilogues_in_place_on_a_slice(cout, lrelu, res):
    from b200sd import ops
    g = torch.Generator().manual_seed(cout + 2 * lrelu + res)
    nb, h, w, c = 2, 23, 150, 128
    buf = torch.randn((nb, h, w, 224), generator=g).half().cuda()
    x = buf[..., 96:96 + c]
    wt = (torch.randn((cout, 9 * c), generator=g) / (9 * c) ** 0.5).half().cuda()
    bias = torch.randn((cout,), generator=g).cuda()
    before = buf.clone()
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), wt.float().reshape(cout, 3, 3, c).permute(0, 3, 1, 2), bias, padding=1)
    ref = ref.permute(0, 2, 3, 1)
    if lrelu:
        ref = F.leaky_relu(ref, 0.2)
    if res:    # D = r + 0.2 * v, residual read from (and D written to) slot [192, 192 + cout) of another buffer
        other = torch.randn((nb, h, w, 256), generator=g).half().cuda()
        out = other[..., 192:192 + cout]
        ref = out.float() + 0.2 * ref
        keep = other.clone()
        ops.conv2d_scaled(x, wt, out, bias=bias, residual=out, res_scale=0.2, lrelu=lrelu)
    else:      # written into channels [0, cout) of the buffer the conv reads, outside the window [96, 224) it reads
        out = buf[..., 0:cout]
        ops.conv2d_scaled(x, wt, out, bias=bias, lrelu=lrelu)
    torch.cuda.synchronize()
    d = (out.float() - ref).abs()
    _record(f"conv2d_scaled cout{cout} lrelu{lrelu} res{res}", max_abs=float(d.max()))
    assert bool((d <= 2e-2 + 2e-3 * ref.abs()).all()), float(d.max())
    if res:
        assert torch.equal(other[..., :192], keep[..., :192]) and torch.equal(other[..., 192 + cout:], keep[..., 192 + cout:])
        assert torch.equal(buf, before)
    else:
        assert torch.equal(buf[..., cout:], before[..., cout:])


def test_scaled_add_and_quantize_unit():
    from b200sd import ops
    g = torch.Generator().manual_seed(5)
    y = torch.randn((7, 33, 96), generator=g).half().cuda()
    x = torch.randn((7, 33, 96), generator=g).half().cuda()
    want = (y[..., 32:].float() + 0.2 * x[..., :64].float()).half()
    ops.scaled_add_(y[..., 32:], x[..., :64], 0.2)
    v = (torch.rand((3, 1000, 32), generator=g) * 1.4 - 0.2).half().cuda()
    q = torch.empty((3, 1000, 3), dtype=torch.uint8, device="cuda")
    ops.quantize_unit_u8(v, q)
    torch.cuda.synchronize()
    assert torch.equal(y[..., 32:], want)
    ref = (255.0 * v[..., :3].float().cpu().clamp(0, 1).numpy()).round().astype(np.uint8)
    assert np.array_equal(q.cpu().numpy(), ref)


@pytest.mark.parametrize("filt", ["lanczos", "nearest"])
def test_resample_equals_pil_bitwise(filt):
    from b200sd import upscale as U
    rng = np.random.default_rng(1)
    pil = Image.LANCZOS if filt == "lanczos" else Image.NEAREST
    for (hh, ww), (h2, w2) in [((512, 512), (1024, 1024)), ((2048, 2048), (1024, 1024)), ((97, 311), (300, 100)),
                               ((600, 173), (29, 1000)), ((64, 64), (64, 200))]:
        imgs = rng.integers(0, 256, (2, hh, ww, 3), dtype=np.uint8)
        got = U.pil_resize(torch.from_numpy(imgs).cuda(), w2, h2, filt).cpu().numpy()
        want = np.stack([np.array(Image.fromarray(im).resize((w2, h2), pil)) for im in imgs])
        assert np.array_equal(got, want), (filt, hh, ww, h2, w2)


@pytest.mark.parametrize("w,h,tile,overlap", [(512, 512, 192, 8), (300, 200, 64, 16), (100, 60, 192, 8)])
def test_combine_tiles_equals_combine_grid_bitwise(w, h, tile, overlap):
    from b200sd import ops, upscale as U
    from oracle import upscale_oracle as UO
    ys, xs = U.split_grid(w, h, tile, tile, overlap)
    rng = np.random.default_rng(w + h)
    tiles = rng.integers(0, 256, (2, len(ys), len(xs), tile, tile, 3), dtype=np.uint8)
    out = torch.empty((2, h, w, 3), dtype=torch.uint8, device="cuda")
    ops.combine_tiles_u8(torch.from_numpy(tiles.reshape(-1, tile, tile, 3)).cuda(), out,
                         torch.tensor(ys, dtype=torch.int32, device="cuda"), torch.tensor(xs, dtype=torch.int32, device="cuda"),
                         torch.from_numpy(U.blend_mask(overlap)).cuda(), overlap)
    for b in range(2):
        grid = UO.Grid([[y, tile, [[x, tile, Image.fromarray(tiles[b, r, c])] for c, x in enumerate(xs)]]
                        for r, y in enumerate(ys)], tile, tile, w, h, overlap)
        assert np.array_equal(out[b].cpu().numpy(), np.array(UO.combine_grid(grid))), b


def test_latent_modes_equal_interpolate():
    from b200sd import upscale as U
    x = torch.randn((3, 4, 64, 48), generator=torch.Generator().manual_seed(2)).cuda()
    lat = x.permute(0, 2, 3, 1).reshape(3, 64 * 48, 4).contiguous()
    for name, (mode, aa) in U.LATENT_MODES.items():
        if name == "Latent":
            continue
        for ho, wo in ((128, 96), (96, 72), (32, 24)):
            want = F.interpolate(x, size=(ho, wo), mode=mode, antialias=aa).permute(0, 2, 3, 1).reshape(3, ho * wo, 4)
            got = U.resize_latents(lat, name, 64, 48, ho, wo)
            torch.cuda.synchronize()
            if mode.startswith("nearest"):
                assert torch.equal(got, want), (name, ho, wo)
            else:
                d = float((got - want).abs().max())
                _record(f"latent {name} {ho}x{wo}", max_abs=d)
                assert d <= 1e-5 * float(want.abs().max()) + 1e-6, (name, ho, wo, d)


# ------------------------------------------------------------------------------------------------ the whole network
def test_rrdbnet_23_blocks_against_the_fp32_oracle():
    from b200sd import upscale as U
    from oracle import upscale_oracle as UO
    sd = U.synthetic_state_dict(23, seed=11)
    wts = U.RRDBWeights(sd, "cuda:0")
    n = 3
    tiles = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (n, 192, 192, 3), dtype=np.uint8)).cuda()
    prog = U.RRDBProgram(wts, n, 192, 192)
    u8 = prog.run(tiles, n).view(n, 768, 768, 3)
    pre = prog.last[..., :3].float()
    torch.cuda.synchronize()
    with torch.no_grad():
        bgr = UO.pil_to_bgr([Image.fromarray(t) for t in tiles.cpu().numpy()]).cuda()
        ref = UO.rrdbnet({k: v.cuda() for k, v in sd.items()}, bgr).flip(1).permute(0, 2, 3, 1)   # RGB NHWC
    rel = float(((pre - ref) ** 2).mean().sqrt() / (ref ** 2).mean().sqrt())
    ref_u8 = (255.0 * ref.clamp(0, 1)).round().to(torch.uint8)
    du8 = (u8.int() - ref_u8.int()).abs().float()
    _record("rrdbnet 23 blocks 3 x 192^2", rel_rms=rel, u8_mean=float(du8.mean()), u8_max=float(du8.max()))
    assert rel <= 5e-3 and float(du8.mean()) <= 0.3 and float(du8.max()) <= 2, (rel, float(du8.mean()), float(du8.max()))


# ------------------------------------------------------------------------------------------------ whole requests
@pytest.fixture(scope="module")
def tiny():
    from b200sd import config as C, engine as E, synth
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=False)
    return cfgs, sd, {k: v.cuda() for k, v in sd.items()}, eng


@pytest.mark.parametrize("name", ["Latent (bicubic antialiased)", "Latent (nearest)", "Lanczos", "None", "Nearest",
                                  "R-ESRGAN 4x+"])
def test_tiny_hires_request_matches_the_oracle(tiny, name, monkeypatch):
    from b200sd import upscale as U
    from oracle import sd_oracle as O, upscale_oracle as UO
    monkeypatch.delenv("B200SD_UPSCALER_DIR", raising=False)
    cfgs, sd, dsd, eng = tiny
    b = 2
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    esd = U.load_state_dict("RealESRGAN_x4plus") if name == "R-ESRGAN 4x+" else None
    with torch.no_grad():
        ref, _ = UO.txt2img_hires(dsd, *cfgs, tok, neg, seed=910, steps=6, cfg_scale=7.0, height=64, width=64, hr_scale=2.0,
                                  hr_steps=8, denoising_strength=0.7, upscaler=name, esrgan_sd=esd, device="cuda")
    got = eng.txt2img_hires(tok, neg, seed=910, steps=6, cfg_scale=7.0, height=64, width=64, hr_scale=2.0, hr_steps=8,
                            denoising_strength=0.7, upscaler=name)
    _u8_check(f"hires tiny {name}", got, ref)


def test_latent_hires_is_the_parent_call_sequence(tiny):
    """"Latent" (the default) runs exactly what the engine ran before the other upscalers existed"""
    from b200sd import ops
    from oracle import sd_oracle as O
    cfgs, sd, dsd, eng = tiny
    b = 2
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    got = eng.txt2img_hires(tok, neg, seed=920, steps=5, height=64, width=128, hr_scale=2.0, hr_steps=6)
    cond, uncond = eng._conds(tok, neg, 128, 64, None, None)
    lat = eng._sample_txt(cond, uncond, 920, b, 8, 16, 5, 7.0, "DDIM", None)
    up = torch.empty((b, 16 * 32, 4), device="cuda", dtype=torch.float32)
    ops.resize_latent_bilinear(lat.contiguous(), up, 8, 16, 16, 32)
    lat2 = eng._sample_from(up.reshape(b, 16, 32, 4).permute(0, 3, 1, 2), cond, uncond, 920, 0.7, 6, 7.0, "DDIM", None)
    assert torch.equal(got, eng.decode(lat2, 16, 32))


def test_esrgan_hires_batch_invariance(tiny, monkeypatch):
    from oracle import sd_oracle as O
    monkeypatch.delenv("B200SD_UPSCALER_DIR", raising=False)
    cfgs, sd, dsd, eng = tiny
    tok, neg = O.random_prompt_tokens(3, vocab_hi=997), O.empty_prompt_tokens(3, vocab_hi=997)
    kw = dict(steps=4, height=128, width=64, hr_scale=2.0, hr_steps=4, upscaler="R-ESRGAN 4x+", upscaler_tile=24,
              upscaler_overlap=4)   # the tiny autoencoder's images are 32 x 16 pixels: 3 x 1 tiles
    batch = eng.txt2img_hires(tok, neg, seed=930, **kw)
    for k in range(3):
        alone = eng.txt2img_hires(tok[k:k + 1], neg[k:k + 1], seed=930 + k, **kw)
        assert torch.equal(alone[0], batch[k]), k


@pytest.mark.parametrize("name", ["Latent (bicubic antialiased)", "Lanczos", "R-ESRGAN 4x+"])
def test_tinyxl_hires_request_matches_the_oracle(name, monkeypatch):
    """SDXL topology in bf16 (reduced width), Euler a: the bf16 VAE decode and encode around a pixel upscaler, the
    second pass conditioned on the large size"""
    from b200sd import config as C, engine as E, synth, upscale as U
    from oracle import sd_oracle as O, upscale_oracle as UO
    monkeypatch.delenv("B200SD_UPSCALER_DIR", raising=False)
    cfgs = (C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP)
    ocfgs = (O.TINYXL_UNET, O.TINYXL_VAE, O.TINYXL_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", dtype=torch.bfloat16, use_graphs=False)
    b, px = 2, 128
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    esd = U.load_state_dict("RealESRGAN_x4plus") if name == "R-ESRGAN 4x+" else None
    got = eng.txt2img_hires(tok, neg, seed=950, steps=6, cfg_scale=7.0, height=px, width=px, hr_scale=2.0, hr_steps=6,
                            denoising_strength=0.7, sampler="Euler a", upscaler=name)
    with torch.no_grad():
        ref, _ = UO.txt2img_hires_xl({k: v.cuda() for k, v in sd.items()}, *ocfgs, tok, neg, seed=950, steps=6,
                                     cfg_scale=7.0, height=px, width=px, hr_scale=2.0, hr_steps=6,
                                     denoising_strength=0.7, upscaler=name, esrgan_sd=esd, sampler="Euler a",
                                     device="cuda")
    _u8_check(f"hires tinyxl {name}", got, ref, bf16=True)


def test_sd15_esrgan_hires_512_to_1024(monkeypatch):
    from b200sd import config as C, engine as E, synth, upscale as U
    from oracle import sd_oracle as O, upscale_oracle as UO
    monkeypatch.delenv("B200SD_UPSCALER_DIR", raising=False)
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    tok, neg = O.random_prompt_tokens(1, vocab_hi=49405), O.empty_prompt_tokens(1, vocab_hi=49405)
    got = eng.txt2img_hires(tok, neg, seed=940, steps=4, height=512, width=512, hr_scale=2.0, hr_steps=4,
                            upscaler="R-ESRGAN 4x+")
    del eng
    torch.cuda.empty_cache()
    with torch.no_grad():
        ref, _ = UO.txt2img_hires({k: v.cuda() for k, v in sd.items()}, *cfgs, tok, neg, seed=940, steps=4, height=512,
                                  width=512, hr_scale=2.0, hr_steps=4, upscaler="R-ESRGAN 4x+",
                                  esrgan_sd=U.load_state_dict("RealESRGAN_x4plus"), device="cuda")
    _u8_check("hires sd15 512->1024 R-ESRGAN 4x+", got, ref)
