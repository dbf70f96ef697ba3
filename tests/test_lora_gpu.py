"""LoRA networks on the GPU: b200sd_lora_merge against fp64 with a rounding-derived bound and its bitwise properties,
then whole requests with merged networks against the oracles on the oracle-merged state dict (oracle/lora_oracle.py),
and the engine's set switching (bitwise)."""
import json
import os

import pytest
import torch

from kutil import OUT_DIR

pytestmark = pytest.mark.gpu


def _record(name, **kw):
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "lora_parity.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **kw)) + "\n")


def _u8_check(name, got, ref, mean=1.5, within2=0.97, within4=0.0):
    """the bounds of the existing request tests: fp16 mean <= 1.5 LSB with >= 97 % within 2 (test_controlnet_gpu);
    bf16 (SDXL) mean <= 2 with >= 95 % within 4 (test_sdxl_gpu)"""
    du8 = (got.cpu().int() - ref.cpu().int()).abs().float()
    rec = dict(u8_mean=float(du8.mean()), u8_max=float(du8.max()), u8_within2=float((du8 <= 2).float().mean()),
               u8_within4=float((du8 <= 4).float().mean()))
    _record(name, **rec)
    assert got.shape == ref.shape
    assert rec["u8_mean"] <= mean and rec["u8_within2"] >= within2 and rec["u8_within4"] >= within4, rec


# ------------------------------------------------------------------------------------------------ kernel
def _half_ulp(v: torch.Tensor, dt) -> torch.Tensor:
    """half an ulp of the output format at magnitude |v| (float64)"""
    mant, emin = (10, -14) if dt == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - mant) / 2


def _case(g, rows, cols, r, dt, ldw=None):
    ldw = ldw or cols
    buf = (torch.randn((rows, ldw), generator=g) * 0.05).to(dt).cuda()
    p = buf.clone()
    u = (torch.randn((rows, r), generator=g) * 0.1).cuda()
    d = (torch.randn((r, cols), generator=g) * 0.1).cuda()
    return buf, p, u, d


def _check_fp64(name, w, p, u, d, dt):
    pv = p.double()
    s = u.double() @ d.double()
    exact = pv + s
    r = u.shape[1]
    # fmaf accumulation over r terms: |s_fp32 - s| <= r 2^-24 sum |u||d| (1.01 for the higher-order terms), the fp32
    # add P + s one more 2^-24, then one rounding to the output format
    delta = 1.01 * r * 2.0 ** -24 * (u.double().abs() @ d.double().abs()) + 2.0 ** -24 * (pv.abs() + s.abs())
    bound = _half_ulp(exact.abs() + delta, dt) + delta
    ratio = float(((w.double() - exact).abs() / bound).max())
    _record(name, worst_ratio=ratio)
    assert ratio <= 1.0, (name, ratio)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("r", [1, 16, 33, 64, 128])
def test_merge_against_fp64(dt, r):
    """ragged rows and columns, a row pitch wider than the columns, many descriptors in one launch, ranks below, at and
    above the 32-rank staging chunk"""
    from b200sd import ops
    g = torch.Generator().manual_seed(r)
    shapes = [(1, 1, None), (63, 129, None), (64, 128, 136), (200, 1000, 1032), (1280, 320, None), (7, 2048, 2056)]
    shapes += [(int(a), int(b), None) for a, b in torch.randint(1, 300, (40, 2), generator=g)]
    cases = [_case(g, rows, cols, r, dt, ldw) for rows, cols, ldw in shapes]
    views = [(w[:, :d.shape[1]], p[:, :d.shape[1]], u, d) for w, p, u, d in cases]
    ops.lora_merge(views)
    torch.cuda.synchronize()
    for (rows, cols, ldw), (w, p, u, d) in zip(shapes, cases):
        _check_fp64(f"merge {dt} r={r} {rows}x{cols}", w[:, :cols], p[:, :cols], u, d, dt)
        if ldw:
            assert torch.equal(w[:, cols:], p[:, cols:]), "columns beyond `cols` are not written"


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_merge_bitwise_properties(dt):
    """R = 0 copies P bitwise (a restore), zero rows of U leave their rows bitwise pristine (padded heads), and two
    launches give bitwise the same weights"""
    from b200sd import ops
    g = torch.Generator().manual_seed(3)
    w, p, u, d = _case(g, 300, 520, 40, dt)
    u[::7] = 0
    w.copy_(torch.randn(w.shape, generator=g).to(dt).cuda())   # garbage to be overwritten
    w0, p0, u0, d0 = _case(g, 129, 77, 0, dt)
    w0.zero_()
    ops.lora_merge([(w, p, u, d), (w0, p0, u0, d0)])
    first = w.clone()
    torch.cuda.synchronize()
    assert torch.equal(w0, p0)
    assert torch.equal(w[::7], p[::7])
    ops.lora_merge([(w, p, u, d)])
    torch.cuda.synchronize()
    assert torch.equal(w, first)


# ------------------------------------------------------------------------------------------------ engine
_ENG = {}


def _engine(size, graphs=True):
    from b200sd import engine as E, factory, synth
    key = (size, graphs)
    if key not in _ENG:
        cfgs = factory.configs(size)
        sd = synth.make_state_dict(*cfgs, seed=0)
        dt = torch.bfloat16 if size.endswith("xl") else torch.float16
        pred = factory.prediction(size)
        _ENG[key] = (E.SDEngine(sd, *cfgs, device="cuda:0", dtype=dt, use_graphs=graphs, prediction=pred), sd, cfgs)
    return _ENG[key]


def _nets(cfgs, specs):
    """specs: [(seed, rank, form, te, unet, dyn)] -> (engine networks, oracle networks)"""
    from b200sd import lora as L, synth
    nets, onets = [], []
    for seed, rank, form, te, unet, dyn in specs:
        sd = synth.make_lora_state_dict(cfgs[0], cfgs[2], seed=seed, rank=rank, form=form)
        nets.append((L.load_state_dict(f"n{seed}", sd, key=("test", seed, rank, form)), L.LoraRef(f"n{seed}", te, unet, dyn)))
        onets.append((sd, te, unet, dyn))
    return nets, onets


TWO = [(11, 8, "diffusers", 0.8, 1.1, None), (12, 16, "compvis", -0.6, 0.7, 8)]
TWO_XL = [(11, 8, "compvis", 0.8, 1.1, None), (12, 16, "compvis", -0.6, 0.7, 8)]


def _tok(b):
    from oracle import sd_oracle as O
    return O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)


def test_tiny_lora_request_matches_the_oracle():
    from oracle import lora_oracle as LO, sd_oracle as O
    eng, sd, cfgs = _engine("tiny")
    nets, onets = _nets(cfgs, TWO)
    b, hw, steps = 2, 16, 8
    tok, neg = _tok(b)
    got = eng.txt2img(tok, neg, seed=41, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, sampler="DDIM",
                      loras=nets)
    merged = LO.merge({k: v.cuda() for k, v in sd.items()}, onets)
    with torch.no_grad():
        ref, _, _ = O.txt2img(merged, *cfgs, tok, neg, seed=41, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8,
                              device="cuda")
        plain, _, _ = O.txt2img({k: v.cuda() for k, v in sd.items()}, *cfgs, tok, neg, seed=41, steps=steps, cfg_scale=7.0,
                                height=hw * 8, width=hw * 8, device="cuda")
    _u8_check("tiny lora DDIM", got, ref)
    assert float((ref.int() - plain.int()).abs().float().mean()) > 5.0, "the networks change the image"


def test_tiny21_lora_request_matches_the_v_oracle():
    from b200sd import engine as E
    from oracle import lora_oracle as LO, v_oracle as V
    eng, sd, cfgs = _engine("tiny21")
    nets, onets = _nets(cfgs, TWO)
    b, hw, steps, seed = 2, 16, 7, 610
    tok, neg = _tok(b)
    merged = LO.merge({k: v.cuda() for k, v in sd.items()}, onets)
    pr = eng.program("Euler a", None, steps)
    nz = E.per_image_noise(seed, b, (4, hw, hw), 1 + pr.draws).cuda()
    cond, unc = V.encode_sd21(merged, cfgs[2], tok.cuda()), V.encode_sd21(merged, cfgs[2], neg.cuda())
    with torch.no_grad():
        ref, _ = V.txt2img(merged, V.TINY21_UNET, V.TINY21_VAE, V.cfg_unet(merged, V.TINY21_UNET), cond, unc, "Euler a",
                           steps, 7.0, nz)
    got = eng.txt2img(tok, neg, seed=seed, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, sampler="Euler a",
                      loras=nets)
    _u8_check("tiny21 lora Euler a", got, ref)


def _xl_ref(O, ocfgs, dsd, tok, neg, hw, steps, seed):
    ctx_c, y_c = O.sdxl_conditioner(dsd, ocfgs[2], tok.cuda(), hw * 8, hw * 8)
    ctx_u, y_u = O.sdxl_conditioner(dsd, ocfgs[2], neg.cuda(), hw * 8, hw * 8, zero_txt=True)
    y = torch.cat([y_c, y_u])
    unet = lambda x, t, c: O.unet_forward(dsd, ocfgs[0], x, t, c, y=y)  # noqa: E731
    from b200sd import engine as E
    nz = E.per_image_noise(seed, tok.shape[0], (4, hw, hw), 1 + steps).cuda()
    with torch.no_grad():
        z = O.run_sampler("Euler a", unet, ctx_c, ctx_u, 7.0, steps, nz[0], list(nz[1:]))
        return O.to_uint8(O.vae_decode(dsd, ocfgs[1], z / ocfgs[1].scale_factor)).cpu()


def test_tinyxl_lora_request_matches_the_oracle():
    from oracle import lora_oracle as LO, sd_oracle as O
    eng, sd, cfgs = _engine("tinyxl")
    nets, onets = _nets(cfgs, TWO_XL)
    b, hw, steps = 2, 16, 6
    tok, neg = _tok(b)
    merged = LO.merge({k: v.cuda() for k, v in sd.items()}, onets)
    ref = _xl_ref(O, (O.TINYXL_UNET, O.TINYXL_VAE, O.TINYXL_CLIP), merged, tok, neg, hw, steps, 77)
    got = eng.txt2img(tok, neg, seed=77, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, sampler="Euler a",
                      loras=nets)
    _u8_check("tinyxl lora Euler a", got, ref, mean=2.0, within2=0.0, within4=0.95)


def test_sd15_512_lora_request_matches_the_oracle():
    from b200sd import config as C, engine as E, synth
    from oracle import lora_oracle as LO, sd_oracle as O
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    nets, onets = _nets(cfgs, [(21, 16, "diffusers", 0.9, 0.8, None), (22, 8, "compvis", 0.5, -0.5, None)])
    tok, neg = O.random_prompt_tokens(1, vocab_hi=49405), O.empty_prompt_tokens(1, vocab_hi=49405)
    got = eng.txt2img(tok, neg, seed=5, steps=10, cfg_scale=7.0, height=512, width=512, sampler="DDIM", loras=nets)
    del eng
    merged = LO.merge({k: v.cuda() for k, v in sd.items()}, onets)
    with torch.no_grad():
        ref, _, _ = O.txt2img(merged, *cfgs, tok, neg, seed=5, steps=10, cfg_scale=7.0, height=512, width=512,
                              device="cuda")
    _u8_check("sd15 512 lora DDIM", got, ref)
    del merged
    torch.cuda.empty_cache()


def test_set_switching_is_bitwise():
    """a plain request after a LoRA request equals the plain request before it; A -> B -> A reproduces A; graphs on equal
    graphs off; the pristine copies are made on the first LoRA request only"""
    eng, _, cfgs = _engine("tiny")
    eng_ng, _, _ = _engine("tiny", graphs=False)
    a, _ = _nets(cfgs, TWO)
    bnets, _ = _nets(cfgs, [(13, 4, "compvis", 1.0, 1.0, None)])
    tok, neg = _tok(2)
    run = lambda e, **kw: e.txt2img(tok, neg, seed=9, steps=5, height=128, width=128, sampler="Euler a", **kw).cpu()  # noqa: E731
    eng.set_loras(())
    plain = run(eng)
    ga = run(eng, loras=a)
    gb = run(eng, loras=bnets)
    ga2 = run(eng, loras=a)
    plain2 = run(eng)
    assert not torch.equal(ga, plain) and not torch.equal(ga, gb)
    assert torch.equal(ga, ga2) and torch.equal(plain, plain2)
    assert torch.equal(run(eng_ng, loras=a), ga)
    assert torch.equal(run(eng_ng), plain)


def test_hires_pass_with_its_own_set_matches_the_oracle():
    import torch.nn.functional as F
    from b200sd import engine as E
    from oracle import lora_oracle as LO, sd_oracle as O
    eng, sd, cfgs = _engine("tiny")
    a, oa = _nets(cfgs, TWO[:1])
    hb, ob = _nets(cfgs, TWO[1:])
    b, hw, steps = 2, 8, 6
    tok, neg = _tok(b)
    got = eng.txt2img_hires(tok, neg, 31, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, hr_scale=2.0,
                            denoising_strength=0.6, sampler="DDIM", loras=a, hr_loras=hb)
    dsd = {k: v.cuda() for k, v in sd.items()}
    sa_, sb_ = LO.merge(dsd, oa), LO.merge(dsd, ob)
    with torch.no_grad():
        unet = lambda s: lambda x, t, c: O.unet_forward(s, cfgs[0], x, t, c)  # noqa: E731
        c1, u1 = O.clip_text_encode(sa_, cfgs[2], tok.cuda()), O.clip_text_encode(sa_, cfgs[2], neg.cuda())
        x = O.sample_ddim(unet(sa_), E.per_image_noise(31, b, (4, hw, hw))[0].cuda(), c1, u1, steps, 7.0)
        up = F.interpolate(x, size=(2 * hw, 2 * hw), mode="bilinear", antialias=False)
        c2, u2 = O.clip_text_encode(sb_, cfgs[2], tok.cuda()), O.clip_text_encode(sb_, cfgs[2], neg.cuda())
        sa, s1a, rows = O.ddim_img2img_coefficients(steps, 0.6)
        x = up * sa + E.per_image_noise(31, b, (4, 2 * hw, 2 * hw))[0].cuda() * s1a
        for (t, c_sa, c_s1a, c_sap, c_s1ap) in rows:
            e = O.cfg_eps(unet(sb_), x, t, c2, u2, 7.0)
            x = c_sap * ((x - c_s1a * e) / c_sa) + c_s1ap * e
        ref = O.to_uint8(O.vae_decode(sb_, cfgs[1], x / cfgs[1].scale_factor))
    _u8_check("tiny hires lora A -> B", got, ref)


@pytest.mark.parametrize("feature", ["controlnet", "tome", "tiling"])
def test_lora_with_other_features_graphs_on_equal_off(feature):
    from b200sd import factory
    eng, _, cfgs = _engine("tiny")
    eng_ng, _, _ = _engine("tiny", graphs=False)
    a, _ = _nets(cfgs, TWO)
    tok, neg = _tok(2)
    hw = 16

    def run(e):
        kw = {}
        if feature == "controlnet":
            cw = factory.controlnet("lora-test-cn", size="tiny", device="cuda:0", dtype=torch.float16)
            hint = torch.randint(0, 256, (hw * 8, hw * 8, 3), generator=torch.Generator().manual_seed(2), dtype=torch.uint8)
            kw["controls"] = [(cw, hint, 0.8, 0.0, 1.0)]
        elif feature == "tome":
            kw["token_merging_ratio"] = 0.5
        else:
            kw["tiling"] = True
        return e.txt2img(tok, neg, seed=3, steps=5, height=hw * 8, width=hw * 8, sampler="DDIM", loras=a, **kw).cpu()

    assert torch.equal(run(eng), run(eng_ng))


def test_a_request_without_tags_allocates_nothing():
    from b200sd import config as C, engine as E, synth
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
    tok, neg = _tok(2)
    eng.txt2img(tok, neg, seed=1, steps=4, height=128, width=128, sampler="DDIM")
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    eng.txt2img(tok, neg, seed=1, steps=4, height=128, width=128, sampler="DDIM")
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before and not eng._pristine
