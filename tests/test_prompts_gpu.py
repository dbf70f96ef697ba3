"""Prompts with sdwui syntax on the GPU: b200sd_attention_varlen, one UNet evaluation of [cond 154 | uncond 77], whole
multi-chunk weighted requests against the chunked fp32 oracle (oracle/prompt_oracle.py: separate cond / uncond UNet calls
when their lengths differ, as sdwui's default), plan growth under CUDA graphs, and the LocalGPUWorker payload path.
Image tolerances are those of test_engine_gpu.py (fp16) and test_sdxl_gpu.py (bf16)."""
import json
import logging
import os

import pytest
import torch

from kutil import OUT_DIR, assert_close

pytestmark = pytest.mark.gpu
U8_MEAN, U8_WITHIN2 = 1.5, 0.97
U8_MEAN_BF16, U8_WITHIN4_BF16 = 2.0, 0.95


def _record(name, **kw):
    os.makedirs(OUT_DIR, exist_ok=True)
    with open(os.path.join(OUT_DIR, "prompt_parity.jsonl"), "a") as f:
        f.write(json.dumps(dict(name=name, **kw)) + "\n")


# ----------------------------------------------------------------------------------------------- kernel
LENS = [1, 63, 64, 65, 77, 128, 154, 231, 520]


def _own(t):
    """a packed copy: [B, S, C] with batch pitch S * C even when S == 1 (.contiguous() keeps a size-1 slice's strides)"""
    return torch.empty(t.shape, device=t.device, dtype=t.dtype).copy_(t)


def _heads(b, s, heads, d, dp, g, dtype, ones):
    t = torch.zeros((b, s, heads, dp), device="cuda", dtype=dtype)
    t[..., :d] = torch.randn((b, s, heads, d), generator=g, device="cuda").to(dtype)
    if ones:
        t[..., d] = 1.0
    return t.reshape(b, s, heads * dp)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("d,dp", [(40, 48), (80, 96), (160, 176), (64, 64)])
def test_attention_varlen(d, dp, dtype):
    """row b attends to its first kv_len[b] keys of a 520-row buffer (1 .. 9 kv tiles, so the 3-slot ring wraps); the rest
    of the buffer holds finite garbage.  Against fp32 per row, and bitwise against a plain call on the sliced keys."""
    from b200sd import ops
    g = torch.Generator(device="cuda").manual_seed(d + dp)
    b, heads, sq, skv = len(LENS), 2, 200, 520
    ones = dp > d
    q = _heads(b, sq, heads, d, dp, g, dtype, False)
    k = _heads(b, skv, heads, d, dp, g, dtype, False)
    v = _heads(b, skv, heads, d, dp, g, dtype, ones)
    lens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    out = torch.full((b, sq, heads * d), float("nan"), device="cuda", dtype=dtype)
    ops.attention(q, k, v, out, heads, d, dp, d ** -0.5, ones, kv_len=lens)
    torch.cuda.synchronize()
    tol = (4e-3, 1e-2) if dtype == torch.float16 else (2e-2, 2e-2)
    for i, n in enumerate(LENS):
        qi, ki, vi = q[i:i + 1], _own(k[i:i + 1, :n]), _own(v[i:i + 1, :n])
        qh, kh, vh = (t.float().reshape(1, -1, heads, dp)[..., :d].permute(0, 2, 1, 3) for t in (qi, ki, vi))
        ref = (torch.softmax(qh @ kh.transpose(-1, -2) * d ** -0.5, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(1, sq, -1)
        assert_close(f"attention_varlen d{d}/{dp} {dtype} len{n}", out[i:i + 1], ref, *tol)
        plain = torch.full_like(out[i:i + 1], float("nan"))
        ops.attention(qi, ki, vi, plain, heads, d, dp, d ** -0.5, ones)
        torch.cuda.synchronize()
        assert torch.equal(out[i:i + 1], plain), (d, dp, dtype, n)


def test_attention_varlen_clamps_lengths():
    from b200sd import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    heads, d, dp, sq, skv = 2, 40, 48, 64, 154
    q = _heads(2, sq, heads, d, dp, g, torch.float16, False)
    k = _heads(2, skv, heads, d, dp, g, torch.float16, False)
    v = _heads(2, skv, heads, d, dp, g, torch.float16, True)
    out = torch.empty((2, sq, heads * d), device="cuda", dtype=torch.float16)
    ops.attention(q, k, v, out, heads, d, dp, 0.2, True, kv_len=torch.tensor([0, 10 ** 6], dtype=torch.int32, device="cuda"))
    for i, n in enumerate((1, skv)):
        plain = torch.empty_like(out[:1])
        ops.attention(q[i:i + 1], _own(k[i:i + 1, :n]), _own(v[i:i + 1, :n]), plain, heads, d, dp, 0.2, True)
        torch.cuda.synchronize()
        assert torch.equal(out[i:i + 1], plain)


# ----------------------------------------------------------------------------------------------- setup
_CACHE = {}


def _setup(size, graphs=False):
    key = (size, graphs)
    if key not in _CACHE:
        _CACHE.clear()
        torch.cuda.empty_cache()
        from b200sd import config as C, engine as E, synth
        from oracle import prompt_oracle as P, sd_oracle as O
        cfgs = {"tiny": (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP), "sd15": (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP),
                "tinyxl": (C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP)}[size]
        sd = synth.make_state_dict(*cfgs, seed=0)
        dtype = torch.bfloat16 if size == "tinyxl" else torch.float16
        eng = E.SDEngine(sd, *cfgs, device="cuda:0", dtype=dtype, use_graphs=graphs)
        _CACHE[key] = (E, O, P, cfgs, sd, {k: v.cuda() for k, v in sd.items()}, eng)
    return _CACHE[key]


def _tokens(vocab, chunks, b=2, neg="(ugly:1.2), [blurry]"):
    """a weighted prompt of `chunks` 77-token chunks (hashed tokeniser) and a 1-chunk weighted negative"""
    from b200sd import factory
    words = {1: 40, 2: 100, 3: 160}[chunks]
    text = "a (red:1.3) house, " + " ".join(f"w{i}" for i in range(words)) + ", [blue] ((sky))"
    ids, mult = factory.tokenize_prompts([text] * b, vocab)
    nids, nmult = factory.tokenize_prompts([neg] * b, vocab)
    assert ids.shape[1] == 77 * chunks and nids.shape[1] == 77
    return ids, mult, nids, nmult


def _u8_check(name, got, ref_u8, bf16=False):
    du8 = (got.cpu().int() - ref_u8.cpu().int()).abs().float()
    rec = dict(u8_mean=float(du8.mean()), u8_max=float(du8.max()), u8_exact=float((du8 == 0).float().mean()),
               u8_within2=float((du8 <= 2).float().mean()), u8_within4=float((du8 <= 4).float().mean()))
    _record(name, **rec)
    assert got.shape == ref_u8.shape
    if bf16:
        assert rec["u8_mean"] <= U8_MEAN_BF16 and rec["u8_within4"] >= U8_WITHIN4_BF16, rec
    else:
        assert rec["u8_mean"] <= U8_MEAN and rec["u8_within2"] >= U8_WITHIN2, rec


# ----------------------------------------------------------------------------------------------- one UNet evaluation
@pytest.mark.parametrize("size,hw", [("tiny", 16), ("sd15", 32)])
def test_unet_eval_cond154_uncond77(size, hw):
    """[cond 154 | uncond 77] in one evaluation == cond alone at 154 and uncond alone at 77 (torch.equal), and within
    test_engine_gpu.py's UNet tolerances of the oracle's separate fp32 calls"""
    from b200sd.unet_exec import UNetProgram
    E, O, P, cfgs, sd, dsd, eng = _setup(size)
    b = 2
    ids, mult, nids, nmult = _tokens(cfgs[2].vocab, 2, b)
    cond = P.encode_sd1(dsd, cfgs[2], ids.cuda(), mult.cuda())
    unc = P.encode_sd1(dsd, cfgs[2], nids.cuda(), nmult.cuda())
    x = O.per_image_noise(1000, b, (4, hw, hw)).cuda()
    t = torch.full((2 * b,), 651.0, device="cuda")
    c, u, lc, lu = P.pad_pair(cond, unc)
    with torch.no_grad():
        ref = P.cfg_unet(dsd, cfgs[0], lc, lu)(torch.cat([x, x]), t, torch.cat([c, u]))
    table = eng.temb.table(torch.tensor([651.0]))

    def run(prog, setup):
        setup()
        prog.cur_bias.copy_(table[0])
        xin = x.permute(0, 2, 3, 1).reshape(b, hw * hw, 4)
        for r in range(prog.n // b):
            prog.xin[r * b:(r + 1) * b, :, :4] = xin.half()
        prog.run()
        torch.cuda.synchronize()
        return prog.eps[..., :4].clone()

    plan = eng.plan(b, hw, hw)
    fused = run(plan.unet, lambda: plan.set_context(cond.half(), unc.half()))
    assert plan.ctx_cap == 154 and plan.kv_len.tolist() == [154] * b + [77] * b
    alone_c = UNetProgram(eng.unet_w, b, hw, hw, 154)
    ec = run(alone_c, lambda: alone_c.set_context(cond.half().contiguous()))
    del alone_c
    alone_u = UNetProgram(eng.unet_w, b, hw, hw, 77)
    eu = run(alone_u, lambda: alone_u.set_context(unc.half().contiguous()))
    del alone_u
    assert torch.equal(fused[:b], ec) and torch.equal(fused[b:], eu)
    got = fused.float().reshape(2 * b, hw, hw, 4).permute(0, 3, 1, 2)
    d = (got - ref).abs()
    rel_max = float(d.max() / ref.abs().max())
    rel_rms = float(d.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
    _record(f"unet_eval cond154/uncond77 {size} hw{hw}", rel_max=rel_max, rel_rms=rel_rms)
    assert rel_max <= 3e-2 and rel_rms <= 5e-3, (rel_max, rel_rms)


# ----------------------------------------------------------------------------------------------- whole requests
@pytest.mark.parametrize("size,chunks,sampler", [
    ("tiny", 2, "DDIM"), ("tiny", 3, "Euler a"), ("tiny", 2, "DPM++ 2M"), ("tiny", 3, "Heun"),
    ("sd15", 2, "DDIM"), ("sd15", 3, "Euler a"),
])
def test_weighted_multichunk_txt2img(size, chunks, sampler):
    E, O, P, cfgs, sd, dsd, eng = _setup(size)
    b, hw, steps = 2, 16 if size == "tiny" else 32, 6
    ids, mult, nids, nmult = _tokens(cfgs[2].vocab, chunks, b)
    got = eng.txt2img(ids, nids, 90, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, sampler=sampler,
                      multipliers=mult, neg_multipliers=nmult)
    pr = eng.program(sampler, None, steps)
    nz = E.per_image_noise(90, b, (4, hw, hw), 1 + pr.draws).cuda()
    with torch.no_grad():
        cond = P.encode_sd1(dsd, cfgs[2], ids.cuda(), mult.cuda())
        unc = P.encode_sd1(dsd, cfgs[2], nids.cuda(), nmult.cuda())
        z = P.sample(dsd, cfgs[0], cond, unc, sampler, steps, 7.0, nz[0], list(nz[1:]))
        ref_u8 = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8_check(f"txt2img {size} {chunks} chunks {sampler}", got, ref_u8)


def test_weighted_img2img_and_hires_tiny():
    E, O, P, cfgs, sd, dsd, eng = _setup("tiny")
    b, hw, steps = 2, 16, 8
    ids, mult, nids, nmult = _tokens(cfgs[2].vocab, 2, b)
    with torch.no_grad():
        cond = P.encode_sd1(dsd, cfgs[2], ids.cuda(), mult.cuda())
        unc = P.encode_sd1(dsd, cfgs[2], nids.cuda(), nmult.cuda())
    # img2img
    g = torch.Generator().manual_seed(5)
    init_u8 = torch.randint(0, 256, (b, hw * 2, hw * 2, 3), generator=g, dtype=torch.uint8)
    got = eng.img2img(ids, nids, 91, init_u8, denoising_strength=0.6, steps=steps, cfg_scale=7.0, sampler="DDIM",
                      multipliers=mult, neg_multipliers=nmult)
    with torch.no_grad():
        init = O.vae_encode_mean(dsd, cfgs[1], O.image_to_model_input(init_u8.cuda())) * cfgs[1].scale_factor
        nz = E.per_image_noise(91, b, tuple(init.shape[1:]), 1).cuda()
        z = P.sample(dsd, cfgs[0], cond, unc, "DDIM", steps, 7.0, nz[0], init=init, denoising_strength=0.6)
        ref_u8 = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8_check("img2img tiny 2 chunks DDIM", got, ref_u8)
    # hires fix (DDIM, "Latent" upscaler)
    got = eng.txt2img_hires(ids, nids, 92, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, hr_scale=2.0,
                            denoising_strength=0.7, sampler="DDIM", multipliers=mult, neg_multipliers=nmult)
    with torch.no_grad():
        x = P.sample(dsd, cfgs[0], cond, unc, "DDIM", steps, 7.0, E.per_image_noise(92, b, (4, hw, hw))[0].cuda())
        up = torch.nn.functional.interpolate(x, size=(2 * hw, 2 * hw), mode="bilinear", antialias=False)
        nz = E.per_image_noise(92, b, (4, 2 * hw, 2 * hw))[0].cuda()
        z = P.sample(dsd, cfgs[0], cond, unc, "DDIM", steps, 7.0, nz, init=up, denoising_strength=0.7)
        ref_u8 = O.to_uint8(O.vae_decode(dsd, cfgs[1], z / cfgs[1].scale_factor))
    _u8_check("hires tiny 2 chunks DDIM", got, ref_u8)


def test_weighted_multichunk_sdxl_tiny():
    """tiny SDXL: emphasis per tower, pooled vector from the first chunk, an empty negative's zero embedding, hires fix"""
    E, O, P, cfgs, sd, dsd, eng = _setup("tinyxl")
    from oracle import sd_oracle
    ocfgs = (sd_oracle.TINYXL_UNET, sd_oracle.TINYXL_VAE, sd_oracle.TINYXL_CLIP)
    b, hw, steps = 2, 16, 6
    ids, mult, nids, nmult = _tokens(cfgs[2].vocab, 2, b, neg="")
    px = hw * 8
    got = eng.txt2img(ids, nids, 93, steps=steps, cfg_scale=7.0, height=px, width=px, sampler="Euler a",
                      multipliers=mult, neg_multipliers=nmult)
    nz = E.per_image_noise(93, b, (4, hw, hw), 1 + steps).cuda()
    with torch.no_grad():
        ctx_c, y_c = P.encode_sdxl(dsd, ocfgs[2], ids.cuda(), mult.cuda(), px, px)
        ctx_u, y_u = P.encode_sdxl(dsd, ocfgs[2], nids.cuda(), nmult.cuda(), px, px, zero_txt=True)
        z = P.sample(dsd, ocfgs[0], ctx_c, ctx_u, "Euler a", steps, 7.0, nz[0], list(nz[1:]), y=torch.cat([y_c, y_u]))
        ref_u8 = O.to_uint8(O.vae_decode(dsd, ocfgs[1], z / ocfgs[1].scale_factor))
    _u8_check("txt2img tinyxl 2 chunks Euler a", got, ref_u8, bf16=True)
    hr = eng.txt2img_hires(ids, nids, 93, steps=steps, cfg_scale=7.0, height=px, width=px, hr_scale=2.0,
                           denoising_strength=0.7, sampler="DDIM", multipliers=mult, neg_multipliers=nmult)
    assert hr.shape == (b, 2 * got.shape[1], 2 * got.shape[2], 3) and eng.plan(b, 2 * hw, 2 * hw).ctx_cap == 154


# ----------------------------------------------------------------------------------------------- invariants
def test_all_one_weights_and_batch_invariance():
    E, O, P, cfgs, sd, dsd, eng = _setup("tiny")
    ids, mult, nids, nmult = _tokens(cfgs[2].vocab, 2, 3)
    kw = dict(steps=5, cfg_scale=7.0, height=128, width=128, sampler="DDIM")
    plain = eng.txt2img(ids, nids, 40, **kw)
    ones = eng.txt2img(ids, nids, 40, multipliers=torch.ones(ids.shape), neg_multipliers=torch.ones(nids.shape), **kw)
    assert torch.equal(plain, ones)
    batch = eng.txt2img(ids, nids, 40, multipliers=mult, neg_multipliers=nmult, **kw)
    for k in range(3):
        alone = eng.txt2img(ids[k:k + 1], nids[k:k + 1], 40 + k, multipliers=mult[k:k + 1],
                            neg_multipliers=nmult[k:k + 1], **kw)
        assert torch.equal(batch[k:k + 1], alone), k


def test_plan_growth_under_graphs():
    """1-, 3- and 2-chunk requests alternating on one engine with CUDA graphs: each equals a fresh engine's result, the
    short request after growth equals the one before it, and the step graphs replay"""
    from b200sd import config as C, engine as E, synth
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
    kw = dict(steps=5, cfg_scale=7.0, height=128, width=128, sampler="Euler a")
    runs = []
    for chunks in (1, 3, 2, 1):
        ids, mult, nids, nmult = _tokens(cfgs[2].vocab, chunks)
        before = eng.graph_replayed_launches
        got = eng.txt2img(ids, nids, 50, multipliers=mult, neg_multipliers=nmult, **kw).clone()
        assert eng.graph_replayed_launches > before
        fresh = E.SDEngine(sd, *cfgs, device="cuda:0", use_graphs=True)
        want = fresh.txt2img(ids, nids, 50, multipliers=mult, neg_multipliers=nmult, **kw)
        del fresh
        assert torch.equal(got, want), chunks
        runs.append(got)
    assert eng.plan(2, 16, 16).ctx_cap == 231 and "vae" in eng.plan(2, 16, 16).graphs
    assert torch.equal(runs[0], runs[3])


def test_local_worker_payload_with_prompt_syntax():
    from b200sd import factory
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker
    E, O, P, cfgs, sd, dsd, eng = _setup("tiny", graphs=True)
    logging.getLogger("distributed").setLevel(logging.ERROR)
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    wk = LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0)
    prompt = "a (word:1.3) BREAK " + " ".join(f"w{i}" for i in range(80))
    payload = {"prompt": prompt, "negative_prompt": "[bad]", "seed": 30, "subseed": 4, "subseed_strength": 0,
               "batch_size": 2, "n_iter": 1, "steps": 5, "width": 128, "height": 128, "sampler_name": "DDIM",
               "cfg_scale": 7.0}
    wk.request(payload, None, False)
    ids, mult = factory.tokenize_prompts([prompt] * 2, cfgs[2].vocab)
    nids, nmult = factory.tokenize_prompts(["[bad]"] * 2, cfgs[2].vocab)
    assert ids.shape[1] == 231
    direct = eng.txt2img(ids, nids, 30, steps=5, cfg_scale=7.0, height=128, width=128, sampler="DDIM", multipliers=mult,
                         neg_multipliers=nmult)
    assert torch.equal(wk.response["tensors"], direct.cpu())
