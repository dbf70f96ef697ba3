"""v-prediction models and the SD 2.x family on the CPU: the v-oracle against diffusion theory, the engine's stage machine
and fused steps (b200sd.ops emulated: tests/ops_emulator.py plus the `_v` fused steps below) against the v-oracle on the
reduced-width SD 2.x model, the OpenCLIP ViT-H tower against transformers, tokenisation with pad id 0, parameter totals and
the factory's family / prediction selection."""
import math

import pytest
import torch

import ops_emulator

ALL = ["DDIM", "Euler", "Euler a", "LMS", "Heun", "DPM2", "DPM2 a", "DPM++ 2S a", "DPM++ 2M", "DPM++ SDE", "DPM fast",
       "DPM adaptive", "LMS Karras", "DPM2 Karras", "DPM2 a Karras", "DPM++ 2S a Karras", "DPM++ 2M Karras",
       "DPM++ SDE Karras", "PLMS"]


# ------------------------------------------------------------------------------------------------ emulated _v steps
def _cfg(v, b, cfg_scale):
    vc, vu = v[:b, :, :4].float(), v[b:, :, :4].float()
    return vu + cfg_scale * (vc - vu)


def cfg_ddim_step_v(v, x, xin, cfg_scale, coef, step_counter):
    """b200sd_cfg_ddim_step_v: eps = sqrt(1 - a_t) x + sqrt(a_t) v with the pre-update x, then the DDIM update"""
    b, s = x.shape[0], int(step_counter.item())
    sa, s1a, sap, s1ap = (float(c) for c in coef[s])
    e = s1a * x + sa * _cfg(v, b, cfg_scale)
    x.copy_(sap * ((x - s1a * e) / sa) + s1ap * e)
    ops_emulator.pack_unet_input(x, xin, 1.0)
    step_counter += 1


def cfg_euler_a_step_v(v, x, noise, xin, cfg_scale, coef8, step_counter):
    """b200sd_cfg_euler_a_step_v: rows {sigma, sigma_down, sigma_up, in_next, kx, kv, 0, 0}"""
    b, s = x.shape[0], int(step_counter.item())
    sigma, sdown, sup, in_next, kx, kv = (float(c) for c in coef8[s][:6])
    e = kx * x + kv * _cfg(v, b, cfg_scale)
    xn = x + e * (sdown - sigma)
    if noise is not None and sup > 0:
        xn = xn + noise[s] * sup
    x.copy_(xn)
    ops_emulator.pack_unet_input(x, xin, in_next)
    step_counter += 1


def cfg_dpmpp_2m_step_v(v, x, old_denoised, xin, cfg_scale, coef8, step_counter):
    """b200sd_cfg_dpmpp_2m_step_v: kx, kv in columns 5, 6"""
    b, s = x.shape[0], int(step_counter.item())
    sigma, a, c1, c2, in_next, kx, kv = (float(c) for c in coef8[s][:7])
    e = kx * x + kv * _cfg(v, b, cfg_scale)
    dn = x - sigma * e
    dd = c1 * dn - c2 * old_denoised if c2 != 0 else dn
    x.copy_(a * x + (1.0 - a) * dd)
    old_denoised.copy_(dn)
    ops_emulator.pack_unet_input(x, xin, in_next)
    step_counter += 1


def _install(monkeypatch):
    from b200sd import engine as E, ops
    ops_emulator.install(monkeypatch, ops)
    for fn in (cfg_ddim_step_v, cfg_euler_a_step_v, cfg_dpmpp_2m_step_v):
        monkeypatch.setattr(ops, fn.__name__, fn)
    monkeypatch.setattr(E.SDEngine, "_require_cuda", False)


@pytest.fixture()
def env(monkeypatch):
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O, v_oracle as V
    _install(monkeypatch)
    cfgs = (C.TINY21_UNET, C.TINY21_VAE, C.TINY21_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2, prediction="v")
    b = 2
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    cond, unc = V.sd21_text_encode(sd, cfgs[2], tok), V.sd21_text_encode(sd, cfgs[2], neg)
    unet = V.cfg_unet(sd, V.TINY21_UNET)
    return E, V, eng, cond, unc, unet, b


# ------------------------------------------------------------------------------------------------ the v-oracle vs theory
# Gaussian data N(0, s^2): the optimal v is sqrt(a) sqrt(1 - a) (1 - s^2) x_t / (a s^2 + 1 - a) (a = alphas_cumprod at t).
# Converted by the v-oracle it must give exactly the optimal eps of tests/test_oracle_pins_cpu.py, so the samplers reach the
# same errors with the same orders; the stochastic samplers end on variance s^2.
_S_DATA = 0.8


def _alpha(t):
    from oracle import sd_oracle as O
    _, log_sig = O.model_sigmas()
    tt = t.double().clamp(0, 999)
    lo = tt.floor().long().clamp(max=998)
    w = tt - lo
    sg = ((1 - w) * log_sig[lo] + w * log_sig[lo + 1]).exp()
    return 1 / (1 + sg * sg)


def _gaussian_v_model(x, t, ctx):
    a, s2 = _alpha(t), _S_DATA ** 2
    k = (torch.sqrt(a) * torch.sqrt(1 - a) * (1 - s2) / (a * s2 + 1 - a)).float()
    return x * k[:, None, None, None]


def _gaussian_eps_model(x, t, ctx):
    a, s2 = _alpha(t), _S_DATA ** 2
    return x * (torch.sqrt(1 - a) / (a * s2 + 1 - a)).float()[:, None, None, None]


def _flow_errors(name, steps, noise0):
    from oracle import sd_oracle as O, v_oracle as V
    c = torch.zeros(noise0.shape[0], 1, 1)
    xv = V.run_sampler(name, _gaussian_v_model, c, c, 1.0, steps, noise0, None)
    xe = (O.sample_ddim(_gaussian_eps_model, noise0, c, c, steps, 1.0) if name == "DDIM" else
          O.run_sampler(name, _gaussian_eps_model, c, c, 1.0, steps, noise0, None))
    s = _S_DATA
    if name in ("DDIM", "PLMS"):
        ac, ts = O.alphas_cumprod().double(), O.ddim_timesteps(steps)
        a_T, a_0 = float(ac[ts[-1]]), float(ac[ts[0]] if name == "DDIM" else ac[0])
        exact = noise0 * math.sqrt((a_0 * s * s + 1 - a_0) / (a_T * s * s + 1 - a_T))
    else:
        karras = name.endswith("Karras") or name == "DPM++ 2M"
        s0 = float((O.sigmas_karras(steps) if karras else O.karras_sigmas_compvis(steps))[0][0])
        exact = noise0 * s0 * s / math.sqrt(s * s + s0 * s0)
    return float((xv - exact).norm() / exact.norm()), float((xe - exact).norm() / exact.norm())


@pytest.mark.parametrize("name,err40,order", [
    ("DDIM", 0.05, 0.75), ("Euler", 0.06, 1), ("Heun", 0.003, 2), ("DPM2", 0.012, 2), ("DPM2 Karras", 0.003, 2),
    ("DPM++ 2M", 0.006, 2), ("DPM++ 2M Karras", 0.006, 2), ("LMS", 5e-4, 3), ("LMS Karras", 2e-3, 3), ("PLMS", 0.008, 1.2)])
def test_v_oracle_solves_the_probability_flow_ode_as_the_eps_model_does(name, err40, order):
    noise0 = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(0))
    (v20, e20), (v40, e40) = _flow_errors(name, 20, noise0), _flow_errors(name, 40, noise0)
    for v, e in ((v20, e20), (v40, e40)):
        assert abs(v - e) <= 1e-4 * e + 1e-6, (name, v, e)
    assert v40 <= err40 and v20 / v40 >= 0.8 * 2 ** order, (name, v20, v40)


@pytest.mark.parametrize("name", ["DPM fast", "DPM adaptive"])
def test_v_oracle_dpm_solvers_match_the_eps_model(name):
    noise0 = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(0))
    v, e = _flow_errors(name, 20, noise0)
    # DPM adaptive's accept / reject decisions on an fp32 error norm amplify rounding: 0.2 % here
    rel = 1e-4 if name == "DPM fast" else 1e-2
    assert abs(v - e) <= rel * e + 1e-6 and v <= (0.01 if name == "DPM fast" else 0.05), (name, v, e)


@pytest.mark.parametrize("name,lo,hi", [("Euler a", 0.80, 1.02), ("DPM2 a", 0.93, 1.10), ("DPM++ 2S a", 0.92, 1.06),
                                        ("DPM++ SDE", 0.90, 1.06)])
def test_v_oracle_stochastic_samplers_end_on_the_data_distribution(name, lo, hi):
    from oracle import v_oracle as V
    g = torch.Generator().manual_seed(1)
    shape = (4, 4, 32, 32)
    noise0 = torch.randn(shape, generator=g)
    draws = [torch.randn(shape, generator=g) for _ in range(160)]
    c = torch.zeros(shape[0], 1, 1)
    x = V.run_sampler(name, _gaussian_v_model, c, c, 1.0, 40, noise0, draws)
    ratio = float(x.var()) / _S_DATA ** 2
    assert lo <= ratio <= hi and abs(float(x.mean())) <= 0.03, (name, ratio, float(x.mean()))


# ------------------------------------------------------------------------------------------------ engine vs v-oracle
def _close(z, ref, name):
    assert float((z - ref).abs().max()) <= 2e-3 * float(ref.abs().max()), name


@pytest.mark.parametrize("name", ALL)
def test_txt2img_v_sampler_matches_v_oracle(env, name):
    E, V, eng, cond, unc, unet, b = env
    hw, steps = 8, 7
    pr = eng.program(name, None, steps)
    nz = E.per_image_noise(4100, b, (4, hw, hw), 1 + pr.draws)
    with torch.no_grad():
        ref = V.run_sampler(name, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]))
    lat = eng.run_program(cond, unc, pr.start(nz[0]), pr, 7.0, noises=nz[1:] if pr.draws else None)
    _close(lat.reshape(b, hw, hw, 4).permute(0, 3, 1, 2), ref, name)


@pytest.mark.parametrize("name", ["DDIM", "Euler a", "DPM++ 2M Karras", "Heun", "DPM2 a Karras", "DPM++ SDE", "LMS",
                                  "DPM fast", "PLMS", "DPM adaptive"])
def test_img2img_half_v_matches_v_oracle(env, name):
    E, V, eng, cond, unc, unet, b = env
    hw, steps, d = 8, 9, 0.6
    init = torch.randn((b, 4, hw, hw), generator=torch.Generator().manual_seed(5)) * 0.7
    pr = eng.program(name, None, steps, denoise=d)
    nz = E.per_image_noise(4200, b, (4, hw, hw), 1 + pr.draws)
    with torch.no_grad():
        ref = V.run_sampler(name, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d)
    lat = eng.run_program(cond, unc, pr.start(nz[0], init), pr, 7.0, noises=nz[1:] if pr.draws else None)
    _close(lat.reshape(b, hw, hw, 4).permute(0, 3, 1, 2), ref, name)


@pytest.mark.parametrize("name", ["DDIM", "Euler a", "DPM++ 2M Karras", "Heun", "PLMS", "DPM++ SDE"])
def test_masked_v_sampling_matches_v_oracle(env, name):
    E, V, eng, cond, unc, unet, b = env
    hw, steps, d = 8, 8, 0.75
    g = torch.Generator().manual_seed(6)
    init = torch.randn((b, 4, hw, hw), generator=g) * 0.7
    nmask = (torch.rand((hw, hw), generator=g) > 0.5).float()
    pr = eng.program(name, None, steps, denoise=d, masked=True)
    nz = E.per_image_noise(4300, b, (4, hw, hw), 1 + pr.draws)
    m = nmask[None, None]
    with torch.no_grad():
        ref = V.run_sampler(name, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d,
                            mask=(init, m))
        ref = ref * m + init * (1 - m)
    lat = eng.run_program(cond, unc, pr.start(nz[0], init), pr, 7.0, noises=nz[1:] if pr.draws else None,
                          inpaint=(init, nmask.reshape(-1)))
    z = lat.reshape(b, hw, hw, 4).permute(0, 3, 1, 2)
    _close(z, ref, name)
    keep = (nmask == 0)[None, None].expand_as(z)
    assert torch.equal(z[keep], init[keep])


def test_v_fused_kernels_equal_their_generic_twins(env):
    """Euler / Euler a / DPM++ 2M on a v model: the fused _v step and the stage list (with its v lincomb) agree"""
    E, V, eng, cond, unc, unet, b = env
    hw, steps = 8, 6
    for name in ("Euler", "Euler a", "DPM++ 2M"):
        fused, twin = eng.program(name, None, steps), eng.program(name, None, steps, masked=True)
        assert fused.fused is not None and len(fused.rows[0]) == 8 and twin.sp is not None
        nz = E.per_image_noise(4400, b, (4, hw, hw), 1 + fused.draws)
        a = eng.run_program(cond, unc, fused.start(nz[0]), fused, 7.0, noises=nz[1:] if fused.draws else None).clone()
        c = eng.run_program(cond, unc, twin.start(nz[0]), twin, 7.0, noises=nz[1:] if twin.draws else None)
        assert float((a - c).abs().max()) <= 1e-4 * float(a.abs().max()), name


def test_v_rows_carry_the_conversion_coefficients():
    from b200sd import engine as E, samplers as S
    st = S.Stage(S.EULER, 500.0, [1.0, -1.0, 0.5], "x", 2.0)
    r = st.row()
    assert r[S.V_COL:S.V_COL + 2] == pytest.approx([2.0 / 5.0, 1 / math.sqrt(5.0)])
    st = S.Stage(S.EULER, 500.0, [1.0, -1.0, 0.5], "x", 0.0, alpha=0.36)
    assert st.row()[S.V_COL:S.V_COL + 2] == pytest.approx([0.8, 0.6])
    rows = E.v_rows("euler_a", [[2.0, 1.0, 0.5, 0.3]])
    assert rows[0] == pytest.approx([2.0, 1.0, 0.5, 0.3, 0.4, 1 / math.sqrt(5.0), 0.0, 0.0])
    rows = E.v_rows("dpmpp_2m", [[2.0, 0.5, 1.0, 0.0, 0.3, 0.0, 0.0, 0.0]])
    assert rows[0] == pytest.approx([2.0, 0.5, 1.0, 0.0, 0.3, 0.4, 1 / math.sqrt(5.0), 0.0])


def test_prediction_must_be_eps_or_v(monkeypatch):
    from b200sd import config as C, engine as E
    monkeypatch.setattr(E.SDEngine, "_require_cuda", False)
    with pytest.raises(ValueError):
        E.SDEngine({}, C.TINY21_UNET, C.TINY21_VAE, C.TINY21_CLIP, device="cpu", prediction="x0")


def test_engine_text_tower_equals_the_v_oracle(env):
    from b200sd import config as C, synth
    from oracle import v_oracle as V, sd_oracle as O
    E, _, eng, _, _, _, b = env
    sd = synth.make_state_dict(C.TINY21_UNET, C.TINY21_VAE, C.TINY21_CLIP, seed=0)
    tok = O.random_prompt_tokens(3, seed=9, vocab_hi=997)
    tok2 = torch.cat([tok, O.random_prompt_tokens(3, seed=10, vocab_hi=997)], dim=1)
    mult = torch.ones_like(tok2, dtype=torch.float32)
    mult[:, 5:9] = 1.3
    with torch.no_grad():
        got = eng.encode_prompts(tok2, multipliers=mult)
        ref = V.encode_sd21(sd, C.TINY21_CLIP, tok2, mult)
    assert got.shape == (3, 154, 64)
    assert float((got - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


# ------------------------------------------------------------------------------------------------ SD 2.x text tower pin
def test_sd21_open_clip_tower_matches_transformers():
    """ldm FrozenOpenCLIPEmbedder(layer="penultimate") is transformers.CLIPTextModel(hidden_act="gelu")'s
    hidden_states[-2] through final_layer_norm, under the open_clip -> HF key mapping of the SDXL pin; the product's tower
    (clip_text.OpenClipText.encode) equals the oracle's"""
    transformers = pytest.importorskip("transformers")
    from b200sd import clip_text, config as C
    from oracle import sd_oracle as O, v_oracle as V
    vocab, width, layers, heads = 1500, 96, 4, 4
    hcfg = transformers.CLIPTextConfig(vocab_size=vocab + 3, hidden_size=width, intermediate_size=4 * width,
                                       num_hidden_layers=layers, num_attention_heads=heads, max_position_embeddings=77,
                                       hidden_act="gelu", layer_norm_eps=1e-5, eos_token_id=vocab + 2,
                                       bos_token_id=vocab + 1, pad_token_id=0)
    torch.manual_seed(15)
    model = transformers.CLIPTextModel(hcfg).eval().float()
    with torch.no_grad():
        for p in model.parameters():
            p.add_(0.05 * torch.randn_like(p))
    hf = {k: v.detach().clone() for k, v in model.state_dict().items()}
    p = C.OPENCLIP_PREFIX
    sd = {p + "token_embedding.weight": hf["text_model.embeddings.token_embedding.weight"],
          p + "positional_embedding": hf["text_model.embeddings.position_embedding.weight"],
          p + "ln_final.weight": hf["text_model.final_layer_norm.weight"],
          p + "ln_final.bias": hf["text_model.final_layer_norm.bias"],
          p + "text_projection": torch.eye(width)}
    for i in range(layers):
        h, o = f"text_model.encoder.layers.{i}.", f"{p}transformer.resblocks.{i}."
        sd[o + "attn.in_proj_weight"] = torch.cat([hf[h + f"self_attn.{n}_proj.weight"] for n in "qkv"])
        sd[o + "attn.in_proj_bias"] = torch.cat([hf[h + f"self_attn.{n}_proj.bias"] for n in "qkv"])
        for a, b_ in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                      ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            sd[o + a + ".weight"], sd[o + a + ".bias"] = hf[h + b_ + ".weight"], hf[h + b_ + ".bias"]
    tokens = O.random_prompt_tokens(3, seed=16, vocab_hi=vocab)
    tokens[:, 40:] = 0   # SD 2.x padding after the EOS
    cfg = C.CLIPConfig(vocab=vocab + 3, width=width, layers=layers, heads=heads, open_clip=True, pad_id=0)
    with torch.no_grad():
        hs = model(input_ids=tokens, output_hidden_states=True).hidden_states[-2]
        want = model.text_model.final_layer_norm(hs)
        ref = V.sd21_text_encode(sd, cfg, tokens)
        got = clip_text.OpenClipText(sd, cfg, "cpu", torch.float32, p).encode(tokens)
    tol = 2e-5 * max(1.0, float(want.abs().max()))
    assert float((ref - want).abs().max()) <= tol
    assert float((got - ref).abs().max()) <= tol


# ------------------------------------------------------------------------------------------------ tokenisation
def test_pad_zero_after_the_first_eos_of_every_chunk():
    from b200sd import factory
    vocab = 1000
    bos, eos = vocab - 2, vocab - 1
    words = " ".join(f"w{i}" for i in range(100))
    ids, mult = factory.tokenize_prompts([f"a (b:1.3) c BREAK {words}", "x"], vocab, pad=0)
    assert ids.shape == (2, 77 * 3)
    for row in ids.tolist():
        for j in range(3):
            ch = row[77 * j:77 * (j + 1)]
            assert ch[0] == bos
            k = ch.index(eos)
            assert all(t == 0 for t in ch[k + 1:]) and eos not in ch[k + 1:]
    assert ids[0, :5].tolist() == [bos, *ids[0, 1:4].tolist(), eos] and ids[0, 5] == 0
    assert float(mult[0, 2]) == pytest.approx(1.3)
    # the empty padding chunks of the shorter prompt: [BOS, EOS, 0, ...]
    assert ids[1, 77:79].tolist() == [bos, eos] and bool((ids[1, 79:154] == 0).all())
    # without a pad id nothing changes: EOS padding, as before
    ids_eos, mult_eos = factory.tokenize_prompts([f"a (b:1.3) c BREAK {words}", "x"], vocab)
    assert torch.equal(mult_eos, mult)
    assert torch.equal(torch.where(ids == 0, torch.full_like(ids, eos), ids), ids_eos)
    plain = factory.synthetic_tokens(["one two three"], vocab, pad=0)
    assert plain[0, :5].tolist()[4] == eos and bool((plain[0, 5:] == 0).all())
    assert torch.equal(factory.tokenize_prompts(["one two three"], vocab, pad=0)[0], plain)


# ------------------------------------------------------------------------------------------------ known answers
def test_sd21_parameter_totals():
    """SD 2.x UNet 865 910 724 and kl-f8 VAE 83 653 863 parameters (shapes only, no storage); real key names"""
    from unittest import mock
    from b200sd import config as C, synth

    def meta_randn(*shape, **kw):
        shape = shape[0] if len(shape) == 1 and not isinstance(shape[0], int) else shape
        return torch.empty(tuple(shape), device="meta")
    with mock.patch.object(torch, "randn", meta_randn):
        sd = synth.make_state_dict(C.SD21_UNET, C.SD21_VAE, C.SD21_CLIP, seed=0)
    count = lambda pre: sum(v.numel() for k, v in sd.items() if k.startswith(pre))  # noqa: E731
    assert count(C.UNET_PREFIX) == 865_910_724
    assert count(C.VAE_PREFIX) == 83_653_863
    assert "cond_stage_model.model.transformer.resblocks.23.attn.in_proj_weight" in sd
    assert tuple(sd["cond_stage_model.model.token_embedding.weight"].shape) == (49408, 1024)
    assert "model.diffusion_model.input_blocks.1.1.proj_in.weight" in sd
    assert tuple(sd["model.diffusion_model.input_blocks.1.1.proj_in.weight"].shape) == (320, 320)
    assert tuple(sd["model.diffusion_model.input_blocks.1.1.transformer_blocks.0.attn2.to_k.weight"].shape) == (320, 1024)


# ------------------------------------------------------------------------------------------------ factory
def test_factory_families_and_prediction(monkeypatch):
    from b200sd import config as C, factory
    monkeypatch.delenv("B200SD_PREDICTION", raising=False)
    assert factory.configs("sd21") == (C.SD21_UNET, C.SD21_VAE, C.SD21_CLIP)
    assert factory.configs("tiny21") == (C.TINY21_UNET, C.TINY21_VAE, C.TINY21_CLIP)
    assert [factory.prediction(f) for f in ("sd15", "sdxl", "tiny", "tinyxl", "sd21", "tiny21")] == \
        ["eps", "eps", "eps", "eps", "v", "v"]
    monkeypatch.setenv("B200SD_PREDICTION", "eps")
    assert factory.prediction("sd21") == "eps"
    monkeypatch.setenv("B200SD_PREDICTION", "v")
    assert factory.prediction("sd15") == "v"
    monkeypatch.setenv("B200SD_PREDICTION", "x0")
    with pytest.raises(ValueError):
        factory.prediction("sd21")
    assert C.SD21_CLIP.pad_id == 0 and C.SD15_CLIP.pad_id is None and C.SD21_VAE.scale_factor == 0.18215


def test_sd_ckpt_is_honoured_for_sd21_only(monkeypatch, tmp_path):
    from b200sd import factory
    loaded = []
    monkeypatch.setattr(factory, "_load_safetensors", lambda p: loaded.append(p) or {"k": torch.zeros(1)})
    monkeypatch.setattr(factory, "make_state_dict", lambda *a, **k: {"synthetic": torch.zeros(1)})
    monkeypatch.setattr(factory, "_STATE", {})
    ckpt = str(tmp_path / "v2-1_768-ema-pruned.safetensors")
    monkeypatch.setenv("SD_CKPT", ckpt)
    assert "k" in factory.state_dict("sd21")
    assert "synthetic" in factory.state_dict("sdxl") and "synthetic" in factory.state_dict("tiny21")
    assert loaded == [ckpt]
    assert factory.model_identity("sd21") == "v2-1_768-ema-pruned.safetensors"
    assert factory.model_identity("sdxl") == "synthetic-sdxl-seed0"
