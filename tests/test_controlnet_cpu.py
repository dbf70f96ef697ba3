"""ControlNet on the CPU: the oracle's pins, the engine's control segments (b200sd.ops emulated: tests/ops_emulator.py plus
the hint conversion below) against the ControlNet oracle on tiny and tiny21, the worker's unit parsing and refusals, the
dispatcher's packing of ControlNet script arguments, and the loader."""
import base64
from collections import OrderedDict
import io
import json

import numpy as np
import pytest
import torch

import ops_emulator
from test_vpred_cpu import cfg_ddim_step_v, cfg_dpmpp_2m_step_v, cfg_euler_a_step_v


def hint_to_nhwc(img_u8, out):
    """b200sd_hint_to_nhwc: channels 0..2 = x / 255, the rest of the row 0"""
    out.zero_()
    out[..., :3] = (img_u8.float() / 255.0).to(out.dtype)
    return out


def _install(monkeypatch):
    from b200sd import engine as E, ops
    ops_emulator.install(monkeypatch, ops)
    for fn in (hint_to_nhwc, cfg_ddim_step_v, cfg_euler_a_step_v, cfg_dpmpp_2m_step_v):
        monkeypatch.setattr(ops, fn.__name__, fn)
    monkeypatch.setattr(E.SDEngine, "_require_cuda", False)


def _hint(seed, hh, ww):
    return torch.randint(0, 256, (hh, ww, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


# ------------------------------------------------------------------------------------------------ oracle pins
@pytest.fixture(scope="module")
def tiny():
    from b200sd import config as C, synth
    sd = synth.make_state_dict(C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP, seed=0)
    csd = synth.make_controlnet_state_dict(C.TINY_UNET, seed=7)
    return C.TINY_UNET, sd, csd


def _inputs(cfg, b=2, hw=8):
    g = torch.Generator().manual_seed(3)
    x = torch.randn((b, 4, hw, hw), generator=g)
    ctx = torch.randn((b, 77, cfg.context_dim), generator=g)
    t = torch.tensor([500.0] * b)
    return x, t, ctx


def test_zero_convs_zero_give_the_plain_unet(tiny):
    from oracle import controlnet_oracle as CN, sd_oracle as O
    cfg, sd, csd = tiny
    z = {k: (torch.zeros_like(v) if ".zero_convs." in k or "middle_block_out" in k else v) for k, v in csd.items()}
    x, t, ctx = _inputs(cfg)
    hint = CN.hint_input(_hint(1, 64, 64)[None])
    with torch.no_grad():
        assert torch.equal(CN.unet_forward(sd, cfg, x, t, ctx, [(z, hint, 1.0)]), O.unet_forward(sd, cfg, x, t, ctx))


def test_unet_copy_with_zero_hint_gives_the_unet_skips(tiny):
    """a ControlNet whose encoder / middle block / time embedding are the UNet's, with the last hint conv zero: its features
    before the zero convs are the UNet's skip tensors hs and middle result (pins the block reuse and the key mapping)"""
    from oracle import controlnet_oracle as CN, sd_oracle as O
    cfg, sd, csd = tiny
    own = dict(csd)
    for k in csd:
        body = k[len("control_model."):]
        if not body.startswith(("input_hint_block", "zero_convs", "middle_block_out")):
            own[k] = sd["model.diffusion_model." + body]
    own["control_model.input_hint_block.14.weight"] = torch.zeros_like(own["control_model.input_hint_block.14.weight"])
    own["control_model.input_hint_block.14.bias"] = torch.zeros_like(own["control_model.input_hint_block.14.bias"])
    x, t, ctx = _inputs(cfg)
    with torch.no_grad():
        feats = CN.controlnet_forward(own, cfg, x, CN.hint_input(_hint(2, 64, 64)[None]), t, ctx, features=True)
        sdp = O._Prefixed(sd, "model.diffusion_model.")
        inputs, middle, _ = O.unet_layout(cfg)
        emb = CN._emb(sdp, cfg, t, x.dtype)
        hs, h = [], x
        for i, blk in enumerate(inputs):
            h = O._run_block(sdp, cfg, f"input_blocks.{i}", blk, h, emb, ctx)
            hs.append(h)
        hs.append(O._run_block(sdp, cfg, "middle_block", middle, h, emb, ctx))
    assert len(feats) == len(hs)
    for f, h in zip(feats, hs):
        assert torch.equal(f, h)


def test_output_is_linear_in_weight(tiny):
    """a unit of weight w adds w times the ControlNet's outputs: the same as weight 1 on zero convs scaled by w (which is
    how the engine applies it)"""
    from oracle import controlnet_oracle as CN
    cfg, sd, csd = tiny
    x, t, ctx = _inputs(cfg)
    hint = CN.hint_input(_hint(3, 64, 64)[None])
    scaled = {k: (0.6 * v if ".zero_convs." in k or "middle_block_out" in k else v) for k, v in csd.items()}
    with torch.no_grad():
        outs = CN.controlnet_forward(csd, cfg, x, hint, t, ctx)
        for a, b in zip(CN.controlnet_forward(scaled, cfg, x, hint, t, ctx), outs):
            assert torch.allclose(a, 0.6 * b, rtol=1e-4, atol=1e-5)
        a = CN.unet_forward(sd, cfg, x, t, ctx, [(csd, hint, 0.6)])
        b = CN.unet_forward(sd, cfg, x, t, ctx, [(scaled, hint, 1.0)])
    assert torch.allclose(a, b, rtol=1e-4, atol=1e-4)


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
    csds = [synth.make_controlnet_state_dict(cfgs[0], seed=s) for s in (11, 12)]
    cws = [ControlNetWeights(c, cfgs[0], "cpu", torch.float32, name=f"cn{k}") for k, c in enumerate(csds)]
    b = 2
    tok, neg = O.random_prompt_tokens(b, vocab_hi=997), O.empty_prompt_tokens(b, vocab_hi=997)
    if pred == "eps":
        cond, unc = O.clip_text_encode(sd, cfgs[2], tok), O.clip_text_encode(sd, cfgs[2], neg)
    else:
        cond, unc = V.sd21_text_encode(sd, cfgs[2], tok), V.sd21_text_encode(sd, cfgs[2], neg)
    return E, eng, sd, cfgs[0], csds, cws, cond, unc, b, pred


def _run(env, name, windows, units=(0,), hw=8, steps=6, d=None, masked=False):
    from oracle import controlnet_oracle as CN
    E, eng, sd, cfg, csds, cws, cond, unc, b, pred = env
    hints = [_hint(20 + k, 8 * hw, 8 * hw) for k in units]
    weights = [0.8, 0.6, 0.5]
    controls = [(cws[k], hints[j], weights[j], *windows[j]) for j, k in enumerate(units)]
    g = torch.Generator().manual_seed(5)
    init = torch.randn((b, 4, hw, hw), generator=g) * 0.7 if d is not None else None
    nmask = (torch.rand((hw, hw), generator=g) > 0.5).float() if masked else None
    pr = eng.program(name, None, steps, denoise=d, masked=masked)
    nz = E.per_image_noise(4100, b, (4, hw, hw), 1 + pr.draws)
    unet = CN.ControlledUNet(sd, cfg, [(csds[k], hints[j], weights[j], *windows[j]) for j, k in enumerate(units)])
    with torch.no_grad():
        ref = CN.run_sampler(name, unet, cond, unc, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d,
                             mask=None if nmask is None else (init, nmask[None, None]), prediction=pred)
    if masked:
        ref = ref * nmask + init * (1 - nmask)
    lat = eng.run_program(cond, unc, pr.start(nz[0], init), pr, 7.0, noises=nz[1:] if pr.draws else None,
                          inpaint=None if nmask is None else (init, nmask.reshape(-1)), controls=controls)
    z = lat.reshape(b, hw, hw, 4).permute(0, 3, 1, 2)
    assert float((z - ref).abs().max()) <= 1e-4 * float(ref.abs().max()), (name, float((z - ref).abs().max()))
    return z


@pytest.mark.parametrize("name", ["DDIM", "Euler a", "DPM++ 2M", "Heun"])
@pytest.mark.parametrize("window", [(0.0, 1.0), (0.0, 0.5), (0.3, 0.8)])
def test_txt2img_with_a_unit_matches_the_oracle(env, name, window):
    _run(env, name, [window])


def test_two_units_of_different_models(env):
    _run(env, "DPM++ 2M", [(0.0, 1.0), (0.2, 0.7)], units=(0, 1))


@pytest.mark.parametrize("name", ["DDIM", "Euler a"])
def test_img2img_with_a_unit_matches_the_oracle(env, name):
    _run(env, name, [(0.0, 0.6)], steps=8, d=0.75)


@pytest.mark.parametrize("name", ["DDIM", "Heun"])
def test_masked_img2img_with_a_unit_matches_the_oracle(env, name):
    _run(env, name, [(0.0, 1.0)], steps=8, d=0.75, masked=True)


def test_a_unit_changes_the_result_and_a_later_request_without_one_does_not_keep_it(env):
    E, eng, sd, cfg, csds, cws, cond, unc, b, pred = env
    pr = eng.program("Euler a", None, 5)
    nz = E.per_image_noise(7, b, (4, 8, 8), 1 + pr.draws)
    plain = eng.run_program(cond, unc, pr.start(nz[0]), pr, 7.0, noises=nz[1:]).clone()
    ctl = eng.run_program(cond, unc, pr.start(nz[0]), pr, 7.0, noises=nz[1:],
                          controls=[(cws[0], _hint(1, 64, 64), 1.0, 0.0, 1.0)]).clone()
    again = eng.run_program(cond, unc, pr.start(nz[0]), pr, 7.0, noises=nz[1:]).clone()
    assert not torch.allclose(plain, ctl) and torch.equal(plain, again)


def test_stage_steps_group_intermediate_evaluations():
    from b200sd import engine as E, samplers as S
    eng = E.SDEngine.__new__(E.SDEngine)
    eng.prediction = "eps"
    pr = E.SDEngine.program(eng, "Heun", None, 5)
    assert S.stage_steps(pr.sp.stages) == [0, 0, 1, 1, 2, 2, 3, 3, 4]
    pr = E.SDEngine.program(eng, "PLMS", None, 6)   # its warm-up step evaluates twice
    n = len(pr.sp.stages)
    assert S.stage_steps(pr.sp.stages) == [0, 0] + list(range(1, n - 1))


# ------------------------------------------------------------------------------------------------ worker / payload
def _png(arr, data_url=False):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, format="PNG")
    s = base64.b64encode(buf.getvalue()).decode()
    return "data:image/png;base64," + s if data_url else s


def _unit(**kw):
    u = {"enabled": True, "model": "control_canny [abc123]", "module": "none",
         "image": _png(np.full((32, 48, 3), 200, np.uint8)), "weight": 0.7}
    u.update(kw)
    return u


def test_parse_units_fields_and_defaults():
    from b200sd import controlnet as CTL
    units = CTL.parse_units({"ControlNet": {"args": [_unit(), _unit(enabled=False), {"enabled": False}]}}, 64, 32)
    assert len(units) == 1
    u = units[0]
    assert u.model == "control_canny" and u.weight == 0.7 and (u.start, u.end) == (0.0, 1.0)
    assert u.image.shape == (32, 64, 3) and u.image.dtype == torch.uint8
    assert CTL.parse_units({}, 64, 64) == [] and CTL.parse_units({"controlnet": {"args": []}}, 64, 64) == []


def test_data_url_and_dict_images_decode_like_base64():
    from b200sd import controlnet as CTL
    arr = np.random.default_rng(0).integers(0, 256, (40, 40, 3), dtype=np.uint8)
    a = CTL.parse_units({"controlnet": {"args": [_unit(image=_png(arr))]}}, 40, 40)[0].image
    b = CTL.parse_units({"controlnet": {"args": [_unit(image=_png(arr, True))]}}, 40, 40)[0].image
    c = CTL.parse_units({"controlnet": {"args": [_unit(image=None, input_image={"image": _png(arr),
                                                                                 "mask": _png(np.zeros_like(arr))})]}},
                        40, 40)[0].image
    assert torch.equal(a, torch.from_numpy(arr)) and torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.parametrize("mode,code", [("Just Resize", 0), ("Crop and Resize", 1)])
@pytest.mark.parametrize("src", [(30, 50), (100, 70)])
def test_resize_modes_against_cv2(mode, code, src):
    import cv2
    from b200sd import controlnet as CTL
    arr = np.random.default_rng(1).integers(0, 256, (*src, 3), dtype=np.uint8)
    w, h = 64, 48
    for rm in (mode, code):
        got = CTL.parse_units({"controlnet": {"args": [_unit(image=_png(arr), resize_mode=rm)]}}, w, h)[0].image.numpy()
        if code == 0:
            interp = cv2.INTER_AREA if w * h < src[0] * src[1] else cv2.INTER_CUBIC
            ref = cv2.resize(arr, (w, h), interpolation=interp)
        else:
            k = max(w / src[1], h / src[0])
            nw, nh = int(np.round(src[1] * k)), int(np.round(src[0] * k))
            big = cv2.resize(arr, (nw, nh), interpolation=cv2.INTER_AREA if k < 1 else cv2.INTER_CUBIC)
            y0, x0 = (nh - h) // 2, (nw - w) // 2
            ref = big[y0:y0 + h, x0:x0 + w]
        assert np.array_equal(got, ref), (rm, src)


@pytest.mark.parametrize("bad,msg", [
    (dict(module="canny"), "preprocessor"), (dict(control_mode="My prompt is more important"), "control mode"),
    (dict(control_mode=2), "control mode"), (dict(resize_mode="Resize and Fill"), "Resize and Fill"),
    (dict(resize_mode=2), "Resize and Fill"), (dict(mask=_png(np.full((32, 48, 3), 255, np.uint8))), "mask"),
    (dict(image=None), "image"), (dict(guidance_start=0.8, guidance_end=0.2), "guidance")])
def test_refused_unit_fields(bad, msg):
    from b200sd import controlnet as CTL
    with pytest.raises(ValueError, match=msg):
        CTL.parse_units({"controlnet": {"args": [_unit(**bad)]}}, 64, 64)


def test_more_than_three_units_are_refused():
    from b200sd import controlnet as CTL
    with pytest.raises(ValueError, match="at most 3"):
        CTL.parse_units({"controlnet": {"args": [_unit()] * 4}}, 64, 64)


# ------------------------------------------------------------------------------------------------ loader
def test_loader_synthetic_fallback_and_cache(monkeypatch, caplog):
    from b200sd import config as C, factory
    from b200sd.unet_exec import ControlNetWeights
    monkeypatch.delenv("B200SD_CONTROLNET_DIR", raising=False)
    monkeypatch.setattr(factory, "_CONTROLNETS", OrderedDict())
    with caplog.at_level("WARNING"):
        a = factory.controlnet("control_canny", "tiny", "cpu", torch.float32)
    assert isinstance(a, ControlNetWeights) and a.name == "control_canny" and "SYNTHETIC" in caplog.text
    assert factory.controlnet("control_canny", "tiny", "cpu", torch.float32) is a
    b = factory.controlnet("control_depth", "tiny", "cpu", torch.float32)
    assert not torch.equal(a.t["zero.0.w"], b.t["zero.0.w"])
    for name in ("c", "d", "e"):
        factory.controlnet(name, "tiny", "cpu", torch.float32)
    assert len([k for k in factory._CONTROLNETS if k[0] == "cpu"]) == factory.MAX_CONTROLNETS


def test_loader_reads_the_directory_with_or_without_the_prefix(monkeypatch, tmp_path):
    from safetensors.torch import save_file
    from b200sd import config as C, factory, synth
    sd = synth.make_controlnet_state_dict(C.TINY_UNET, seed=4)
    save_file(sd, str(tmp_path / "with.safetensors"))
    save_file({k[len("control_model."):]: v for k, v in sd.items()}, str(tmp_path / "bare.safetensors"))
    save_file({"controlnet_cond_embedding.conv_in.weight": torch.zeros(1)}, str(tmp_path / "diffusers.safetensors"))
    monkeypatch.setenv("B200SD_CONTROLNET_DIR", str(tmp_path))
    monkeypatch.setattr(factory, "_CONTROLNETS", OrderedDict())
    a = factory.controlnet("with", "tiny", "cpu", torch.float32)
    b = factory.controlnet("bare", "tiny", "cpu", torch.float32)
    assert all(torch.equal(a.t[k], b.t[k]) for k in a.t)
    with pytest.raises(FileNotFoundError):
        factory.controlnet("missing", "tiny", "cpu", torch.float32)
    with pytest.raises(ValueError, match="diffusers"):
        factory.controlnet("diffusers", "tiny", "cpu", torch.float32)


# ------------------------------------------------------------------------------------------------ worker / dispatcher
@pytest.fixture()
def worker(monkeypatch):
    import logging
    from b200sd import config as C, engine as E, factory, synth
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker
    logging.getLogger("distributed").setLevel(logging.ERROR)
    _install(monkeypatch)
    monkeypatch.delenv("B200SD_CONTROLNET_DIR", raising=False)
    monkeypatch.setenv("B200SD_MODEL", "tiny")
    monkeypatch.setattr(factory, "_CONTROLNETS", OrderedDict())
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cpu", dtype=torch.float32, use_graphs=False,
                     vae_chunk=2)
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    return LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0), eng


def _payload(**kw):
    p = {"prompt": "a b", "negative_prompt": "", "seed": 30, "subseed": 4, "subseed_strength": 0, "batch_size": 2,
         "n_iter": 1, "steps": 4, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0}
    p.update(kw)
    return p


def test_worker_serves_units_and_leaves_plain_payloads_as_they_were(worker, monkeypatch):
    wk, eng = worker
    calls = []
    real = eng.txt2img
    monkeypatch.setattr(eng, "txt2img", lambda *a, **k: calls.append(k) or real(*a, **k))
    wk.request(_payload(alwayson_scripts={"Sampler": {"args": []}}), None, False)
    plain = wk.response["tensors"].clone()
    assert "controls" not in calls[-1]
    wk.request(_payload(alwayson_scripts={"ControlNet": {"args": [_unit(resize_mode="Just Resize")]}}), None, False)
    ctl = calls[-1]["controls"]
    assert len(ctl) == 1 and ctl[0][0].name == "control_canny" and ctl[0][2] == 0.7
    assert tuple(ctl[0][1].shape) == (64, 64, 3) and not torch.equal(wk.response["tensors"], plain)


@pytest.mark.parametrize("extra", [dict(enable_hr=True), dict(alwayson_scripts={"controlnet": {"args": [_unit(module="depth")]}})])
def test_worker_refusals_are_invalid_responses(worker, extra):
    from scripts.spartan.worker import InvalidWorkerResponse
    wk, eng = worker
    p = _payload(alwayson_scripts={"controlnet": {"args": [_unit()]}})
    p.update(extra)
    with pytest.raises(InvalidWorkerResponse):
        wk.request(p, None, False)
    assert wk.response is None


def test_worker_refuses_a_missing_model(worker, monkeypatch, tmp_path):
    from scripts.spartan.worker import InvalidWorkerResponse
    wk, eng = worker
    monkeypatch.setenv("B200SD_CONTROLNET_DIR", str(tmp_path))
    with pytest.raises(InvalidWorkerResponse):
        wk.request(_payload(alwayson_scripts={"controlnet": {"args": [_unit()]}}), None, False)


def test_local_worker_advertises_controlnet(worker):
    wk, _ = worker
    assert wk.query_scripts() == {"txt2img": ["controlnet"], "img2img": ["controlnet"]}


class ControlNetUnit:   # the name sd-webui-controlnet's unit objects carry
    def __init__(self, **kw):
        self.__dict__.update(kw)


class _Mode:
    def __init__(self, value):
        self.value = value


def test_dispatcher_packs_enabled_units_for_local_and_http_workers(worker):
    import modules.processing as processing
    import modules.scripts as mscripts
    from scripts.distributed import DistributedScript
    from scripts.spartan.worker import Worker
    wk, eng = worker
    arr = np.random.default_rng(3).integers(0, 256, (64, 64, 3), dtype=np.uint8)

    class FakeControlNet(mscripts.Script):
        def title(self):
            return "ControlNet"

    script, cn = DistributedScript(), FakeControlNet()
    script.args_from = script.args_to = 0
    cn.args_from, cn.args_to = 0, 3
    args = [ControlNetUnit(enabled=True, module="none", model="control_canny [ab12]", weight=0.8,
                           image={"image": arr, "mask": np.zeros_like(arr)}, resize_mode=_Mode("Crop and Resize"),
                           control_mode=_Mode("Balanced"), guidance_start=0.0, guidance_end=1.0, save_detected_map=True),
            ControlNetUnit(enabled=False, module="none", model="control_depth", image=arr),
            {"enabled": True, "module": "none", "model": "control_depth", "image": _png(arr), "weight": 0.5}]
    p = processing.StableDiffusionProcessingTxt2Img(
        prompt="a b", negative_prompt="", seed=7, subseed=3, subseed_strength=0, batch_size=2, n_iter=1, steps=4,
        width=64, height=64, sampler_name="DDIM", cfg_scale=7.0, scripts=mscripts.ScriptRunner([script, cn]),
        script_args=args)
    packed = script._pack_script_args(p)
    units = packed["ControlNet"]["args"]
    assert [u["model"] for u in units] == ["control_canny [ab12]", "control_depth"]
    u = units[0]
    assert u["image"] == u["input_image"] and u["image"].startswith("data:image/png;base64,")
    assert "mask" not in u and u["resize_mode"] == "Crop and Resize" and u["save_detected_map"] is False
    json.dumps(packed)
    # a local GPU worker serves them ...
    wk.request(_payload(alwayson_scripts=packed), None, False)
    assert wk.response is not None
    from b200sd import controlnet as CTL
    got = CTL.parse_units(packed, 64, 64)
    assert torch.equal(got[0].image, torch.from_numpy(arr)) and got[0].model == "control_canny" and got[1].weight == 0.5
    # ... and an HTTP worker that reports the script sends them as they are
    http = Worker(address="10.0.0.9", port=7860, label="http", verify_remotes=False)
    http.supported_scripts = {"txt2img": ["controlnet"], "img2img": ["controlnet"]}
    payload = _payload(alwayson_scripts=packed)
    assert http._scrub_payload(payload) == "txt2img"
    assert json.loads(json.dumps(payload))["alwayson_scripts"]["ControlNet"]["args"] == units
