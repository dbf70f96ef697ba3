"""LoRA networks named in prompts, on the CPU: tag parsing and module names against the restatement of sdwui's Lora
extension (oracle/lora_oracle.py) and a hand-written table, the packers' placements through an fp64 emulation of the
merge against the packing of the oracle-merged state dict, and the worker's handling of tags with an engine double."""
import json
import os
import types

import pytest
import torch

from oracle import lora_oracle as LO

HERE = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------------------ tags
CORPUS = [
    "a cat <lora:style:0.8>",
    "<lora:a:0.5:0.25> x, <lora:b> y",
    "x <lora:n:te=0.3:unet=1.5> y",
    "x <lora:n:0.7:unet=0.1:dyn=4>",
    "x <lora:n:1:0.5:8> y",
    "<lyco:lc:0.6> z",
    "<hypernet:h:1> kept <lora:l:2>",
    "[cat:<lora:dog:0.5> dog:0.5] x",
    "a (red:1.2) <lora:s:0.9>, BREAK b",
    "\\(x\\) <lora:e:1> \\[y\\]",
    "  <lora:sp:1>  ,  <lora:sp2:1>  ",
    "no tags at all",
    "<lora:w:1:te=0.5>",
    "a <notatag> <lora:> b",
]


@pytest.mark.parametrize("text", CORPUS)
def test_tags_match_the_oracle(text):
    from b200sd import lora as L
    body, refs = L.parse_prompt(text)
    obody, onets = LO.networks_of(text)
    assert body == obody
    assert sorted((r.name, r.te, r.unet, r.dyn) for r in refs) == sorted(onets)


def test_tag_arguments():
    from b200sd import lora as L
    body, refs = L.parse_prompt("a <lora:x:0.5>, b <lora:y:te=0.2:unet=3:dyn=2> <lyco:z:1:0.5:4>")
    assert body == "a , b  "
    assert refs == [L.LoraRef("x", 0.5, 0.5), L.LoraRef("y", 0.2, 3.0, 2), L.LoraRef("z", 1.0, 0.5, 4)]


# ------------------------------------------------------------------------------------------------ module names
def _model(size):
    from b200sd import config as C, factory, synth
    from b200sd.clip_text import ClipText, OpenClipText
    from b200sd.unet_exec import UNetWeights
    u, v, c = factory.configs(size)
    sd = synth.make_state_dict(u, v, c, seed=0)
    uw = UNetWeights(sd, u, "cpu", torch.float32)
    if c.xl_width:
        towers = [("t0", ClipText(sd, c, "cpu", torch.float32, C.XL_PREFIX0)),
                  ("t1", OpenClipText(sd, c, "cpu", torch.float32, C.XL_PREFIX1))]
        cut = "conditioner.embedders."
    elif c.open_clip:
        towers, cut = [("t0", OpenClipText(sd, c, "cpu", torch.float32, C.OPENCLIP_PREFIX))], "cond_stage_model."
    else:
        towers, cut = [("t0", ClipText(sd, c, "cpu", torch.float32))], "cond_stage_model."
    return types.SimpleNamespace(sd=sd, cfgs=(u, v, c), uw=uw, towers=dict(towers), cut=cut)


@pytest.fixture(scope="module")
def models():
    return {s: _model(s) for s in ("tiny", "tiny21", "tinyxl")}


def _table(m):
    from b200sd import lora as L
    owners = [("unet", m.uw.place, "model.", False)] + [(n, t.place, m.cut, True) for n, t in m.towers.items()]
    return L.KeyTable(owners, m.cfgs[0], m.cfgs[2].open_clip)


def test_sd15_diffusers_names_convert_as_sdwui_converts_them():
    """every diffusers-form name of a full SD1.5 LoRA and SD 2.x text names: the layout-derived conversion equals sdwui's
    block arithmetic"""
    from b200sd import config as C, lora as L, synth
    blocks = L.diffusers_blocks(C.SD15_UNET)
    names = [k.split(".")[0] for k in synth.make_lora_state_dict(C.TINY_UNET, C.TINY_CLIP, rank=1) if k.endswith("alpha")]
    assert len(names) > 250
    for n in names:
        assert L.to_compvis(n, blocks, False) == LO.convert_diffusers_name_to_compvis(n, False), n
    for n in ("lora_te_text_model_encoder_layers_5_self_attn_q_proj", "lora_te_text_model_encoder_layers_5_mlp_fc1",
              "lora_te_text_model_encoder_layers_23_mlp_fc2", "lora_te2_text_model_encoder_layers_31_self_attn_out_proj"):
        assert L.to_compvis(n, blocks, True) == LO.convert_diffusers_name_to_compvis(n, True), n


@pytest.mark.parametrize("size", ["tiny", "tiny21", "tinyxl"])
def test_key_table_matches_the_oracle_and_the_golden_pairs(models, size):
    from b200sd import synth
    m = models[size]
    table = _table(m)
    mapping = LO.layer_mapping(m.sd)
    is_sd2 = m.cfgs[2].open_clip
    forms = ("compvis",) if size == "tinyxl" else ("diffusers", "compvis")   # sdwui's diffusers arithmetic is SD1's
    for form in forms:
        for k in synth.make_lora_state_dict(m.cfgs[0], m.cfgs[2], rank=1, form=form):
            name = k.split(".")[0]
            t = table.find(name)
            _, ok, ob = LO.match_key(mapping, name, is_sd2)
            assert t is not None and (t.ldm_key, t.block) == (ok, ob), name
    with open(os.path.join(HERE, "golden", "lora_key_pairs.json")) as f:
        pairs = json.load(f)[size]
    for name, key, block in pairs:
        t = table.find(name)
        assert t is not None and (t.ldm_key, t.block) == (key, block), name
    assert table.find("lora_unet_not_a_module") is None


# ------------------------------------------------------------------------------------------------ placements
def _emulate(m, nets):
    """fp64 merge of the packed fp32 weights through lora.resolve / lora.plan -> {(owner, tensor): merged}"""
    from b200sd import lora as L
    packed = {"unet": m.uw.t, **{n: t.w for n, t in m.towers.items()}}
    place = {"unet": m.uw.place, **{n: t.place for n, t in m.towers.items()}}
    groups = L.plan(L.resolve(_table(m), nets), place, packed, "cpu")
    out = {}
    for (owner, name), gs in groups.items():
        w = packed[owner][name].double().clone()
        assert sum(g.hi - g.lo for g in gs) == w.shape[0] and gs[0].lo == 0
        for g in gs:
            if g.U is not None:
                w[g.lo:g.hi] += g.U.double() @ g.D.double()
        out[(owner, name)] = w
    return out, packed


@pytest.mark.parametrize("size", ["tiny", "tiny21", "tinyxl"])
def test_placements_carry_the_merge_into_every_packed_tensor(models, size):
    """two stacked networks (te + unet + LoCon; diffusers and compvis names where both apply, dyn on one): merged packed
    weights = packing of the oracle-merged fp32 state dict, for every touched tensor — conv tap order, head padding,
    the GEGLU interleave, qkv / kv / emb_all concatenation, OpenCLIP's in_proj row blocks"""
    from b200sd import lora as L, synth
    from b200sd.clip_text import ClipText, OpenClipText
    from b200sd.unet_exec import UNetWeights
    m = models[size]
    u, _, c = m.cfgs
    sd_a = synth.make_lora_state_dict(u, c, seed=5, rank=4, form="compvis")
    sd_b = synth.make_lora_state_dict(u, c, seed=6, rank=6, form="compvis" if c.xl_width else "diffusers")
    nets = [(L.load_state_dict("a", sd_a), L.LoraRef("a", 0.7, 1.3)),
            (L.load_state_dict("b", sd_b), L.LoraRef("b", -0.5, 0.8, 4))]
    got, packed = _emulate(m, nets)
    merged = LO.merge(m.sd, [(sd_a, 0.7, 1.3, None), (sd_b, -0.5, 0.8, 4)])
    uw = UNetWeights(merged, u, "cpu", torch.float32)
    towers = {n: (ClipText if isinstance(t, ClipText) else OpenClipText)(merged, c, "cpu", torch.float32, t.prefix)
              for n, t in m.towers.items()}
    ref = {"unet": uw.t, **{n: t.w for n, t in towers.items()}}
    kinds = set()
    for (owner, name), w in got.items():
        r = ref[owner][name].double()
        scale = float(r.abs().max())
        assert float((w - r).abs().max()) <= 2e-6 * scale, (owner, name)
        assert not torch.equal(w, packed[owner][name].double()), (owner, name)
        kinds.add(name.rsplit(".", 2)[-2] if owner == "unet" else name.rsplit(".", 2)[-2])
    untouched = [(o, n) for o in ref for n in ref[o] if (o, n) not in got and n.endswith(("w", "weight"))
                 and torch.is_tensor(ref[o][n]) and ref[o][n].dim() == 2]
    for o, n in untouched:
        assert torch.equal(ref[o][n], packed[o][n]), (o, n)
    need = {"qkv", "kv", "q", "ff1", "emb_all", "conv1", "conv2", "skip"}
    assert need <= kinds, need - kinds
    if c.open_clip or c.xl_width:
        assert any(k.endswith("in_proj_weight") for (_, k) in got)


def test_openclip_attention_needs_all_four_modules(models):
    """sdwui applies q / k / v / out_proj to a MultiheadAttention only together: a network without out_proj leaves the
    attention alone (in the oracle and here)"""
    from b200sd import lora as L, synth
    m = models["tiny21"]
    u, _, c = m.cfgs
    sd = {k: v for k, v in synth.make_lora_state_dict(u, c, seed=2, rank=2, unet_modules=False).items()
          if "layers_0_self_attn_out_proj" not in k}
    got, _ = _emulate(m, [(L.load_state_dict("x", sd), L.LoraRef("x"))])
    assert ("t0", "transformer.resblocks.0.attn.in_proj_weight") not in got
    assert ("t0", "transformer.resblocks.1.attn.in_proj_weight") in got
    merged = LO.merge(m.sd, [(sd, 1.0, 1.0, None)])
    k0 = "cond_stage_model.model.transformer.resblocks.0.attn.in_proj_weight"
    assert torch.equal(merged[k0], m.sd[k0])


@pytest.mark.parametrize("part,what", [("hada_w1_a", "LoHa"), ("lokr_w1", "LoKr"), ("on_input", "IA3"),
                                       ("oft_blocks", "OFT"), ("dora_scale", "DoRA"), ("lora_mid.weight", "mid"),
                                       ("diff", "diff"), ("lora_A.weight", "PEFT")])
def test_unserved_network_types_are_refused(part, what):
    from b200sd import lora as L
    sd = {"lora_unet_conv_in.lora_up.weight": torch.zeros(4, 2, 1, 1),
          "lora_unet_conv_in.lora_down.weight": torch.zeros(2, 4, 3, 3), f"lora_unet_conv_out.{part}": torch.zeros(2)}
    with pytest.raises(ValueError, match=what):
        L.load_state_dict("bad", sd)


def test_a_module_that_does_not_fit_is_skipped_with_a_warning(models, caplog):
    from b200sd import lora as L
    m = models["tiny"]
    sd = {"lora_unet_conv_in.lora_up.weight": torch.ones(7, 2, 1, 1),
          "lora_unet_conv_in.lora_down.weight": torch.ones(2, 4, 3, 3),
          "lora_unet_nothing_here.lora_up.weight": torch.ones(7, 2), "lora_unet_nothing_here.lora_down.weight": torch.ones(2, 3)}
    with caplog.at_level("WARNING", logger="distributed"):
        entries = L.resolve(_table(m), [(L.load_state_dict("x", sd), L.LoraRef("x"))])
    assert entries == [[]] and "do not fit" in caplog.text


# ------------------------------------------------------------------------------------------------ worker
@pytest.fixture
def worker(monkeypatch, tmp_path):
    import logging
    from b200sd import config as C
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker

    class Eng:
        interrupted = False
        clip_cfg = C.TINY_CLIP
        unet_cfg = C.TINY_UNET
        inpainting = False
        vae_cfg = types.SimpleNamespace(ch_mult=(1, 2, 2, 2))

        def __init__(self):
            self.calls = []

        def _out(self, name, tok, kw):
            self.calls.append((name, kw))
            h, w = kw.get("height", 64), kw.get("width", 64)
            return torch.zeros((tok.shape[0], h, w, 3), dtype=torch.uint8)

        def txt2img(self, tok, neg, seed, **kw):
            return self._out("txt2img", tok, dict(kw, tok=tok, neg=neg))

        def img2img(self, tok, neg, seed, init, **kw):
            return self._out("img2img", tok, dict(kw, tok=tok, neg=neg))

        def txt2img_hires(self, tok, neg, seed, **kw):
            return self._out("txt2img_hires", tok, dict(kw, tok=tok, neg=neg))

    logging.getLogger("distributed").setLevel(logging.WARNING)
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    monkeypatch.delenv("B200SD_LORA_DIR", raising=False)
    from b200sd import factory
    factory.refresh_loras()
    eng = Eng()
    return LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0), eng


def _payload(**kw):
    p = {"prompt": "a b", "negative_prompt": "", "seed": 30, "subseed": 4, "subseed_strength": 0, "batch_size": 2,
         "n_iter": 1, "steps": 4, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0}
    p.update(kw)
    return p


def test_a_payload_without_tags_reaches_the_engine_with_todays_arguments(worker):
    wk, eng = worker
    wk.request(_payload(), None, False)
    assert set(eng.calls[-1][1]) == {"steps", "cfg_scale", "height", "width", "sampler", "scheduler", "tok", "neg"}
    wk.request(_payload(enable_hr=True, hr_scale=2.0, hr_prompt="c d"), None, False)
    assert "loras" not in eng.calls[-1][1] and "hr_loras" not in eng.calls[-1][1]


def test_tags_are_stripped_exactly_and_passed_as_a_set(worker):
    from b200sd.factory import tokenize_prompts
    wk, eng = worker
    wk.request(_payload(prompt="a <lora:s1:0.5>, b <hypernet:h:1><lora:s2:te=0.2>", negative_prompt="<lora:n:1> ugly"),
               None, False)
    kw = eng.calls[-1][1]
    assert torch.equal(kw["tok"], tokenize_prompts(["a , b "] * 2, 1000)[0])
    assert torch.equal(kw["neg"], tokenize_prompts(["<lora:n:1> ugly"] * 2, 1000)[0])   # sdwui leaves it as it is
    assert [(f.name, r.te, r.unet) for f, r in kw["loras"]] == [("s1", 0.5, 0.5), ("s2", 0.2, 0.2)]
    info = json.loads(wk.response["info"])
    assert info["all_prompts"][0] == "a <lora:s1:0.5>, b <hypernet:h:1><lora:s2:te=0.2>"


def test_a_missing_file_warns_and_is_skipped(worker, monkeypatch, tmp_path, caplog):
    from safetensors.torch import save_file
    from b200sd import config as C, synth
    wk, eng = worker
    monkeypatch.setenv("B200SD_LORA_DIR", str(tmp_path))
    save_file(synth.make_lora_state_dict(C.TINY_UNET, C.TINY_CLIP, seed=1, rank=2), str(tmp_path / "here.safetensors"))
    with caplog.at_level("WARNING", logger="distributed"):
        wk.request(_payload(prompt="x <lora:gone:1> <lora:here:0.5>"), None, False)
    assert "Networks not found: gone" in caplog.text
    assert [f.name for f, _ in eng.calls[-1][1]["loras"]] == ["here"]
    wk.request(_payload(prompt="x <lora:gone:1>"), None, False)
    assert "loras" not in eng.calls[-1][1]


def test_a_loha_file_is_refused_before_the_engine_runs(worker, monkeypatch, tmp_path):
    from safetensors.torch import save_file
    from scripts.spartan.worker import InvalidWorkerResponse
    wk, eng = worker
    monkeypatch.setenv("B200SD_LORA_DIR", str(tmp_path))
    save_file({"lora_unet_conv_in.hada_w1_a": torch.zeros(2, 2), "lora_unet_conv_in.hada_w1_b": torch.zeros(2, 2)},
              str(tmp_path / "loha.safetensors"))
    n = len(eng.calls)
    with pytest.raises(InvalidWorkerResponse):
        wk.request(_payload(prompt="x <lora:loha:1>"), None, False)
    assert len(eng.calls) == n


def test_the_hires_pass_gets_hr_prompts_set(worker):
    wk, eng = worker
    wk.request(_payload(prompt="a <lora:one:1>", enable_hr=True, hr_scale=2.0), None, False)
    kw = eng.calls[-1][1]
    assert [f.name for f, _ in kw["loras"]] == ["one"] and "hr_loras" not in kw   # empty hr_prompt: the same set
    wk.request(_payload(prompt="a <lora:one:1>", enable_hr=True, hr_scale=2.0, hr_prompt="a <lora:two:0.5>"), None, False)
    kw = eng.calls[-1][1]
    assert [f.name for f, _ in kw["loras"]] == ["one"] and [(f.name, r.te) for f, r in kw["hr_loras"]] == [("two", 0.5)]
    wk.request(_payload(prompt="a <lora:one:1>", enable_hr=True, hr_scale=2.0, hr_prompt="a "), None, False)
    kw = eng.calls[-1][1]
    assert kw["hr_loras"] == [] and "hr_schedule" not in kw
    wk.request(_payload(prompt="a", enable_hr=True, hr_scale=2.0, hr_prompt="a <lora:two:1>"), None, False)
    kw = eng.calls[-1][1]
    assert "loras" not in kw and [f.name for f, _ in kw["hr_loras"]] == ["two"]


def test_refresh_drops_the_file_cache(worker):
    from b200sd import factory
    wk, eng = worker
    wk.request(_payload(prompt="a <lora:one:1>"), None, False)
    assert factory._LORAS
    wk.refresh_checkpoints()
    assert not factory._LORAS
