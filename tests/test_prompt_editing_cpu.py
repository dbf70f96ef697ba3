"""Prompt editing `[from:to:when]` and alternation `[a|b]` on the CPU: the hand-written parser against the lark
restatement of sdwui's grammar (oracle/prompt_schedule_oracle.py), the entry each model evaluation takes, and the engine's
per-evaluation context switch on emulated ops (tests/ops_emulator.py plus select_context below) against the schedule
oracle, which runs the unchanged sd / ControlNet / SDXL oracle samplers under an evaluation-counting shim."""
import random
import re
import types

import pytest
import torch

import ops_emulator
from oracle import prompt_schedule_oracle as PSO


# ------------------------------------------------------------------------------------------------ parser
KNOWN = [  # sdwui's doctests of get_learned_conditioning_prompt_schedules, steps 10
    ("test", None, [(10, "test")]),
    ("a [b:3]", None, [(3, "a "), (10, "a b")]),
    ("a [b: 3]", None, [(3, "a "), (10, "a b")]),
    ("a [[[b]]:2]", None, [(2, "a "), (10, "a [[b]]")]),
    ("[(a:2):3]", None, [(3, ""), (10, "(a:2)")]),
    ("a [b : c : 1] d", None, [(1, "a b  d"), (10, "a  c  d")]),
    ("a[b:[c:d:2]:1]e", None, [(1, "abe"), (2, "ace"), (10, "ade")]),
    ("a [unbalanced", None, [(10, "a [unbalanced")]),
    ("a [b:.5] c", None, [(5, "a  c"), (10, "a b c")]),
    ("((a][:b:c [d:3]", None, [(3, "((a][:b:c "), (10, "((a][:b:c d")]),
    ("[a|(b:1.1)]", None, [(s, "a" if s % 2 else "(b:1.1)") for s in range(1, 11)]),
    ("[fe|]male", None, [(s, "female" if s % 2 else "male") for s in range(1, 11)]),
    ("[fe|||]male", None, [(s, "female" if s % 4 == 1 else "male") for s in range(1, 11)]),
    ("a [b:.5] c", 10, [(10, "a b c")]),
    ("a [b:1.5] c", 10, [(5, "a  c"), (10, "a b c")]),
]


@pytest.mark.parametrize("text,hires,want", KNOWN)
def test_known_answers(text, hires, want):
    from b200sd.prompts import prompt_schedule
    assert prompt_schedule(text, 10, hires) == want


@pytest.mark.parametrize("text,hires,want", KNOWN)
def test_known_answers_of_the_lark_restatement(text, hires, want):
    pytest.importorskip("lark")
    assert [tuple(e) for e in PSO.get_learned_conditioning_prompt_schedules([text], 10, hires)[0]] == want


_WORDS = ["a", "cat", "red hat", " ", "  ", "x y", "BREAK", "1", "2.5", ",", "\\(", "\\]", "\\\\", "\\:", "\\|"]
_WHEN = ["0", "1", "3", "5", "12", "-2", "+4", ".5", "0.25", "1.5", "2.", "-0.5", "1e1", "0.0", " 3 ", "  .7", "4 "]


def _random_prompt(rng: random.Random, depth: int = 0) -> str:
    """nesting, edits inside alternations and the reverse, escapes, (x:1.2) next to [x:1.2], [a::5], [:b:5], [a|],
    whitespace around numbers, negative and zero `when`, unbalanced and stray brackets (a stray is followed by text:
    see test_random_prompts_match_the_lark_restatement)"""
    parts = []
    for _ in range(rng.randint(0, 4)):
        r = rng.random()
        if depth < 3 and r < 0.2:
            before = _random_prompt(rng, depth + 1) + ":" if rng.random() < 0.6 else ""
            parts.append("[" + before + _random_prompt(rng, depth + 1) + ":" + rng.choice(_WHEN) + "]")
        elif depth < 3 and r < 0.32:
            parts.append("[" + "|".join(_random_prompt(rng, depth + 1) for _ in range(rng.randint(1, 4))) + "]")
        elif depth < 3 and r < 0.42:
            w = ":" + rng.choice(["1.2", "0.8", "x"]) if rng.random() < 0.5 else ""
            parts.append("(" + _random_prompt(rng, depth + 1) + w + ")")
        elif depth < 3 and r < 0.48:
            parts.append("[" + _random_prompt(rng, depth + 1) + (":1.2" if rng.random() < 0.3 else "") + "]")
        elif r < 0.56:
            parts.append(rng.choice(["[", "]", "(", ")", ":", "|", "\\"]) + rng.choice(_WORDS[:6]))
        else:
            parts.append(rng.choice(_WORDS))
    return "".join(parts)


# a closer followed by two more bracket / colon characters: see test_random_prompts_match_the_lark_restatement
_EARLEY_CORNER = re.compile(r"[\])][\[\]():]{2}")


def test_random_prompts_match_the_lark_restatement():
    """2,400 seeded prompts, every step count / hires / old-scheduling combination.  One corner is left out: lark's
    Earley parser resolves the ambiguity between a group and a run of two or more stray bracket or colon characters
    right after its closer by an order that depends on the rest of the prompt (`[a:1]::` is left unparsed, `[a:1]:`
    and `[a:1]:::x` are parsed); prompt_schedule always parses such a group."""
    pytest.importorskip("lark")
    from b200sd.prompts import prompt_schedule
    rng = random.Random(20261018)
    scheduled = n = 0
    while n < 2400:
        text = _random_prompt(rng)
        if _EARLEY_CORNER.search(text):
            continue
        n += 1
        steps, hires, old = rng.choice([1, 4, 10, 20]), rng.choice([None, None, 7]), rng.random() < 0.2
        want = [tuple(e) for e in PSO.get_learned_conditioning_prompt_schedules([text], steps, hires, old)[0]]
        assert prompt_schedule(text, steps, hires, old) == want, (text, steps, hires, old)
        scheduled += len(want) > 1
    assert scheduled > 150


def test_unparsable_prompts_are_used_as_they_are():
    from b200sd.prompts import prompt_schedule
    assert prompt_schedule("a|b [c:2]", 10) == [(10, "a|b [c:2]")]
    assert prompt_schedule("x [c:2] \\", 10, 6) == [(6, "x [c:2] \\")]


# ------------------------------------------------------------------------------------------------ evaluations
def test_second_order_samplers_count_two_evaluations_per_step():
    from b200sd import engine as E
    assert set(E.SECOND_ORDER) == set(PSO.SECOND_ORDER)
    for name in E.SAMPLERS:
        assert E.total_steps(name, 10) == PSO.total_steps(name, 10)
    assert E.total_steps("Heun", 10) == 20 and E.total_steps("DPM++ 2M", 10) == 10


@pytest.mark.parametrize("name", ["DDIM", "Euler a", "Euler", "DPM++ 2M", "Heun", "DPM2", "DPM2 a", "DPM++ 2S a",
                                  "DPM++ SDE", "LMS", "DPM fast", "PLMS", "DPM2 Karras", "DPM++ SDE Karras"])
def test_every_evaluation_takes_sdwuis_entry(name):
    from b200sd import engine as E
    from b200sd.prompts import prompt_schedule, schedule_index
    steps = 8
    sch = prompt_schedule("a [b:c:0.5] [d|e]", E.total_steps(name, steps))
    pr = E.SDEngine.program(types.SimpleNamespace(prediction="eps"), name, None, steps)
    for i in range(pr.n_evals + 3):   # beyond the last entry (DPM adaptive): entry 0
        assert schedule_index(sch, i) == PSO.reconstruct_index(sch, i)
    assert schedule_index([(3, "x"), (6, "y")], 7) == 0 and schedule_index([(3, "x"), (6, "y")], 3) == 0


# ------------------------------------------------------------------------------------------------ engine (emulated ops)
def select_context(bank, entry_len, sched, step_counter, ctx, kv_len):
    """b200sd_select_context: row r copies entry sched[step, r] up to its length and zero-fills to the capacity"""
    for row in range(ctx.shape[0]):
        e = int(sched[int(step_counter.item()), row])
        n = int(entry_len[e])
        ctx[row].zero_()
        ctx[row, :n] = bank[e, :n]
        kv_len[row] = n
    return ctx


def _install(monkeypatch):
    from b200sd import engine as E, ops
    from test_controlnet_cpu import hint_to_nhwc
    from test_prompts_cpu import attention_varlen
    ops_emulator.install(monkeypatch, ops)
    for fn in (select_context, hint_to_nhwc):
        monkeypatch.setattr(ops, fn.__name__, fn)
    monkeypatch.setattr(ops, "attention", attention_varlen)
    monkeypatch.setattr(E.SDEngine, "_require_cuda", False)


LONG = "a dog " + " ".join(f"w{i}" for i in range(80))   # two chunks


@pytest.fixture
def env(monkeypatch):
    from b200sd import config as C, engine as E, synth
    _install(monkeypatch)
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2)
    switches = []
    real = E.Plan.switch_context
    monkeypatch.setattr(E.Plan, "switch_context", lambda plan, slots: switches.append(int(plan.step)) or real(plan, slots))
    return types.SimpleNamespace(E=E, eng=eng, sd=sd, cfgs=cfgs, switches=switches, b=2)


def _sched(texts, ends, vocab=1000):
    from b200sd.engine import PromptSchedule
    from b200sd.factory import tokenize_prompts
    ids, mult = tokenize_prompts(texts, vocab)
    return PromptSchedule(list(ends), ids, mult if bool((mult != 1).any()) else None)


def _of(text, steps, hires=None, base=None):
    """PromptSchedule of a prompt, as the worker builds it"""
    from b200sd.prompts import prompt_schedule
    sch = prompt_schedule(text, base if hires else steps, hires)
    return _sched([t for _, t in sch], [e for e, _ in sch])


def _tok(text, b=2, vocab=1000):
    from b200sd.factory import tokenize_prompts
    return tokenize_prompts([text] * b, vocab)[0]


def _oracle(env, name, steps, sched, nz, init=None, d=None, nmask=None, units=()):
    """the unchanged ControlNet / sd oracle samplers under the schedule oracle's evaluation-counting shim"""
    from oracle import controlnet_oracle as CN, prompt_oracle as P, sd_oracle as O
    cs, us = sched
    inner = CN.ControlledUNet(env.sd, env.cfgs[0], list(units))
    unet = PSO.Scheduled(lambda x, t, c, y: inner(x, t, c), P.encode_sd1(env.sd, env.cfgs[2], cs.tokens, cs.multipliers),
                         P.encode_sd1(env.sd, env.cfgs[2], us.tokens, us.multipliers), cs.ends, us.ends, inner=inner)
    c, u = unet.placeholders(env.b)
    mask = None if nmask is None else (init, nmask[None, None])
    with torch.no_grad():
        if name == "DPM adaptive":
            z = O.run_sampler(name, unet, c, u, 7.0, steps, nz[0], list(nz[1:]), init, d, mask)
        else:
            z = CN.run_sampler(name, unet, c, u, 7.0, steps, nz[0], list(nz[1:]), init=init, denoising_strength=d,
                               mask=mask)
    if nmask is not None:
        z = z * nmask + init * (1 - nmask)
    return z, unet.entries


def _check(env, hw, ref):
    lat = env.eng.plan(env.b, hw, hw).x.reshape(env.b, hw, hw, 4).permute(0, 3, 1, 2)
    assert float((lat - ref).abs().max()) <= 1e-3 * float(ref.abs().max())


def _switch_points(entries):
    return [k for k, e in enumerate(entries) if k == 0 or e != entries[k - 1]]


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "DPM++ 2M", "Heun", "PLMS", "DPM adaptive"])
def test_txt2img_matches_the_schedule_oracle(env, sampler):
    """a cond edit to a two-chunk entry and an uncond edit from the empty prompt: cond and uncond of different lengths
    and entries that change at different evaluations; DPM adaptive runs past the steps (entry 0 again)"""
    hw, steps = 8, 6
    total = env.E.total_steps(sampler, steps)
    sched = (_of(f"a [cat:{LONG}:0.5]", total), _of("[:ugly:2]", total))
    assert sched[0].tokens.shape[1] == 154 and sched[1].tokens.shape[1] == 77
    pr = env.eng.program(sampler, None, steps)
    nz = env.E.per_image_noise(41, env.b, (4, hw, hw), 1 + pr.draws)
    env.eng.txt2img(_tok("x"), _tok(""), 41, steps=steps, height=8 * hw, width=8 * hw, sampler=sampler, schedule=sched)
    ref, entries = _oracle(env, sampler, steps, sched, nz)
    _check(env, hw, ref)
    assert len(set(entries)) >= 3 and env.eng.last_unet_evals == len(entries)
    if sampler != "DPM adaptive":   # its device counter restarts with every attempt
        assert env.switches == _switch_points(entries)
    assert env.eng.plan(env.b, hw, hw).kv_len.tolist() == [154] * 2 + [77] * 2


def test_alternation_matches_the_schedule_oracle(env):
    hw, steps = 8, 6
    sched = (_of("a [cat|dog|cow]", steps), _of("", steps))
    nz = env.E.per_image_noise(5, env.b, (4, hw, hw), 1 + steps)
    env.eng.txt2img(_tok("x"), _tok(""), 5, steps=steps, height=8 * hw, width=8 * hw, sampler="Euler a", schedule=sched)
    ref, entries = _oracle(env, "Euler a", steps, sched, nz)
    _check(env, hw, ref)
    assert env.switches == _switch_points(entries) == [0, 2, 3, 4, 5]


def test_masked_img2img_matches_the_schedule_oracle(env):
    from oracle import sd_oracle as O
    hw, steps, d = 8, 8, 0.75
    sched = (_of("a [cat:dog:0.5]", steps), _of("[ugly:3]", steps))
    init_u8 = torch.randint(0, 256, (env.b, 8 * hw, 8 * hw, 3), generator=torch.Generator().manual_seed(9),
                            dtype=torch.uint8)
    f = 2 ** (len(env.cfgs[1].ch_mult) - 1)
    init_u8 = init_u8[:, :f * hw, :f * hw].contiguous()
    nmask = (torch.rand((hw, hw), generator=torch.Generator().manual_seed(5)) > 0.5).float()
    pr = env.eng.program("Euler a", None, steps, denoise=d, masked=True)
    nz = env.E.per_image_noise(31, env.b, (4, hw, hw), 1 + pr.draws)
    env.eng.img2img(_tok("x"), _tok(""), 31, init_u8, denoising_strength=d, steps=steps, sampler="Euler a",
                    latmask=nmask.reshape(-1), schedule=sched)
    with torch.no_grad():
        init = O.vae_encode_mean(env.sd, env.cfgs[1], O.image_to_model_input(init_u8)) * env.cfgs[1].scale_factor
    ref, entries = _oracle(env, "Euler a", steps, sched, nz, init=init, d=d, nmask=nmask)
    _check(env, hw, ref)
    assert len(set(entries)) >= 2 and env.switches == _switch_points(entries)


def test_hires_fix_with_its_own_prompt_matches_the_schedule_oracle(env):
    """first pass `a [cat:dog:0.5]`, second pass hr_prompt `b [c:1.5]` over the hires steps (an edit halfway)"""
    from oracle import upscale_oracle as UO
    hw, steps, hr_steps, d = 8, 5, 8, 0.9
    first = (_of("a [cat:dog:0.5]", steps), _of("", steps))
    second = (_of("b [c:1.5]", steps, hr_steps, steps), _of("", steps, hr_steps, steps))
    assert second[0].ends == [4, 8]   # (1.5 - 1) x 8; DDIM at strength 0.9 evaluates 6 of them
    env.eng.txt2img_hires(_tok("x"), _tok(""), 77, steps=steps, height=8 * hw, width=8 * hw, hr_scale=2.0,
                          hr_steps=hr_steps, denoising_strength=d, schedule=first, hr_schedule=second)
    nz1 = env.E.per_image_noise(77, env.b, (4, hw, hw), 1)
    nz2 = env.E.per_image_noise(77, env.b, (4, 2 * hw, 2 * hw), 1)
    z1, e1 = _oracle(env, "DDIM", steps, first, nz1)
    _check(env, hw, z1)
    with torch.no_grad():
        up = UO.hires_upscale(env.sd, env.cfgs[1], z1, 2 * hw, 2 * hw, "Latent")
    ref, e2 = _oracle(env, "DDIM", hr_steps, second, nz2, init=up, d=d)
    _check(env, 2 * hw, ref)
    assert env.switches == _switch_points(e1) + _switch_points(e2) and len(set(e2)) == 2


def test_controlnet_unit_matches_the_schedule_oracle(env):
    from b200sd import synth
    from b200sd.unet_exec import ControlNetWeights
    from test_controlnet_cpu import _hint
    hw, steps = 8, 6
    csd = synth.make_controlnet_state_dict(env.cfgs[0], seed=11)
    cw = ControlNetWeights(csd, env.cfgs[0], "cpu", torch.float32, name="cn0")
    hint = _hint(20, 8 * hw, 8 * hw)
    sched = (_of("a [cat:dog:0.5]", steps), _of("", steps))
    pr = env.eng.program("Euler a", None, steps)
    nz = env.E.per_image_noise(12, env.b, (4, hw, hw), 1 + pr.draws)
    env.eng.txt2img(_tok("x"), _tok(""), 12, steps=steps, height=8 * hw, width=8 * hw, sampler="Euler a",
                    controls=[(cw, hint, 0.8, 0.0, 0.6)], schedule=sched)
    ref, entries = _oracle(env, "Euler a", steps, sched, nz, units=[(csd, hint, 0.8, 0.0, 0.6)])
    _check(env, hw, ref)
    assert env.switches == _switch_points(entries)


def test_a_new_controlnet_model_drops_the_ctx_graph_of_its_slot(env):
    from b200sd import synth
    from b200sd.unet_exec import ControlNetWeights
    from test_controlnet_cpu import _hint
    plan = env.eng.plan(env.b, 8, 8)
    cws = [ControlNetWeights(synth.make_controlnet_state_dict(env.cfgs[0], seed=s), env.cfgs[0], "cpu", torch.float32,
                             name=f"cn{s}") for s in (1, 2)]
    env.eng._set_controls(plan, [(cws[0], _hint(1, 64, 64), 1.0, 0.0, 1.0)])
    plan.graphs.update({"ctx|cn0=cn1": None, "ctx": None, "vae": None})
    env.eng._set_controls(plan, [(cws[1], _hint(1, 64, 64), 1.0, 0.0, 1.0)])
    assert set(plan.graphs) == {"ctx", "vae"}
    plan.graphs["ctx|cn0=cn2"] = None
    plan.ensure_context(154)
    assert set(plan.graphs) == {"vae"}


def test_unscheduled_requests_keep_their_program(env):
    """the plain request after a scheduled one: same op list, same images as on a fresh engine, no schedule state"""
    from b200sd import engine as E
    kw = dict(steps=4, height=64, width=64, sampler="DDIM")
    fresh = E.SDEngine(env.sd, *env.cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2)
    want = fresh.txt2img(_tok("a cat"), _tok(""), 3, **kw)
    ops_before = [(op[0].__qualname__, len(op[1])) for op in fresh.plan(2, 8, 8).unet.ops]
    env.eng.txt2img(_tok("x"), _tok(""), 3, schedule=(_of("a [cat:dog:0.5]", 4), _of("", 4)), **kw)
    got = env.eng.txt2img(_tok("a cat"), _tok(""), 3, **kw)
    assert torch.equal(got, want) and env.eng._entries is None
    assert [(op[0].__qualname__, len(op[1])) for op in env.eng.plan(2, 8, 8).unet.ops] == ops_before


def test_collapsed_schedule_takes_the_plain_path(env):
    """[a:b:0] is the prompt b: one entry per side, no switch"""
    from b200sd.prompts import prompt_schedule
    kw = dict(seed=11, steps=6, height=64, width=64, sampler="DDIM")
    assert prompt_schedule("a [cat:dog:0]", 6) == [(6, "a dog")]
    plain = env.eng.txt2img(_tok("a dog"), _tok(""), **kw)
    got = env.eng.txt2img(_tok("x"), _tok(""), schedule=(_of("a [cat:dog:0]", 6), _of("", 6)), **kw)
    assert torch.equal(got, plain) and env.switches == []


def test_entries_of_a_prompt_share_one_chunk_count():
    """one chunk and two chunks: the short entry gets an empty second chunk, as sdwui pads the entries it encodes
    together"""
    sch = _of(f"[short:{LONG}:0.5]", 10)
    assert sch.tokens.shape == (2, 154)
    assert torch.equal(sch.tokens[0, :77], _tok("short", 1)[0]) and torch.equal(sch.tokens[0, 77:], _tok("", 1)[0])


# ------------------------------------------------------------------------------------------------ SDXL
@pytest.mark.parametrize("negative,zeroed", [("[:ugly:2]", False), ("[:  :2]", True)])
def test_tiny_sdxl_matches_the_schedule_oracle(monkeypatch, negative, zeroed):
    """each evaluation's vector conditioning comes from its entries; the negative prompt is zeroed only when every entry
    of its schedule is empty"""
    from b200sd import config as C, engine as E, synth
    from b200sd.prompts import prompt_schedule
    from oracle import sd_oracle as O
    _install(monkeypatch)
    cfgs = (C.TINYXL_UNET, C.TINYXL_VAE, C.TINYXL_CLIP)
    ocfgs = (O.TINYXL_UNET, O.TINYXL_VAE, O.TINYXL_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2)
    b, hw, steps = 2, 8, 5
    assert len(prompt_schedule(negative, steps)) == 2
    sched = (_of("a [cat:dog:1]", steps), _of(negative, steps))
    with torch.no_grad():
        cc, yc = O.sdxl_conditioner(sd, ocfgs[2], sched[0].tokens, 8 * hw, 8 * hw)
        cu, yu = O.sdxl_conditioner(sd, ocfgs[2], sched[1].tokens, 8 * hw, 8 * hw, zero_txt=zeroed)
    unet = PSO.Scheduled(lambda x, t, c, y: O.unet_forward(sd, ocfgs[0], x, t, c, y=y), cc, cu, sched[0].ends,
                         sched[1].ends, yc, yu)
    nz = E.per_image_noise(77, b, (4, hw, hw), 1 + steps)
    c, u = unet.placeholders(b)
    with torch.no_grad():
        z = O.run_sampler("Euler a", unet, c, u, 7.0, steps, nz[0], list(nz[1:]))
    eng.txt2img(_tok("x"), _tok(""), 77, steps=steps, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler="Euler a",
                schedule=sched)
    lat = eng.plan(b, hw, hw).x.reshape(b, hw, hw, 4).permute(0, 3, 1, 2)
    assert float((lat - z).abs().max()) <= 1e-3 * float(z.abs().max())
    assert len(set(unet.entries)) >= 3


# ------------------------------------------------------------------------------------------------ worker
@pytest.fixture
def worker(monkeypatch):
    import logging
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker

    class Eng:
        interrupted = False
        clip_cfg = types.SimpleNamespace(vocab=1000)
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

        def txt2img_hires(self, tok, neg, seed, **kw):
            return self._out("txt2img_hires", tok, dict(kw, tok=tok, neg=neg))

    logging.getLogger("distributed").setLevel(logging.ERROR)
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    eng = Eng()
    return LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0), eng


def _payload(**kw):
    p = {"prompt": "a b", "negative_prompt": "", "seed": 30, "subseed": 4, "subseed_strength": 0, "batch_size": 2,
         "n_iter": 1, "steps": 4, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0}
    p.update(kw)
    return p


def test_a_payload_without_syntax_reaches_the_engine_with_todays_arguments(worker):
    from b200sd.factory import tokenize_prompts
    wk, eng = worker
    wk.request(_payload(prompt="a (b:1.2)"), None, False)
    name, kw = eng.calls[-1]
    assert name == "txt2img" and "schedule" not in kw
    assert set(kw) == {"steps", "cfg_scale", "height", "width", "sampler", "scheduler", "multipliers", "tok", "neg"}
    assert torch.equal(kw["tok"], tokenize_prompts(["a (b:1.2)"] * 2, 1000)[0])
    wk.request(_payload(enable_hr=True, hr_scale=2.0), None, False)
    assert eng.calls[-1][0] == "txt2img_hires" and "hr_schedule" not in eng.calls[-1][1]


def test_worker_builds_the_schedules(worker):
    from b200sd.factory import tokenize_prompts
    wk, eng = worker
    wk.request(_payload(prompt="a [cat:dog:0.5]", negative_prompt="[:ugly:2]", sampler_name="Heun"), None, False)
    kw = eng.calls[-1][1]
    cs, us = kw["schedule"]
    assert cs.ends == [4, 8] and us.ends == [2, 8]   # Heun: 2 x 4 steps
    assert torch.equal(cs.tokens, tokenize_prompts(["a cat", "a dog"], 1000)[0])
    info = wk.response["info"]
    assert "a [cat:dog:0.5]" in info
    wk.request(_payload(prompt="a [cat:dog:0]"), None, False)
    kw = eng.calls[-1][1]
    assert "schedule" not in kw and torch.equal(kw["tok"], tokenize_prompts(["a dog"] * 2, 1000)[0])


def test_worker_gives_the_hires_pass_its_own_prompt(worker):
    wk, eng = worker
    wk.request(_payload(enable_hr=True, hr_scale=2.0, hr_prompt="x [y:1.5]"), None, False)
    kw = eng.calls[-1][1]
    assert "schedule" not in kw
    hc, hu = kw["hr_schedule"]
    assert hc.ends == [2, 4] and hu.ends == [4]
    wk.request(_payload(enable_hr=True, hr_scale=2.0, prompt="p [q:0.5]", override_settings={"use_old_scheduling": True}),
               None, False)
    kw = eng.calls[-1][1]
    assert kw["schedule"][0].ends == [2, 4] and kw["hr_schedule"][0].ends == [2, 4]


def test_rest_server_passes_the_prompt_fields_through():
    import json
    from fastapi.testclient import TestClient
    from server.sdapi import create_app

    class Eng:
        interrupted = False
        clip_cfg = types.SimpleNamespace(vocab=1000)
        calls = []

        def txt2img_hires(self, tok, neg, seed, **kw):
            self.calls.append(kw)
            return torch.zeros((tok.shape[0], 128, 128, 3), dtype=torch.uint8)

    eng = Eng()
    client = TestClient(create_app(lambda device: eng, [0]))
    body = {"prompt": "a [b|c]", "steps": 2, "width": 64, "height": 64, "sampler_name": "DDIM", "enable_hr": True,
            "hr_scale": 2.0, "hr_prompt": "d [e:1]"}
    r = client.post("/sdapi/v1/txt2img", json=body)
    assert r.status_code == 200
    kw = eng.calls[-1]
    assert kw["schedule"][0].ends == [1, 2] and kw["hr_schedule"][0].ends == [2]   # [e:1] lies in the first pass
    assert json.loads(r.json()["info"])["all_prompts"][0] == "a [b|c]"


def test_a_scheduled_hires_request_needs_the_second_pass_schedule(env):
    with pytest.raises(ValueError, match="hr_schedule"):
        env.eng.txt2img_hires(_tok("x"), _tok(""), 1, steps=4, height=64, width=64,
                              schedule=(_of("a [b:c:0.5]", 4), _of("", 4)))
