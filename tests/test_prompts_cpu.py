"""sdwui prompt syntax on the CPU: the emphasis / BREAK parser, 77-token chunking with comma backtracking, the hashed
tokeniser's agreement with synthetic_tokens, and multi-chunk weighted prompts through the engine with b200sd.ops
emulated (tests/ops_emulator.py, plus attention_varlen below for the per-row key counts), against the chunked oracle
with sdwui's separate cond / uncond evaluation."""
import logging

import pytest
import torch

import ops_emulator


def attention_varlen(q, k, v, out, heads, d, d_pad, scale, v_ones_col=False, kv_len=None):
    """CPU emulation of b200sd.ops.attention with its kv_len argument: row i is the emulator's plain attention on its first
    kv_len[i] keys (clamped to [1, Skv], as the kernel does); without kv_len it is the plain emulation"""
    if kv_len is None:
        return ops_emulator.attention(q, k, v, out, heads, d, d_pad, scale, v_ones_col)
    skv = k.shape[1]
    for i, n in enumerate(kv_len.tolist()):
        n = min(max(int(n), 1), skv)
        ops_emulator.attention(q[i:i + 1], k[i:i + 1, :n], v[i:i + 1, :n], out[i:i + 1], heads, d, d_pad, scale,
                               v_ones_col)
    return out


def _same(got, want):
    assert len(got) == len(want), (got, want)
    for (t, w), (t2, w2) in zip(got, want):
        assert t == t2 and abs(w - w2) < 1e-9, (got, want)


# ------------------------------------------------------------------------------------------------ parser
@pytest.mark.parametrize("text,want", [
    ("an (important) word", [("an ", 1.0), ("important", 1.1), (" word", 1.0)]),
    ("(unbalanced", [("unbalanced", 1.1)]),
    ("\\(literal\\]", [("(literal]", 1.0)]),
    ("(unnecessary)(parens)", [("unnecessaryparens", 1.1)]),
    ("a (((house:1.3)) [on] a (hill:0.5), sun, (((sky))).",
     [("a ", 1.0), ("house", 1.573), (" ", 1.1), ("on", 1.0), (" a ", 1.1), ("hill", 0.55), (", sun, ", 1.1),
      ("sky", 1.4641), (".", 1.1)]),
    ("a BREAK b", [("a", 1.0), ("BREAK", -1), ("b", 1.0)]),
    ("", [("", 1.0)]),
    ("[a]", [("a", 1 / 1.1)]),
    ("a) b]", [("a) b]", 1.0)]),
])
def test_parse_prompt_attention(text, want):
    from b200sd.prompts import parse_prompt_attention
    _same(parse_prompt_attention(text), want)


# ------------------------------------------------------------------------------------------------ chunking
BOS, EOS, COMMA = 900, 901, 5


def _chunks(ids, weight=1.0):
    from b200sd.prompts import chunk_tokens
    return chunk_tokens([(ids, weight, False)], BOS, EOS, COMMA)


def _body(chunk):
    """the prompt tokens of a chunk: between BOS and the EOS padding"""
    assert chunk[0] == BOS and chunk[-1] == EOS and len(chunk) == 77
    body = chunk[1:-1]
    while body and body[-1] == EOS:
        body = body[:-1]
    return body


@pytest.mark.parametrize("n,k", [(0, 1), (1, 1), (75, 1), (76, 2), (150, 2), (151, 3)])
def test_chunk_count(n, k):
    ids = [10 + i for i in range(n)]
    chunks, mults = _chunks(ids)
    assert len(chunks) == len(mults) == k
    assert sum((_body(c) for c in chunks), []) == ids


@pytest.mark.parametrize("comma_at,moved", [(60, True), (55, True), (54, False), (40, False)])
def test_comma_backtrack(comma_at, moved):
    """a full chunk followed by a non-comma token: the tokens after the chunk's last comma move to the next chunk when the
    comma is within its last 20 tokens (75 - 55 = 20 moves, 75 - 54 = 21 does not)"""
    ids = [10 + i for i in range(80)]
    ids[comma_at] = COMMA
    chunks, _ = _chunks(ids)
    assert len(chunks) == 2
    first = _body(chunks[0])
    assert first == (ids[:comma_at + 1] if moved else ids[:75])
    assert first + _body(chunks[1]) == ids


def test_no_backtrack_when_a_comma_follows_the_full_chunk():
    ids = [10 + i for i in range(75)] + [COMMA, 99]
    ids[70] = COMMA
    chunks, _ = _chunks(ids)
    assert _body(chunks[0]) == ids[:75] and _body(chunks[1]) == [COMMA, 99]


def _tok(text):
    return [ord(w[0]) for w in text.split()]


@pytest.mark.parametrize("text,bodies", [
    ("BREAK a", [[], [ord("a")]]),
    ("a BREAK b", [[ord("a")], [ord("b")]]),
    ("a BREAK", [[ord("a")]]),
    ("a BREAK BREAK b", [[ord("a")], [], [ord("b")]]),
    ("", [[]]),
])
def test_break(text, bodies):
    from b200sd.prompts import tokenize_prompt
    chunks, mults = tokenize_prompt(text, _tok, BOS, EOS, COMMA)
    assert [_body(c) for c in chunks] == bodies
    assert all(len(m) == 77 for m in mults)


def test_multipliers_line_up_with_tokens():
    from b200sd.prompts import tokenize_prompt
    chunks, mults = tokenize_prompt("x (a b) c [d] (e:1.5)", _tok, BOS, EOS, COMMA)
    assert len(chunks) == 1
    got = dict(zip(chunks[0][1:6], mults[0][1:6]))
    want = {ord("x"): 1.0, ord("a"): 1.1, ord("b"): 1.1, ord("c"): 1.0, ord("d"): 1 / 1.1}
    assert chunks[0][1:7] == [ord(t) for t in "xabcde"]
    assert all(abs(got[k] - v) < 1e-12 for k, v in want.items()) and abs(mults[0][6] - 1.5) < 1e-12
    assert mults[0][0] == 1.0 and all(m == 1.0 for m in mults[0][7:])   # BOS, EOS and padding


# ------------------------------------------------------------------------------------------------ tokenisers
@pytest.mark.parametrize("prompts", [["a b c"], ["", ""], ["a photo of a cat, highly detailed: 8k"],
                                     [" ".join(f"w{i}" for i in range(75))], ["one", "two words"]])
def test_hashed_tokenize_prompts_equals_synthetic_tokens(monkeypatch, prompts):
    from b200sd import factory
    monkeypatch.delenv("SD_TOKENIZER", raising=False)
    ids, mult = factory.tokenize_prompts(prompts, 1000)
    assert torch.equal(ids, factory.synthetic_tokens(prompts, 1000))
    assert bool((mult == 1.0).all()) and mult.dtype == torch.float32


def test_hashed_tokenize_prompts_long_and_weighted(monkeypatch):
    from b200sd import factory
    monkeypatch.delenv("SD_TOKENIZER", raising=False)
    long = " ".join(f"w{i}" for i in range(100))
    ids, mult = factory.tokenize_prompts([long, "(a:1.3) BREAK b"], 1000)
    assert ids.shape == mult.shape == (2, 154)
    plain = factory.synthetic_tokens([long], 1000)[0]
    assert torch.equal(ids[0, :77], plain)                         # the first 75 words, as today
    assert int(ids[0, 77]) == 998 and int(ids[1, 77]) == 998        # BOS of the second chunk
    assert abs(float(mult[1, 1]) - 1.3) < 1e-6 and float(mult[1, 2]) == 1.0


# ------------------------------------------------------------------------------------------------ engine, emulated ops
@pytest.fixture()
def env(monkeypatch):
    from b200sd import config as C, engine as E, ops, synth
    from oracle import prompt_oracle as P, sd_oracle as O
    monkeypatch.delenv("SD_TOKENIZER", raising=False)
    ops_emulator.install(monkeypatch, ops)
    monkeypatch.setattr(ops, "attention", attention_varlen)
    monkeypatch.setattr(E.SDEngine, "_require_cuda", False)
    cfgs = (C.TINY_UNET, C.TINY_VAE, C.TINY_CLIP)
    sd = synth.make_state_dict(*cfgs, seed=0)
    eng = E.SDEngine(sd, *cfgs, device="cpu", dtype=torch.float32, use_graphs=False, vae_chunk=2)
    return E, O, P, cfgs, sd, eng


def test_emulated_varlen_attention_matches_masked_softmax():
    g = torch.Generator().manual_seed(0)
    b, heads, sq, skv, d, dp = 3, 2, 5, 154, 8, 16
    q, k, v = (torch.randn((b, s, heads * dp), generator=g) for s in (sq, skv, skv))
    lens = torch.tensor([1, 77, 154], dtype=torch.int32)
    out = torch.zeros((b, sq, heads * d))
    attention_varlen(q, k, v, out, heads, d, dp, 0.3, kv_len=lens)
    qh, kh, vh = (t.reshape(b, -1, heads, dp)[..., :d].permute(0, 2, 1, 3) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) * 0.3
    s = s.masked_fill(torch.arange(skv)[None, None, None, :] >= lens[:, None, None, None], float("-inf"))
    ref = (torch.softmax(s, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(b, sq, heads * d)
    assert torch.allclose(out, ref, atol=1e-5, rtol=1e-5)


def _prompts(E, vocab):
    from b200sd import factory
    long = "a (red:1.3) house " + " ".join(f"w{i}" for i in range(90)) + ", [blue] sky"
    return factory.tokenize_prompts([long] * 2, vocab), factory.tokenize_prompts(["(ugly) text"] * 2, vocab)


@pytest.mark.parametrize("sampler", ["DDIM", "Euler a", "Heun"])
def test_two_chunk_weighted_prompt_matches_oracle(env, sampler):
    E, O, P, cfgs, sd, eng = env
    (ids, mult), (nids, nmult) = _prompts(E, cfgs[2].vocab)
    assert ids.shape[1] == 154 and nids.shape[1] == 77 and bool((mult != 1).any()) and bool((nmult != 1).any())
    b, hw, steps = 2, 8, 4
    cond = P.encode_sd1(sd, cfgs[2], ids, mult)
    unc = P.encode_sd1(sd, cfgs[2], nids, nmult)
    assert torch.allclose(eng.encode_prompts(ids, multipliers=mult), cond, atol=1e-4, rtol=1e-4)
    assert torch.allclose(eng.encode_prompts(nids, multipliers=nmult), unc, atol=1e-4, rtol=1e-4)
    pr = eng.program(sampler, None, steps)
    nz = E.per_image_noise(77, b, (4, hw, hw), 1 + pr.draws)
    with torch.no_grad():
        ref = P.sample(sd, cfgs[0], cond, unc, sampler, steps, 7.0, nz[0],
                       draws=list(nz[1:]))
    got = eng.txt2img(ids, nids, 77, steps=steps, cfg_scale=7.0, height=hw * 8, width=hw * 8, sampler=sampler,
                      multipliers=mult, neg_multipliers=nmult)
    plan = eng.plan(b, hw, hw)
    assert plan.ctx_cap == 154 and plan.kv_len.tolist() == [154, 154, 77, 77]
    z = plan.x.reshape(b, hw, hw, 4).permute(0, 3, 1, 2)
    assert float((z - ref).abs().max()) <= 1e-3 * float(ref.abs().max())
    assert got.shape[0] == b and got.dtype == torch.uint8


def test_separate_cfg_differs_from_padded_batch(env):
    """the oracle's separate cond / uncond calls are not the same as one call on zero-padded contexts: the engine must
    not silently attend to the padding"""
    E, O, P, cfgs, sd, eng = env
    (ids, mult), (nids, nmult) = _prompts(E, cfgs[2].vocab)
    cond, unc = P.encode_sd1(sd, cfgs[2], ids, mult), P.encode_sd1(sd, cfgs[2], nids, nmult)
    c, u, lc, lu = P.pad_pair(cond, unc)
    x = O.per_image_noise(5, 2, (4, 8, 8))
    t = torch.full((4,), 500.0)
    with torch.no_grad():
        sep = P.cfg_unet(sd, cfgs[0], lc, lu)(torch.cat([x, x]), t, torch.cat([c, u]))
        pad = O.unet_forward(sd, cfgs[0], torch.cat([x, x]), t, torch.cat([c, u]))
    assert torch.allclose(sep[:2], pad[:2], atol=1e-5) and not torch.allclose(sep[2:], pad[2:], atol=1e-4)
    plan = eng.plan(2, 8, 8)
    plan.set_context(cond, unc)
    plan.table[:1].copy_(eng.temb.table(torch.tensor([500.0])))
    plan.x.copy_(x.permute(0, 2, 3, 1).reshape(2, 64, 4))
    from b200sd import ops
    ops.pack_unet_input(plan.x, plan.unet.xin, 1.0)
    ops.select_step(plan.table, plan.step, plan.unet.cur_bias)
    plan.unet.run()
    got = plan.unet.eps[..., :4].reshape(4, 8, 8, 4).permute(0, 3, 1, 2)
    assert float((got - sep).abs().max()) <= 2e-4 * float(sep.abs().max())


def test_short_request_after_growth_matches_fresh_engine(env):
    E, O, P, cfgs, sd, eng = env
    from b200sd import factory
    tok, neg = factory.synthetic_tokens(["a b"] * 2, 1000), factory.synthetic_tokens([""] * 2, 1000)
    kw = dict(steps=3, cfg_scale=7.0, height=64, width=64, sampler="DDIM")
    before = eng.txt2img(tok, neg, 5, **kw)
    (ids, mult), _ = _prompts(E, 1000)
    eng.txt2img(ids, neg, 5, multipliers=mult, **kw)
    assert eng.plan(2, 8, 8).ctx_cap == 154
    after = eng.txt2img(tok, neg, 5, **kw)
    assert eng.plan(2, 8, 8).kv_len.tolist() == [77] * 4
    assert (after.int() - before.int()).abs().max() <= 1


def test_all_one_multipliers_are_the_unweighted_path(env):
    E, O, P, cfgs, sd, eng = env
    (ids, _), _ = _prompts(E, 1000)
    a = eng.encode_prompts(ids)
    assert torch.equal(a, eng.encode_prompts(ids, multipliers=torch.ones(ids.shape)))


def test_worker_interprets_prompt_syntax(monkeypatch, env):
    E, O, P, cfgs, sd, eng = env
    from b200sd import factory
    from scripts.spartan import pmodels, shared as sh
    from scripts.spartan.local_worker import LocalGPUWorker
    logging.getLogger("distributed").setLevel(logging.ERROR)
    sh.benchmark_payload = pmodels.Benchmark_Payload()
    wk = LocalGPUWorker(0, lambda d: eng, avg_ipm=600.0)
    prompt = "a (word:1.3) BREAK " + " ".join(f"w{i}" for i in range(80))
    payload = {"prompt": prompt, "negative_prompt": "[bad]", "seed": 30, "subseed": 4, "subseed_strength": 0,
               "batch_size": 2, "n_iter": 1, "steps": 3, "width": 64, "height": 64, "sampler_name": "DDIM", "cfg_scale": 7.0}
    wk.request(payload, None, False)
    ids, mult = factory.tokenize_prompts([prompt] * 2, 1000)
    nids, nmult = factory.tokenize_prompts(["[bad]"] * 2, 1000)
    assert ids.shape[1] == 231
    direct = eng.txt2img(ids, nids, 30, steps=3, cfg_scale=7.0, height=64, width=64, sampler="DDIM", multipliers=mult,
                         neg_multipliers=nmult)
    assert torch.equal(wk.response["tensors"], direct.to(torch.uint8))
