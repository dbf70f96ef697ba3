"""Time prompt editing `[a:b:0.5]` and alternation `[a|b]` against the plain prompt.

  * Requests: SD1.5 512x512, batch 32, 20 DDIM steps, and SDXL 1024x1024, batch 16, 30 Euler a steps; the prompt plain
    ("a cat in a garden"), edited halfway ("a [cat:dog:0.5] in a garden": one switch after evaluation 0) and alternated
    ("a [cat|dog] in a garden": a switch before every evaluation), the modes alternated within each of `--reps` rounds.
    CFG 7, CUDA graphs, seeded synthetic weights.  Each timed request follows a release of the plans and an untimed
    warm-up of its mode; CUDA events around the whole call; the median gives images/s.
  * The `ctx` graph alone (select_context and the K/V projections of every attn2): CUDA events around `--iters` replays,
    median of 5 rounds, at each workload's shape.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing.

    python tools/bench_prompt_editing.py [--reps 3] [--skip-sd15] [--skip-sdxl]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-diffusion-webui-distributed_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_prompt_lengths import card  # noqa: E402

PROMPTS = {"plain": "a cat in a garden", "edit": "a [cat:dog:0.5] in a garden", "alternate": "a [cat|dog] in a garden"}


def _events():
    import torch
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def _schedule(text, steps, b, vocab):
    """(tokens [b, 77k], schedule or None) as LocalGPUWorker builds them"""
    from b200sd.engine import PromptSchedule
    from b200sd.factory import tokenize_prompts
    from b200sd.prompts import prompt_schedule
    sch = prompt_schedule(text, steps)
    ids, _ = tokenize_prompts([t for _, t in sch], vocab)
    neg, _ = tokenize_prompts([""], vocab)
    if len(sch) == 1:
        return ids.expand(b, -1).contiguous(), None
    return ids[:1].expand(b, -1).contiguous(), (PromptSchedule([e for e, _ in sch], ids),
                                                 PromptSchedule([steps], neg))


def time_requests(eng, call, b, reps):
    import torch
    times = {m: [] for m in PROMPTS}
    for _ in range(reps):
        for m in PROMPTS:
            eng.release()
            call(m)
            torch.cuda.synchronize()
            e0, e1 = _events()
            e0.record()
            call(m)
            e1.record()
            torch.cuda.synchronize()
            times[m].append(e0.elapsed_time(e1))
    out = {}
    for m in PROMPTS:
        med = statistics.median(times[m])
        out[m] = {"ms_median": round(med, 1), "ms_min": round(min(times[m]), 1), "ms_max": round(max(times[m]), 1),
                  "images_per_s": round(b / (med / 1000.0), 3)}
    for m in ("edit", "alternate"):
        out[m]["vs_plain"] = round(out[m]["images_per_s"] / out["plain"]["images_per_s"], 4)
    return out


def time_ctx_graph(eng, b, hw, iters):
    """ms of one replay of the plan's ctx graph (the last scheduled request left it captured)"""
    import torch
    plan = eng.plan(b, hw, hw)
    name = next(n for n in plan.graphs if n.startswith("ctx"))
    g = plan.graphs[name]
    plan.step.zero_()
    for _ in range(3):
        g.replay()
    rounds = []
    for _ in range(5):
        e0, e1 = _events()
        e0.record()
        for _ in range(iters):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        rounds.append(e0.elapsed_time(e1) / iters)
    return {"graph": name, "kernels": plan.graph_launches[name], "ms_median": round(statistics.median(rounds), 4)}


def run(eng, b, hw, steps, sampler, vocab, reps, iters):
    cases = {m: _schedule(t, steps, b, vocab) for m, t in PROMPTS.items()}
    neg = _schedule("", steps, b, vocab)[0]

    def call(m):
        tok, sched = cases[m]
        return eng.txt2img(tok, neg, 1234, steps=steps, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler=sampler,
                           schedule=sched)
    res = time_requests(eng, call, b, reps)
    call("alternate")
    res["ctx_graph"] = time_ctx_graph(eng, b, hw, iters)
    res["ctx_switches"] = {"edit": 2, "alternate": eng.last_unet_evals - 1}   # evaluation 0 and the change points
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed requests per mode and model")
    ap.add_argument("--iters", type=int, default=50, help="ctx graph replays per timing round")
    ap.add_argument("--skip-sd15", action="store_true")
    ap.add_argument("--skip-sdxl", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import config as C, engine as E, synth
    res = {"card": card(), "reps": args.reps}

    if not args.skip_sd15:
        cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
        eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
        res["sd15"] = {"workload": "SD1.5 txt2img 512x512 batch 32, 20 DDIM steps, CFG 7, fp16, CUDA graphs",
                       **run(eng, 32, 64, 20, "DDIM", cfgs[2].vocab, args.reps, args.iters)}
        eng.release()
        del eng
        torch.cuda.empty_cache()

    if not args.skip_sdxl:
        cfgs = (C.SDXL_UNET, C.SDXL_VAE, C.SDXL_CLIP)
        eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True,
                         dtype=torch.bfloat16)
        res["sdxl"] = {"workload": "SDXL txt2img 1024x1024 batch 16, 30 Euler a steps, CFG 7, bf16, CUDA graphs",
                       **run(eng, 16, 128, 30, "Euler a", cfgs[2].vocab, args.reps, args.iters)}
        eng.release()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
