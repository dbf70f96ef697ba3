"""Time requests with LoRA networks merged against requests without, and the merge itself.

  * Requests: SD1.5 512x512, batch 32, 20 DDIM steps, and SDXL 1024x1024, batch 16, 30 Euler a steps, with no LoRA, one
    LoRA and three stacked (seeded synthetic kohya LoCon networks of rank 32 on every UNet and text-tower layer), the
    modes alternated within each of `--reps` rounds.  CFG 7, CUDA graphs.  Each timed request follows an untimed one of
    the same mode, so the networks are merged already (what a client repeating a style pays); CUDA events around the
    whole call; the median gives images/s.
  * The merge per set switch (the ops.lora_merge call: descriptor upload and launch, device events around it; plain ->
    one LoRA -> three -> plain, median of `--reps` rounds), with its bytes (pristine reads + weight writes + factor reads) and FLOPs
    (2 x rows x cols x R per target), and the bound they give at the H100 SXM data sheet's 3.35 TB/s and 67 TFLOP/s fp32.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing.

    python tools/bench_lora.py [--reps 3] [--skip-sd15] [--skip-sdxl]
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

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12


def _events():
    import torch
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def _nets(eng, n, rank):
    from b200sd import lora as L, synth
    form = "compvis" if eng.clip_cfg.xl_width else "diffusers"
    out = []
    for i in range(n):
        sd = synth.make_lora_state_dict(eng.unet_cfg, eng.clip_cfg, seed=100 + i, rank=rank, form=form)
        out.append((L.load_state_dict(f"bench{i}", sd, key=("bench", i, rank)), L.LoraRef(f"bench{i}", 0.7, 0.7)))
    return out


def _merge_work(eng, nets):
    """(bytes, flops) of the launch that merges `nets` from pristine weights"""
    from b200sd import lora as L
    owners = eng._lora_owners()
    groups = L.plan(L.resolve(eng.lora_key_table(), nets), {n: pl for n, (_, pl) in owners.items()},
                    {n: t for n, (t, _) in owners.items()}, eng.device)
    nbytes = flops = 0
    for (owner, name), gs in groups.items():
        w = owners[owner][0][name]
        nbytes += 2 * w.numel() * w.element_size()
        for g in gs:
            if g.U is not None:
                nbytes += 4 * (g.U.numel() + g.D.numel())
                flops += 2 * (g.hi - g.lo) * w.shape[1] * g.U.shape[1]
    return nbytes, flops


def time_merge(eng, sets, reps):
    """device ms of the b200sd_lora_merge launch alone for each switch of the cycle plain -> 1 -> 3 -> plain"""
    import torch
    from b200sd import ops
    real = ops.lora_merge
    times = {}

    def timed(targets):
        e0, e1 = _events()
        e0.record()
        buf = real(targets)
        e1.record()
        timed.last.append((e0, e1))
        return buf

    eng.set_loras(())
    ops.lora_merge = timed
    try:
        for _ in range(reps):
            for name, nets in sets:
                timed.last = []
                eng.set_loras(nets)
                torch.cuda.synchronize()
                times.setdefault(name, []).append(sum(a.elapsed_time(b) for a, b in timed.last))
    finally:
        ops.lora_merge = real
    return {k: round(statistics.median(v), 3) for k, v in times.items()}


def run(eng, b, hw, steps, sampler, reps, rank):
    import torch
    from b200sd.factory import tokenize_prompts
    vocab = eng.clip_cfg.vocab
    tok = tokenize_prompts(["a cat in a garden"] * b, vocab)[0]
    neg = tokenize_prompts([""] * b, vocab)[0]
    one, three = _nets(eng, 1, rank), _nets(eng, 3, rank)
    modes = {"none": None, "one": one, "three": three}

    def call(m):
        return eng.txt2img(tok, neg, 1234, steps=steps, cfg_scale=7.0, height=8 * hw, width=8 * hw, sampler=sampler,
                           loras=modes[m])

    times = {m: [] for m in modes}
    for _ in range(reps):
        for m in modes:
            call(m)
            torch.cuda.synchronize()
            e0, e1 = _events()
            e0.record()
            call(m)
            e1.record()
            torch.cuda.synchronize()
            times[m].append(e0.elapsed_time(e1))
    res = {}
    for m in modes:
        med = statistics.median(times[m])
        res[m] = {"ms_median": round(med, 1), "ms_min": round(min(times[m]), 1), "ms_max": round(max(times[m]), 1),
                  "images_per_s": round(b / (med / 1000.0), 3)}
    for m in ("one", "three"):
        res[m]["vs_none"] = round(res[m]["images_per_s"] / res["none"]["images_per_s"], 4)
    merge_ms = time_merge(eng, [("plain->one", one), ("one->three", three), ("three->plain", ())], reps)
    res["merge"] = {}
    for name, nets, key in (("one", one, "plain->one"), ("three", three, "one->three")):
        nbytes, flops = _merge_work(eng, nets)
        bound = max(nbytes / HBM_BPS, flops / FP32_FLOPS) * 1e3
        res["merge"][name] = {"ms": merge_ms[key], "GB": round(nbytes / 1e9, 3), "GFLOP": round(flops / 1e9, 2),
                              "bound_ms": round(bound, 3), "bound_by": "bytes" if nbytes / HBM_BPS > flops / FP32_FLOPS
                              else "fp32 FLOPs", "share_of_bound": round(bound / merge_ms[key], 3)}
    res["merge"]["restore_ms"] = merge_ms["three->plain"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed requests per mode and model")
    ap.add_argument("--rank", type=int, default=32)
    ap.add_argument("--skip-sd15", action="store_true")
    ap.add_argument("--skip-sdxl", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import config as C, engine as E, synth
    out = {"card": card(), "rank": args.rank}
    if not args.skip_sd15:
        cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
        eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
        out["sd15_512_b32_ddim20"] = run(eng, 32, 64, 20, "DDIM", args.reps, args.rank)
        eng.release()
        del eng
        torch.cuda.empty_cache()
    if not args.skip_sdxl:
        cfgs = (C.SDXL_UNET, C.SDXL_VAE, C.SDXL_CLIP)
        eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", dtype=torch.bfloat16,
                         use_graphs=True)
        out["sdxl_1024_b16_euler_a30"] = run(eng, 16, 128, 30, "Euler a", args.reps, args.rank)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
