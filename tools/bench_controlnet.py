"""Time SD1.5 txt2img with 0, 1 and 2 ControlNet units (seeded synthetic UNet and ControlNets).

  * Requests: the SD1.5 workload of bench.py — 512x512, batch 32, 20 DDIM steps, CFG 7, fp16, CUDA graphs — with 0, 1 and
    2 units (weight 1, window [0, 1], one 512x512 control map each).  The three configurations alternate within each of
    `--reps` rounds after one warm-up request each; every request is timed with CUDA events around the whole call; the
    median gives images/s.
  * UNet evaluation: one [cond | uncond] evaluation with the same units active, captured in a CUDA graph and replayed
    `--iters` times between CUDA events (median of 5 rounds).
  * FLOPs: the ControlNet's share of one evaluation, from the algorithmic FLOPs of the program's GEMM / conv /
    attention launches (op_flops, the rule of bench.py's roofline).

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing.

    python tools/bench_controlnet.py [--reps 3] [--batch 32] [--steps 20]
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


def program_flops(op_list, op_flops) -> float:
    """algorithmic FLOPs of a list of (fn, args, kwargs) launches: 2 M N K of linears and convs (or their recorded
    algo_flops), 4 B heads Sq Skv d of attention"""
    total = 0.0
    for (fn, a, k), algo in zip(op_list, op_flops):
        name = getattr(fn, "__name__", "op")
        if name in ("linear", "conv2d"):
            m = (a[0].numel() // a[0].shape[-1]) if name == "linear" else (a[2].numel() // a[2].shape[-1])
            total += 2.0 * m * a[1].shape[0] * a[1].shape[1] if algo is None else algo
        elif name == "attention":
            total += 4.0 * a[0].shape[0] * a[4] * a[0].shape[1] * a[1].shape[1] * a[5]
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed requests per configuration")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=10, help="graph replays per UNet-evaluation timing round")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import config as C, engine as E, ops, synth
    from b200sd.unet_exec import ControlNetWeights
    from oracle import sd_oracle as O
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    dev = torch.device("cuda:0")
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
    cws = [ControlNetWeights(synth.make_controlnet_state_dict(C.SD15_UNET, seed=s), C.SD15_UNET, dev, name=f"cn{s}")
           for s in (1, 2)]
    b, px = args.batch, 512
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    g = torch.Generator().manual_seed(0)
    hints = [torch.randint(0, 256, (px, px, 3), generator=g, dtype=torch.uint8) for _ in cws]
    configs = {n: [(cws[k], hints[k], 1.0, 0.0, 1.0) for k in range(n)] for n in (0, 1, 2)}

    def request(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.txt2img(tok, neg, 1234, steps=args.steps, cfg_scale=7.0, height=px, width=px, sampler="DDIM",
                    controls=configs[n] or None)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    times = {n: [] for n in configs}
    for n in configs:
        request(n)
    for _ in range(args.reps):
        for n in configs:
            times[n].append(request(n))
    evals = eng.last_unet_evals
    plan = eng.plan(b, px // 8, px // 8)
    unet = plan.unet
    base = program_flops(unet.ops, unet.op_flops)
    res = {"workload": f"SD1.5 txt2img {px}x{px} batch {b}, {args.steps} DDIM steps ({evals} UNet evaluations), CFG 7, "
                       "fp16, synthetic weights, CUDA graphs", "card": card(), "reps": args.reps}
    stream = torch.cuda.Stream(device=dev)
    for n in configs:
        active = tuple(range(n))
        eng._set_controls(plan, configs[n])   # the last request's units stay in their slots; refreshed for clarity
        gr = torch.cuda.CUDAGraph()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            ops.select_step(plan.table, plan.step, unet.cur_bias)
            unet.run(active)
        torch.cuda.current_stream().wait_stream(stream)
        with torch.cuda.graph(gr, stream=stream):
            unet.run(active)
        rounds = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            rounds.append(e0.elapsed_time(e1) / args.iters)
        del gr
        cn = sum(program_flops(unet.segments[s].ops, unet.segments[s].op_flops) for s in active)
        med = statistics.median(times[n])
        res[f"units_{n}"] = {"ms_median": round(med, 1), "ms_min": round(min(times[n]), 1),
                             "ms_max": round(max(times[n]), 1), "images_per_s": round(b / (med / 1000.0), 3),
                             "ms_per_unet_eval": round(statistics.median(rounds), 2),
                             "eval_tflop": round((base + cn) / 1e12, 3),
                             "controlnet_flop_share": round(cn / (base + cn), 4)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
