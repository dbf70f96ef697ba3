"""Time SD 2.x (768-v) txt2img at 768x768 with seeded synthetic weights, and each eps fused step against its v twin.

  * Requests: batch 16, 20 steps, CFG 7, CUDA graphs on, for "DDIM", "Euler a" and "DPM++ 2M Karras" on an SDEngine with
    prediction="v".  Each request is timed with CUDA events around the whole call (text encoding, sampling, decode),
    after one warm-up request per sampler; the median of `--reps` (3) gives images/s.
  * Fused steps: at the same shape (2 x 16 UNet outputs of 96 x 96 pixels), b200sd_cfg_{ddim,euler_a,dpmpp_2m}_step and
    their _v twins, `--iters` launches each (CUDA events, median of 5 rounds), fp16.

Prints one JSON line with the card's name and power limit.  Writes nothing.

    python tools/bench_sd21.py [--reps 3] [--batch 16] [--steps 20]
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


def time_steps(b: int, hw: int, iters: int):
    """us per launch of each fused step kernel and its v twin"""
    import torch
    from b200sd import ops
    dev = "cuda:0"
    v = torch.randn((2 * b, hw, 32), device=dev).half()
    x = torch.randn((b, hw, 4), device=dev)
    old = torch.zeros_like(x)
    xin = torch.zeros((2 * b, hw, 64), device=dev, dtype=torch.float16)
    noise = torch.randn((1, b, hw, 4), device=dev)
    step = torch.zeros((1,), device=dev, dtype=torch.int32)
    c4 = torch.tensor([[0.5, 0.8, 0.6, 0.7]], device=dev)
    c8 = torch.tensor([[2.0, 1.5, 0.5, 0.2, 0.4, 0.4, 0.45, 0.0]], device=dev)
    c8e = torch.tensor([[2.0, 1.5, 0.5, 0.2, 0.4, 0.0, 0.0, 0.0]], device=dev)
    calls = {
        "ddim": lambda: ops.cfg_ddim_step(v, x, xin, 7.0, c4, step),
        "ddim_v": lambda: ops.cfg_ddim_step_v(v, x, xin, 7.0, c4, step),
        "euler_a": lambda: ops.cfg_euler_a_step(v, x, noise, xin, 7.0, c4, step),
        "euler_a_v": lambda: ops.cfg_euler_a_step_v(v, x, noise, xin, 7.0, c8, step),
        "dpmpp_2m": lambda: ops.cfg_dpmpp_2m_step(v, x, old, xin, 7.0, c8e, step),
        "dpmpp_2m_v": lambda: ops.cfg_dpmpp_2m_step_v(v, x, old, xin, 7.0, c8, step),
    }
    res = {}
    for _ in range(5):
        for name, fn in calls.items():
            for _ in range(10):
                step.zero_()
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                step.zero_()   # one coefficient row: every launch reads row 0
                fn()
            e1.record()
            torch.cuda.synchronize()
            res.setdefault(name, []).append(e0.elapsed_time(e1) * 1000.0 / iters)
    return {k: round(statistics.median(t), 2) for k, t in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed requests per sampler")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=200, help="launches per fused-step timing round")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O
    cfgs = (C.SD21_UNET, C.SD21_VAE, C.SD21_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True, prediction="v")
    b, px = args.batch, 768
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    neg[:, 2:] = 0   # SD 2.x pads with id 0 after the first EOS

    def request(sampler):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.txt2img(tok, neg, 1234, steps=args.steps, cfg_scale=7.0, height=px, width=px, sampler=sampler)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    res = {"workload": f"SD 2.x 768-v txt2img {px}x{px} batch {b}, {args.steps} steps, CFG 7, fp16, synthetic weights, "
                       "CUDA graphs", "card": card(), "reps": args.reps}
    for sampler in ("DDIM", "Euler a", "DPM++ 2M Karras"):
        request(sampler)
        ts = [request(sampler) for _ in range(args.reps)]
        med = statistics.median(ts)
        res[sampler] = {"ms_median": round(med, 1), "ms_min": round(min(ts), 1), "ms_max": round(max(ts), 1),
                        "images_per_s": round(b / (med / 1000.0), 3), "unet_evals": eng.last_unet_evals}
    eng.release()
    res["fused_step_us"] = time_steps(b, (px // 8) ** 2, args.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
