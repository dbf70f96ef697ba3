"""Time seamless tiling (circular padding of every 3x3 conv) against the same requests without it.

  * Requests: SD1.5 512x512, batch 32, 20 DDIM steps, and SDXL-base 1024x1024, batch 16, Euler a (30 steps by default),
    CFG 7, CUDA graphs, seeded synthetic weights.  Per model, tiling off and on alternate within each of `--reps` rounds;
    each timed request follows an untimed warm-up of its mode on freshly built plans, and is timed with CUDA events around
    the whole call (UNet steps and VAE decode); the median gives images/s.
  * Peak device memory: torch.cuda.max_memory_allocated over the warm-up request of each mode, the other mode's plan
    released (weights included in both).
  * b200sd_pad_circular at the UNet's conv-input shapes (batch 32 with CFG: 64 rows) and the VAE decoder's (chunk of 8):
    CUDA events around `--iters` launches, median of 5 rounds; bytes moved = input read + padded output written, and
    that rate against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing.

    python tools/bench_tiling.py [--reps 3] [--sdxl-steps 30] [--skip-sdxl]
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

HBM_BYTES_PER_S = 3.35e12
# (N, H, W, C) of conv inputs: SD1.5 UNet at 512^2, batch 32 with CFG; the VAE decoder at 512^2, chunk of 8 images
PAD_SHAPES = {"unet": [(64, 64, 64, 320), (64, 64, 64, 640), (64, 64, 64, 960), (64, 32, 32, 640), (64, 16, 16, 1280),
                       (64, 8, 8, 1280)],
              "vae": [(8, 64, 64, 512), (8, 128, 128, 512), (8, 256, 256, 256), (8, 512, 512, 128)]}


def _events():
    import torch
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def time_requests(eng, call, b, reps):
    """per mode: ms per request and peak bytes of call(tiling), off and on alternated.  Only one mode's plan is resident
    at a time (two SDXL plans at batch 16 do not fit in 80 GB together): each timed request follows a release of the
    plans and one untimed warm-up request that builds the mode's plan and graphs."""
    import torch
    times, peak = {False: [], True: []}, {}
    for _ in range(reps):
        for tiling in (False, True):
            eng.release()
            torch.cuda.reset_peak_memory_stats()
            call(tiling)
            torch.cuda.synchronize()
            peak[tiling] = max(peak.get(tiling, 0), torch.cuda.max_memory_allocated())
            e0, e1 = _events()
            e0.record()
            call(tiling)
            e1.record()
            torch.cuda.synchronize()
            times[tiling].append(e0.elapsed_time(e1))
    out = {}
    for tiling in (False, True):
        med = statistics.median(times[tiling])
        out["tiling_on" if tiling else "tiling_off"] = {
            "ms_median": round(med, 1), "ms_min": round(min(times[tiling]), 1), "ms_max": round(max(times[tiling]), 1),
            "images_per_s": round(b / (med / 1000.0), 3), "peak_alloc_gib": round(peak[tiling] / 2 ** 30, 2)}
    out["on_over_off_images_per_s"] = round(out["tiling_on"]["images_per_s"] / out["tiling_off"]["images_per_s"], 4)
    return out


def time_pads(iters):
    import torch
    from b200sd import ops
    res = {}
    for kind, shapes in PAD_SHAPES.items():
        for n, h, w, c in shapes:
            x = torch.randn((n, h, w, c), device="cuda", dtype=torch.float16)
            y = torch.empty((n, h + 2, w + 2, c), device="cuda", dtype=torch.float16)
            for _ in range(3):
                ops.pad_circular(x, y, 1)
            rounds = []
            for _ in range(5):
                e0, e1 = _events()
                e0.record()
                for _ in range(iters):
                    ops.pad_circular(x, y, 1)
                e1.record()
                torch.cuda.synchronize()
                rounds.append(e0.elapsed_time(e1) / iters)
            ms = statistics.median(rounds)
            nbytes = 2 * (x.numel() + y.numel())
            res[f"{kind} {n}x{h}x{w}x{c}"] = {"us": round(ms * 1000, 1), "bytes": nbytes,
                                               "tb_per_s": round(nbytes / (ms / 1000) / 1e12, 3),
                                               "share_of_3.35": round(nbytes / (ms / 1000) / HBM_BYTES_PER_S, 3)}
            del x, y
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed requests per mode and model")
    ap.add_argument("--sdxl-steps", type=int, default=30)
    ap.add_argument("--iters", type=int, default=50, help="pad launches per timing round")
    ap.add_argument("--skip-sdxl", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O
    res = {"card": card(), "reps": args.reps, "pad_circular": time_pads(args.iters)}

    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
    b = 32
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    sd15 = lambda tiling: eng.txt2img(tok, neg, 1234, steps=20, cfg_scale=7.0, height=512, width=512,  # noqa: E731
                                      sampler="DDIM", tiling=tiling)
    res["sd15"] = {"workload": "SD1.5 txt2img 512x512 batch 32, 20 DDIM steps, CFG 7, fp16, CUDA graphs",
                   **time_requests(eng, sd15, b, args.reps)}
    eng.release()
    del eng
    torch.cuda.empty_cache()

    if not args.skip_sdxl:
        cfgs = (C.SDXL_UNET, C.SDXL_VAE, C.SDXL_CLIP)
        eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", dtype=torch.bfloat16,
                         use_graphs=True)
        b = 16
        tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
        xl = lambda tiling: eng.txt2img(tok, neg, 1234, steps=args.sdxl_steps, cfg_scale=7.0, height=1024,  # noqa: E731
                                        width=1024, sampler="Euler a", tiling=tiling)
        res["sdxl"] = {"workload": f"SDXL-base txt2img 1024x1024 batch 16, {args.sdxl_steps} Euler a steps, CFG 7, bf16, "
                                   "CUDA graphs", **time_requests(eng, xl, b, args.reps)}
        eng.release()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
