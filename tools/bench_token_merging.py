"""Time token merging (sdwui's token_merging_ratio) against the same requests without it.

  * Requests: SD1.5 512x512, batch 32, 20 DDIM steps, and SD 2.x 768x768 (N = 9216 level-0 tokens), batch 16, 20 DDIM
    steps (v-prediction), at ratios 0 / 0.3 / 0.5 alternated within each of `--reps` rounds; the hires fix 512 -> 1024
    ("Latent"), batch 16, 20 + 20 DDIM steps, at ratio_hr 0 and 0.5 (first pass unmerged).  CFG 7, CUDA graphs, seeded
    synthetic weights.  Each timed request follows a release of the plans and an untimed warm-up of its mode; CUDA events
    around the whole call; the median gives images/s.
  * Peak device memory: torch.cuda.max_memory_allocated over the warm-up request of each mode (weights included).
  * Kernel times (CUDA events around `--iters` launches, median of 5 rounds) at the SD1.5 level-0 shapes (64 rows =
    batch 32 with CFG, 64x64 tokens, C = 320, 8 heads of d = 40): tome_match, tome_merge, tome_unmerge_add, and the
    self-attention with N and with N - r tokens.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing.

    python tools/bench_token_merging.py [--reps 3] [--skip-sd21] [--skip-hires]
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


def _events():
    import torch
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def time_requests(eng, call, b, modes, reps):
    """per mode: ms per request and peak bytes of call(mode), the modes alternated"""
    import torch
    times, peak = {m: [] for m in modes}, {}
    for _ in range(reps):
        for m in modes:
            eng.release()
            torch.cuda.reset_peak_memory_stats()
            call(m)
            torch.cuda.synchronize()
            peak[m] = max(peak.get(m, 0), torch.cuda.max_memory_allocated())
            e0, e1 = _events()
            e0.record()
            call(m)
            e1.record()
            torch.cuda.synchronize()
            times[m].append(e0.elapsed_time(e1))
    out = {}
    for m in modes:
        med = statistics.median(times[m])
        out[f"ratio_{m}"] = {"ms_median": round(med, 1), "ms_min": round(min(times[m]), 1),
                             "ms_max": round(max(times[m]), 1), "images_per_s": round(b / (med / 1000.0), 3),
                             "peak_alloc_gib": round(peak[m] / 2 ** 30, 2)}
    base = out[f"ratio_{modes[0]}"]["images_per_s"]
    for m in modes[1:]:
        out[f"ratio_{m}"]["speedup"] = round(out[f"ratio_{m}"]["images_per_s"] / base, 4)
    return out


def _time(fn, iters):
    import torch
    for _ in range(3):
        fn()
    rounds = []
    for _ in range(5):
        e0, e1 = _events()
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        rounds.append(e0.elapsed_time(e1) / iters)
    return round(statistics.median(rounds) * 1000, 1)


def time_kernels(iters):
    import torch
    from b200sd import ops
    from b200sd.unet_exec import _pad64
    nb, h, w, c, heads = 64, 64, 64, 320, 8
    d = c // heads
    dp = _pad64(d)
    n = h * w
    x = torch.randn((nb, n, c), device="cuda", dtype=torch.float16)
    res = {"shape": f"{nb} rows x {h}x{w} tokens x C={c}"}
    for ratio in (0.3, 0.5):
        r = min(n - n // 4, int(n * ratio))
        nm = n - r
        slot, members = (torch.zeros((nb, n), dtype=torch.int32, device="cuda") for _ in range(2))
        seg = torch.zeros((nb, nm + 1), dtype=torch.int32, device="cuda")
        ws = torch.empty((ops.tome_workspace_bytes(nb, h, w, c),), dtype=torch.uint8, device="cuda")
        y = torch.empty((nb, nm, c), device="cuda", dtype=torch.float16)
        o = torch.empty_like(x)
        res[f"ratio_{ratio}"] = {
            "r": r,
            "match_us": _time(lambda: ops.tome_match(x, h, w, r, slot, members, seg, ws), iters),
            "merge_us": _time(lambda: ops.tome_merge(x, members, seg, y), iters),
            "unmerge_add_us": _time(lambda: ops.tome_unmerge_add(x, y, slot, o), iters),
        }
    for ratio in (0.0, 0.3, 0.5):
        s = n - min(n - n // 4, int(n * ratio))
        qkv = torch.randn((nb, s, 3 * heads * dp), device="cuda", dtype=torch.float16)
        qkv.reshape(nb, s, 3, heads, dp)[:, :, 2, :, d] = 1.0
        q, k, v = (qkv[..., j * heads * dp:(j + 1) * heads * dp] for j in range(3))
        out = torch.empty((nb, s, c), device="cuda", dtype=torch.float16)
        res[f"self_attention_S{s}_us"] = _time(lambda: ops.attention(q, k, v, out, heads, d, dp, d ** -0.5, dp > d), iters)
        del qkv, out
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed requests per mode and model")
    ap.add_argument("--iters", type=int, default=20, help="kernel launches per timing round")
    ap.add_argument("--skip-sd21", action="store_true")
    ap.add_argument("--skip-hires", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import config as C, engine as E, synth
    from oracle import sd_oracle as O
    res = {"card": card(), "reps": args.reps, "kernels": time_kernels(args.iters)}
    modes = (0.0, 0.3, 0.5)

    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
    b = 32
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    sd15 = lambda m: eng.txt2img(tok, neg, 1234, steps=20, cfg_scale=7.0, height=512, width=512,  # noqa: E731
                                 sampler="DDIM", token_merging_ratio=m)
    res["sd15"] = {"workload": "SD1.5 txt2img 512x512 batch 32, 20 DDIM steps, CFG 7, fp16, CUDA graphs",
                   **time_requests(eng, sd15, b, modes, args.reps)}
    if not args.skip_hires:
        b = 16
        tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
        hr = lambda m: eng.txt2img_hires(tok, neg, 1234, steps=20, cfg_scale=7.0, height=512, width=512,  # noqa: E731
                                         hr_scale=2.0, denoising_strength=0.7, sampler="DDIM",
                                         token_merging_ratio_hr=m)
        res["sd15_hires"] = {"workload": "SD1.5 hires fix 512 -> 1024 (Latent) batch 16, 20 + 20 DDIM steps, CFG 7, "
                                         "ratio_hr", **time_requests(eng, hr, b, (0.0, 0.5), args.reps)}
    eng.release()
    del eng
    torch.cuda.empty_cache()

    if not args.skip_sd21:
        cfgs = (C.SD21_UNET, C.SD21_VAE, C.SD21_CLIP)
        eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True,
                         prediction="v")
        b = 16
        tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
        sd21 = lambda m: eng.txt2img(tok, neg, 1234, steps=20, cfg_scale=7.0, height=768, width=768,  # noqa: E731
                                     sampler="DDIM", token_merging_ratio=m)
        res["sd21"] = {"workload": "SD 2.x txt2img 768x768 batch 16, 20 DDIM steps, CFG 7, v-prediction, fp16, CUDA graphs",
                       **time_requests(eng, sd21, b, modes, args.reps)}
        eng.release()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
