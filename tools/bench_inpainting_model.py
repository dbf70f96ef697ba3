"""Time an SD1.5 inpainting checkpoint (9-channel UNet) against the plain SD1.5 model on the same requests.

  * Requests: SD1.5 512x512, batch 32, 20 DDIM steps, CFG 7, fp16, CUDA graphs, seeded synthetic weights:
      - img2img inpainting, "whole picture", denoising 0.75, one mask for the batch (the inpainting model also encodes
        the masked init images: one more VAE encode of 32 images);
      - txt2img (the inpainting model also encodes one gray image).
    Per workload, `sd15` and `sd15-inpainting` alternate within each of `--reps` rounds; each timed request follows a
    release of both engines' plans and one untimed warm-up request that rebuilds the configuration's plan and graphs, and
    is timed with CUDA events around the whole call (encodes, UNet steps, VAE decode); the median gives images/s.
  * Peak device memory: torch.cuda.max_memory_allocated over each warm-up request (both engines' weights are resident).

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing.

    python tools/bench_inpainting_model.py [--reps 3]
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


def time_configs(engines, call, b, reps):
    """per configuration: ms per request and peak bytes of call(engine), the configurations alternated"""
    import torch
    times, peak = {n: [] for n in engines}, {}
    for _ in range(reps):
        for name, eng in engines.items():
            for e in engines.values():
                e.release()
            torch.cuda.reset_peak_memory_stats()
            call(eng)
            torch.cuda.synchronize()
            peak[name] = max(peak.get(name, 0), torch.cuda.max_memory_allocated())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call(eng)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    out = {}
    for name in engines:
        med = statistics.median(times[name])
        out[name] = {"ms_median": round(med, 1), "ms_min": round(min(times[name]), 1),
                     "ms_max": round(max(times[name]), 1), "images_per_s": round(b / (med / 1000.0), 3),
                     "peak_alloc_gib": round(peak[name] / 2 ** 30, 2)}
    names = list(engines)
    out["inpainting_over_plain_images_per_s"] = round(out[names[1]]["images_per_s"] / out[names[0]]["images_per_s"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed requests per configuration and workload")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import engine as E, factory, synth
    from oracle import sd_oracle as O
    res = {"card": card(), "reps": args.reps}
    engines = {}
    for fam in ("sd15", "sd15-inpainting"):
        cfgs = factory.configs(fam)
        engines[fam] = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
    b = 32
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    init_u8 = torch.randint(0, 256, (b, 512, 512, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
    image_mask = torch.zeros((512, 512), dtype=torch.uint8)
    image_mask[128:384, 96:352] = 255
    latmask = (image_mask[::8, ::8] >= 128).float().reshape(-1)

    def inpaint(eng):
        kw = {"image_mask": image_mask, "inpainting_mask_weight": 1.0} if eng.inpainting else {}
        return eng.img2img(tok, neg, 1234, init_u8, denoising_strength=0.75, steps=20, cfg_scale=7.0, sampler="DDIM",
                           latmask=latmask, **kw)

    def txt2img(eng):
        return eng.txt2img(tok, neg, 1234, steps=20, cfg_scale=7.0, height=512, width=512, sampler="DDIM")

    res["img2img_inpaint"] = {"workload": "SD1.5 img2img inpainting 512x512 batch 32, whole picture, denoising 0.75, "
                                          "20 DDIM steps, CFG 7, fp16, CUDA graphs",
                              **time_configs(engines, inpaint, b, args.reps)}
    res["txt2img"] = {"workload": "SD1.5 txt2img 512x512 batch 32, 20 DDIM steps, CFG 7, fp16, CUDA graphs",
                      **time_configs(engines, txt2img, b, args.reps)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
