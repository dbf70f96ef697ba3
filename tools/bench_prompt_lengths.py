"""Time SD1.5 txt2img requests whose prompts span 1, 2 and 3 chunks of 77 tokens against a 1-chunk negative prompt.

512x512, batch 32, 20 DDIM steps, CFG 7, seeded synthetic weights, CUDA graphs on: the bench workload with longer
prompts.  A 2- or 3-chunk prompt makes the cond context 154 or 231 tokens long while the uncond one stays at 77, so the
cross-attention runs b200sd_attention_varlen on the plan's grown K/V buffers.

  * "1_chunk_fresh": 1-chunk requests on a plan that never grew (capacity 77, the plain attention call).
  * then every length is warmed up (the plan grows to 231) and timed in alternating rounds: "1_chunk", "2_chunks",
    "3_chunks" (the 1-chunk requests now take the varlen path with 77 keys per row).

Each request is timed with CUDA events around the whole call (text encoding, sampling, decode).  Prints one JSON line with
the card's name and power limit.  Writes nothing.

    python tools/bench_prompt_lengths.py [--reps 5] [--batch 32]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-diffusion-webui-distributed_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed requests per prompt length and phase")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    os.environ.pop("SD_TOKENIZER", None)   # hashed tokens: the chunk counts below do not depend on a vocabulary file
    from b200sd import config as C, engine as E, factory, synth
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
    b, vocab = args.batch, cfgs[2].vocab
    words = {1: 60, 2: 130, 3: 200}
    prompts = {k: factory.tokenize_prompts(["a (red:1.2) house, " + " ".join(f"w{i}" for i in range(n))] * b, vocab)
               for k, n in words.items()}
    neg = factory.tokenize_prompts(["(blurry), [text]"] * b, vocab)
    assert all(prompts[k][0].shape[1] == 77 * k for k in prompts) and neg[0].shape[1] == 77

    def request(k):
        ids, mult = prompts[k]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.txt2img(ids, neg[0], 1234, steps=args.steps, cfg_scale=7.0, height=512, width=512, sampler="DDIM",
                    multipliers=mult, neg_multipliers=neg[1])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    times = {"1_chunk_fresh": [], "1_chunk": [], "2_chunks": [], "3_chunks": []}
    for _ in range(2):
        request(1)
    assert eng.plan(b, 64, 64).ctx_cap == 77
    times["1_chunk_fresh"] = [request(1) for _ in range(args.reps)]
    for k in (2, 3, 1, 2, 3):
        request(k)
    assert eng.plan(b, 64, 64).ctx_cap == 231
    names = {1: "1_chunk", 2: "2_chunks", 3: "3_chunks"}
    for _ in range(args.reps):
        for k in (1, 2, 3):
            times[names[k]].append(request(k))
    res = {"workload": f"SD1.5 txt2img 512x512 batch {b}, {args.steps} DDIM steps, 1-chunk negative, CUDA graphs",
           "card": card(), "reps": args.reps}
    for name, ts in times.items():
        med = statistics.median(ts)
        res[name] = {"ms_median": round(med, 2), "ms_min": round(min(ts), 2), "ms_max": round(max(ts), 2),
                     "images_per_s": round(b / (med / 1000.0), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
