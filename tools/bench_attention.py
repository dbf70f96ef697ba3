"""Time every attention shape of one UNet evaluation at the bench's batch sizes through the C ABI.

  * SD1.5, batch 32 (UNet batch 64 with CFG), 8 heads: self-attention 4096/d40, 1024/d80, 256/d160 (5 each) and the
    middle block's 64/d160 (1), plus the cross-attention of each to the 77-token context.
  * SDXL, batch 16 (UNet batch 32), 64-wide heads: 4096 tokens x 10 heads (10 per evaluation) and 1024 tokens x 20 heads
    (60), self and cross.

Each shape is timed with CUDA events over --iters back-to-back launches per round; the median round is reported as ms
per call, with unpadded TFLOP/s (4 B H Sq Skv d), T exp/s (one exponential per score) and the fraction of the MUFU.EX2
peak at the SM clock sampled during the run.  Inputs are seeded; heads use the UNet's padded pitch.

--baseline-lib PATH loads a second libb200sd.so (ctypes loads it RTLD_LOCAL, so both coexist), alternates the two
libraries round by round on identical inputs and reports the max |difference| of their outputs and the speed-up.
Prints one JSON line with the card's name and power limit.  Writes nothing.

    python tools/bench_attention.py [--baseline-lib build/parent/libb200sd.so] [--iters 20] [--rounds 5]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-diffusion-webui-distributed_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

# (model, label, UNet batch, heads, Sq, Skv, d, calls per evaluation)
SHAPES = [
    ("sd15", "self 4096/d40", 64, 8, 4096, 4096, 40, 5),
    ("sd15", "cross 4096/d40", 64, 8, 4096, 77, 40, 5),
    ("sd15", "self 1024/d80", 64, 8, 1024, 1024, 80, 5),
    ("sd15", "cross 1024/d80", 64, 8, 1024, 77, 80, 5),
    ("sd15", "self 256/d160", 64, 8, 256, 256, 160, 5),
    ("sd15", "cross 256/d160", 64, 8, 256, 77, 160, 5),
    ("sd15", "self 64/d160", 64, 8, 64, 64, 160, 1),
    ("sd15", "cross 64/d160", 64, 8, 64, 77, 160, 1),
    ("sdxl", "self 4096/d64", 32, 10, 4096, 4096, 64, 10),
    ("sdxl", "cross 4096/d64", 32, 10, 4096, 77, 64, 10),
    ("sdxl", "self 1024/d64", 32, 20, 1024, 1024, 64, 60),
    ("sdxl", "cross 1024/d64", 32, 20, 1024, 77, 64, 60),
]
DTYPE = {"sd15": "float16", "sdxl": "bfloat16"}


def load(path):
    lib = ctypes.CDLL(path)   # RTLD_LOCAL: a second copy of the library keeps its own symbols
    lib.b200sd_attention.restype = ctypes.c_int
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None, help="a second libb200sd.so to compare against")
    ap.add_argument("--iters", type=int, default=20, help="launches per timed round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--model", choices=["sd15", "sdxl", "all"], default="all")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from b200sd import _lib
    from b200sd.unet_exec import _pad64
    from bench import MUFU_EXP_PER_CLK_SM, NUM_SMS, ClockSampler
    from bench_prompt_lengths import card

    libs = {"new": load(_lib.LIB_PATH)}
    if args.baseline_lib:
        libs["baseline"] = load(os.path.abspath(args.baseline_lib))
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev)

    def call(lib, q, k, v, out, b, heads, sq, skv, d, d_pad, is_bf16):
        rc = lib.b200sd_attention(
            ctypes.c_void_p(q.data_ptr()), ctypes.c_longlong(q.stride(1)), ctypes.c_void_p(k.data_ptr()),
            ctypes.c_longlong(k.stride(1)), ctypes.c_void_p(v.data_ptr()), ctypes.c_longlong(v.stride(1)),
            ctypes.c_void_p(out.data_ptr()), ctypes.c_longlong(out.stride(1)), b, heads, sq, skv, d, d_pad,
            ctypes.c_float(d ** -0.5), 0, int(is_bf16), ctypes.c_void_p(stream.cuda_stream))
        if rc != 0:
            raise RuntimeError(f"b200sd_attention failed rc={rc} (B={b} heads={heads} Sq={sq} Skv={skv} d={d})")

    clk = ClockSampler(0)
    clk.start()
    rows = []
    for model, label, b, heads, sq, skv, d, per_eval in SHAPES:
        if args.model not in ("all", model):
            continue
        dt = getattr(torch, DTYPE[model])
        d_pad = _pad64(d)
        g = torch.Generator(device=dev).manual_seed(sq * 131 + skv * 7 + d)

        def heads_tensor(s):
            t = torch.zeros((b, s, heads, d_pad), device=dev, dtype=dt)
            t[..., :d] = torch.randn((b, s, heads, d), generator=g, device=dev).to(dt)
            return t.reshape(b, s, heads * d_pad)

        q, k, v = heads_tensor(sq), heads_tensor(skv), heads_tensor(skv)
        outs = {name: torch.empty((b, sq, heads * d), device=dev, dtype=dt) for name in libs}
        for name, lib in libs.items():   # warm-up: module load, smem opt-in, clocks
            for _ in range(3):
                call(lib, q, k, v, outs[name], b, heads, sq, skv, d, d_pad, dt == torch.bfloat16)
        torch.cuda.synchronize()
        times = {name: [] for name in libs}
        for _ in range(args.rounds):
            for name, lib in libs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    call(lib, q, k, v, outs[name], b, heads, sq, skv, d, d_pad, dt == torch.bfloat16)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / args.iters)
        flop = 4.0 * b * heads * sq * skv * d
        exps = float(b) * heads * sq * skv
        row = {"model": model, "shape": label, "batch": b, "heads": heads, "Sq": sq, "Skv": skv, "d": d, "d_pad": d_pad,
               "dtype": DTYPE[model], "calls_per_eval": per_eval}
        for name in libs:
            ms = statistics.median(times[name])
            row[name] = {"ms": round(ms, 4), "ms_min": round(min(times[name]), 4), "ms_max": round(max(times[name]), 4),
                         "tflops": round(flop / (ms * 1e-3) / 1e12, 2), "t_exp_per_s": round(exps / (ms * 1e-3) / 1e12, 4)}
        if "baseline" in libs:
            diff = (outs["new"].float() - outs["baseline"].float()).abs()
            row["max_abs_diff"] = float(diff.max())
            row["mean_abs_diff"] = float(diff.mean())
            row["speedup"] = round(row["baseline"]["ms"] / row["new"]["ms"], 3)
        rows.append(row)
        del q, k, v, outs
    c = clk.stop()
    sm_mhz = c.get("sm_mhz")
    if sm_mhz:
        exp_peak = NUM_SMS * MUFU_EXP_PER_CLK_SM * sm_mhz * 1e6 / 1e12
        for row in rows:
            for name in libs:
                row[name]["mufu_frac"] = round(row[name]["t_exp_per_s"] / exp_peak, 4)
    per_eval = {}
    for row in rows:
        for name in libs:
            key = f"{row['model']}_{name}_ms"
            per_eval[key] = round(per_eval.get(key, 0.0) + row[name]["ms"] * row["calls_per_eval"], 3)
    print(json.dumps({"card": card(), "clocks": c, "iters": args.iters, "rounds": args.rounds,
                      "mufu_peak_source": f"{NUM_SMS} SMs x {MUFU_EXP_PER_CLK_SM} MUFU.EX2/clk x sampled SM clock",
                      "attention_ms_per_unet_eval": per_eval, "shapes": rows}))


if __name__ == "__main__":
    main()
