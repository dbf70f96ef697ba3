"""Time SD1.5 hires-fix requests with the "Latent", "Lanczos" and "R-ESRGAN 4x+" upscalers (seeded synthetic weights).

  * Requests: SD1.5 512x512 -> 1024x1024, batch `--batch` (16), 20 + 20 DDIM steps, denoising 0.7, CFG 7, fp16, CUDA
    graphs.  The three configurations alternate within each of `--reps` rounds after one warm-up request each; every
    request is timed with CUDA events around the whole call; the median gives images/s.
  * Upscaler alone: R-ESRGAN 4x+ on the batch's decoded 512x512 images (9 tiles of 192^2 each, overlap 8), timed with
    CUDA events, median of `--reps`.  Two FLOP counts, both including the tile overlap: "useful" is the network's own
    convolutions (useful_flops_per_tile); "executed" is what the kernels run, with conv_first's 64 padded input
    channels, the RDB convs' zero weight columns and conv_last's 32 padded outputs (RRDBWeights.flops_per_tile).
  * Comparator: the fp32 oracle's RRDBNet (oracle/upscale_oracle.rrdbnet) run by stock PyTorch in fp16, cuDNN,
    channels_last, on the same tiles, timed the same way; cuDNN runs no padding, so its rate is over the useful count.

Prints one JSON line with the card's name and power limit, read in the same run.  Writes nothing.

    python tools/bench_hires_upscalers.py [--reps 3] [--batch 16] [--steps 20]
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


def useful_flops_per_tile(num_block: int, h: int, w: int) -> float:
    """FLOPs of basicsr RRDBNet(3, 3, scale 4, 64 features, growth 32) on one h x w tile: 2 * 9 * Cin * Cout per pixel"""
    px = h * w
    rdb = sum(9 * cin * 32 for cin in (64, 96, 128, 160)) + 9 * 192 * 64
    macs = px * (9 * 3 * 64 + num_block * 3 * rdb + 9 * 64 * 64) + 4 * px * 9 * 64 * 64 + \
        16 * px * (2 * 9 * 64 * 64 + 9 * 64 * 3)
    return 2.0 * macs


def timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    from b200sd import config as C, engine as E, synth, upscale as U
    from oracle import sd_oracle as O, upscale_oracle as UO
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    os.environ.pop("B200SD_UPSCALER_DIR", None)
    cfgs = (C.SD15_UNET, C.SD15_VAE, C.SD15_CLIP)
    eng = E.SDEngine(synth.make_state_dict(*cfgs, seed=0), *cfgs, device="cuda:0", use_graphs=True)
    b = args.batch
    tok, neg = O.random_prompt_tokens(b), O.empty_prompt_tokens(b)
    names = ["Latent", "Lanczos", "R-ESRGAN 4x+"]

    def request(name):
        return eng.txt2img_hires(tok, neg, seed=1, steps=args.steps, cfg_scale=7.0, height=512, width=512,
                                 hr_scale=2.0, hr_steps=args.steps, denoising_strength=0.7, upscaler=name)

    times = {n: [] for n in names}
    for n in names:
        request(n)
    for _ in range(args.reps):
        for n in names:
            times[n].append(timed(lambda: request(n))[0])

    # the upscaler alone on decoded first-pass images
    imgs = request("Latent")[:, ::2, ::2].contiguous()   # any 512x512 uint8 batch: the cost does not depend on content
    wts = U.model("RealESRGAN_x4plus", eng.device)
    U.upscale_with_model(wts, imgs)
    esr = statistics.median(timed(lambda: U.upscale_with_model(wts, imgs))[0] for _ in range(args.reps))
    ys, xs = U.split_grid(512, 512, 192, 192, 8)
    n_tiles = b * len(ys) * len(xs)
    flops = n_tiles * wts.flops_per_tile(192, 192)
    useful = n_tiles * useful_flops_per_tile(wts.num_block, 192, 192)

    sd = {k: v.to("cuda", torch.float16).to(memory_format=torch.channels_last) if v.dim() == 4 else v.to("cuda", torch.float16)
          for k, v in U.load_state_dict("RealESRGAN_x4plus").items()}
    tiles = U.crop_tiles(imgs, ys, xs, 192, 192).permute(0, 3, 1, 2).flip(1).half().div(255)
    tiles = tiles.contiguous(memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True

    def stock():
        with torch.no_grad():
            for i in range(0, n_tiles, 16):
                UO.rrdbnet(sd, tiles[i:i + 16])

    stock()
    ref = statistics.median(timed(stock)[0] for _ in range(args.reps))
    ips = {n: b / (statistics.median(t) / 1e3) for n, t in times.items()}
    print(json.dumps({
        "workload": f"SD1.5 512->1024 hires, batch {b}, {args.steps}+{args.steps} DDIM, denoise 0.7, graphs",
        "images_per_s": {n: round(v, 3) for n, v in ips.items()},
        "request_ms_median": {n: round(statistics.median(t), 1) for n, t in times.items()},
        "esrgan_ms_per_image": round(esr / b, 2), "esrgan_tiles": n_tiles,
        "esrgan_useful_flops_per_image": useful / b, "esrgan_executed_flops_per_image": flops / b,
        "esrgan_useful_tflops": round(useful / (esr / 1e3) / 1e12, 1),
        "esrgan_executed_tflops": round(flops / (esr / 1e3) / 1e12, 1),
        "stock_pytorch_fp16_ms_per_image": round(ref / b, 2),
        "stock_pytorch_fp16_useful_tflops": round(useful / (ref / 1e3) / 1e12, 1),
        "card": card()}))


if __name__ == "__main__":
    main()
