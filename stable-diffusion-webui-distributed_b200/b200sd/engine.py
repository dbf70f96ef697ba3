"""SDEngine — the local executor a Worker binds instead of POST /sdapi/v1/txt2img (reference worker.py:432-435).

One engine per GPU: packed weights, per-shape execution plans (UNet step graph, VAE decode graph), samplers.
Images of one request are independent given (prompt, seed + k) — the property the reference's seed offsetting
relies on (scripts/distributed.py:297-305) — so a request's batch is sharded across engines with no per-step
exchange; results meet once, at the end (bench: one NCCL all-gather; plugin path: the collector thread join).
"""
import contextlib
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from . import lora as L
from . import ops
from . import samplers as S
from .clip_text import CAPTURE_LOCK as _CAPTURE_LOCK, Cond, Conditioner
from .config import UNET_PREFIX, CLIPConfig, UNetConfig, VAEConfig
from .prompts import schedule_index
from .unet_exec import MAX_CONTROLS, ControlNetWeights, TimeEmbedding, UNetProgram, UNetWeights
from .vae_exec import VAEDecoderProgram, VAEDecoderWeights, VAEEncoderProgram, VAEEncoderWeights

MAX_STEPS = 256
MAX_PLANS = 6        # distinct (batch, latent h, w) kept per engine; the least recently used one is dropped beyond that
MAX_GRAPHS = 48      # step graphs kept per plan (one per sampler stage structure x cfg scale): oldest dropped beyond that
CHUNK = 77           # tokens per prompt chunk (sdwui: [BOS] + 75 + [EOS]); contexts are 77 * k tokens long
NOISE_SAMPLERS = ("Euler a", "stage")   # graph-name prefixes of the step graphs that may read Plan.noise
PREDICTIONS = ("eps", "v")   # what the UNet predicts: the noise (SD1.x, SDXL, SD 2.x-base) or v (SD 2.x 768-v)
# UNet input channels served: the latents (4), or latents + mask + masked-image latents (9, inpainting checkpoints)
IN_CHANNELS = (4, 9)
# _CAPTURE_LOCK (imported): CUDA graph captures are serialised across the per-device worker threads


# ------------------------------------------------------------------------------------------------ schedules
def alphas_cumprod() -> torch.Tensor:
    """ldm linear schedule (linear_start 0.00085, linear_end 0.012, 1000 steps), fp64 math, fp32 storage."""
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float64) ** 2
    return torch.cumprod(1.0 - betas, dim=0).to(torch.float32)


def ddim_plan(steps: int) -> Tuple[List[float], List[List[float]]]:
    """sdwui sd_samplers_timesteps(_impl).ddim, eta = 0.  Returns (timesteps, coef rows) in execution order;
    `steps` timesteps give steps-1 UNet evaluations (index len-1 .. 1)."""
    ac = alphas_cumprod().double()
    ts = torch.clamp(torch.arange(0, 1000, 1000 // steps) + 1, 0, 999)
    a = ac[ts]
    a_prev = ac[torch.cat([ts.new_zeros(1), ts[:-1]])]
    t_out, rows = [], []
    for i in range(len(ts) - 1, 0, -1):
        at, ap = float(a[i]), float(a_prev[i])
        t_out.append(float(ts[i]))
        rows.append([math.sqrt(at), math.sqrt(1 - at), math.sqrt(ap), math.sqrt(1 - ap)])
    return t_out, rows


def ddim_img2img_plan(steps: int, denoising_strength: float):
    """sdwui sd_samplers_timesteps.sample_img2img: t_enc = int(min(d, 0.999) * steps); DDIM runs on timesteps[:t_enc]
    (t_enc - 1 UNet evaluations) from x = init * sqrt(a[ts[t_enc]]) + noise * sqrt(1 - a[ts[t_enc]]).
    Returns (sqrt_a_start, sqrt_1m_a_start, timesteps, coef rows)."""
    ac = alphas_cumprod().double()
    ts = torch.clamp(torch.arange(0, 1000, 1000 // steps) + 1, 0, 999)
    t_enc = max(1, min(int(min(denoising_strength, 0.999) * steps), len(ts) - 1))
    a_start = float(ac[ts[t_enc]])
    sub = ts[:t_enc]
    a = ac[sub]
    a_prev = ac[torch.cat([sub.new_zeros(1), sub[:-1]])]
    t_out, rows = [], []
    for i in range(len(sub) - 1, 0, -1):
        at, ap = float(a[i]), float(a_prev[i])
        t_out.append(float(sub[i]))
        rows.append([math.sqrt(at), math.sqrt(1 - at), math.sqrt(ap), math.sqrt(1 - ap)])
    return math.sqrt(a_start), math.sqrt(1 - a_start), t_out, rows


def euler_a_plan(steps: int, scheduler: str = "uniform", sigmas=None):
    """k-diffusion sample_euler_ancestral over CompVisDenoiser sigmas.  Returns (timesteps, coef rows, sigma0):
    row = [sigma, sigma_down, sigma_up, c_in of the NEXT step].  `sigmas` = (table ending in 0, log-sigma table of the
    model) runs an explicit schedule instead (img2img: the tail of the full one)."""
    sig, log_sig = sigmas if sigmas is not None else kdiffusion_sigmas(steps, scheduler)
    steps = len(sig) - 1

    t_out, rows = [], []
    for i in range(steps):
        s, sn = float(sig[i]), float(sig[i + 1])
        up = min(sn, (sn ** 2 * (s ** 2 - sn ** 2) / s ** 2) ** 0.5)
        down = (sn ** 2 - up ** 2) ** 0.5
        t_out.append(sigma_to_t(s, log_sig))
        rows.append([s, down, up, 1.0 / math.sqrt(sn * sn + 1.0)])
    return t_out, rows, float(sig[0])


def euler_plan(steps: int, scheduler: str = "uniform", sigmas=None):
    """k-diffusion sample_euler (s_churn = 0) on the same sigmas: the ancestral step with sigma_up = 0, i.e.
    sigma_down = sigma_next and no noise — same coefficient rows, same kernel."""
    t_out, rows, sigma0 = euler_a_plan(steps, scheduler, sigmas)
    for i, r in enumerate(rows):
        sn = (r[1] ** 2 + r[2] ** 2) ** 0.5   # sigma_next = sqrt(down^2 + up^2)
        rows[i] = [r[0], sn, 0.0, r[3]]
    return t_out, rows, sigma0


def kdiffusion_sigmas(steps: int, scheduler: str = "uniform") -> Tuple[torch.Tensor, torch.Tensor]:
    """sigmas[steps + 1] (last 0) as sdwui's KDiffusionSampler.get_sigmas builds them, and the model's log-sigma table.
    "uniform": k-diffusion DiscreteSchedule.get_sigmas (timesteps linspace(999, 0, steps), log-sigma interpolation);
    "karras": get_sigmas_karras(steps, sigma_min = sigmas[0], sigma_max = sigmas[-1], rho = 7);
    "exponential" (= "polyexponential", rho 1): get_sigmas_exponential — log-sigmas equally spaced between the same bounds;
    "sgm_uniform": sdwui sd_schedulers.sgm_uniform — timesteps linspace(t(sigma_max), t(sigma_min), steps + 1)[:-1]."""
    ac = alphas_cumprod().double()
    sig_all = ((1 - ac) / ac) ** 0.5
    log_sig = sig_all.log()
    if scheduler == "karras":
        ramp = torch.linspace(0, 1, steps, dtype=torch.float64)
        lo, hi = float(sig_all[0]) ** (1 / 7.0), float(sig_all[-1]) ** (1 / 7.0)
        sig = (hi + ramp * (lo - hi)) ** 7.0
    elif scheduler in ("exponential", "polyexponential"):
        sig = torch.linspace(math.log(float(sig_all[-1])), math.log(float(sig_all[0])), steps, dtype=torch.float64).exp()
    elif scheduler in ("uniform", "sgm_uniform"):
        # t(sigma_max) = 999 and t(sigma_min) = 0 on the model's own table
        tt = torch.linspace(999, 0, steps + 1, dtype=torch.float64)[:-1] if scheduler == "sgm_uniform" else \
            torch.linspace(999, 0, steps, dtype=torch.float64)
        lo, hi = tt.floor().long(), tt.ceil().long()
        wgt = tt - lo
        sig = ((1 - wgt) * log_sig[lo] + wgt * log_sig[hi]).exp()
    else:
        raise ValueError(f"scheduler {scheduler!r} is not implemented")
    return torch.cat([sig, sig.new_zeros(1)]), log_sig


def sigma_to_t(s: float, log_sig: torch.Tensor) -> float:
    """k-diffusion DiscreteSchedule.sigma_to_t (quantize = False)"""
    ls = math.log(s)
    dists = ls - log_sig
    low = int((dists >= 0).cumsum(0).argmax().clamp(max=len(log_sig) - 2))
    l0, h0 = float(log_sig[low]), float(log_sig[low + 1])
    w = min(max((l0 - ls) / (l0 - h0), 0.0), 1.0)
    return (1 - w) * low + w * (low + 1)


def kdiffusion_img2img_sigmas(steps: int, denoising_strength: float, scheduler: str):
    """sdwui KDiffusionSampler.sample_img2img: t_enc = int(min(d, 0.999) * steps); the sampler runs on
    sigmas[steps - t_enc - 1:] (t_enc + 1 UNet evaluations) from x = init + noise * sigma_sched[0]."""
    sig, log_sig = kdiffusion_sigmas(steps, scheduler)
    t_enc = int(min(denoising_strength, 0.999) * steps)
    return sig[steps - t_enc - 1:], log_sig


def dpmpp_2m_plan(steps: int, scheduler: str = "karras", sigmas=None):
    """k-diffusion sample_dpmpp_2m.  Returns (timesteps, coef rows of 8, sigma0);
    row = [sigma, sigma_next / sigma, c1, c2, c_in of the NEXT step, 0, 0, 0] with denoised_d = c1 * denoised - c2 * old."""
    sig, log_sig = sigmas if sigmas is not None else kdiffusion_sigmas(steps, scheduler)
    steps = len(sig) - 1
    t_out, rows = [], []
    for i in range(steps):
        s, sn = float(sig[i]), float(sig[i + 1])
        c1, c2 = 1.0, 0.0
        if i > 0 and sn > 0:
            h = math.log(s / sn)
            h_last = math.log(float(sig[i - 1]) / s)
            r = h_last / h
            c1, c2 = 1.0 + 1.0 / (2.0 * r), 1.0 / (2.0 * r)
        t_out.append(sigma_to_t(s, log_sig))
        rows.append([s, sn / s, c1, c2, 1.0 / math.sqrt(sn * sn + 1.0), 0.0, 0.0, 0.0])
    return t_out, rows, float(sig[0])


def v_rows(fused: str, rows: List[List[float]]) -> List[List[float]]:
    """coefficient rows of the fused k-diffusion steps for a v-prediction model: {kx, kv} of the row's sigma join them,
    eps = kx x + kv v (CompVisVDenoiser, sigma_data 1).  Euler (a): 8-float rows {sigma, sigma_down, sigma_up, in_next,
    kx, kv, 0, 0}; DPM++ 2M: columns 5, 6.  DDIM rows already hold sqrt(a_t), sqrt(1 - a_t)."""
    if fused == "ddim":
        return rows
    out = []
    for r in rows:
        s = r[0]
        kx, kv = s / (s * s + 1.0), 1.0 / math.sqrt(s * s + 1.0)
        out.append(list(r[:4]) + [kx, kv, 0.0, 0.0] if fused in ("euler_a", "euler") else list(r[:5]) + [kx, kv, 0.0])
    return out


# sampler names of the sdwui API -> (method, scheduler).  sdwui >= 1.9 sends the scheduler separately ("scheduler" key,
# "Automatic" = the sampler's default, which is Karras for DPM++ 2M); older versions fold it into the name.
SAMPLERS = {"DDIM": ("ddim", None), "Euler a": ("euler_a", "uniform"), "Euler": ("euler", "uniform"),
            "DPM++ 2M": ("dpmpp_2m", "karras"), "DPM++ 2M Karras": ("dpmpp_2m", "karras"), **S.GENERIC}


# sdwui's samplers flagged second_order (sd_samplers_kdiffusion.samplers_k_diffusion): two model evaluations per step,
# and SamplerData.total_steps counts both, so prompt schedules run over steps x 2
SECOND_ORDER = ("Heun", "DPM2", "DPM2 a", "DPM++ 2S a", "DPM++ SDE", "DPM2 Karras", "DPM2 a Karras",
                "DPM++ 2S a Karras", "DPM++ SDE Karras")


def total_steps(sampler: str, steps: int) -> int:
    """sdwui SamplerData.total_steps: the steps a prompt schedule of the request is built over"""
    return steps * 2 if sampler in SECOND_ORDER else steps


# API scheduler labels (sdwui >= 1.9 sd_schedulers.schedulers: label or name) -> kdiffusion_sigmas scheduler
SCHEDULERS = {"Uniform": "uniform", "uniform": "uniform", "Karras": "karras", "karras": "karras",
              "Exponential": "exponential", "exponential": "exponential", "Polyexponential": "polyexponential",
              "polyexponential": "polyexponential", "SGM Uniform": "sgm_uniform", "sgm_uniform": "sgm_uniform"}


def resolve_sampler(name: str, scheduler: Optional[str] = None):
    """(method, scheduler) for an API sampler name + optional API scheduler label; ValueError if not implemented."""
    if name not in SAMPLERS:
        raise ValueError(f"sampler {name!r} is not implemented on the local executor")
    method, default = SAMPLERS[name]
    if default is not None and scheduler not in (None, "", "Automatic"):   # DDIM takes no sigma schedule
        label = SCHEDULERS.get(scheduler, SCHEDULERS.get(str(scheduler).lower()))
        if label is None:
            raise ValueError(f"scheduler {scheduler!r} is not implemented on the local executor")
        return method, label
    return method, default


def slerp(val: float, low: torch.Tensor, high: torch.Tensor) -> torch.Tensor:
    """sdwui modules/rng.py slerp, applied to one image's [C, H, W] noise (norms and angles along dim 1, as upstream)"""
    low_norm = low / torch.norm(low, dim=1, keepdim=True)
    high_norm = high / torch.norm(high, dim=1, keepdim=True)
    dot = (low_norm * high_norm).sum(1)
    if float(dot.mean()) > 0.9995:
        return low * val + high * (1 - val)
    omega = torch.acos(dot)
    so = torch.sin(omega)
    return (torch.sin((1.0 - val) * omega) / so).unsqueeze(1) * low + (torch.sin(val * omega) / so).unsqueeze(1) * high


def per_image_noise(seed: int, n: int, shape, draws: int = 1, subseed: Optional[int] = None,
                    subseed_strength: float = 0.0) -> torch.Tensor:
    """sdwui ImageRNG with randn_source = 'CPU': image k owns torch.Generator('cpu').manual_seed(all_seeds[k]);
    `draws` successive tensors per image (x_T, then ancestral noises).  processing.py: all_seeds[k] = seed + k when
    subseed_strength == 0, but seed for EVERY image when variation seeds are on (only all_subseeds[k] = subseed + k
    varies; the reference dispatcher mirrors this by not offsetting `seed`, scripts/distributed.py:297-305).
    Variation seeds (ImageRNG.first): the FIRST draw is slerp(strength, noise(seed), noise(subseed + k)).
    Returns [draws, n, *shape] fp32 (host)."""
    out = torch.empty((draws, n, *shape), dtype=torch.float32)
    variation = subseed is not None and subseed_strength != 0
    for k in range(n):
        g = torch.Generator(device="cpu").manual_seed(int(seed) + (0 if variation else k))
        for d in range(draws):
            out[d, k] = torch.randn(shape, generator=g, dtype=torch.float32)
        if variation:
            sg = torch.Generator(device="cpu").manual_seed(int(subseed) + k)
            out[0, k] = slerp(float(subseed_strength), out[0, k], torch.randn(shape, generator=sg, dtype=torch.float32))
    return out


@dataclass
class Program:
    """what one sampling run executes (SDEngine.program)"""
    sampler: str
    method: str
    fused: Optional[str] = None          # "ddim" | "euler_a" | "euler" | "dpmpp_2m": the fused per-step kernels
    ts: List[float] = field(default_factory=list)      # fused: timestep per evaluation
    rows: List[List[float]] = field(default_factory=list)   # fused: coefficient row per evaluation
    sp: Optional[S.SamplerPlan] = None   # generic stage list
    adaptive: Optional[tuple] = None     # DPM adaptive: (sigma_min, sigma_max, sigma -> timestep)
    draws: int = 0                       # N(0,1) draws per image after the start noise
    init_scale: float = 0.0              # start latents = init * init_scale + noise * noise_scale
    noise_scale: float = 1.0
    in0: float = 1.0                     # scale of the first UNet input
    timestep_sampler: bool = False
    steps: int = 0                       # sampler steps requested (DPM adaptive: the n of ControlNet windows)

    def start(self, noise0: torch.Tensor, init: Optional[torch.Tensor] = None) -> torch.Tensor:
        x = noise0 * self.noise_scale
        return x if init is None else x + init * self.init_scale

    @property
    def n_evals(self) -> Optional[int]:
        return len(self.ts) if self.fused else (len(self.sp.stages) if self.sp is not None else None)


@dataclass
class PromptSchedule:
    """one prompt's sdwui schedule (prompts.prompt_schedule) for a sampling pass: the entries' token ids, tokenized
    together so that they have one chunk count, and the step each entry ends at"""
    ends: List[int]                              # end_at_step per entry, increasing
    tokens: torch.Tensor                         # [E, 77 * k]
    multipliers: Optional[torch.Tensor] = None   # [E, 77 * k] emphasis weights (None: all 1)


# ------------------------------------------------------------------------------------------------ plans
class Plan:
    """Everything shape-dependent for (images per call b, latent h x w) on one device.  tiling: the UNet's and the VAE
    decoder's 3x3 convs pad circularly (sdwui's tiling option).  token_merging: r tokens merged in the UNet's
    full-resolution self-attention (sdwui's token merging ratio, SDEngine.merged_tokens)."""

    def __init__(self, eng: "SDEngine", b: int, h: int, w: int, vae_chunk: int, tiling: bool = False,
                 token_merging: int = 0):
        dev = eng.device
        self.b, self.h, self.w = b, h, w
        self.unet = UNetProgram(eng.unet_w, 2 * b, h, w, CHUNK, tiling=tiling, token_merging=token_merging)
        self.kv_len = self.unet.kv_len   # int32 [2b] on the device: context tokens of every [cond | uncond] row
        self.vae_chunk = min(vae_chunk, b)
        self.vae = VAEDecoderProgram(eng.vae_w, self.vae_chunk, h, w, tiling=tiling)
        self.x = torch.zeros((b, h * w, 4), device=dev, dtype=torch.float32)
        self.step = torch.zeros((1,), device=dev, dtype=torch.int32)
        self.coef = torch.zeros((MAX_STEPS, 4), device=dev, dtype=torch.float32)
        self.table = torch.zeros((MAX_STEPS, self.unet.cur_bias.numel()), device=dev, dtype=torch.float32)
        self.coef8 = torch.zeros((MAX_STEPS, 8), device=dev, dtype=torch.float32)   # DPM++ 2M rows
        self.old = torch.zeros((b, h * w, 4), device=dev, dtype=torch.float32)        # its previous x0 prediction
        self.init = torch.zeros((b, h * w, 4), device=dev, dtype=torch.float32)     # inpainting: clean init latents
        self.latmask = torch.ones((h * w,), device=dev, dtype=torch.float32)        # ... and the latent mask (1 = repaint)
        # generic stage machine (b200sd/samplers.py): named fp32 latents, coefficient rows selected by `step`
        self.lat = {"x": self.x}
        for name in ("e", "u", "h1", "h2", "h3", "d"):
            self.lat[name] = torch.zeros((b, h * w, 4), device=dev, dtype=torch.float32)
        self.coefL = torch.zeros((MAX_STEPS, S.COEF_LD), device=dev, dtype=torch.float32)
        self.noise = None            # [rows, b, h*w, 4] fp32, persistent: captured graphs bake its address
        # prompt editing (SDEngine._switch): the request's encoded entries [E, cap, ctx], their lengths, the entry of
        # every [cond | uncond] row per evaluation [MAX_STEPS, 2b], and the context the "ctx" graph selects into
        self.bank = self.bank_len = self.sched = self.ctx_stage = None
        self.graphs: Dict[str, torch.cuda.CUDAGraph] = {}
        self.graph_launches: Dict[str, int] = {}
        self.stage_ids: Dict[tuple, int] = {}   # (lincomb structure, evaluated latent) of a generic stage -> graph-name id
        self.vpred = eng.prediction == "v"      # the UNet output is v: the _v fused steps, one more lincomb per stage

    def noise_rows(self, rows: int) -> torch.Tensor:
        """the request's per-step noises live in ONE buffer per plan (the step graphs hold its raw address); it grows in
        powers of two, and growing drops the graphs that captured the old address"""
        if self.noise is None or self.noise.shape[0] < rows:
            cap = 32
            while cap < rows:
                cap *= 2
            self.noise = torch.zeros((cap, self.b, self.h * self.w, 4), device=self.x.device, dtype=torch.float32)
            for name in [n for n in self.graphs if n.split(":")[0] in NOISE_SAMPLERS]:  # incl. every "stage" graph
                del self.graphs[name]
                self.graph_launches.pop(name, None)
        return self.noise

    def set_bank(self, cond_bank: torch.Tensor, uncond_bank: torch.Tensor):
        """encoded schedule entries [Ec, Lc, ctx] and [Eu, Lu, ctx] -> the bank (cond entries first).  The bank grows in
        powers of two and follows the context capacity; reallocating drops the "ctx" graphs that captured it."""
        (ec, lc, c), (eu, lu, _) = cond_bank.shape, uncond_bank.shape
        self.ensure_context(max(lc, lu))
        cap, e = self.ctx_cap, ec + eu
        if self.bank is None or self.bank.shape[0] < e or self.bank.shape[1] != cap:
            rows = 4
            while rows < e:
                rows *= 2
            dev, dt = self.x.device, self.unet.dt
            self.bank = torch.zeros((rows, cap, c), device=dev, dtype=dt)
            self.bank_len = torch.ones((rows,), device=dev, dtype=torch.int32)
            self.ctx_stage = torch.zeros((2 * self.b, cap, c), device=dev, dtype=dt)
            for name in [n for n in self.graphs if n.startswith("ctx")]:
                del self.graphs[name]
                self.graph_launches.pop(name, None)
        if self.sched is None:
            self.sched = torch.zeros((MAX_STEPS, 2 * self.b), device=self.x.device, dtype=torch.int32)
        self.bank[:ec, :lc].copy_(cond_bank)
        self.bank[ec:e, :lu].copy_(uncond_bank)
        self.bank_len[:e].copy_(torch.tensor([lc] * ec + [lu] * eu, dtype=torch.int32))

    def set_sched(self, row0: int, entries):
        """rows row0.. of the schedule table: (cond entry, uncond entry) per evaluation, bank indices"""
        rows = [[c] * self.b + [u] * self.b for c, u in entries]
        self.sched[row0:row0 + len(rows)].copy_(torch.tensor(rows, dtype=torch.int32))

    def switch_context(self, slots):
        """the switch: select this evaluation's entries (device step counter) into the staging context, then project
        the K/V of every attn2 of the UNet and of the ControlNet segments in `slots`"""
        ops.select_context(self.bank, self.bank_len, self.sched, self.step, self.ctx_stage, self.unet.kv_len)
        self.unet.project_context(self.ctx_stage, [self.unet.segments[s] for s in slots])

    @property
    def ctx_cap(self) -> int:
        """context capacity: rows per image of the cross-attention K/V buffers (a multiple of 77)"""
        return self.unet.ctx_len

    def ensure_context(self, tokens: int):
        """grow the K/V buffers in whole 77-token chunks to hold a `tokens`-long context; growing drops the step graphs
        that captured the old buffers (the "vae" graph does not read them).  Activation buffers are not duplicated."""
        if tokens > self.ctx_cap:
            self.unet.grow_context(-(-tokens // CHUNK) * CHUNK)
            for name in [n for n in self.graphs if n != "vae"]:
                del self.graphs[name]
                self.graph_launches.pop(name, None)

    def set_context(self, cond_ctx: torch.Tensor, uncond_ctx: torch.Tensor):
        """[cond | uncond] contexts -> the UNet's cross-attention K/V.  Equal lengths take the plain batched call; different
        lengths (sdwui then runs two UNet calls) are zero-padded to the longer one and attend to their own lengths."""
        b, lc, c = cond_ctx.shape
        lu = uncond_ctx.shape[1]
        self.ensure_context(max(lc, lu))
        if lc == lu:
            self.unet.set_context(torch.cat([cond_ctx, uncond_ctx]).to(self.unet.dt).contiguous())
            return
        ctx = torch.zeros((2 * b, max(lc, lu), c), device=self.x.device, dtype=self.unet.dt)
        ctx[:b, :lc] = cond_ctx
        ctx[b:, :lu] = uncond_ctx
        self.unet.set_context(ctx, [lc] * b + [lu] * b)

    def _unet(self, active):
        """one UNet evaluation with the ControlNet slots `active`; without any, the same call as ever"""
        if active:
            self.unet.run(active)
        else:
            self.unet.run()

    # one sampler step = select this step's biases, UNet on [cond | uncond], CFG + update + repack
    def step_ddim(self, cfg_scale: float, active=()):
        ops.select_step(self.table, self.step, self.unet.cur_bias)
        self._unet(active)
        if self.vpred:
            ops.cfg_ddim_step_v(self.unet.eps, self.x, self.unet.xin, cfg_scale, self.coef, self.step)
        else:
            ops.cfg_ddim_step(self.unet.eps, self.x, self.unet.xin, cfg_scale, self.coef, self.step)

    def step_ddim_masked(self, cfg_scale: float, active=()):
        """inpainting (sdwui CFGDenoiserTimesteps, mask_before_denoising): the kept region of x is replaced by the clean
        init latent before every model call"""
        ops.blend_latent(self.x, self.init, self.latmask)
        ops.pack_unet_input(self.x, self.unet.xin, 1.0)
        self.step_ddim(cfg_scale, active)

    def step_euler_a(self, cfg_scale: float, active=()):
        ops.select_step(self.table, self.step, self.unet.cur_bias)
        self._unet(active)
        if self.vpred:
            ops.cfg_euler_a_step_v(self.unet.eps, self.x, self.noise, self.unet.xin, cfg_scale, self.coef8, self.step)
        else:
            ops.cfg_euler_a_step(self.unet.eps, self.x, self.noise, self.unet.xin, cfg_scale, self.coef, self.step)

    def step_euler(self, cfg_scale: float, active=()):  # sigma_up == 0 in every coefficient row: the kernel needs no noise
        ops.select_step(self.table, self.step, self.unet.cur_bias)
        self._unet(active)
        if self.vpred:
            ops.cfg_euler_a_step_v(self.unet.eps, self.x, None, self.unet.xin, cfg_scale, self.coef8, self.step)
        else:
            ops.cfg_euler_a_step(self.unet.eps, self.x, None, self.unet.xin, cfg_scale, self.coef, self.step)

    def stage(self, lcs, ev: str, cfg_scale: float, masked: bool, timestep_sampler: bool, active=()):
        """one model evaluation of a generic sampler program + its linear combinations (samplers.Stage.lcs)"""
        lat = self.lat
        if masked and timestep_sampler:   # sdwui CFGDenoiser, mask_before_denoising: the evaluated tensor is blended first
            ops.blend_latent(lat[ev], self.init, self.latmask)
            ops.pack_unet_input(lat[ev], self.unet.xin, 1.0)
        ops.select_step(self.table, self.step, self.unet.cur_bias)
        self._unet(active)
        ops.cfg_eps(self.unet.eps, lat["e"], cfg_scale)
        if self.vpred:   # e holds the CFG-combined v: eps = kx ev + kv v, in fp32 next to the latents
            ops.latent_lincomb(lat["e"], [lat[ev], lat["e"]], self.coefL, S.V_COL, self.step)
        if masked and not timestep_sampler:
            # k-diffusion samplers: denoised = denoised * nmask + init_latent * mask (CFGDenoiser.forward's last lines);
            # re-expressed on e = (ev - denoised) / sigma
            ops.latent_lincomb(lat["d"], [lat[ev], lat["e"]], self.coefL, S.MASK_COL, self.step)
            ops.blend_latent(lat["d"], self.init, self.latmask)
            ops.latent_lincomb(lat["e"], [lat[ev], lat["d"]], self.coefL, S.MASK_COL + 2, self.step)
        col = 0
        for dst, srcs, pack in lcs:
            ops.latent_lincomb(lat[dst], [self.noise if n == "n" else lat[n] for n in srcs], self.coefL, col, self.step,
                               self.unet.xin if pack else None, S.IDX_COL if "n" in srcs else -1)
            col += len(srcs) + int(pack)
        ops.bump_step(self.step)

    def step_dpmpp_2m(self, cfg_scale: float, active=()):
        ops.select_step(self.table, self.step, self.unet.cur_bias)
        self._unet(active)
        if self.vpred:
            ops.cfg_dpmpp_2m_step_v(self.unet.eps, self.x, self.old, self.unet.xin, cfg_scale, self.coef8, self.step)
        else:
            ops.cfg_dpmpp_2m_step(self.unet.eps, self.x, self.old, self.unet.xin, cfg_scale, self.coef8, self.step)


class SDEngine:
    _require_cuda = True  # tests/test_programs_cpu.py flips this together with an emulated ops module

    def _ctx(self):
        return torch.cuda.device(self.device) if self.device.type == "cuda" else contextlib.nullcontext()

    def __init__(self, sd: Dict[str, torch.Tensor], unet_cfg: UNetConfig, vae_cfg: VAEConfig, clip_cfg: CLIPConfig,
                 device="cuda:0", dtype=torch.float16, use_graphs: bool = True, vae_chunk: int = 8,
                 prediction: str = "eps"):
        """prediction: "eps" (the UNet predicts the noise) or "v" (v-parameterisation, SD 2.x 768-v and v finetunes)"""
        if prediction not in PREDICTIONS:
            raise ValueError(f"prediction {prediction!r} is not one of {PREDICTIONS}")
        if unet_cfg.in_channels not in IN_CHANNELS:
            raise ValueError(f"a UNet with {unet_cfg.in_channels} input channels is not served: only 4-channel models and "
                             f"9-channel inpainting models are (not instruct-pix2pix's 8 or depth2img's 5)")
        self.prediction = prediction
        self.device = torch.device(device)
        if self.device.type != "cuda" and self._require_cuda:
            raise RuntimeError("SDEngine needs a CUDA device: the hot path is sm_90a kernels only (no CPU fallback)")
        w_in = sd[UNET_PREFIX + "input_blocks.0.0.weight"].shape[1]
        if w_in != unet_cfg.in_channels:
            raise ValueError(f"the UNet config takes {unet_cfg.in_channels} input channels but the checkpoint's conv_in "
                             f"takes {w_in}")
        self.dtype = dtype
        self.unet_cfg, self.vae_cfg, self.clip_cfg = unet_cfg, vae_cfg, clip_cfg
        self.use_graphs = use_graphs
        self.vae_chunk = vae_chunk
        with self._ctx():
            self.unet_w = UNetWeights(sd, unet_cfg, self.device, dtype)
            self.vae_w = VAEDecoderWeights(sd, vae_cfg, self.device, dtype)
            self.vae_enc_w = VAEEncoderWeights(sd, vae_cfg, self.device, dtype)
            self.clip = Conditioner(sd, clip_cfg, self.device, dtype, use_graphs=use_graphs)
            self.temb = TimeEmbedding(self.unet_w)
        self.plans: Dict[Tuple[int, int, int], Plan] = {}
        self.encoders: Dict[Tuple[int, int, int], VAEEncoderProgram] = {}
        self.interrupted = False
        self.variation = (None, 0.0)   # (subseed, subseed_strength) of the request being served: sdwui variation seeds
        self._y = None                 # SDXL vector conditioning of the run in progress
        self._windows = []             # (guidance_start, guidance_end) of the run's ControlNet unit in each slot
        self._entries = None           # prompt editing: (cond ends, uncond ends, cond entries) of the run in progress
        self._ybank = None             # ... and the entries' SDXL vector conditionings (cond, uncond)
        self._last_entry = None        # (cond, uncond) bank entries the K/V buffers hold
        self._cap_stream = None
        self.last_unet_evals = 0
        self.graph_replayed_launches = 0   # b200sd kernels launched through graph replays (bench.py gpu_launches)
        self._lora_set = ()            # identity of the LoRA networks merged into the weights; () = pristine weights
        self._lora_touched = set()     # (owner, packed tensor) the merged set rewrote
        self._pristine: Dict[tuple, torch.Tensor] = {}   # their pristine copies, made when a LoRA first touches one
        self._lora_keys = None         # lora.KeyTable of this model, built on the first LoRA request

    @property
    def inpainting(self) -> bool:
        """a 9-channel inpainting UNet: every sampling run packs its image conditioning (mask, masked-image latents)"""
        return self.unet_cfg.in_channels == 9

    def _capture_stream(self):
        """torch.cuda.graph's default capture stream is ONE process-wide stream, created on whichever device captured
        first — a second engine on another device would capture (and then run) its kernels on that other device.
        Every engine captures on a stream of its own device."""
        if self._cap_stream is None:
            self._cap_stream = torch.cuda.Stream(device=self.device)
        return self._cap_stream

    def merged_tokens(self, h: int, w: int, ratio: float) -> int:
        """r of sdwui's token merging at `ratio` for an h x w latent: tomesd's int(N * ratio) of the N = h*w tokens of the
        full-resolution transformer blocks, capped at the 3/4 N src tokens of the 2x2 grid.  0 for a ratio <= 0 (sdwui
        patches nothing) and for a UNet without attention at full resolution (SDXL)."""
        if not ratio > 0 or not self.unet_cfg.depth(0):
            return 0
        n = h * w
        return min(n - (h // 2) * (w // 2), int(n * ratio))

    def plan(self, b: int, h: int, w: int, tiling: bool = False, token_merging_ratio: float = 0.0) -> Plan:
        """the plan of (b, h, w); tiled plans are kept apart under (b, h, w, "tiling"), and plans that merge r > 0 tokens
        under the same key + ("tome", r)"""
        r = self.merged_tokens(h, w, token_merging_ratio)
        key = (b, h, w, "tiling") if tiling else (b, h, w)
        if r:
            key += ("tome", r)
        down = 2 ** (len(self.unet_cfg.channel_mult) - 1)
        if b < 1 or h < down or w < down or h % down or w % down:
            # the UNet halves the latent len(channel_mult) - 1 times and concatenates skip tensors on the way up: upstream
            # ldm fails with a size mismatch for other sizes, here it is refused before any buffer is built
            raise ValueError(f"latent size {h}x{w} (batch {b}) is not a positive multiple of {down}: image sides must be "
                             f"multiples of {8 * down} pixels")
        if key not in self.plans:
            while len(self.plans) >= MAX_PLANS:   # LRU: a client varying sizes must not walk the device out of memory
                old = self.plans.pop(next(iter(self.plans)))
                old.graphs.clear()
            with self._ctx():
                self.plans[key] = Plan(self, b, h, w, self.vae_chunk, tiling, r)
        else:
            self.plans[key] = self.plans.pop(key)   # most recently used last
        return self.plans[key]

    def release(self):
        """drop every plan, graph and encoder program (factory.evict / LocalGPUWorker.restart); merged LoRA networks are
        taken out of the weights first and the pristine copies freed"""
        self.set_loras(())
        self._pristine.clear()
        for p in self.plans.values():
            p.graphs.clear()
        self.plans.clear()
        self.encoders.clear()
        if self.device.type == "cuda":
            with self._ctx():
                torch.cuda.empty_cache()

    # ------------------------------------------------------------------------------------------ LoRA networks
    def _lora_owners(self):
        """{owner: (packed tensors, placements)}: the UNet and the text towers (ControlNets and the VAE are never touched)"""
        towers = [("t0", self.clip.t0)] + ([("t1", self.clip.t1)] if self.clip.xl else [])
        return {"unet": (self.unet_w.t, self.unet_w.place), **{n: (t.w, t.place) for n, t in towers}}

    def lora_key_table(self) -> "L.KeyTable":
        """sdwui's network_layer_mapping of this model: UNet names without `model.`, text towers without
        `cond_stage_model.` (SD1.x, SD 2.x) or `conditioner.embedders.` (SDXL)"""
        if self._lora_keys is None:
            cut = "conditioner.embedders." if self.clip.xl else "cond_stage_model."
            owners = [("unet", self.unet_w.place, UNET_PREFIX[:-len("diffusion_model.")], False)]
            owners += [(n, pl, cut, True) for n, (_, pl) in self._lora_owners().items() if n != "unet"]
            self._lora_keys = L.KeyTable(owners, self.unet_cfg, self.clip_cfg.open_clip)
        return self._lora_keys

    @torch.no_grad()
    def set_loras(self, nets=()):
        """Merge the LoRA networks `nets` [(lora.LoraFile, lora.LoraRef)] into the packed UNet and text-tower weights, in
        place on this engine's stream (captured graphs stay valid); () restores the pristine weights.  The set merged now
        costs nothing; another set rewrites, from the pristine copies, only the tensors the old or the new set touches.
        A tensor's pristine copy is made the first time a network touches it (an engine without LoRA requests holds
        none).  Every output is bitwise the same on every device (ops.lora_merge)."""
        key = tuple((f.key or (f.name, id(f)), r.te, r.unet, r.dyn) for f, r in nets)
        if key == self._lora_set:
            return
        owners = self._lora_owners()
        packed = {n: t for n, (t, _) in owners.items()}
        with self._ctx():
            groups = L.plan(L.resolve(self.lora_key_table(), list(nets)) if nets else [],
                            {n: pl for n, (_, pl) in owners.items()}, packed, self.device)
            touched = set(groups)
            for k in self._lora_touched - touched:
                groups[k] = [L.Group(0, packed[k[0]][k[1]].shape[0])]
            targets = []
            for (owner, name), gs in groups.items():
                w = packed[owner][name]
                p = self._pristine.get((owner, name))
                if p is None:
                    p = self._pristine[(owner, name)] = w.clone()
                for g in gs:
                    u = g.U if g.U is not None else torch.zeros((g.hi - g.lo, 0), device=self.device)
                    d = g.D if g.D is not None else torch.zeros((0, w.shape[1]), device=self.device)
                    targets.append((w[g.lo:g.hi], p[g.lo:g.hi], u, d))
            ops.lora_merge(targets)
        self._lora_set, self._lora_touched = key, touched

    def _use_loras(self, loras):
        """a request's networks: None (a request without tags) restores pristine weights if a set is merged, else
        nothing happens"""
        if loras is not None or self._lora_set:
            self.set_loras(loras or ())

    @torch.no_grad()
    def encode_prompts(self, tokens: torch.Tensor, width: int = 512, height: int = 512, zero_txt: bool = False,
                       multipliers: Optional[torch.Tensor] = None):
        """tokens [b, 77 * k] (k chunks of [BOS] + 75 + [EOS], factory.tokenize_prompts) -> cross-attention context
        [b, 77 * k, ctx] (SD1.x), or Cond(ctx, vector conditioning) for SDXL.  multipliers [b, 77 * k]: sdwui emphasis
        weights of the tokens (None: all 1)."""
        with self._ctx():
            c = self.clip(tokens, width, height, zero_txt, multipliers)
            return c if c.y is not None else c.ctx

    def _conds(self, tokens: torch.Tensor, neg_tokens: torch.Tensor, width: int, height: int, multipliers=None,
               neg_multipliers=None):
        """(cond, uncond) of a request.  SDXL: an all-empty negative prompt ([BOS] + EOS padding in every row) gets zero
        text embeddings, as sdwui's sd_models_xl.get_learned_conditioning does (force_zero_embeddings=['txt'])."""
        empty_neg = self.clip.xl and bool((neg_tokens[:, 1:] == neg_tokens[:, -1:]).all())
        return (self.encode_prompts(tokens, width, height, multipliers=multipliers),
                self.encode_prompts(neg_tokens, width, height, zero_txt=empty_neg, multipliers=neg_multipliers))

    def _pass_conds(self, tokens, neg_tokens, width: int, height: int, multipliers, neg_multipliers, schedule):
        """(cond, uncond, run_program's schedule) of one sampling pass.  schedule = (cond PromptSchedule, uncond
        PromptSchedule) or None (the tokens).  Schedules of one entry per side are encoded as that entry for every image
        and run as an unscheduled pass; otherwise every entry is encoded once and the pass switches between them."""
        if schedule is None:
            return (*self._conds(tokens, neg_tokens, width, height, multipliers, neg_multipliers), None)
        cs, us = schedule
        if len(cs.ends) == 1 and len(us.ends) == 1:
            b = tokens.shape[0]
            rows = lambda t: None if t is None else t[:1].expand(b, -1)  # noqa: E731
            return (*self._conds(rows(cs.tokens), rows(us.tokens), width, height, rows(cs.multipliers),
                                 rows(us.multipliers)), None)
        if len(cs.ends) > MAX_STEPS or len(us.ends) > MAX_STEPS:
            raise ValueError("too many prompt schedule entries")
        cond, uncond = self._conds(cs.tokens, us.tokens, width, height, cs.multipliers, us.multipliers)
        return cond, uncond, (cs.ends, us.ends)

    def _graph(self, plan: Plan, name: str, fn):
        """Run fn eagerly once (per-device kernel attribute setup must not happen under capture), then capture."""
        if not self.use_graphs or self.device.type != "cuda":
            return None
        if name not in plan.graphs:
            # eager warm-up on scratch state: save what a step mutates (x, counter, UNet input, and the generic stage
            # machine's latents — a multistep stage SHIFTS its history, which must not happen twice)
            state = [plan.x, plan.step, plan.unet.xin, plan.old] + [v for k, v in plan.lat.items() if k != "x"]
            saved = [t.clone() for t in state]
            s = torch.cuda.Stream(device=self.device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn()
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            # One LocalGPUWorker thread per device may be building its graphs at the same time: capture one at a time,
            # and in thread-local error mode so that another thread's allocations / launches on ITS device do not
            # invalidate this capture (the default "global" mode does).
            with _CAPTURE_LOCK:
                l0 = ops.LAUNCHES
                with torch.cuda.graph(g, stream=self._capture_stream(), capture_error_mode="thread_local"):
                    fn()
                plan.graph_launches[name] = ops.LAUNCHES - l0   # b200sd kernels inside one replay
            # a client walking through cfg scales / samplers must not accumulate graphs without bound ("vae" stays)
            while len(plan.graphs) >= MAX_GRAPHS:
                victim = next(n for n in plan.graphs if n != "vae")
                del plan.graphs[victim]
                plan.graph_launches.pop(victim, None)
            plan.graphs[name] = g
            for t, v in zip(state, saved):
                t.copy_(v)
        else:
            plan.graphs[name] = plan.graphs.pop(name)   # most recently used last
        return plan.graphs[name]

    # ------------------------------------------------------------------------------------------ sampler programs
    def program(self, sampler: str, scheduler: Optional[str], steps: int, denoise: Optional[float] = None,
                masked: bool = False) -> "Program":
        """(sampler name, API scheduler, steps[, img2img denoising strength]) -> what to run: the fused per-step kernels
        for DDIM / Euler a / Euler / DPM++ 2M, a stage list (b200sd/samplers.py) for every other sampler of the
        reference's table.  With `denoise` the program is the img2img half: the sampler's schedule from t_enc on
        (sdwui sd_samplers_timesteps.sample_img2img / KDiffusionSampler.sample_img2img)."""
        method, sched = resolve_sampler(sampler, scheduler)
        pr = Program(sampler, method, steps=steps)
        if method in ("ddim", "plms"):
            ac = alphas_cumprod().double()
            ts_all = torch.clamp(torch.arange(0, 1000, 1000 // steps) + 1, 0, 999)
            if denoise is None:
                sub = ts_all
            else:
                t_enc = max(1, min(int(min(denoise, 0.999) * steps), len(ts_all) - 1))
                a_start = float(ac[ts_all[t_enc]])
                pr.init_scale, pr.noise_scale = math.sqrt(a_start), math.sqrt(1 - a_start)
                sub = ts_all[:t_enc]
            if method == "ddim":
                pr.fused = "ddim"
                a = ac[sub]
                a_prev = ac[torch.cat([sub.new_zeros(1), sub[:-1]])]
                for i in range(len(sub) - 1, 0, -1):
                    at, ap = float(a[i]), float(a_prev[i])
                    pr.ts.append(float(sub[i]))
                    pr.rows.append([math.sqrt(at), math.sqrt(1 - at), math.sqrt(ap), math.sqrt(1 - ap)])
            else:
                pr.sp = S.plms([int(t) for t in sub], [float(v) for v in ac])
            pr.timestep_sampler = True
            return pr
        sig, log_sig = kdiffusion_sigmas(steps, sched)
        if denoise is not None:
            t_enc = int(min(denoise, 0.999) * steps)
            sig = sig[steps - t_enc - 1:]
            pr.init_scale, pr.noise_scale = 1.0, float(sig[0])
        else:
            pr.noise_scale = float(sig[0])
        pr.in0 = S.c_in(float(sig[0]))
        if method in ("euler_a", "euler", "dpmpp_2m") and not masked:   # with a mask: the same sampler as stages
            pr.fused = method
            fn = {"euler_a": euler_a_plan, "euler": euler_plan, "dpmpp_2m": dpmpp_2m_plan}[method]
            pr.ts, pr.rows, _ = fn(len(sig) - 1, sched, (sig, log_sig))
            if self.prediction == "v":
                pr.rows = v_rows(method, pr.rows)
            pr.draws = len(pr.rows) if method == "euler_a" else 0
            return pr
        sg = [float(v) for v in sig]
        t_of = lambda v: sigma_to_t(v, log_sig)  # noqa: E731
        if method in ("dpm_fast", "dpm_adaptive"):
            # sdwui passes sigma_min / sigma_max instead of a schedule: the model's own extremes for txt2img, the ends
            # of the (positive part of the) tail for img2img; DPM fast spends n = steps evaluations
            sig_all = log_sig.exp()
            lo, hi = (float(sig_all[0]), float(sig_all[-1])) if denoise is None else (sg[-2], sg[0])
            if method == "dpm_fast":
                pr.sp = S.dpm_fast(lo, hi, len(sg) - 1, t_of)
            else:
                pr.adaptive = (lo, hi, t_of)
            return pr
        pr.sp = S.BUILDERS[method](sg, t_of)
        pr.draws = pr.sp.draws
        return pr

    def _stage_graph(self, plan: Plan, st, cfg_scale: float, masked: bool, ts_sampler: bool, active=()):
        sid = plan.stage_ids.setdefault((st.lcs, st.ev), len(plan.stage_ids))   # exact structure -> id (no hash collisions)
        name = f"stage:{sid}:{cfg_scale}:{int(masked)}{int(ts_sampler)}" + self._control_name(plan, active)
        fn = lambda: plan.stage(st.lcs, st.ev, cfg_scale, masked, ts_sampler, active)  # noqa: E731
        return name, fn, self._graph(plan, name, fn)

    # ------------------------------------------------------------------------------------------ ControlNet
    def _set_controls(self, plan: Plan, controls):
        """controls: [(ControlNetWeights, hint uint8 [8h, 8w, 3], weight, guidance_start, guidance_end)], unit k in slot k.
        Builds the slots' segments (dropping the graphs that ran a slot's previous model), runs each hint block and
        scales the slots' zero convs; returns the (start, end) windows."""
        if len(controls) > MAX_CONTROLS:
            raise ValueError(f"{len(controls)} ControlNet units: at most {MAX_CONTROLS} are served")
        windows = []
        for slot, (cw, hint, weight, start, end) in enumerate(controls):
            if not isinstance(cw, ControlNetWeights) or cw.cfg != self.unet_cfg:
                raise ValueError(f"ControlNet {getattr(cw, 'name', cw)!r} does not match this engine's UNet")
            if tuple(hint.shape) != (8 * plan.h, 8 * plan.w, 3) or hint.dtype != torch.uint8:
                raise ValueError(f"control map {tuple(hint.shape)} {hint.dtype}: expected uint8 "
                                 f"({8 * plan.h}, {8 * plan.w}, 3)")
            if plan.unet.set_control(slot, cw, MAX_STEPS, plan.step):
                for name in [n for n in plan.graphs if f"|cn{slot}=" in n]:
                    del plan.graphs[name]
                    plan.graph_launches.pop(name, None)
            plan.unet.segments[slot].set_hint(hint.to(self.device), float(weight))
            windows.append((float(start), float(end)))
        return windows

    def _active(self, i: int, n: int) -> tuple:
        """slots whose unit is active at sampler step i of n: guidance_start <= i / n <= guidance_end"""
        return tuple(s for s, (a, b) in enumerate(self._windows) if a <= i / n <= b)

    @staticmethod
    def _control_name(plan: Plan, active) -> str:
        """graph-name suffix of the active slots and their models (empty without ControlNet: today's names)"""
        return "".join(f"|cn{s}={plan.unet.segments[s].w.name}" for s in active)

    def _control_tables(self, plan: Plan, ts: torch.Tensor):
        """each unit's own time-embedding rows for the evaluations' timesteps"""
        for s in range(len(self._windows)):
            seg = plan.unet.segments[s]
            seg.table[:ts.numel()].copy_(TimeEmbedding(seg.w).table(ts))

    @torch.no_grad()
    def run_program(self, cond: torch.Tensor, uncond: torch.Tensor, x_start: torch.Tensor, pr: "Program", cfg_scale: float,
                    noises: Optional[torch.Tensor] = None, inpaint=None, controls=None,
                    tiling: bool = False, image_cond=None, token_merging_ratio: float = 0.0,
                    schedule=None) -> torch.Tensor:
        """cond/uncond [b, 77 * k, ctx] on device (cond and uncond may have different k); x_start [b, 4, h, w] fp32 (host or device) = Program.start(...): the start
        latents in the sampler's own space; noises [pr.draws, b, 4, h, w]: the per-image N(0,1) draws after the first;
        inpaint = (clean init latents [b, 4, h, w], latent mask [h * w]).  controls: ControlNet units, see _set_controls
        (None: no ControlNet).  tiling: the UNet's convs pad circularly (its own plan).  image_cond = (masked-image
        latents fp32 [b, 4, h, w], pixel mask uint8 [f*h, f*w] or None for all ones): an inpainting model's extra UNet
        input channels, packed once before sampling (required for a 9-channel UNet, refused for a 4-channel one).
        token_merging_ratio: sdwui's token merging (its own plan; see merged_tokens).  schedule = (cond ends, uncond
        ends): prompt editing — cond / uncond are then the encoded entries of the two schedules [E, 77 * k, ctx] and
        every model evaluation attends to its own entries (sdwui reconstruct_cond_batch).  Returns the final latents fp32
        [b, h*w, 4] (NHWC, a view of plan state)."""
        b, _, h, w = x_start.shape
        if pr.draws and (noises is None or noises.shape[0] < pr.draws):
            raise ValueError(f"{pr.sampler} needs {pr.draws} per-image noise draws")
        if (image_cond is not None) != self.inpainting:
            raise ValueError("an inpainting model samples with its image conditioning" if self.inpainting else
                             "image conditioning is for 9-channel inpainting models only")
        if inpaint is not None and pr.fused not in (None, "ddim"):
            # the fused Euler / Euler a / DPM++ 2M kernels do not carry the mask: same sampler, generic stages
            raise ValueError("masked sampling of a fused sampler must be requested through a generic program")
        cond = cond if isinstance(cond, Cond) else Cond(cond)
        uncond = uncond if isinstance(uncond, Cond) else Cond(uncond)
        with self._ctx():
            plan = self.plan(b, h, w, tiling, token_merging_ratio)
            if controls and cond.y is not None:
                raise ValueError("ControlNet is not served for SDXL")
            self._windows = self._set_controls(plan, controls) if controls else []
            if schedule is None:
                self._entries = self._ybank = None
                plan.set_context(cond.ctx, uncond.ctx)
                # SDXL: the vector conditioning of [cond | uncond] enters through the time-embedding table (per-sample
                # rows)
                self._y = None if cond.y is None else torch.cat([cond.y, uncond.y]).to(self.device)
            else:
                self._entries = (list(schedule[0]), list(schedule[1]), cond.ctx.shape[0])
                self._ybank = None if cond.y is None else (cond.y.to(self.device), uncond.y.to(self.device))
                self._y = None
                self._last_entry = None
                plan.set_bank(cond.ctx, uncond.ctx)
            masked = inpaint is not None
            if masked:   # (clean init latents [b, 4, h, w], latent mask [h * w])
                plan.init.copy_(inpaint[0].to(self.device, torch.float32).permute(0, 2, 3, 1).reshape(b, h * w, 4))
                plan.latmask.copy_(inpaint[1].to(self.device, torch.float32).reshape(-1))
            if image_cond is not None:   # channels 4..8 of [cond | uncond]; the step kernels write channels 0..3 only
                z, m = image_cond
                ops.pack_image_cond(z.to(self.device, torch.float32).permute(0, 2, 3, 1).reshape(b, h * w, 4).contiguous(),
                                    None if m is None else m.to(self.device, torch.uint8).contiguous(), plan.unet.xin, h, w)
            plan.x.copy_(x_start.to(self.device, torch.float32).permute(0, 2, 3, 1).reshape(b, h * w, 4))
            plan.step.zero_()
            ops.pack_unet_input(plan.x, plan.unet.xin, pr.in0)
            self.last_unet_evals = 0
            if pr.adaptive is not None:
                self._run_dpm_adaptive(plan, pr, cfg_scale, masked)
            elif pr.fused is not None:
                self._run_fused(plan, pr, cfg_scale, noises, masked)
            else:
                self._run_stages(plan, pr.sp, cfg_scale, noises, masked)
            if masked:   # processing.py sample(): samples * nmask + init_latent * mask
                ops.blend_latent(plan.x, plan.init, plan.latmask)
            return plan.x

    # ------------------------------------------------------------------------------------------ prompt editing
    def _entry(self, i: int) -> tuple:
        """(cond, uncond) bank entries of model evaluation i"""
        cond_ends, uncond_ends, ec = self._entries
        return (schedule_index([(e, None) for e in cond_ends], i),
                ec + schedule_index([(e, None) for e in uncond_ends], i))

    def _set_sched(self, plan: Plan, i0: int, n: int):
        """schedule-table rows 0..n-1 <- the entries of evaluations i0..i0+n-1 (no-op without a schedule)"""
        if self._entries is not None and n:
            plan.set_sched(0, [self._entry(i0 + k) for k in range(n)])

    def _emb_table(self, plan: Plan, ts: torch.Tensor, i0: int) -> torch.Tensor:
        """time-embedding rows of evaluations i0..: SDXL under a schedule takes each evaluation's vector conditioning
        from its entries, one table per distinct entry pair"""
        if self._ybank is None:
            return self.temb.table(ts, self._y)
        yc, yu = self._ybank
        ec = self._entries[2]
        groups: Dict[tuple, List[int]] = {}
        for k in range(ts.numel()):
            groups.setdefault(self._entry(i0 + k), []).append(k)
        out = torch.empty((ts.numel(), plan.table.shape[1]), device=self.device, dtype=torch.float32)
        for (c, u), idx in groups.items():
            y = torch.cat([yc[c:c + 1].expand(plan.b, -1), yu[u - ec:u - ec + 1].expand(plan.b, -1)])
            out[torch.tensor(idx, device=self.device)] = self.temb.table(ts[idx], y)
        return out

    def _switch(self, plan: Plan, i: int):
        """before model evaluation i: replay the "ctx" graph when its entries differ from the ones the K/V buffers hold.
        The graph reads the device step counter, i.e. the schedule-table row _set_sched filled for evaluation i."""
        if self._entries is None:
            return
        e = self._entry(i)
        if e == self._last_entry:
            return
        self._last_entry = e
        slots = tuple(range(len(self._windows)))
        name = "ctx" + self._control_name(plan, slots)
        fn = lambda: plan.switch_context(slots)  # noqa: E731
        g = self._graph(plan, name, fn)
        if g is not None:
            g.replay()
            self.graph_replayed_launches += plan.graph_launches[name]
        else:
            fn()

    def _upload_noises(self, plan: Plan, noises: torch.Tensor, mix=None):
        """draws [D, b, 4, h, w] (host) -> rows of the plan's persistent noise stack, mixed as the program says"""
        d = noises.to(torch.float32)
        if mix is not None:
            d = torch.stack([sum(w * d[i] for i, w in row) for row in mix]) if mix else d[:0]
        n = d.shape[0]
        if n:
            plan.noise_rows(n)[:n].copy_(d.to(self.device).permute(0, 1, 3, 4, 2).reshape(n, plan.b, plan.h * plan.w, 4))
        elif plan.noise is None:
            plan.noise_rows(1)

    def _run_fused(self, plan: Plan, pr: "Program", cfg_scale: float, noises, masked: bool):
        n_evals = len(pr.ts)
        if n_evals > MAX_STEPS:
            raise ValueError("too many steps")
        if n_evals == 0:   # img2img at a very low denoising strength runs zero evaluations: the noised init comes back
            return
        name = f"{pr.sampler if pr.fused != 'ddim' else 'DDIM'}:{cfg_scale}"
        if pr.fused == "ddim":
            step_fn = (lambda a=(): plan.step_ddim_masked(cfg_scale, a)) if masked else \
                (lambda a=(): plan.step_ddim(cfg_scale, a))
            name += ":mask" if masked else ""
        elif pr.fused == "euler_a":
            self._upload_noises(plan, noises[:n_evals])
            name = f"Euler a:{cfg_scale}"
            step_fn = lambda a=(): plan.step_euler_a(cfg_scale, a)  # noqa: E731
        elif pr.fused == "euler":
            step_fn = lambda a=(): plan.step_euler(cfg_scale, a)  # noqa: E731
        else:
            step_fn = lambda a=(): plan.step_dpmpp_2m(cfg_scale, a)  # noqa: E731
        ts = torch.tensor(pr.ts, dtype=torch.float32)
        self._set_sched(plan, 0, n_evals)
        plan.table[:n_evals].copy_(self._emb_table(plan, ts, 0))
        self._control_tables(plan, ts)
        (plan.coef8 if len(pr.rows[0]) == 8 else plan.coef)[:n_evals].copy_(torch.tensor(pr.rows, dtype=torch.float32))
        steps = {}   # active ControlNet slots -> (graph name, step function, graph); no units: () for every evaluation
        for i in range(n_evals):
            if self.interrupted:
                break
            active = self._active(i, n_evals)
            if active not in steps:
                fn = (lambda a: lambda: step_fn(a))(active) if active else step_fn
                gname = name + self._control_name(plan, active)
                steps[active] = (gname, fn, self._graph(plan, gname, fn))
            gname, fn, g = steps[active]
            self._switch(plan, i)
            if g is not None:
                g.replay()
                self.graph_replayed_launches += plan.graph_launches[gname]
            else:
                fn()
            self.last_unet_evals += 1

    def _run_stages(self, plan: Plan, sp, cfg_scale: float, noises, masked: bool):
        stages = sp.stages
        if len(stages) > MAX_STEPS:
            raise ValueError("too many model evaluations")
        if not stages:
            return
        self._upload_noises(plan, noises if noises is not None else torch.zeros((0, plan.b, 4, plan.h, plan.w)), sp.mix)
        ts = torch.tensor([st.t for st in stages], dtype=torch.float32)
        self._set_sched(plan, 0, len(stages))
        plan.table[:len(stages)].copy_(self._emb_table(plan, ts, 0))
        self._control_tables(plan, ts)
        plan.coefL[:len(stages)].copy_(torch.tensor([st.row() for st in stages], dtype=torch.float32))
        step_of = S.stage_steps(stages)
        for st, i in zip(stages, step_of):
            if self.interrupted:
                break
            name, fn, g = self._stage_graph(plan, st, cfg_scale, masked, sp.timestep_sampler,
                                            self._active(i, step_of[-1] + 1))
            self._switch(plan, self.last_unet_evals)
            if g is not None:
                g.replay()
                self.graph_replayed_launches += plan.graph_launches[name]
            else:
                fn()
            self.last_unet_evals += 1

    def _run_dpm_adaptive(self, plan: Plan, pr: "Program", cfg_scale: float, masked: bool):
        """k-diffusion sample_dpm_adaptive -> DPMSolver.dpm_solver_adaptive(order 3, rtol 0.05, atol 0.0078, h_init 0.05,
        PI controller icoeff 1, accept_safety 0.81, eta 0): the step size depends on an error norm over the WHOLE batch, so
        the host reads one scalar per attempted step (3 evaluations) and rewrites three coefficient / time-embedding rows.
        (Being batch-coupled upstream, this sampler is the one whose images depend on how the request was sharded.)"""
        sigma_min, sigma_max, t_of = pr.adaptive
        t_start, t_end = -math.log(sigma_max), -math.log(sigma_min)
        rtol, atol, order = 0.05, 0.0078, 3
        pid = S.PIDStepSizeController(0.05, 0.0, 1.0, 0.0, order, 0.81)
        s = t_start
        accepted = 0   # the sampler step of an attempt (ControlNet windows: of the requested steps)
        x_prev = plan.x.clone()
        if plan.noise is None:
            plan.noise_rows(1)
        while s < t_end - 1e-5:
            if self.interrupted:
                break
            t = min(t_end, s + pid.h)
            stages = S.dpm_adaptive_attempt(s, t, t_of)
            ts = torch.tensor([st.t for st in stages], dtype=torch.float32)
            self._set_sched(plan, self.last_unet_evals, 3)
            plan.table[:3].copy_(self._emb_table(plan, ts, self.last_unet_evals))
            self._control_tables(plan, ts)
            plan.coefL[:3].copy_(torch.tensor([st.row() for st in stages], dtype=torch.float32))
            active = self._active(accepted, max(pr.steps, 1)) if self._windows else ()
            plan.step.zero_()
            ops.pack_unet_input(plan.x, plan.unet.xin, S.c_in(math.exp(-s)))
            for st in stages:
                name, fn, g = self._stage_graph(plan, st, cfg_scale, masked, False, active)
                self._switch(plan, self.last_unet_evals)
                if g is not None:
                    g.replay()
                    self.graph_replayed_launches += plan.graph_launches[name]
                else:
                    fn()
                self.last_unet_evals += 1
            x_low, x_high = plan.lat["h3"], plan.lat["u"]
            delta = torch.maximum(torch.full_like(x_low, atol), rtol * torch.maximum(x_low.abs(), x_prev.abs()))
            error = float(torch.linalg.norm((x_low - x_high) / delta) / x_low.numel() ** 0.5)
            if pid.propose_step(error):
                x_prev.copy_(x_low)
                plan.x.copy_(x_high)
                s = t
                accepted += 1

    @torch.no_grad()
    def sample(self, cond: torch.Tensor, uncond: torch.Tensor, x_T: torch.Tensor, steps: int, cfg_scale: float,
               sampler: str = "DDIM", noises: Optional[torch.Tensor] = None, schedule=None,
               scheduler: Optional[str] = None, sigmas=None, inpaint=None) -> torch.Tensor:
        """txt2img sampling from unit noise x_T [b, 4, h, w] (the historical entry point; tests drive it directly).
        `schedule` = (timesteps, coef rows) overrides the DDIM schedule and `sigmas` = (sigma table ending in 0, model
        log-sigmas) the k-diffusion one — x_T is then the ALREADY NOISED start.  Requests go through program() /
        run_program()."""
        pr = self.program(sampler, scheduler, steps)
        if schedule is not None:
            pr.ts, pr.rows = list(schedule[0]), list(schedule[1])
            pr.noise_scale = 1.0
        if sigmas is not None:
            fn = {"euler_a": euler_a_plan, "euler": euler_plan, "dpmpp_2m": dpmpp_2m_plan}[pr.fused]
            pr.ts, pr.rows, sigma0 = fn(len(sigmas[0]) - 1, None, sigmas)
            if self.prediction == "v":
                pr.rows = v_rows(pr.fused, pr.rows)
            pr.noise_scale, pr.in0 = 1.0, S.c_in(sigma0)
            pr.draws = len(pr.rows) if pr.fused == "euler_a" else 0
        return self.run_program(cond, uncond, x_T.to(torch.float32) * pr.noise_scale, pr, cfg_scale, noises, inpaint)

    @torch.no_grad()
    def decode(self, latents: torch.Tensor, h: int, w: int, tiling: bool = False,
               token_merging_ratio: float = 0.0) -> torch.Tensor:
        """latents fp32 [b, h*w, 4] (scaled) -> uint8 [b, 8h, 8w, 3] on device.  tiling: circular convs (the tiled plan's
        decoder).  token_merging_ratio: the decoder of the plan that sampled them (merging does not touch the VAE; the
        request then builds one plan, not two)."""
        b = latents.shape[0]
        with self._ctx():
            plan = self.plan(b, h, w, tiling, token_merging_ratio)
            vae = plan.vae
            out = torch.empty((b, vae.out_h * vae.out_w, 3), device=self.device, dtype=torch.uint8)
            c = plan.vae_chunk
            for i in range(0, b, c):
                chunk = latents[i:i + c]
                if chunk.shape[0] < c:  # ragged tail: pad with the last latent, drop the surplus images
                    chunk = torch.cat([chunk, chunk[-1:].expand(c - chunk.shape[0], -1, -1)]).contiguous()
                vae.set_latents(chunk.contiguous(), self.vae_cfg.scale_factor)
                if self.use_graphs and self.device.type == "cuda":
                    if "vae" not in plan.graphs:
                        vae.run()
                        torch.cuda.current_stream().synchronize()
                        g = torch.cuda.CUDAGraph()
                        with _CAPTURE_LOCK:
                            l0 = ops.LAUNCHES
                            with torch.cuda.graph(g, stream=self._capture_stream(), capture_error_mode="thread_local"):
                                vae.run()
                            plan.graph_launches["vae"] = ops.LAUNCHES - l0
                        plan.graphs["vae"] = g
                    plan.graphs["vae"].replay()
                    self.graph_replayed_launches += plan.graph_launches["vae"]
                else:
                    vae.run()
                n = min(c, b - i)
                out[i:i + n].copy_(vae.u8[:n])
            return out.reshape(b, vae.out_h, vae.out_w, 3)

    @torch.no_grad()
    def encode(self, images_u8: torch.Tensor, tiling: bool = False) -> torch.Tensor:
        """images uint8 [b, H, W, 3] (host or device) -> scaled latents fp32 [b, 4, H/f, W/f] (posterior mean), in
        chunks of `vae_chunk` images.  tiling: circular convs (an encoder program of its own)."""
        return self._encode(images_u8, tiling)

    @torch.no_grad()
    def encode_conditioning(self, images_u8: torch.Tensor, mask_u8: Optional[torch.Tensor] = None, weight: float = 1.0,
                            tiling: bool = False) -> torch.Tensor:
        """the masked-image half of an inpainting model's conditioning (sdwui inpainting_image_conditioning): uint8
        images [b, H, W, 3] and the pixel mask uint8 [H, W] (None: all ones) -> scaled latents fp32 [b, 4, H/f, W/f] of
        s * (1 - weight * [mask >= 128]), s = 2x/255 - 1, encoded as `encode` encodes init images"""
        return self._encode(images_u8, tiling, (mask_u8, weight))

    def _encode(self, images_u8: torch.Tensor, tiling: bool, condition=None) -> torch.Tensor:
        """encode / encode_conditioning; condition = (mask, weight) runs the masked encoder program of the size"""
        b, hh, ww, _ = images_u8.shape
        with self._ctx():
            c = min(self.vae_chunk, b)
            key = (c, hh, ww, "tiling") if tiling else (c, hh, ww)
            if condition is not None:
                key = key + ("masked",)
            if key not in self.encoders:
                while len(self.encoders) >= MAX_PLANS:
                    self.encoders.pop(next(iter(self.encoders)))
                self.encoders[key] = VAEEncoderProgram(self.vae_enc_w, c, hh, ww, tiling=tiling,
                                                       masked=condition is not None)
            enc = self.encoders[key]
            if condition is not None:
                mask, weight = condition
                enc.set_condition(None if mask is None else mask.to(self.device, torch.uint8), weight)
            imgs = images_u8.to(self.device).reshape(b, hh * ww, 3)
            out = torch.empty((b, enc.lat_h * enc.lat_w, 4), device=self.device, dtype=torch.float32)
            for i in range(0, b, c):
                chunk = imgs[i:i + c]
                n = chunk.shape[0]
                enc.img_u8[:n].copy_(chunk)
                if n < c:
                    enc.img_u8[n:].copy_(chunk[-1:].expand(c - n, -1, -1))
                enc.run()
                out[i:i + n].copy_(enc.latents[:n])
            return out.reshape(b, enc.lat_h, enc.lat_w, 4).permute(0, 3, 1, 2).contiguous()

    @torch.no_grad()
    def img2img(self, tokens: torch.Tensor, neg_tokens: torch.Tensor, seed: int, init_u8: torch.Tensor,
                denoising_strength: float = 0.75, steps: int = 20, cfg_scale: float = 7.0, sampler: str = "DDIM",
                scheduler: Optional[str] = None, latmask: Optional[torch.Tensor] = None,
                inpainting_fill: int = 1, multipliers: Optional[torch.Tensor] = None,
                neg_multipliers: Optional[torch.Tensor] = None, controls=None, tiling: bool = False,
                image_mask: Optional[torch.Tensor] = None, inpainting_mask_weight: float = 1.0,
                token_merging_ratio: float = 0.0, schedule=None, loras=None) -> torch.Tensor:
        """img2img: VAE-encode the init images (posterior mean), noise them to t_enc, run the remaining part of the
        sampler's schedule, decode.  init_u8 uint8 [b, H, W, 3].  Returns uint8 [b, H, W, 3] on device.
        `latmask` fp32 [h * w] (b200sd.inpaint.prepare_mask): inpainting — the region with latmask 0 is held to the init
        latents (timestep samplers: blended into x before every model call; k-diffusion samplers: blended into the
        denoised prediction, as sdwui's CFGDenoiser does); the caller composites the original pixels back
        (inpaint.apply_overlays).
        `inpainting_fill` 2 ("latent noise") / 3 ("latent nothing") replace the repainted region of the init latents by
        the request's start noise / by zeros first (sdwui Img2Img.init); 0 ("fill") is image-space work the caller does
        before the call (inpaint.fill_masked), 1 keeps the original content.
        `controls`: ControlNet units [(ControlNetWeights, control map uint8 [H, W, 3], weight, guidance_start,
        guidance_end)], at most 3 (None: none).
        `tiling`: sdwui's tiling option — every 3x3 conv of the UNet and the VAE pads circularly (ControlNet's do
        not).
        Inpainting models (9 input channels) are conditioned on the mask and the VAE latents of
        init * (1 - inpainting_mask_weight * mask) (sdwui img2img_image_conditioning): `image_mask` uint8 [H, W] is the
        processed pixel mask (inpaint.InpaintMask.fill_mask), required with `latmask`; without a mask it is all ones.
        Other models ignore both arguments.
        `token_merging_ratio`: sdwui's token merging (tomesd) in the UNet's full-resolution self-attention; <= 0 does not
        merge.
        `schedule` = (cond PromptSchedule, uncond PromptSchedule): prompt editing / alternation (sdwui's prompt
        schedules over the sampler's total steps); tokens / neg_tokens then give only the batch size.  None: the
        tokens for every step.
        `loras`: LoRA networks [(lora.LoraFile, lora.LoraRef)] merged for this request (set_loras); None: pristine
        weights."""
        b = tokens.shape[0]
        self._use_loras(loras)
        cond, uncond, sched = self._pass_conds(tokens, neg_tokens, init_u8.shape[2], init_u8.shape[1], multipliers,
                                               neg_multipliers, schedule)
        init = self.encode(init_u8, tiling)
        _, _, h, w = init.shape
        image_cond = None
        if self.inpainting:
            if latmask is not None and image_mask is None:
                raise ValueError("masked img2img on an inpainting model needs the pixel mask (image_mask)")
            image_cond = (self.encode_conditioning(init_u8, image_mask, inpainting_mask_weight, tiling), image_mask)
        if latmask is not None and inpainting_fill in (2, 3):
            nm = latmask.to(self.device, torch.float32).reshape(1, 1, h, w)
            init = init * (1.0 - nm)
            if inpainting_fill == 2:   # create_random_tensors(shape, seeds): the same first draw the sampler starts from
                init = init + per_image_noise(seed, b, (4, h, w), 1, *self.variation)[0].to(self.device) * nm
        lat = self._sample_from(init, cond, uncond, seed, denoising_strength, steps, cfg_scale, sampler, scheduler,
                                inpaint=None if latmask is None else (init, latmask), controls=controls, tiling=tiling,
                                image_cond=image_cond, token_merging_ratio=token_merging_ratio, schedule=sched)
        return self.decode(lat, h, w, tiling, token_merging_ratio)

    def _txt2img_cond(self, b: int, h: int, w: int, tiling: bool):
        """sdwui txt2img_image_conditioning of an inpainting model at latent size h x w: an all-ones mask over a gray image
        (0 in [-1, 1]).  Weight 1 under the all-ones mask zeroes every pixel, so one image of any content (255: +0) is
        encoded and shared by the b images."""
        f = 2 ** (len(self.vae_cfg.ch_mult) - 1)
        gray = torch.full((1, f * h, f * w, 3), 255, device=self.device, dtype=torch.uint8)
        return self.encode_conditioning(gray, None, 1.0, tiling).expand(b, -1, -1, -1), None

    def _sample_from(self, init: torch.Tensor, cond, uncond, seed: int, denoising_strength: float, steps: int,
                     cfg_scale: float, sampler: str, scheduler: Optional[str], inpaint=None, controls=None,
                     tiling: bool = False, image_cond=None, token_merging_ratio: float = 0.0,
                     schedule=None) -> torch.Tensor:
        """the img2img half of a sampler (also the second pass of the hires fix): `init` [b, 4, h, w] latents on the device,
        fresh per-image noise from `seed`, start at the noise level of t_enc.
        DDIM / PLMS: sdwui sd_samplers_timesteps.sample_img2img; k-diffusion samplers: KDiffusionSampler.sample_img2img."""
        b, _, h, w = init.shape
        pr = self.program(sampler, scheduler, steps, denoise=denoising_strength, masked=inpaint is not None)
        nz = per_image_noise(seed, b, (4, h, w), 1 + pr.draws, *self.variation)
        return self.run_program(cond, uncond, pr.start(nz[0].to(self.device), init), pr, cfg_scale,
                                noises=nz[1:] if pr.draws else None, inpaint=inpaint, controls=controls, tiling=tiling,
                                image_cond=image_cond, token_merging_ratio=token_merging_ratio, schedule=schedule)

    @torch.no_grad()
    def txt2img_hires(self, tokens: torch.Tensor, neg_tokens: torch.Tensor, seed: int, steps: int = 20,
                      cfg_scale: float = 7.0, height: int = 512, width: int = 512, hr_scale: float = 2.0,
                      hr_steps: int = 0, denoising_strength: float = 0.7, sampler: str = "DDIM",
                      scheduler: Optional[str] = None, multipliers: Optional[torch.Tensor] = None,
                      neg_multipliers: Optional[torch.Tensor] = None, upscaler: str = "Latent",
                      upscaler_tile: int = 192, upscaler_overlap: int = 8, tiling: bool = False,
                      inpainting_mask_weight: float = 1.0, token_merging_ratio: float = 0.0,
                      token_merging_ratio_hr: float = 0.0, schedule=None, hr_schedule=None, loras=None,
                      hr_loras=None) -> torch.Tensor:
        """txt2img with sdwui's hires fix (StableDiffusionProcessingTxt2Img.sample / sample_hr_pass): first pass at
        (height, width), the `upscaler` to hr_scale x, a fresh per-image noise of the large shape from the same seeds,
        then the same sampler's img2img half from t_enc with `hr_steps` (0 = `steps`) steps, decode at the large size.
        `upscaler` (b200sd.upscale): a "Latent ..." mode resizes the latents (F.interpolate); any other name decodes the
        first pass, resizes the uint8 images as sdwui's images.resize_image does (ESRGAN tiles of `upscaler_tile` pixels
        overlapping by `upscaler_overlap`) and VAE-encodes the result as img2img encodes init images.  `tiling` holds for
        both passes and the VAE decode / encode between them (the pixel upscalers are not part of the model).
        Inpainting models: the first pass and a "Latent" second pass get txt2img's conditioning, a pixel upscaler's second
        pass the upscaled images' under an all-ones mask, s * (1 - inpainting_mask_weight).  sdwui conditions a "Latent"
        second pass with a weight below 1 on the float decode of the upscaled latents: refused.
        Token merging: the first pass (and its decode) at `token_merging_ratio`, the second at `token_merging_ratio_hr`.
        `schedule` as for img2img, for the first pass; `hr_schedule` the second pass's own (sdwui hr_prompt /
        hr_negative_prompt over the hires steps, with the first pass's steps as the base of its offsets), required with
        `schedule`; without both the second pass takes the first pass's prompts.
        `loras` as for img2img, for the first pass; `hr_loras` the second pass's own networks (sdwui
        hr_extra_network_data; () for none), which re-encode its prompts; None: the first pass's.
        Returns uint8 [b, H*hr, W*hr, 3] on device."""
        from . import upscale
        if schedule is not None and hr_schedule is None:
            raise ValueError("a scheduled first pass needs the second pass's own schedule (hr_schedule): sdwui builds it "
                             "over the hires steps")
        kind, _ = upscale.kind(upscaler)
        if self.inpainting and kind == "latent" and inpainting_mask_weight < 1:
            raise ValueError(f"hires upscaler {upscaler!r} with inpainting_mask_weight {inpainting_mask_weight} < 1 is not "
                             f"served on an inpainting model")
        b = tokens.shape[0]
        self._use_loras(loras)
        h, w = height // 8, width // 8
        h2, w2 = int(height * hr_scale) // 8, int(width * hr_scale) // 8
        if kind != "latent" and (int(height * hr_scale) % 8 or int(width * hr_scale) % 8):
            raise ValueError(f"hires upscaler {upscaler!r}: the target size must be a multiple of 8")
        cond, uncond, sched = self._pass_conds(tokens, neg_tokens, width, height, multipliers, neg_multipliers, schedule)
        lat = self._sample_txt(cond, uncond, seed, b, h, w, steps, cfg_scale, sampler, scheduler, tiling=tiling,
                               image_cond=self._txt2img_cond(b, h, w, tiling) if self.inpainting else None,
                               token_merging_ratio=token_merging_ratio, schedule=sched)
        image_cond = None
        if kind == "latent":
            with self._ctx():
                if upscaler == "Latent":
                    up = torch.empty((b, h2 * w2, 4), device=self.device, dtype=torch.float32)
                    ops.resize_latent_bilinear(lat.contiguous(), up, h, w, h2, w2)
                else:
                    up = upscale.resize_latents(lat, upscaler, h, w, h2, w2)
            init = up.reshape(b, h2, w2, 4).permute(0, 3, 1, 2)
            if self.inpainting:
                image_cond = self._txt2img_cond(b, h2, w2, tiling)
        else:
            images = self.decode(lat, h, w, tiling, token_merging_ratio)
            f = 2 ** (len(self.vae_cfg.ch_mult) - 1)   # 8 for the kl-f8 autoencoder: the target is then W*hr x H*hr
            with self._ctx():
                images = upscale.resize_image(images, w2 * f, h2 * f, upscaler, upscaler_tile, upscaler_overlap)
            init = self.encode(images.contiguous(), tiling)
            if self.inpainting:
                image_cond = (self.encode_conditioning(images.contiguous(), None, inpainting_mask_weight, tiling), None)
        if hr_loras is not None:
            self.set_loras(hr_loras)
        if hr_schedule is not None:
            cond, uncond, sched = self._pass_conds(tokens, neg_tokens, w2 * 8, h2 * 8, None, None, hr_schedule)
        elif self.clip.xl or hr_loras is not None:   # SDXL's vector conditioning carries the target size: the second pass gets its own (sdwui hr_c / hr_uc)
            cond, uncond, sched = self._pass_conds(tokens, neg_tokens, w2 * 8, h2 * 8, multipliers, neg_multipliers,
                                                   schedule)
        lat2 = self._sample_from(init, cond, uncond, seed, denoising_strength, hr_steps or steps, cfg_scale, sampler, scheduler,
                                 tiling=tiling, image_cond=image_cond, token_merging_ratio=token_merging_ratio_hr,
                                 schedule=sched)
        return self.decode(lat2, h2, w2, tiling, token_merging_ratio_hr)

    def _sample_txt(self, cond, uncond, seed: int, b: int, h: int, w: int, steps: int, cfg_scale: float, sampler: str,
                    scheduler: Optional[str], controls=None, tiling: bool = False, image_cond=None,
                    token_merging_ratio: float = 0.0, schedule=None) -> torch.Tensor:
        pr = self.program(sampler, scheduler, steps)
        nz = per_image_noise(seed, b, (4, h, w), 1 + pr.draws, *self.variation)
        return self.run_program(cond, uncond, pr.start(nz[0]), pr, cfg_scale, noises=nz[1:] if pr.draws else None,
                                controls=controls, tiling=tiling, image_cond=image_cond,
                                token_merging_ratio=token_merging_ratio, schedule=schedule)

    @torch.no_grad()
    def txt2img(self, tokens: torch.Tensor, neg_tokens: torch.Tensor, seed: int, steps: int = 20, cfg_scale: float = 7.0,
                height: int = 512, width: int = 512, sampler: str = "DDIM", scheduler: Optional[str] = None,
                multipliers: Optional[torch.Tensor] = None, neg_multipliers: Optional[torch.Tensor] = None,
                controls=None, tiling: bool = False, inpainting_mask_weight: float = 1.0,
                token_merging_ratio: float = 0.0, schedule=None, loras=None) -> torch.Tensor:
        """Whole request for this engine's share: returns uint8 [b, H, W, 3] on device.  tokens [b, 77 * k] and
        neg_tokens [b, 77 * k'] with their optional emphasis multipliers of the same shapes (factory.tokenize_prompts).
        `controls`: ControlNet units as for img2img (None: none); `tiling` as for img2img.  An inpainting model gets
        sdwui's txt2img conditioning, which inpainting_mask_weight does not enter (it is taken for a uniform call).
        `token_merging_ratio`, `schedule` and `loras` as for img2img."""
        b = tokens.shape[0]
        self._use_loras(loras)
        h, w = height // 8, width // 8
        cond, uncond, sched = self._pass_conds(tokens, neg_tokens, width, height, multipliers, neg_multipliers, schedule)
        lat = self._sample_txt(cond, uncond, seed, b, h, w, steps, cfg_scale, sampler, scheduler, controls, tiling,
                               self._txt2img_cond(b, h, w, tiling) if self.inpainting else None, token_merging_ratio,
                               sched)
        return self.decode(lat, h, w, tiling, token_merging_ratio)
