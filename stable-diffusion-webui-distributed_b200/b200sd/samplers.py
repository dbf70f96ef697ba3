"""Sampler programs: every sampler of the reference's ETA table (scripts/spartan/worker.py:75-94) as a list of STAGES.

A stage is one model evaluation plus the latent arithmetic that follows it.  For an eps-prediction model behind
k-diffusion's CompVisDenoiser, `denoised = x - sigma * eps` and `to_d(x, sigma, denoised) = eps`, so every update of
every sampler below is a LINEAR COMBINATION of a handful of fp32 latent tensors — x, the CFG-combined eps `e` of this
evaluation, an intermediate point `u`, up to three history tensors `h1..h3`, a noise draw `n` — with coefficients that
depend on the step only.  The executor therefore needs two kernels beyond the UNet: `b200sd_cfg_eps` and
`b200sd_latent_lincomb` (coefficient row selected on the device by the evaluation counter), and a stage's STRUCTURE (which
tensors are combined into which) is a CUDA graph that replays for every evaluation with that structure.

A v-prediction model (SD 2.x 768-v) changes one thing: the CFG-combined UNet output in `e` is v, and one more linear
combination per evaluation, e = kx * ev + kv * e with the coefficients of the evaluated noise level (V_COL), turns it into
the eps the stages below expect (k-diffusion CompVisVDenoiser / sdwui CompVisTimestepsVDenoiser, see Stage.row).

This module is host arithmetic only (float64): it turns (sampler, sigma schedule | DDIM timesteps) into
    stages[i] = (structure, timestep for the time embedding, coefficient row)
and says how many noise draws per image it needs and how they are mixed into the rows of the noise stack.

Upstream (not in /root/reference): k-diffusion sampling.py sample_heun / sample_dpm_2 / sample_dpm_2_ancestral /
sample_dpmpp_2s_ancestral / sample_dpmpp_sde / sample_lms / DPMSolver.dpm_solver_fast / dpm_solver_adaptive; sdwui
sd_samplers_timesteps_impl.plms.  oracle/sd_oracle.py restates the same algorithms step by step (not as coefficient
algebra) and tests/ compare the two.
"""
import math
from dataclasses import dataclass, field
from typing import Callable, List, Sequence, Tuple

COEF_LD = 32           # floats per coefficient row
IDX_COL = COEF_LD - 1  # the row's last float = which tensor of the noise stack this stage reads
MASK_COL = 24          # 4 floats {1, -sigma, 1/sigma, -1/sigma}: denoised = ev - sigma e and back (masked k-diffusion sampling)
V_COL = 28             # 2 floats {kx, kv}: v-prediction models, eps = kx * ev + kv * v (Stage.row)

# one linear combination: (dst, (src, ...), pack) — pack: the result, times one more coefficient, becomes the UNet input
LC = Tuple[str, Tuple[str, ...], bool]


@dataclass
class Stage:
    lcs: Tuple[LC, ...]          # structure (the graph key)
    t: float                     # timestep fed to the time embedding (k-diffusion: sigma_to_t(sigma))
    coefs: List[float]           # concatenated coefficients of the lcs (pack scale after each packed one)
    ev: str = "x"                # which tensor the model was evaluated on (inpainting masks act on it / its denoised)
    sigma: float = 0.0           # its noise level (k-diffusion samplers; 0 for the timestep samplers)
    noise: int = -1              # row of the noise stack read by an 'n' source
    alpha: float = 0.0           # alphas_cumprod at the evaluated timestep (timestep samplers; 0 for k-diffusion)

    def row(self) -> List[float]:
        assert len(self.coefs) <= MASK_COL, "coefficient row overflow"
        r = list(self.coefs) + [0.0] * (COEF_LD - len(self.coefs))
        if self.sigma > 0:
            r[MASK_COL:MASK_COL + 4] = [1.0, -self.sigma, 1.0 / self.sigma, -1.0 / self.sigma]
            # v -> eps for sigma-space ev: ev * c_in is the UNet input and alphas_cumprod = 1 / (sigma^2 + 1)
            r[V_COL:V_COL + 2] = [self.sigma / (self.sigma ** 2 + 1.0), 1.0 / math.sqrt(self.sigma ** 2 + 1.0)]
        elif self.alpha > 0:
            # v -> eps for latent-space ev (the UNet input itself): eps = sqrt(1 - a) ev + sqrt(a) v
            r[V_COL:V_COL + 2] = [math.sqrt(1.0 - self.alpha), math.sqrt(self.alpha)]
        r[IDX_COL] = float(max(self.noise, 0))
        return r


@dataclass
class SamplerPlan:
    stages: List[Stage]
    x_scale0: float = 1.0        # start latents = x_T * x_scale0 (k-diffusion: sigma_max; skipped for img2img starts)
    in0: float = 1.0             # scale of the first UNet input (c_in of the first sigma)
    draws: int = 0               # N(0, 1) draws per image AFTER the start noise
    mix: List[List[Tuple[int, float]]] = field(default_factory=list)   # noise-stack row r = sum w * draw[i]
    timestep_sampler: bool = False   # DDIM / PLMS: inpainting masks blend the evaluated tensor BEFORE the model call


def c_in(sigma: float) -> float:
    return 1.0 / math.sqrt(sigma * sigma + 1.0)


def ancestral_step(s: float, sn: float, eta: float = 1.0) -> Tuple[float, float]:
    """k-diffusion get_ancestral_step -> (sigma_down, sigma_up)"""
    if not eta:
        return sn, 0.0
    up = min(sn, eta * (sn ** 2 * (s ** 2 - sn ** 2) / s ** 2) ** 0.5)
    return (sn ** 2 - up ** 2) ** 0.5, up


X_E = ("x", "e")
EULER: Tuple[LC, ...] = (("x", X_E, True),)                       # x = a x + b e
MID: Tuple[LC, ...] = (("u", X_E, True),)                         # u = a x + b e
MID_KEEP: Tuple[LC, ...] = (("u", X_E, True), ("h1", ("e",), False))
FROM_H1: Tuple[LC, ...] = (("x", ("x", "h1", "e"), True),)        # x = a x + b h1 + c e
ANC: Tuple[LC, ...] = (("x", ("x", "e", "n"), True),)
S2_B: Tuple[LC, ...] = (("x", ("x", "u", "e", "n"), True),)
SDE_A: Tuple[LC, ...] = (("u", ("x", "e", "n"), True), ("h1", ("e",), False))
SDE_B: Tuple[LC, ...] = (("x", ("x", "h1", "u", "e", "n"), True),)
MULTISTEP: Tuple[LC, ...] = (("x", ("x", "e", "h1", "h2", "h3"), True), ("h3", ("h2",), False), ("h2", ("h1",), False),
                             ("h1", ("e",), False))
F3_B: Tuple[LC, ...] = (("u", ("x", "h1", "e"), True),)            # u = a x + b h1 + c e


def _euler_to(s: float, sn: float, t: float, ev: str = "x") -> Stage:
    """x += d * (sn - s); the next evaluation (if any) is at sn"""
    return Stage(EULER, t, [1.0, sn - s, c_in(sn)], ev, s)


# ------------------------------------------------------------------------------------------------ k-diffusion samplers
def heun(sig: Sequence[float], t_of: Callable[[float], float]) -> SamplerPlan:
    """sample_heun, s_churn = 0: d = to_d(x); x2 = x + d dt; d2 = to_d(x2, sigma_next); x += (d + d2) / 2 dt; the step to
    sigma 0 is an Euler step."""
    st = []
    for i in range(len(sig) - 1):
        s, sn = sig[i], sig[i + 1]
        if sn == 0:
            st.append(_euler_to(s, sn, t_of(s)))
            continue
        dt = sn - s
        st.append(Stage(MID_KEEP, t_of(s), [1.0, dt, c_in(sn), 1.0], "x", s))
        st.append(Stage(FROM_H1, t_of(sn), [1.0, dt / 2, dt / 2, c_in(sn)], "u", sn))
    return SamplerPlan(st, sig[0], c_in(sig[0]))


def dpm_2(sig, t_of) -> SamplerPlan:
    """sample_dpm_2, s_churn = 0: midpoint in log sigma"""
    st = []
    for i in range(len(sig) - 1):
        s, sn = sig[i], sig[i + 1]
        if sn == 0:
            st.append(_euler_to(s, sn, t_of(s)))
            continue
        mid = math.exp(0.5 * (math.log(s) + math.log(sn)))
        st.append(Stage(MID, t_of(s), [1.0, mid - s, c_in(mid)], "x", s))
        st.append(Stage(EULER, t_of(mid), [1.0, sn - s, c_in(sn)], "u", mid))
    return SamplerPlan(st, sig[0], c_in(sig[0]))


def dpm_2_ancestral(sig, t_of) -> SamplerPlan:
    """sample_dpm_2_ancestral, eta = 1: DPM2 to sigma_down, then + noise * sigma_up (not on the Euler step to 0)"""
    st, draws = [], 0
    for i in range(len(sig) - 1):
        s, sn = sig[i], sig[i + 1]
        down, up = ancestral_step(s, sn)
        if down == 0:
            st.append(_euler_to(s, 0.0, t_of(s)))
            continue
        mid = math.exp(0.5 * (math.log(s) + math.log(down)))
        st.append(Stage(MID, t_of(s), [1.0, mid - s, c_in(mid)], "x", s))
        st.append(Stage(ANC, t_of(mid), [1.0, down - s, up, c_in(sn)], "u", mid, noise=draws))
        draws += 1
    return SamplerPlan(st, sig[0], c_in(sig[0]), draws, [[(k, 1.0)] for k in range(draws)])


def dpmpp_2s_ancestral(sig, t_of) -> SamplerPlan:
    """sample_dpmpp_2s_ancestral, eta = 1, r = 1/2"""
    st, draws = [], 0
    for i in range(len(sig) - 1):
        s, sn = sig[i], sig[i + 1]
        down, up = ancestral_step(s, sn)
        if down == 0:
            st.append(_euler_to(s, 0.0, t_of(s)))
            continue
        t, t_next = -math.log(s), -math.log(down)
        h = t_next - t
        sm = math.exp(-(t + 0.5 * h))                 # sigma_fn(s)
        a1 = -math.expm1(-h * 0.5)                    # x_2 = (sm / s) x + a1 * denoised,  denoised = x - s e
        st.append(Stage(MID, t_of(s), [sm / s + a1, -a1 * s, c_in(sm)], "x", s))
        a2 = -math.expm1(-h)                          # x = (down / s) x + a2 * denoised_2,  denoised_2 = u - sm e
        st.append(Stage(S2_B, t_of(sm), [down / s, a2, -a2 * sm, up if sn > 0 else 0.0, c_in(sn)], "u", sm, noise=draws))
        draws += 1
    return SamplerPlan(st, sig[0], c_in(sig[0]), draws, [[(k, 1.0)] for k in range(draws)])


def dpmpp_sde(sig, t_of) -> SamplerPlan:
    """sample_dpmpp_sde, eta = 1, s_noise = 1, r = 1/2.  Upstream draws its noise from a torchsde BrownianTree
    (BrownianTreeNoiseSampler: (W(t1) - W(t0)) / sqrt|t1 - t0| on the sigma axis; torchsde is not installable offline);
    the two intervals of a step overlap — [sigma_s, sigma] inside [sigma_next, sigma] — so the two noises are correlated.
    Restated with two independent N(0,1) draws per step and image, z1 for [sigma_s, sigma] and z2 for [sigma_next, sigma_s]:
    n1 = z1,  n2 = (sqrt(sigma - sigma_s) z1 + sqrt(sigma_s - sigma_next) z2) / sqrt(sigma - sigma_next) — the same joint
    distribution, not the same numbers."""
    st, draws, mix = [], 0, []
    r, fac = 0.5, 1.0
    for i in range(len(sig) - 1):
        s, sn = sig[i], sig[i + 1]
        if sn == 0:
            st.append(_euler_to(s, 0.0, t_of(s)))
            continue
        t, t_next = -math.log(s), -math.log(sn)
        h = t_next - t
        ss = math.exp(-(t + h * r))                   # sigma_fn(s)
        sd, su = ancestral_step(s, ss)
        a = -math.expm1(t - (-math.log(sd)))          # x_2 = (sd / s) x + a denoised + n1 su
        st.append(Stage(SDE_A, t_of(s), [sd / s + a, -a * s, su, c_in(ss), 1.0], "x", s, noise=len(mix)))
        mix.append([(draws, 1.0)])
        sd2, su2 = ancestral_step(s, sn)
        b = -math.expm1(t - (-math.log(sd2)))         # x = (sd2 / s) x + b ((1 - fac) den + fac den2) + n2 su2
        st.append(Stage(SDE_B, t_of(ss), [sd2 / s + b * (1 - fac), -b * (1 - fac) * s, b * fac, -b * fac * ss, su2, c_in(sn)],
                        "u", ss, noise=len(mix)))
        w1, w2 = math.sqrt(s - ss), math.sqrt(ss - sn)
        mix.append([(draws, w1 / math.sqrt(s - sn)), (draws + 1, w2 / math.sqrt(s - sn))])
        draws += 2
    return SamplerPlan(st, sig[0], c_in(sig[0]), draws, mix)


def euler(sig, t_of) -> SamplerPlan:
    """sample_euler (s_churn 0) as stages — the fused kernel's twin, used when a mask rides along"""
    return SamplerPlan([_euler_to(sig[i], sig[i + 1], t_of(sig[i])) for i in range(len(sig) - 1)], sig[0], c_in(sig[0]))


def euler_ancestral(sig, t_of) -> SamplerPlan:
    """sample_euler_ancestral as stages (one draw per step, unused on the step to 0)"""
    st = []
    for i in range(len(sig) - 1):
        s, sn = sig[i], sig[i + 1]
        down, up = ancestral_step(s, sn)
        st.append(Stage(ANC, t_of(s), [1.0, down - s, up, c_in(sn)], "x", s, noise=i))
    n = len(st)
    return SamplerPlan(st, sig[0], c_in(sig[0]), n, [[(k, 1.0)] for k in range(n)])


DPMPP_2M: Tuple[LC, ...] = (("h2", X_E, False), ("x", ("x", "h2", "h1"), True), ("h1", ("h2",), False))


def dpmpp_2m(sig, t_of) -> SamplerPlan:
    """sample_dpmpp_2m as stages: h2 = denoised = x - sigma e; x = a x + (1 - a)(c1 h2 - c2 h1); h1 = h2"""
    st = []
    for i in range(len(sig) - 1):
        s, sn = sig[i], sig[i + 1]
        c1, c2 = 1.0, 0.0
        if i > 0 and sn > 0:
            r = math.log(sig[i - 1] / s) / math.log(s / sn)
            c1, c2 = 1.0 + 1.0 / (2.0 * r), 1.0 / (2.0 * r)
        a = sn / s
        st.append(Stage(DPMPP_2M, t_of(s), [1.0, -s, a, (1 - a) * c1, -(1 - a) * c2, c_in(sn), 1.0], "x", s))
    return SamplerPlan(st, sig[0], c_in(sig[0]))


def lms_coeff(order: int, t: Sequence[float], i: int, j: int) -> float:
    """k-diffusion linear_multistep_coeff: integral of the j-th Lagrange basis over [t_i, t_{i+1}] (scipy quad, epsrel 1e-4)"""
    from scipy import integrate
    if order - 1 > i:
        raise ValueError(f"Order {order} too high for step {i}")

    def fn(tau):
        prod = 1.0
        for k in range(order):
            if j == k:
                continue
            prod *= (tau - t[i - k]) / (t[i - j] - t[i - k])
        return prod

    return integrate.quad(fn, t[i], t[i + 1], epsrel=1e-4)[0]


def lms(sig, t_of, order: int = 4) -> SamplerPlan:
    """sample_lms: x += sum_j coeff_j * d_{i-j} over the last min(i + 1, 4) derivatives"""
    st = []
    for i in range(len(sig) - 1):
        cur = min(i + 1, order)
        c = [lms_coeff(cur, sig, i, j) for j in range(cur)] + [0.0] * (order - cur)
        st.append(Stage(MULTISTEP, t_of(sig[i]), [1.0, *c, c_in(sig[i + 1]), 1.0, 1.0, 1.0], "x", sig[i]))
    return SamplerPlan(st, sig[0], c_in(sig[0]))


def dpm_fast(sigma_min: float, sigma_max: float, n: int, t_of) -> SamplerPlan:
    """sample_dpm_fast -> DPMSolver.dpm_solver_fast(x, t(sigma_max), t(sigma_min), nfe = n), eta = 0: DPM-Solver-3 steps
    on a uniform grid in t = -log sigma, the last ones of order 2 / 1 so that exactly n evaluations are spent.  It ends at
    sigma_min (no final step to 0)."""
    t_start, t_end = -math.log(sigma_max), -math.log(sigma_min)
    m = n // 3 + 1
    ts = [t_start + (t_end - t_start) * k / m for k in range(m + 1)]
    orders = [3] * (m - 2) + [2, 1] if n % 3 == 0 else [3] * (m - 1) + [n % 3]
    st = []
    for i, order in enumerate(orders):
        t, tn = ts[i], ts[i + 1]
        st.extend(_dpm_solver_step(order, t, tn, t_of, 1 / 3 if order == 3 else 1 / 2))
    return SamplerPlan(st, sigma_max, c_in(sigma_max))


def _dpm_solver_step(order: int, t: float, tn: float, t_of, r1: float, r2: float = 2 / 3, dst: str = "x") -> List[Stage]:
    """DPMSolver.dpm_solver_{1,2,3}_step with eps = to_d = e.  The last stage writes `dst`."""
    sg = lambda tt: math.exp(-tt)  # noqa: E731
    h = tn - t
    if order == 1:
        lcs = EULER if dst == "x" else ((dst, X_E, True),)
        return [Stage(lcs, t_of(sg(t)), [1.0, -sg(tn) * math.expm1(h), c_in(sg(tn))], "x", sg(t))]
    last = FROM_H1 if dst == "x" else ((dst, ("x", "h1", "e"), True),)
    if order == 2:
        s1 = t + r1 * h
        k = sg(tn) / (2 * r1) * math.expm1(h)
        return [Stage(MID_KEEP, t_of(sg(t)), [1.0, -sg(s1) * math.expm1(r1 * h), c_in(sg(s1)), 1.0], "x", sg(t)),
                Stage(last, t_of(sg(s1)), [1.0, -sg(tn) * math.expm1(h) + k, -k, c_in(sg(tn))], "u", sg(s1))]
    s1, s2 = t + r1 * h, t + r2 * h
    k2 = sg(s2) * (r2 / r1) * (math.expm1(r2 * h) / (r2 * h) - 1)
    k3 = sg(tn) / r2 * (math.expm1(h) / h - 1)
    return [Stage(MID_KEEP, t_of(sg(t)), [1.0, -sg(s1) * math.expm1(r1 * h), c_in(sg(s1)), 1.0], "x", sg(t)),
            Stage(F3_B, t_of(sg(s1)), [1.0, -sg(s2) * math.expm1(r2 * h) + k2, -k2, c_in(sg(s2))], "u", sg(s1)),
            Stage(last, t_of(sg(s2)), [1.0, -sg(tn) * math.expm1(h) + k3, -k3, c_in(sg(tn))], "u", sg(s2))]


# ------------------------------------------------------------------------------------------------ timestep samplers
def plms(ts: Sequence[int], ac: Sequence[float]) -> SamplerPlan:
    """sdwui sd_samplers_timesteps_impl.plms over timesteps `ts` (ascending; alphas_prev pads with alphas_cumprod[0]):
    index runs len(ts)-1 .. 1; pseudo linear multistep on eps with a 2-evaluation warm-up step."""
    a = [ac[t] for t in ts]
    a_prev = [ac[0]] + [ac[t] for t in ts[:-1]]
    st = []
    n_old = 0
    for index in range(len(ts) - 1, 0, -1):
        at, ap = a[index], a_prev[index]
        cx = math.sqrt(ap) / math.sqrt(at)                                    # x_prev = cx * x + ce * e_t
        ce = math.sqrt(1 - ap) - math.sqrt(ap) * math.sqrt(1 - at) / math.sqrt(at)
        t_here, t_next = float(ts[index]), float(ts[max(index - 1, 0)])
        if n_old == 0:
            st.append(Stage(MID_KEEP, t_here, [cx, ce, 1.0, 1.0], "x", 0.0, alpha=at))
            st.append(Stage(FROM_H1, t_next, [cx, ce / 2, ce / 2, 1.0], "u", 0.0, alpha=ap))   # ap = ac[t_next]
            n_old = 1
            continue
        w = {1: [3 / 2, -1 / 2, 0, 0], 2: [23 / 12, -16 / 12, 5 / 12, 0], 3: [55 / 24, -59 / 24, 37 / 24, -9 / 24]}[min(n_old, 3)]
        st.append(Stage(MULTISTEP, t_here, [cx, *[ce * v for v in w], 1.0, 1.0, 1.0, 1.0], "x", 0.0, alpha=at))
        n_old += 1
    return SamplerPlan(st, 1.0, 1.0, timestep_sampler=True)


# sampler names of the sdwui API handled by the generic stage machine -> (builder key, default sigma schedule)
GENERIC = {
    "Heun": ("heun", "uniform"), "DPM2": ("dpm_2", "uniform"), "DPM2 a": ("dpm_2_ancestral", "uniform"),
    "DPM++ 2S a": ("dpmpp_2s_ancestral", "uniform"), "DPM++ SDE": ("dpmpp_sde", "uniform"), "LMS": ("lms", "uniform"),
    "DPM fast": ("dpm_fast", "uniform"), "DPM adaptive": ("dpm_adaptive", "uniform"), "PLMS": ("plms", None),
    "LMS Karras": ("lms", "karras"), "DPM2 Karras": ("dpm_2", "karras"), "DPM2 a Karras": ("dpm_2_ancestral", "karras"),
    "DPM++ 2S a Karras": ("dpmpp_2s_ancestral", "karras"), "DPM++ SDE Karras": ("dpmpp_sde", "karras"),
}
BUILDERS = {"euler": euler, "euler_a": euler_ancestral, "dpmpp_2m": dpmpp_2m, "heun": heun, "dpm_2": dpm_2, "dpm_2_ancestral": dpm_2_ancestral, "dpmpp_2s_ancestral": dpmpp_2s_ancestral,
            "dpmpp_sde": dpmpp_sde, "lms": lms}


# ------------------------------------------------------------------------------------------------ DPM adaptive
class PIDStepSizeController:
    """k-diffusion PIDStepSizeController (h, pcoeff, icoeff, dcoeff, order, accept_safety, eps = 1e-8)"""

    def __init__(self, h, pcoeff, icoeff, dcoeff, order=1, accept_safety=0.81, eps=1e-8):
        self.h = h
        self.b1 = (pcoeff + icoeff + dcoeff) / order
        self.b2 = -(pcoeff + 2 * dcoeff) / order
        self.b3 = dcoeff / order
        self.accept_safety = accept_safety
        self.eps = eps
        self.errs = []

    @staticmethod
    def limiter(x):
        return 1 + math.atan(x - 1)

    def propose_step(self, error: float) -> bool:
        inv_error = 1 / (float(error) + self.eps)
        if not self.errs:
            self.errs = [inv_error, inv_error, inv_error]
        self.errs[0] = inv_error
        factor = self.errs[0] ** self.b1 * self.errs[1] ** self.b2 * self.errs[2] ** self.b3
        factor = self.limiter(factor)
        accept = factor >= self.accept_safety
        if accept:
            self.errs[2] = self.errs[1]
            self.errs[1] = self.errs[0]
        self.h *= factor
        return accept


def dpm_adaptive_attempt(s: float, t: float, t_of) -> List[Stage]:
    """one attempted step of DPMSolver.dpm_solver_adaptive (order 3, eta 0) from s to t in t = -log sigma: eps at (x, s);
    x_low = dpm_solver_2_step(r1 = 1/3) -> 'h3'; x_high = dpm_solver_3_step -> 'u' (shares eps and eps_r1 with x_low, as
    upstream's eps_cache does).  3 evaluations; the caller accepts (x_prev = x_low, x = x_high) or rejects."""
    sg = lambda tt: math.exp(-tt)  # noqa: E731
    h = t - s
    r1, r2 = 1 / 3, 2 / 3
    s1, s2 = s + r1 * h, s + r2 * h
    k_low = sg(t) / (2 * r1) * math.expm1(h)
    k2 = sg(s2) * (r2 / r1) * (math.expm1(r2 * h) / (r2 * h) - 1)
    k3 = sg(t) / r2 * (math.expm1(h) / h - 1)
    a = (("u", X_E, True), ("h1", ("e",), False))
    b = (("h3", ("x", "h1", "e"), False), ("u", ("x", "h1", "e"), True))       # x_low, then u2
    c = (("u", ("x", "h1", "e"), True),)                                         # x_high
    return [Stage(a, t_of(sg(s)), [1.0, -sg(s1) * math.expm1(r1 * h), c_in(sg(s1)), 1.0], "x", sg(s)),
            Stage(b, t_of(sg(s1)), [1.0, -sg(t) * math.expm1(h) + k_low, -k_low,
                                    1.0, -sg(s2) * math.expm1(r2 * h) + k2, -k2, c_in(sg(s2))], "u", sg(s1)),
            Stage(c, t_of(sg(s2)), [1.0, -sg(t) * math.expm1(h) + k3, -k3, c_in(sg(t))], "u", sg(s2))]
