"""sdwui prompt editing `[from:to:when]` and alternation `[a|b]`, restated from sdwui >= 1.9 (parity unpinned, DESIGN §2).

  * prompt_parser.get_learned_conditioning_prompt_schedules: the lark grammar below (`schedule_parser`), its
    CollectSteps visitor (the step boundaries) and AtStep transformer (the text at a boundary).  This restatement is the
    arbiter of b200sd.prompts.prompt_schedule; it needs lark, which only the tests import.
  * processing.setup_conds / calculate_hr_conds: the schedules are built over SamplerData.total_steps(steps) (steps x 2
    for the samplers sdwui flags second_order), the hires pass's with base_steps = the first pass's steps.
  * prompt_parser.reconstruct_cond_batch: CFGDenoiser.step counts model evaluations from 0; evaluation `step` takes the
    first entry with step <= end_at_step, entry 0 when there is none.

`Scheduled` runs the unchanged sd / v / ControlNet / SDXL oracle samplers under such a schedule: it is the unet(x, t, c)
they call once per model evaluation, counts the calls and evaluates call k on its own entries, as sdwui's CFGDenoiser
does (one call when the two contexts have one length, cond and uncond apart otherwise).
"""
from typing import List, Optional

import torch

SCHEDULE_GRAMMAR = r"""
!start: (prompt | /[][():]/+)*
prompt: (emphasized | scheduled | alternate | plain | WHITESPACE)*
!emphasized: "(" prompt ")"
        | "(" prompt ":" prompt ")"
        | "[" prompt "]"
scheduled: "[" [prompt ":"] prompt ":" [WHITESPACE] NUMBER [WHITESPACE] "]"
alternate: "[" prompt ("|" [prompt])+ "]"
WHITESPACE: /\s+/
plain: /([^\\\[\]():|]|\\.)+/
%import common.SIGNED_NUMBER -> NUMBER
"""

_PARSER = None

# sd_samplers_kdiffusion.samplers_k_diffusion entries with second_order=True (Karras variants share the flag)
SECOND_ORDER = ("Heun", "DPM2", "DPM2 a", "DPM++ 2S a", "DPM++ SDE", "DPM2 Karras", "DPM2 a Karras",
                "DPM++ 2S a Karras", "DPM++ SDE Karras")


def total_steps(sampler: str, steps: int) -> int:
    """SamplerData.total_steps"""
    return steps * 2 if sampler in SECOND_ORDER else steps


def get_learned_conditioning_prompt_schedules(prompts: List[str], base_steps: int, hires_steps: Optional[int] = None,
                                              use_old_scheduling: bool = False):
    import lark
    global _PARSER
    if _PARSER is None:
        _PARSER = lark.Lark(SCHEDULE_GRAMMAR)

    if hires_steps is None or use_old_scheduling:
        int_offset, flt_offset, steps = 0, 0, base_steps
    else:
        int_offset, flt_offset, steps = base_steps, 1.0, hires_steps

    def collect_steps(steps, tree):
        res = [steps]

        class CollectSteps(lark.Visitor):
            def scheduled(self, tree):
                s = tree.children[-2]
                v = float(s)
                if use_old_scheduling:
                    v = v * steps if v < 1 else v
                else:
                    if "." in s:
                        v = (v - flt_offset) * steps
                    else:
                        v = (v - int_offset)
                tree.children[-2] = min(steps, int(v))
                if tree.children[-2] >= 1:
                    res.append(tree.children[-2])

            def alternate(self, tree):
                res.extend(range(1, steps + 1))

        CollectSteps().visit(tree)
        return sorted(set(res))

    def at_step(step, tree):
        class AtStep(lark.Transformer):
            def scheduled(self, args):
                before, after, _, when, _ = args
                yield before or () if step <= when else after

            def alternate(self, args):
                args = ["" if not arg else arg for arg in args]
                yield args[(step - 1) % len(args)]

            def start(self, args):
                def flatten(x):
                    if isinstance(x, str):
                        yield x
                    else:
                        for gen in x:
                            yield from flatten(gen)
                return "".join(flatten(args))

            def plain(self, args):
                yield args[0].value

            def __default__(self, data, children, meta):
                for child in children:
                    yield child
        return AtStep().transform(tree)

    def get_schedule(prompt):
        try:
            tree = _PARSER.parse(prompt)
        except lark.exceptions.LarkError:
            return [[steps, prompt]]
        return [[t, at_step(t, tree)] for t in collect_steps(steps, tree)]

    promptdict = {prompt: get_schedule(prompt) for prompt in set(prompts)}
    return [promptdict[prompt] for prompt in prompts]


def reconstruct_index(schedule, step: int) -> int:
    """prompt_parser.reconstruct_cond_batch's choice for one prompt: [(end_at_step, text)], evaluation `step`"""
    for i, (end, _) in enumerate(schedule):
        if step <= end:
            return i
    return 0


class Scheduled:
    """unet(x, t, c) for the oracle samplers under prompt schedules.  forward(x, t, c, y) is one UNet call on contexts of
    one length (y: SDXL vector conditioning, else None); cond [Ec, Lc, C] / uncond [Eu, Lu, C] are the encoded entries,
    cond_ends / uncond_ends their end_at_step values, y_cond / y_uncond their SDXL vectors.  The context a sampler hands
    in is ignored.  `inner`: a ControlNet oracle unet whose `units` / `active` the ControlNet sampler reads and sets.
    `entries` records the (cond, uncond) entry of every evaluation."""

    def __init__(self, forward, cond, uncond, cond_ends, uncond_ends, y_cond=None, y_uncond=None, inner=None):
        self.forward, self.cond, self.uncond = forward, cond, uncond
        self.cond_ends = [(e, None) for e in cond_ends]
        self.uncond_ends = [(e, None) for e in uncond_ends]
        self.y_cond, self.y_uncond, self.inner = y_cond, y_uncond, inner
        self.entries = []

    @property
    def units(self):
        return self.inner.units

    @property
    def active(self):
        return self.inner.active

    @active.setter
    def active(self, value):
        self.inner.active = value

    def placeholders(self, b: int):
        """(cond, uncond) [b, L, C] of one length for the samplers' torch.cat; never evaluated"""
        n = max(self.cond.shape[1], self.uncond.shape[1])
        z = self.cond.new_zeros((b, n, self.cond.shape[2]))
        return z, z.clone()

    def __call__(self, x, t, c):
        k = len(self.entries)
        ic, iu = reconstruct_index(self.cond_ends, k), reconstruct_index(self.uncond_ends, k)
        self.entries.append((ic, iu))
        b = x.shape[0] // 2
        cc = self.cond[ic:ic + 1].expand(b, -1, -1)
        cu = self.uncond[iu:iu + 1].expand(b, -1, -1)
        yc = yu = None
        if self.y_cond is not None:
            yc, yu = self.y_cond[ic:ic + 1].expand(b, -1), self.y_uncond[iu:iu + 1].expand(b, -1)
        if cc.shape[1] == cu.shape[1]:
            y = None if yc is None else torch.cat([yc, yu])
            return self.forward(x, t, torch.cat([cc, cu]), y)
        return torch.cat([self.forward(x[:b], t[:b], cc, yc), self.forward(x[b:], t[b:], cu, yu)])
