"""fp32 oracle of sdwui's tiling option, built from the unchanged sd_oracle, v_oracle and controlnet_oracle functions.

sdwui's `model_hijack.apply_circular(True)` sets padding_mode = 'circular' on every torch.nn.Conv2d of the loaded sd
model (UNet, VAE decoder and encoder).  Here the oracle functions run under a conv shim: for the duration of the call the
`F` those modules use is replaced by one whose conv2d, for padding > 0, pads circularly with F.pad and convolves with
padding 0 — what nn.Conv2d(padding_mode='circular') does.  Convs with padding 0 (1x1 convs, and the VAE encoder's
downsample after its constant F.pad) are untouched.  sd-webui-controlnet's model is not part of the sd model: the
ControlNet forward (hint block, encoder copy, zero convs) runs outside the shim, zero padded.
"""
import contextlib

import torch.nn.functional as F

from oracle import controlnet_oracle as CN
from oracle import sd_oracle as O

_MODULES = (O, CN)   # the modules whose `F` carries the model's convs (sd_oracle; CN.unet_forward's out.2)


class _CircularF:
    """torch.nn.functional with conv2d padding circularly"""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def conv2d(x, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
        if padding:
            p = padding
            x = F.pad(x, (p, p, p, p), mode="circular")
        return F.conv2d(x, weight, bias, stride, 0, dilation, groups)


CIRCULAR_F = _CircularF()


@contextlib.contextmanager
def _functional(f):
    saved = [m.F for m in _MODULES]
    for m in _MODULES:
        m.F = f
    try:
        yield
    finally:
        for m, s in zip(_MODULES, saved):
            m.F = s


def _zero_padded(fn):
    def call(*a, **k):
        with _functional(F):
            return fn(*a, **k)
    return call


@contextlib.contextmanager
def circular(on: bool = True):
    """inside: the oracle's sd-model convs pad circularly (on) or as they always do (off); the ControlNet model never"""
    if not on:
        yield
        return
    forward = CN.controlnet_forward
    CN.controlnet_forward = _zero_padded(forward)
    try:
        with _functional(CIRCULAR_F):
            yield
    finally:
        CN.controlnet_forward = forward


def run(fn, *a, tiling: bool = True, **k):
    """fn(*a, **k) — any sd_oracle / v_oracle / controlnet_oracle / upscale_oracle entry point — with sdwui's tiling
    setting `tiling`"""
    with circular(tiling):
        return fn(*a, **k)
