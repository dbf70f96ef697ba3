"""Kernel parity against fp64 at the shapes SDXL (bf16) and SD1.5 (fp16) run: the GEMM / implicit-GEMM conv epilogues,
the VAE's row softmax, the eps-prediction fused sampler steps, GroupNorm / LayerNorm and two packing kernels.

The reference is fp64 arithmetic on exactly the stored inputs (a bias stays the fp32 values the kernel reads), so neither
the rounding of the inputs nor the TF32 settings enter it.  An output element passes when it is the correctly rounded
value, in the output dtype, of some real number within delta of the exact result y:

    RN(y - delta) <= got <= RN(y + delta)

For the GEMM / conv, delta = C_ACC * sqrt(K) * 2^-24 * S with S = sum_k |a_k w_k| + |bias| + |residual| (fp32
accumulation in any order), the exact result follows the epilogue order of gemm_conv_tc_body (bias, GEGLU, residual,
SiLU), an activation scales delta by its Lipschitz constant and adds its documented approximation error.  That is tight
enough to catch one extra rounding to the output dtype anywhere in the epilogue, a wrong bias row or a gate one column
group off, and loose enough for any fp32 accumulation order.  Every case records its worst |got - y| / (ulp/2 + delta)
and the smallest C_ACC it would have needed in kernel_fp64.jsonl under kutil.OUT_DIR.
"""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kutil import OUT_DIR

pytestmark = pytest.mark.gpu

DTS = [torch.float16, torch.bfloat16]
U = 2.0 ** -24            # unit roundoff of fp32
C_ACC = 1.0               # accumulation constant of the GEMM / conv bound (module docstring)
GELU_ABS = 9e-7           # gelu_erf's documented absolute error (gemm_conv_tc.cu)
GELU_LIP = 1.13           # sup |gelu'|
SILU_LIP = 1.1            # sup |silu'|
N_RANDOM_ROWS = 4096


@pytest.fixture(scope="module")
def ops():
    from b200sd import ops as _ops
    return _ops


def _gen(seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return g


def _rand(shape, g, scale=1.0, dt=torch.float16, offset=0.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale + offset).to(dt)


def _dname(dt):
    return "f16" if dt == torch.float16 else "bf16"


# ----------------------------------------------------------------------------------------------- rounding-window check
def _half_ulp(v, dt):
    """half the spacing of dt at |v| (fp64 tensor), subnormals included"""
    mant, emin = (10, -14) if dt == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** emin)))
    return torch.exp2(e - mant - 1)


def _rn(v, dt, up):
    """RN_dt(v) of an fp64 tensor, never on the wrong side: torch casts fp64 -> fp32 -> dt, so the fp32 step is made
    directed (towards the outside of the window) and the second rounding is then monotone"""
    f = v.float()
    fd = f.double()
    inf = torch.full_like(f, math.inf if up else -math.inf)
    f = torch.where((fd < v) if up else (fd > v), torch.nextafter(f, inf), f)
    return f.to(dt)


def _record(rep):
    try:
        os.makedirs(OUT_DIR, exist_ok=True)
        with open(os.path.join(OUT_DIR, "kernel_fp64.jsonl"), "a") as f:
            f.write(json.dumps(rep) + "\n")
    except OSError:
        pass


def _window_report(name, got, y, delta, dt, rows=None, delta_unit=None, extra=None):
    """got [R, N] (dt), y / delta [R, N] fp64.  rows: global output row of each of the R rows (for localisation);
    delta_unit: the part of delta that C_ACC multiplies (records the smallest constant that would have passed)."""
    g = got.double()
    lo = _rn(y - delta, dt, False).double()
    hi = _rn(y + delta, dt, True).double()
    finite = torch.isfinite(g)
    bad = (g < lo) | (g > hi) | ~finite
    hu = _half_ulp(y.abs() + delta, dt)
    err = (g - y).abs()
    ratio = torch.where(finite, err / (hu + delta), torch.full_like(err, math.inf))
    rep = {"name": name, "dtype": _dname(dt), "shape": list(got.shape), "n_bad": int(bad.sum()),
           "worst_ratio": float(ratio.max()) if ratio.numel() else 0.0, "has_nonfinite": bool((~finite).any())}
    if delta_unit is not None:
        rest = delta - C_ACC * delta_unit
        need = ((err - hu - rest).clamp_min(0) / delta_unit.clamp_min(1e-300)).max()
        rep["c_needed"] = float(need) if ratio.numel() else 0.0
    if extra:
        rep.update(extra)
    if rep["n_bad"]:
        idx = torch.nonzero(bad)
        r_ids = idx[:, 0] if rows is None else rows[idx[:, 0]]
        rep["bad_rows_first"] = sorted(set(int(r) for r in r_ids[:4096].tolist()))[:16]
        rep["bad_cols_first"] = sorted(set(int(c) for c in idx[:4096, 1].tolist()))[:16]
        rep["bad_col_groups_of_32"] = sorted(set(int(c) // 32 for c in idx[:, 1].tolist()))[:32]
        rep["samples"] = [[int(r_ids[i]), int(idx[i, 1]), float(g[idx[i, 0], idx[i, 1]]), float(y[idx[i, 0], idx[i, 1]]),
                           float(delta[idx[i, 0], idx[i, 1]])] for i in range(min(6, idx.shape[0]))]
    _record(rep)
    return rep


def _assert_window(*args, **kw):
    rep = _window_report(*args, **kw)
    assert rep["n_bad"] == 0, json.dumps(rep)
    return rep


# ----------------------------------------------------------------------------------------------- GEMM / conv reference
def _expect(a, w, bias=None, res=None, geglu=False, silu=False):
    """exact epilogue(a @ w^T) in fp64 and its bound.  a [R, K] and w [N, K] in the storage dtype (w in the upstream
    layout: for GEGLU the value rows first, then the gate rows), bias [R, N] fp32 (already one row per output row),
    res [R, N_out].  Returns (y, delta, delta_unit) with delta = C_ACC * delta_unit + activation error."""
    k = a.shape[1]
    ad, wd = a.double(), w.double()
    acc = ad @ wd.t()
    s = ad.abs() @ wd.abs().t()
    if bias is not None:
        acc = acc + bias.double()
        s = s + bias.double().abs()
    unit = math.sqrt(k) * U
    du = unit * s                           # per accumulated column
    act = torch.zeros_like(acc)
    if geglu:
        n = acc.shape[1] // 2
        v, gt = acc[:, :n], acc[:, n:]
        ge = 0.5 * gt * (1.0 + torch.erf(gt / math.sqrt(2.0)))
        y = v * ge
        # d(v * gelu(g)) <= |gelu(g)| dv + |v| (1.13 dg + 9e-7) (+ the product of both); one fp32 rounding of the product
        du_out = ge.abs() * du[:, :n] + v.abs() * GELU_LIP * du[:, n:] + GELU_LIP * du[:, :n] * du[:, n:]
        act = v.abs() * GELU_ABS + U * y.abs()
        du = du_out
    else:
        y = acc
    if res is not None:
        r = res.double()
        y = y + r
        du = du + unit * r.abs()
    if silu:
        # __fdividef(v, 1 + __expf(-v)): __expf is within (2 + 1.173 |v|) ulp, __fdividef within 2 ulp
        sig = torch.sigmoid(y)
        out = y * sig
        act = SILU_LIP * act + y.abs() / 4 * (2.0 + 1.173 * y.abs()) * 2 * U + 4 * U * out.abs()
        du = SILU_LIP * du
        y = out
    return y, C_ACC * du + act, du


def _expect_chunked(a_of, nrows, w, k, bias_of=None, res_of=None, geglu=False, silu=False):
    """_expect over row chunks (a_of(lo, hi) -> a rows), so an im2col of many rows never sits in fp64 at once"""
    step = max(256, (1 << 25) // max(k, 1))
    ys, ds, us = [], [], []
    for lo in range(0, nrows, step):
        hi = min(nrows, lo + step)
        y, d, u = _expect(a_of(lo, hi), w, None if bias_of is None else bias_of(lo, hi),
                          None if res_of is None else res_of(lo, hi), geglu, silu)
        ys.append(y)
        ds.append(d)
        us.append(u)
    return torch.cat(ys), torch.cat(ds), torch.cat(us)


def _gemm_rows(m, n_cols, rng_seed, max_ctas=0, n_n_tiles=1):
    """output rows to check: all when small; else the first and last 128-row tile, the first and last tile of every
    CTA's walk and a seeded sample of interior rows"""
    if m * n_cols <= (1 << 23):
        return torch.arange(m, device="cuda")
    tiles = (m + 127) // 128
    sel = [0, tiles - 1]
    if max_ctas:
        items = tiles * n_n_tiles
        grid = min(items, 132, max_ctas)
        for b in range(grid):
            sel += [b // n_n_tiles, (b + (items - 1 - b) // grid * grid) // n_n_tiles]
    rows = [torch.arange(t * 128, min(m, t * 128 + 128), device="cuda") for t in sorted(set(sel))]
    gr = torch.Generator(device="cuda").manual_seed(rng_seed)
    rows.append(torch.randint(0, m, (N_RANDOM_ROWS,), generator=gr, device="cuda"))
    return torch.unique(torch.cat(rows))


def _out_slice(rows, cols, dt, lpad=32, rpad=32):
    """an output that is a column slice of a NaN-filled wider buffer (the sentinel)"""
    buf = torch.full((rows, lpad + cols + rpad), float("nan"), device="cuda", dtype=dt)
    return buf, buf[:, lpad:lpad + cols]


def _check_slice_untouched(buf, lpad, cols):
    assert bool(torch.isnan(buf[:, :lpad]).all()) and bool(torch.isnan(buf[:, lpad + cols:]).all()), \
        "written outside the output slice"
    assert not bool(torch.isnan(buf[:, lpad:lpad + cols]).any()), "NaN (or unwritten element) in the output"


# ----------------------------------------------------------------------------------------------- linear
def _linear_case(ops, name, dt, m, n, k, bias="one", residual=False, geglu=False, silu=False, block_n=None,
                 max_ctas=0, a_nonneg=False, seed=0):
    g = _gen(seed + m * 3 + n * 7 + k)
    if a_nonneg:   # probabilities (the P.V GEMM of the VAE attention)
        a = (torch.rand((m, k), generator=g, device="cuda") * (2.0 / k)).to(dt)
    else:
        a = _rand((m, k), g, 1.0, dt)
    w = _rand((n, k), g, 1.0 / math.sqrt(k), dt)
    n_out = n // 2 if geglu else n
    b = None
    if bias == "one":
        b = torch.randn(n, generator=g, device="cuda")
    elif bias == "group":
        b = torch.randn(4, n, generator=g, device="cuda")
    res = _rand((m, n_out), g, 1.0, dt) if residual else None
    flags = (ops.EPI_GEGLU if geglu else 0) | (ops.EPI_SILU if silu else 0)
    wk, bk = w, b
    if geglu:
        from b200sd.weights import pack_geglu
        wk, bk = pack_geglu(w, b, block_n or ops.pick_block_n(n, True))
    buf, out = _out_slice(m, n_out, dt)
    grp = (m + 3) // 4 if bias == "group" else 0
    ops.linear(a, wk, out, bias=bk, bias_group_rows=grp, residual=res, flags=flags, block_n=block_n, max_ctas=max_ctas)
    torch.cuda.synchronize()
    _check_slice_untouched(buf, 32, n_out)
    bn_used = block_n or ops.pick_block_n(n, geglu, m)
    rows = _gemm_rows(m, n_out, seed + 1, max_ctas, n // bn_used)

    def bias_of(lo, hi):
        r = rows[lo:hi]
        return (b[r // grp] if grp else b.expand(hi - lo, n)) if b is not None else None
    y, d, u = _expect_chunked(lambda lo, hi: a[rows[lo:hi]], rows.numel(), w, k,
                              None if b is None else bias_of, None if res is None else (lambda lo, hi: res[rows[lo:hi]]),
                              geglu, silu)
    _assert_window(f"linear {name} m{m} n{n} k{k} bn{bn_used} ctas{max_ctas}", out[rows], y, d, dt, rows=rows,
                   delta_unit=u, extra={"op": "linear", "block_n": bn_used})


SDXL_LINEARS = {   # name: (m, n, k, kwargs); m for two images at SDXL's 832x1216 bucket where it is per token
    "ff1_geglu": (1976, 10240, 1280, dict(geglu=True)),
    "ff2_residual": (1976, 1280, 5120, dict(residual=True)),
    "ff2_tail1": (1025, 1280, 5120, dict(residual=True)),
    "ff2_tail127": (1151, 1280, 5120, dict(residual=True)),
    "attn2_kv": (154, 2560, 2048, dict(bias=None)),
    "label_emb0_silu": (2, 1280, 2816, dict(silu=True)),
    "time_emb_residual_silu": (2, 1280, 1280, dict(residual=True, silu=True)),
    "group_bias_silu": (1151, 640, 320, dict(bias="group", silu=True)),
}


@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("case", list(SDXL_LINEARS))
def test_linear_sdxl_epilogues(ops, case, dt):
    m, n, k, kw = SDXL_LINEARS[case]
    _linear_case(ops, case, dt, m, n, k, **kw)


@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_linear_geglu_block_n(ops, bn, dt):
    """ff1 of SDXL's level-2 transformer (GEGLU, K 1280, N 10240) at every GEGLU tile width, with an M tail of 127"""
    _linear_case(ops, "ff1_geglu", dt, 1151, 10240, 1280, geglu=True, block_n=bn)


@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("bn,max_ctas", [(32, 0), (64, 1), (96, 0), (128, 0), (160, 3), (192, 0), (224, 0), (256, 3)])
def test_linear_every_block_n(ops, bn, max_ctas, dt):
    """bias + residual at every tile width on N = 26880 (all eight divide it), M = 257 (one row past two tiles), including
    the spilling 192 / 224 / 256 that pick_block_n never chooses; max_ctas 1 / 3 make persistent CTAs walk many tiles"""
    _linear_case(ops, "every_bn", dt, 257, 26880, 128, residual=True, block_n=bn, max_ctas=max_ctas)


@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("s", [4096, 15808, 16384])
def test_linear_vae_attention(ops, s, dt):
    """the VAE mid-block attention's two GEMMs per image: S = q k^T (M = N = s, K = 512) and O = P V (M = s, N = 512,
    K = s) at 512^2 / 832x1216 / 1024^2 (checked on selected rows)"""
    _linear_case(ops, "vae_scores", dt, s, s, 512, bias=None)
    _linear_case(ops, "vae_pv", dt, s, 512, s, bias=None, a_nonneg=True)


@pytest.mark.parametrize("op", ["linear", "conv2d"])
def test_inplace_residual_channel_slice(ops, op):
    """ControlNet zero convs: D += epi(A W^T) in place (residual is the output), the output a channel slice of a wider
    buffer whose other columns must keep their sentinel"""
    dt = torch.float16
    g = _gen(71 if op == "linear" else 72)
    nb, h, w_, c, cout = 2, 26, 38, 320, 640
    m = nb * h * w_
    x = _rand((nb, h, w_, c), g, 1.0, dt)
    k = c if op == "linear" else 9 * c
    wt = _rand((cout, k), g, 1.0 / math.sqrt(k), dt)
    bias = torch.randn(cout, generator=g, device="cuda")
    buf = torch.full((m, 64 + cout + 320), float("nan"), device="cuda", dtype=dt)
    out = buf[:, 64:64 + cout]
    out.copy_(_rand((m, cout), g, 1.0, dt))
    before = out.clone()
    if op == "linear":
        ops.linear(x.reshape(m, c), wt, out, bias=bias, residual=out)
        a = x.reshape(m, c)
    else:
        ops.conv2d(x, wt, out, ksize=3, bias=bias, residual=out)
        a = _im2col(F.pad(x, (0, 0, 1, 1, 1, 1)), torch.arange(m, device="cuda"), h, w_, 3, 1)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:, :64]).all()) and bool(torch.isnan(buf[:, 64 + cout:]).all())
    y, d, u = _expect(a, wt, bias.expand(m, cout), before)
    _assert_window(f"inplace_residual {op}", out, y, d, dt, delta_unit=u, extra={"op": op})


# ----------------------------------------------------------------------------------------------- conv
def _conv_geometry(nb, ho, wo):
    """the output-pixel box of conv_tc: as much of a row as fits in 128, then rows, then images"""
    bw = min(wo, 128)
    bh = max(1, min(128 // bw, ho))
    bn = max(1, min(128 // (bw * bh), nb))
    return bw, bh, bn, -(-wo // bw), -(-ho // bh), -(-nb // bn)


def _conv_rows(nb, ho, wo, n_n_tiles, max_ctas, seed):
    """every row of every tile that touches an image edge or is ragged, the first and last tile of every CTA's walk
    when max_ctas is set, and a seeded sample of rows"""
    bw, bh, bn, tx, ty, tn = _conv_geometry(nb, ho, wo)
    t = torch.arange(tx * ty * tn, device="cuda")
    x0, y0, n0 = (t % tx) * bw, ((t // tx) % ty) * bh, (t // (tx * ty)) * bn
    keep = (x0 == 0) | (x0 + bw >= wo) | (y0 == 0) | (y0 + bh >= ho) | (n0 + bn > nb)
    if max_ctas:
        items = tx * ty * tn * n_n_tiles
        grid = min(items, 132, max_ctas)
        for b in range(grid):
            for it in (b, b + (items - 1 - b) // grid * grid):
                keep[it // n_n_tiles] = True
    t = t[keep]
    r = torch.arange(bw * bh * bn, device="cuda")
    xs = x0[keep][:, None] + r % bw
    ys = y0[keep][:, None] + (r // bw) % bh
    ns = n0[keep][:, None] + r // (bw * bh)
    valid = (xs < wo) & (ys < ho) & (ns < nb)
    rows = ((ns * ho + ys) * wo + xs)[valid]
    gr = torch.Generator(device="cuda").manual_seed(seed)
    rows = torch.cat([rows, torch.randint(0, nb * ho * wo, (N_RANDOM_ROWS,), generator=gr, device="cuda")])
    return torch.unique(rows)


def _im2col(xp, rows, ho, wo, k, s):
    """the K = k*k*C operand row of each selected output pixel, gathered from the zero-padded NHWC input"""
    n = rows // (ho * wo)
    y = (rows // wo) % ho
    x = rows % wo
    dy = torch.arange(k, device="cuda").repeat_interleave(k)
    dx = torch.arange(k, device="cuda").repeat(k)
    patch = xp[n[:, None], y[:, None] * s + dy[None], x[:, None] * s + dx[None]]
    return patch.reshape(rows.numel(), -1)


CONVS = {   # name: (nb, h, w, c, cout, ksize, stride, pad, pad_end, bias, residual, block_n, max_ctas, in_pitch)
    "unet_128x128": (2, 128, 128, 320, 320, 3, 1, 1, 1, "image", True, None, 0, 0),
    "unet_104x152": (2, 104, 152, 320, 320, 3, 1, 1, 1, "image", True, None, 0, 0),
    "unet_152x104": (2, 152, 104, 320, 320, 3, 1, 1, 1, "image", True, None, 0, 0),
    "unet_52x76": (2, 52, 76, 640, 640, 3, 1, 1, 1, "image", True, None, 0, 0),
    "unet_26x38": (2, 26, 38, 1280, 1280, 3, 1, 1, 1, "image", True, None, 3, 0),
    "unet_down_104x152": (2, 104, 152, 320, 320, 3, 2, 1, 1, "one", False, None, 0, 0),
    "unet_down_52x76": (2, 52, 76, 640, 640, 3, 2, 1, 1, "one", False, None, 0, 0),
    "unet_skipcat_slice": (2, 52, 76, 1920, 640, 3, 1, 1, 1, "image", True, None, 0, 2560),
    "unet_skip_1x1": (2, 52, 76, 1920, 640, 1, 1, 0, 0, "one", False, None, 0, 2560),
    "vae_104x152": (1, 104, 152, 512, 512, 3, 1, 1, 1, "one", True, None, 0, 0),
    "vae_208x304": (1, 208, 304, 512, 512, 3, 1, 1, 1, "one", True, None, 0, 0),
    "vae_416x608": (1, 416, 608, 512, 256, 3, 1, 1, 1, "one", False, None, 0, 0),
    "vae_832x1216": (1, 832, 1216, 256, 128, 3, 1, 1, 1, "one", False, None, 0, 0),
    "vae_conv_out": (1, 832, 1216, 128, 32, 3, 1, 1, 1, "one", False, 32, 0, 0),
    "vae_enc_down": (1, 832, 1216, 128, 128, 3, 2, 0, 1, "one", False, None, 0, 0),
}


@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("case", list(CONVS))
def test_conv_real_geometry(ops, case, dt):
    """UNet / VAE convolutions at SDXL's 1024^2 and 832x1216 latent sizes and their VAE widths: ragged boxes in x
    (Wo > 128, Wo % 128 != 0) and in y (26x38: bw 38, bh 3), stride 2 with pad (1, 1) and (0, 1), a channel-slice input,
    a per-image bias (bias_group_rows = Ho*Wo) and a residual"""
    nb, h, w_, c, cout, ks, st, pad, pad_end, bias_kind, residual, bn, max_ctas, pitch = CONVS[case]
    g = _gen(101 * list(CONVS).index(case) + 7)
    if pitch:
        xbuf = _rand((nb, h, w_, pitch), g, 1.0, dt)
        x = xbuf[..., pitch - c:]
    else:
        x = _rand((nb, h, w_, c), g, 1.0, dt)
    k = ks * ks * c
    wt = _rand((cout, k), g, 1.0 / math.sqrt(k), dt)
    ho = (h + pad + pad_end - ks) // st + 1
    wo = (w_ + pad + pad_end - ks) // st + 1
    m = nb * ho * wo
    if bias_kind == "image":
        bias, grp = torch.randn(nb, cout, generator=g, device="cuda"), ho * wo
    else:
        bias, grp = torch.randn(cout, generator=g, device="cuda"), 0
    res = _rand((m, cout), g, 1.0, dt) if residual else None
    buf, out = _out_slice(m, cout, dt)
    ops.conv2d(x, wt, out, ksize=ks, stride=st, pad=pad, pad_end=pad_end, bias=bias, bias_group_rows=grp,
               residual=res, block_n=bn, max_ctas=max_ctas)
    torch.cuda.synchronize()
    _check_slice_untouched(buf, 32, cout)
    bn_used = bn or ops.pick_block_n(cout, False, m)
    rows = _conv_rows(nb, ho, wo, cout // bn_used, max_ctas, 5)
    xp = F.pad(x, (0, 0, pad, pad_end, pad, pad_end))
    y, d, u = _expect_chunked(
        lambda lo, hi: _im2col(xp, rows[lo:hi], ho, wo, ks, st), rows.numel(), wt, k,
        lambda lo, hi: bias[rows[lo:hi] // grp] if grp else bias.expand(hi - lo, cout),
        None if res is None else (lambda lo, hi: res[rows[lo:hi]]))
    bw, bh, bnb, tx, ty, tn = _conv_geometry(nb, ho, wo)
    rep = _assert_window(f"conv {case} {h}x{w_} c{c}->{cout} k{ks} s{st}", out[rows], y, d, dt, rows=rows,
                         delta_unit=u, extra={"op": "conv2d", "block_n": bn_used, "box": [bw, bh, bnb],
                                              "tiles": [tx, ty, tn], "rows_checked": int(rows.numel()),
                                              "rows_total": m})
    assert rep["rows_checked"] >= min(m, N_RANDOM_ROWS // 2)


# ----------------------------------------------------------------------------------------------- softmax_rows
@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("cols", [77, 4096, 15808, 16384, 36864])
def test_softmax_rows_fp64(ops, cols, dt):
    """the VAE mid-block attention's row softmax at its lengths up to a 1536^2 hires pass (36864), rows of a pitched
    buffer, logits whose scaled values overflow exp() unless the row maximum is subtracted (and rows far below 0)"""
    rows, scale = 48, 512 ** -0.5
    g = _gen(cols)
    lpad = 64
    buf = torch.full((rows, lpad + cols + 40), float("nan"), device="cuda", dtype=dt)
    s = buf[:, lpad:lpad + cols]
    centre = torch.linspace(-3000.0, 3200.0, rows, device="cuda")[:, None]   # scaled: about -133 .. +141
    logits = centre + 40.0 * torch.randn((rows, cols), generator=g, device="cuda")
    s.copy_(logits.to(dt))
    x = s.double()
    ops.softmax_rows_(s, scale)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:, :lpad]).all()) and bool(torch.isnan(buf[:, lpad + cols:]).all())
    # the kernel's exponent: (x - max) * fl32(fl32(scale) * fl32(log2 e)), base 2
    sl2 = float(np.float32(np.float32(scale) * np.float32(1.4426950408889634)))
    t = (x - x.max(dim=1, keepdim=True).values) * sl2
    p = torch.exp2(t)
    p = p / p.sum(dim=1, keepdim=True)
    # rounding of t (|t| ln2 u, and of the row term in the sum), exp2f (2 ulp), the sum of positive terms (a chain of
    # cols/256 + 5 + 8 fp32 additions), 1/sum and the final product (1 rounding each)
    tmax = t.abs().max(dim=1, keepdim=True).values
    eps = (math.log(2.0) * (t.abs() + tmax) + 4 + 4 + (cols / 256 + 13) + 2) * U
    _assert_window(f"softmax_rows cols{cols}", s, p, p * eps, dt, extra={"op": "softmax_rows"})


# ----------------------------------------------------------------------------------------------- fused sampler steps
def _lin(absmode, *pairs):
    """sum of c * v; with absmode the magnitude sum |c| |v| that bounds the rounding errors of the same expression"""
    if absmode:
        return sum(abs(c) * v.abs() for c, v in pairs)
    return sum(c * v for c, v in pairs)


@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("kind", ["ddim", "euler_a", "dpmpp_2m"])
def test_eps_step_kernels_against_fp64(ops, kind, dt):
    """two steps (coefficient rows 1 and 2) of a fused eps-prediction step kernel on B = 3 images of HW = 37 pixels,
    against an fp64 restatement; the second Euler a call passes NULL noise, DPM++ 2M's row 1 has c2 = 0.  Bound: the
    kernel evaluates each step in at most 12 fp32 roundings, so |x - x_ref| <= 32 u * M with M the same two steps
    evaluated on magnitudes (|coefficient| * |input| everywhere)."""
    g = torch.Generator().manual_seed(41)
    b, hw, steps, cfg = 3, 37, 4, 6.5
    eps = torch.randn((2 * b, hw, 32), generator=g).to(dt).cuda()
    x0 = (torch.randn((b, hw, 4), generator=g) * 3.0).float()
    old0 = torch.randn((b, hw, 4), generator=g).float()
    noise = torch.randn((steps, b, hw, 4), generator=g).float()
    rows = []
    for i in range(steps):
        s = 10.0 / (i + 1)
        if kind == "ddim":
            a, ap = 0.2 + 0.15 * i, 0.3 + 0.15 * i
            rows.append([a ** 0.5, (1 - a) ** 0.5, ap ** 0.5, (1 - ap) ** 0.5])
        elif kind == "euler_a":
            sn = s / 2
            up = (sn ** 2 * (s ** 2 - sn ** 2) / s ** 2) ** 0.5
            rows.append([s, (sn ** 2 - up ** 2) ** 0.5, up, 1 / (sn * sn + 1) ** 0.5])
        else:
            c1, c2 = (1.0, 0.0) if i == 1 else (1.4, 0.4)
            rows.append([s, 0.5, c1, c2, 0.7, 0.0, 0.0, 0.0])
    coef = torch.tensor(rows, dtype=torch.float32)
    x, old = x0.cuda(), old0.cuda()
    xin = torch.zeros((2 * b, hw, 64), dtype=dt, device="cuda")
    step = torch.ones((1,), dtype=torch.int32, device="cuda")
    nz = noise.cuda()
    for k in range(2):
        if kind == "ddim":
            ops.cfg_ddim_step(eps, x, xin, cfg, coef.cuda(), step)
        elif kind == "euler_a":
            ops.cfg_euler_a_step(eps, x, None if k == 1 else nz, xin, cfg, coef.cuda(), step)
        else:
            ops.cfg_dpmpp_2m_step(eps, x, old, xin, cfg, coef.cuda(), step)
    torch.cuda.synchronize()
    assert int(step.item()) == 3

    ed = eps[..., :4].double().cpu()
    ec, eu = ed[:b], ed[b:]
    fp = {}
    for am in (False, True):
        xr, oldr, in_next = x0.double(), old0.double(), 1.0
        if am:
            xr, oldr = xr.abs(), oldr.abs()
        e = _lin(am, (1.0 - cfg, eu), (cfg, ec))
        for k, r in enumerate(coef.double()[1:3].tolist()):
            if kind == "ddim":
                sa, s1a, sap, s1ap = r
                x0p = _lin(am, (1.0 / sa, xr), (-s1a / sa, e))
                xr = _lin(am, (sap, x0p), (s1ap, e))
            elif kind == "euler_a":
                s, down, up, in_next = r
                xr = _lin(am, (1.0, xr), (down - s, e)) + (0.0 if k == 1 else 1.0) * _lin(am, (up, noise[1 + k].double()))
            else:
                s, a, c1, c2, in_next = r[:5]
                dn = _lin(am, (1.0, xr), (-s, e))
                dd = _lin(am, (c1, dn), (-c2, oldr)) if c2 != 0 else dn
                xr, oldr = _lin(am, (a, xr), (1.0 - a, dd)), dn
        fp[am] = (xr, oldr, in_next)
    (xr, oldr, in_next), (xm, om, _) = fp[False], fp[True]
    tol = 32 * U * (xm + 1e-30)
    xg = x.cpu().double()
    rep = {"name": f"step {kind}", "dtype": _dname(dt), "op": "fused_step",
           "worst_ratio": float(((xg - xr).abs() / tol).max())}
    if kind == "dpmpp_2m":
        rep["worst_ratio_old"] = float(((old.cpu().double() - oldr).abs() / (32 * U * (om + 1e-30))).max())
    _record(rep)
    assert rep["worst_ratio"] <= 1.0 and rep.get("worst_ratio_old", 0.0) <= 1.0, json.dumps(rep)
    # the packed next UNet input: both CFG halves are RN(x * in_scale_next) of the kernel's own fp32 x, and within one
    # ulp (+ the bound above) of the fp64 value; channels >= 4 stay zero
    xs = x * torch.tensor(np.float32(in_next), device="cuda") if kind != "ddim" else x
    want = xs.to(dt)
    for half in (xin[:b], xin[b:]):
        assert torch.equal(half[..., :4], want), kind
        assert not bool(half[..., 4:].any())
        got = half[..., :4].double().cpu()
        assert bool(((got - xr * in_next).abs() <= 2 * _half_ulp(xr * in_next, dt) + tol * in_next).all()), kind


# ----------------------------------------------------------------------------------------------- GroupNorm / LayerNorm
K_SIGMA = 6.0   # the statistics' rounding error is a sum of many independent roundings: bounded at six standard deviations


def _gn_sum_sigma(hw, c, groups, m0):
    """standard deviation of the fp32 rounding error of one (image, group) sum of hw * C/G terms of magnitude m0, in the
    order of groupnorm_stats_kernel (gn_geometry restated: 96 KB of one image per CTA, 4-pixel unroll): per thread a
    chain over its pixels, then over the block's rows (PY), over the group's channels, and across CTAs in at most 8
    slices.  A sequential chain of n terms of size m has partial sums k m; each rounding is uniform within u |partial|."""
    vx = c // 8
    py = max(1, min(512 // vx, hw))
    quantum = py * 4
    ppc = max(quantum, -(-(96 * 1024 // (2 * c)) // quantum) * quantum)
    parts = -(-hw // ppc)
    cpg = c // groups
    ppt = ppc / py

    def chain(n, m):
        return m * m * n ** 3 / 3.0
    v = (hw * cpg / ppt) * chain(ppt, m0) + parts * cpg * chain(py, ppt * m0) + parts * chain(cpg, ppc * m0)
    if parts > 1:
        slices = max(1, min(vx * py // (2 * groups), 8))
        per = -(-parts // slices)
        v += slices * chain(per, ppc * cpg * m0) + chain(slices, per * ppc * cpg * m0)
    return U * math.sqrt(v / 3.0)


def _silu_with_bound(t, dt_):
    """silu(t) and its error bound given |error of t| <= dt_: the Lipschitz constant, the approximate exp2 and
    reciprocal (2 ulp each) and the rounding of t * log2(e)"""
    sig = torch.sigmoid(t)
    out = t * sig
    return out, SILU_LIP * dt_ + t.abs() / 4 * (t.abs() + 8.0) * U + 8 * U * out.abs()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("dt", DTS, ids=_dname)
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("mean_over_std", [0.0, 8.0, 64.0])
@pytest.mark.parametrize("hw,c", [(128 * 128, 512), (512 * 512, 256), (1024 * 1024, 128), (4096, 640)])
def test_groupnorm_fp64(ops, hw, c, mean_over_std, silu, dt):
    """GroupNorm(32) at the VAE's decoder shapes up to 1024^2 and one UNet shape, on inputs of mean/std 0, 8 and 64: the
    kernel takes var = E[x^2] - mean^2 in fp32, whose error grows with (mean/std)^2.  delta follows that algorithm: the
    summation error of both statistics (K_SIGMA standard deviations of the rounding in the kernel's summation order),
    the cancellation in E[x^2] - mean^2, rsqrtf (2 ulp), the fp32 rounding of the folded scale / shift and of the fma,
    and for SiLU its approximations."""
    g = _gen(hw + c + int(mean_over_std))
    nb, groups, eps = 1, 32, 1e-6
    x = _rand((nb, hw, c), g, 1.0, dt, offset=mean_over_std)
    gamma = torch.randn(c, generator=g, device="cuda")
    beta = torch.randn(c, generator=g, device="cuda")
    out = torch.empty_like(x)
    stats = torch.zeros((ops.groupnorm_stats_floats(nb, hw, c, groups),), device="cuda")
    ops.groupnorm(x, out, stats, gamma, beta, groups, eps, silu)
    torch.cuda.synchronize()
    xd = x.double().reshape(nb, hw, groups, c // groups)
    cnt = hw * (c // groups)
    s1 = xd.sum(dim=(1, 3))
    s2 = (xd * xd).sum(dim=(1, 3))
    mu = s1 / cnt
    ex2 = s2 / cnt
    var = ex2 - mu * mu
    d_s1 = K_SIGMA * torch.tensor([[_gn_sum_sigma(hw, c, groups, float(a)) for a in row]
                                   for row in (xd.abs().sum(dim=(1, 3)) / cnt).tolist()], dtype=torch.float64, device="cuda")
    d_s2 = K_SIGMA * torch.tensor([[_gn_sum_sigma(hw, c, groups, float(a)) for a in row] for row in ex2.tolist()],
                                  dtype=torch.float64, device="cuda")
    got_stats = stats[:nb * groups * 2].double().reshape(nb, groups, 2)
    stat_ratio = max(float(((got_stats[..., 0] - s1).abs() / d_s1).max()), float(((got_stats[..., 1] - s2).abs() / d_s2).max()))
    mu_k = got_stats[..., 0] / cnt
    rstd_err = float(((got_stats[..., 1] / cnt - mu_k * mu_k + eps) / (var + eps)).rsqrt().sub(1).abs().max())
    d_mu = d_s1 / cnt + 2 * U * mu.abs()
    d_var = d_s2 / cnt + 2 * mu.abs() * d_mu + 3 * U * (ex2 + mu * mu) + U * var.abs()
    rstd = 1.0 / torch.sqrt(var + eps)
    e_r = 0.5 * d_var / (var + eps) + 5 * U
    rep_g = lambda t: t.repeat_interleave(c // groups, dim=1)[:, None, :]  # noqa: E731  [nb, 1, c]
    scale = rep_g(rstd) * gamma.double()
    xm = x.double() - rep_g(mu)
    y = xm * scale + beta.double()
    d = (xm.abs() * scale.abs() * (rep_g(e_r) + U) + scale.abs() * rep_g(d_mu)
         + U * (2 * (rep_g(mu) * scale).abs() + beta.double().abs() + 2 * y.abs()))
    if silu:
        y, d = _silu_with_bound(y, d)
    rep = _window_report(f"groupnorm hw{hw} c{c} mean/std{mean_over_std} silu{int(silu)}", out.reshape(-1, c),
                         y.reshape(-1, c), d.reshape(-1, c), dt,
                         extra={"op": "groupnorm", "stats_worst_ratio": stat_ratio, "rstd_rel_err": rstd_err,
                                "rstd_bound_rel": float(e_r.max())})
    assert stat_ratio <= 1.0, json.dumps(rep)
    assert rep["n_bad"] == 0, json.dumps(rep)


@pytest.mark.parametrize("rows,c", [(4133, 640), (4133, 1280), (1000, 2048)])
def test_layernorm_bf16_fp64(ops, rows, c):
    """LayerNorm in bf16 with an offset (mean/std 4): the staged kernel (C <= 1376) and the register kernel (C 2048).
    Both centre before squaring; delta is the worst case of their fp32 sums (C terms), rsqrtf (2 ulp) and the roundings
    of the normalise-scale-shift"""
    dt = torch.bfloat16
    g = _gen(rows + c)
    x = _rand((rows, c), g, 1.0, dt, offset=4.0)
    gamma = torch.randn(c, generator=g, device="cuda")
    beta = torch.randn(c, generator=g, device="cuda")
    out = torch.empty_like(x)
    ops.layernorm(x, out, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    xd = x.double()
    mu = xd.mean(dim=1, keepdim=True)
    xm = xd - mu
    var = (xm * xm).mean(dim=1, keepdim=True)
    d_mu = (c + 2) * U * xd.abs().mean(dim=1, keepdim=True)
    # sum (x - mean_k)^2 with mean_k = mean + e: the first-order term in e vanishes (sum (x - mean) = 0)
    d_var = (c + 4) * U * var + d_mu * d_mu
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    e_r = 0.5 * d_var / (var + 1e-5) + 5 * U
    sc = rstd * gamma.double()
    y = xm * sc + beta.double()
    d = xm.abs() * sc.abs() * (e_r + 2 * U) + sc.abs() * (d_mu + U * xm.abs()) + U * (beta.double().abs() + 2 * y.abs())
    _assert_window(f"layernorm rows{rows} c{c}", out, y, d, dt, extra={"op": "layernorm"})


# ----------------------------------------------------------------------------------------------- packing kernels (bf16)
def test_unpack_latent_and_image_to_nhwc_bf16(ops):
    """bitwise: x = mean * scale (one fp32 multiply) and 2 x / 255 - 1 (one fp32 fma: nvcc contracts the multiply-add)"""
    g = torch.Generator(device="cuda").manual_seed(9)
    b, hw = 2, 3001
    mom = _rand((b, hw, 32), _gen(8), 2.0, torch.bfloat16)
    x = torch.empty((b, hw, 4), device="cuda")
    ops.unpack_latent(mom, x, 0.13025)
    img = torch.randint(0, 256, (b, hw, 3), generator=g, device="cuda", dtype=torch.uint8)
    img[0, :256, 0] = torch.arange(256, device="cuda", dtype=torch.uint8)
    out = torch.full((b, hw, 32), 7.0, device="cuda", dtype=torch.bfloat16)
    ops.image_to_nhwc(img, out)
    torch.cuda.synchronize()
    assert torch.equal(x, mom[..., :4].float() * torch.tensor(np.float32(0.13025), device="cuda"))
    c = float(np.float32(2.0 / 255.0))
    ref = (img.double() * c - 1.0).float().to(torch.bfloat16)   # exact product, one rounding: the fma
    assert torch.equal(out[..., :3], ref)
    assert bool((out[..., 3:] == 7.0).all())
