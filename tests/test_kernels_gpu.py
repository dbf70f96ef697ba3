"""GPU parity tests of every C-ABI op against a plain PyTorch fp32 reference of the same op.

Tolerances (fp16 operands, fp32 accumulation): outputs are fp16, so one rounding of the result (rel 2^-11)
plus accumulation-order differences; atol scales with sqrt(K) * |a| * |w|.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from kutil import assert_close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from b200sd import ops as _ops
    return _ops


def _rand(shape, gen, scale=1.0, dtype=torch.float16):
    return (torch.randn(shape, generator=gen, device="cuda", dtype=torch.float32) * scale).to(dtype)


def _gen(seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return g


# ----------------------------------------------------------------------------------------------- linear
@pytest.mark.parametrize("m,n,k,bn", [
    (128, 64, 64, 64), (256, 128, 128, 128), (300, 256, 192, 256), (77, 320, 768, 160), (4096, 320, 320, 160),
    (2048, 1280, 1280, 256), (1000, 960, 320, 192), (512, 96, 64, 32), (20, 1280, 320, 256),
])
def test_linear_plain(ops, m, n, k, bn):
    g = _gen(m * 7 + n)
    a = _rand((m, k), g)
    w = _rand((n, k), g, 1.0 / math.sqrt(k))
    out = torch.full((m, n), float("nan"), device="cuda", dtype=torch.float16)
    ops.linear(a, w, out, block_n=bn)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t()
    assert_close(f"linear_plain m{m} n{n} k{k} bn{bn}", out, ref, atol=2e-2, rtol=2e-3)


@pytest.mark.parametrize("residual", [False, True])
def test_linear_many_short_tiles_per_cta(ops, residual):
    """Persistent CTAs walking many tiles whose MMA phase is one k-block long, with an odd number of 32-column chunks
    per epilogue group (bn = 160 -> 3 + 2): the TMA store of a tile's last chunk is still in flight when the next
    tile's first chunk is staged.  Regression test for the staging-buffer reuse across tiles (exact compare, repeated)."""
    g = _gen(11)
    m, n, k = 148 * 128 * 8, 320, 64
    a = _rand((m, k), g)
    w = _rand((n, k), g, 1.0 / math.sqrt(k))
    res = _rand((m, n), g) if residual else None
    ref = a.float() @ w.float().t()
    if residual:
        ref = ref + res.float()
    ref16 = ref.half()
    out = torch.empty((m, n), device="cuda", dtype=torch.float16)
    worst = 0
    for _ in range(5):
        out.fill_(float("nan"))
        ops.linear(a, w, out, residual=res, block_n=160)
        torch.cuda.synchronize()
        # fp32 accumulation of a 64-term dot product rounds to the same half as the reference up to 1 ulp
        bad = int(((out.float() - ref16.float()).abs() > 2e-3 * ref16.float().abs() + 2e-3).sum())
        worst = max(worst, bad)
    assert worst == 0, f"{worst} corrupted outputs"


def test_linear_bias_residual_pitched(ops):
    g = _gen(1)
    m, n, k = 1024, 640, 640
    abuf = _rand((m, k + 64), g)
    a = abuf[:, 64:]  # pitched A (lda = k + 64), 128-byte aligned column offset
    w = _rand((n, k), g, 1.0 / math.sqrt(k))
    bias = torch.randn(n, generator=g, device="cuda")
    res = _rand((m, n), g)
    obuf = torch.zeros((m, n + 320), device="cuda", dtype=torch.float16)
    out = obuf[:, 320:]
    ops.linear(a, w, out, bias=bias, residual=res)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias + res.float()
    assert_close("linear_bias_residual_pitched", out, ref, atol=2e-2, rtol=2e-3)
    assert float(obuf[:, :320].abs().max()) == 0.0


def test_linear_group_bias_silu(ops):
    g = _gen(2)
    m, n, k = 512, 256, 128
    a = _rand((m, k), g)
    w = _rand((n, k), g, 1.0 / math.sqrt(k))
    bias = torch.randn(4, n, generator=g, device="cuda")  # one bias row per 128 output rows
    out = torch.empty((m, n), device="cuda", dtype=torch.float16)
    ops.linear(a, w, out, bias=bias, bias_group_rows=128, flags=ops.EPI_SILU)
    torch.cuda.synchronize()
    ref = F.silu(a.float() @ w.float().t() + bias.repeat_interleave(128, dim=0))
    assert_close("linear_group_bias_silu", out, ref, atol=2e-2, rtol=2e-3)


@pytest.mark.parametrize("m,c,bn", [(512, 320, 256), (1024, 640, 128)])
def test_linear_geglu(ops, m, c, bn):
    """FeedForward GEGLU: proj(x).chunk(2) -> a * gelu(g); weight rows interleaved per tile (value half, gate half)."""
    g = _gen(3)
    inner = 4 * c
    a = _rand((m, c), g)
    w = _rand((2 * inner, c), g, 1.0 / math.sqrt(c))   # upstream layout: rows [0,inner) value, [inner,2inner) gate
    b = torch.randn(2 * inner, generator=g, device="cuda")
    from b200sd.weights import pack_geglu
    wp, bp = pack_geglu(w, b, bn)
    out = torch.empty((m, inner), device="cuda", dtype=torch.float16)
    ops.linear(a, wp, out, bias=bp, flags=ops.EPI_GEGLU, block_n=bn)
    torch.cuda.synchronize()
    y = a.float() @ w.float().t() + b
    ref = y[:, :inner] * F.gelu(y[:, inner:])
    assert_close(f"linear_geglu m{m} c{c}", out, ref, atol=3e-2, rtol=3e-3)


def test_linear_bf16(ops):
    g = _gen(4)
    m, n, k = 384, 256, 256
    a = _rand((m, k), g, dtype=torch.bfloat16)
    w = _rand((n, k), g, 1.0 / math.sqrt(k), dtype=torch.bfloat16)
    out = torch.empty((m, n), device="cuda", dtype=torch.bfloat16)
    ops.linear(a, w, out)
    torch.cuda.synchronize()
    assert_close("linear_bf16", out, a.float() @ w.float().t(), atol=5e-2, rtol=1e-2)


# ----------------------------------------------------------------------------------------------- conv
def _conv_ref(x_nhwc, w_packed, ksize, stride, pad, pad_end, bias=None):
    nb, h, w_, c = x_nhwc.shape
    cout = w_packed.shape[0]
    wt = w_packed.float().reshape(cout, ksize, ksize, c).permute(0, 3, 1, 2)
    x = x_nhwc.float().permute(0, 3, 1, 2)
    x = F.pad(x, (pad, pad_end, pad, pad_end))
    y = F.conv2d(x, wt, bias=bias, stride=stride)
    return y.permute(0, 2, 3, 1).reshape(-1, cout)


@pytest.mark.parametrize("nb,h,w,c,cout,k,s,bn", [
    (2, 16, 16, 64, 64, 3, 1, 64), (2, 64, 64, 320, 320, 3, 1, 160), (3, 8, 8, 1280, 1280, 3, 1, 256),
    (2, 32, 32, 640, 640, 3, 1, 128), (1, 128, 128, 128, 128, 3, 1, 128), (1, 4, 256, 64, 128, 3, 1, 128),
    (1, 2, 512, 128, 128, 3, 1, 128), (2, 32, 32, 128, 128, 3, 2, 128), (2, 64, 64, 320, 320, 3, 2, 160),
    (2, 16, 16, 640, 320, 1, 1, 160), (1, 24, 40, 64, 64, 3, 1, 64), (5, 8, 8, 64, 32, 3, 1, 32),
])
def test_conv2d(ops, nb, h, w, c, cout, k, s, bn):
    g = _gen(nb * 100 + h + c)
    x = _rand((nb, h, w, c), g)
    wt = _rand((cout, k * k * c), g, 1.0 / math.sqrt(k * k * c))
    bias = torch.randn(cout, generator=g, device="cuda")
    pad = 1 if k == 3 else 0
    ho = (h + 2 * pad - k) // s + 1
    wo = (w + 2 * pad - k) // s + 1
    out = torch.full((nb * ho * wo, cout), float("nan"), device="cuda", dtype=torch.float16)
    ops.conv2d(x, wt, out, ksize=k, stride=s, pad=pad, bias=bias, block_n=bn)
    torch.cuda.synchronize()
    ref = _conv_ref(x, wt, k, s, pad, pad, bias)
    assert_close(f"conv nb{nb} {h}x{w} c{c}->{cout} k{k} s{s}", out, ref, atol=2e-2, rtol=2e-3)


def test_conv2d_asym_pad_stride2(ops):
    """VAE encoder Downsample: pad (0,1,0,1) then 3x3 stride 2, no padding."""
    g = _gen(11)
    x = _rand((1, 64, 64, 128), g)
    wt = _rand((128, 9 * 128), g, 1.0 / math.sqrt(9 * 128))
    out = torch.empty((32 * 32, 128), device="cuda", dtype=torch.float16)
    ops.conv2d(x, wt, out, ksize=3, stride=2, pad=0, pad_end=1)
    torch.cuda.synchronize()
    assert_close("conv_asym_pad_s2", out, _conv_ref(x, wt, 3, 2, 0, 1), atol=2e-2, rtol=2e-3)


def test_conv2d_per_image_bias_residual_channel_slice(ops):
    """ResBlock conv1 (+ per-image time-embedding bias) reading a channel slice of a wider skip-concat buffer."""
    g = _gen(12)
    nb, h, w, c, cout = 4, 16, 16, 128, 192
    buf = _rand((nb, h, w, c + 64), g)
    x = buf[..., 64:]
    wt = _rand((cout, 9 * c), g, 1.0 / math.sqrt(9 * c))
    bias = torch.randn(nb, cout, generator=g, device="cuda")
    res = _rand((nb * h * w, cout), g)
    out = torch.empty((nb * h * w, cout), device="cuda", dtype=torch.float16)
    ops.conv2d(x, wt, out, ksize=3, bias=bias, bias_group_rows=h * w, residual=res, block_n=64)
    torch.cuda.synchronize()
    ref = _conv_ref(x, wt, 3, 1, 1, 1) + bias.repeat_interleave(h * w, dim=0) + res.float()
    assert_close("conv_per_image_bias_residual_slice", out, ref, atol=2e-2, rtol=2e-3)


# ----------------------------------------------------------------------------------------------- attention
def _attn_ref(q, k, v, heads, d, d_pad, scale):
    b, sq, _ = q.shape
    skv = k.shape[1]
    qh = q.float().reshape(b, sq, heads, d_pad)[..., :d].permute(0, 2, 1, 3)
    kh = k.float().reshape(b, skv, heads, d_pad)[..., :d].permute(0, 2, 1, 3)
    vh = v.float().reshape(b, skv, heads, d_pad)[..., :d].permute(0, 2, 1, 3)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    return (p @ vh).permute(0, 2, 1, 3).reshape(b, sq, heads * d)


def _padded_heads(b, s, heads, d, d_pad, g, ones_col=False):
    t = torch.zeros((b, s, heads, d_pad), device="cuda", dtype=torch.float16)
    t[..., :d] = _rand((b, s, heads, d), g)
    if ones_col:
        t[..., d] = 1.0
    return t.reshape(b, s, heads * d_pad)


@pytest.mark.parametrize("ones_col", [False, True])
@pytest.mark.parametrize("b,heads,sq,skv,d", [
    (1, 2, 128, 128, 64), (2, 8, 4096, 4096, 40), (2, 8, 1024, 1024, 80), (2, 8, 256, 256, 160), (3, 8, 64, 64, 160),
    (2, 8, 4096, 77, 40), (2, 8, 1024, 77, 80), (1, 8, 256, 77, 160), (1, 10, 1024, 1024, 64), (1, 4, 200, 300, 40),
    # resident-K/V mode (Skv <= 128) with several Q tiles per CTA: 8, 8, 4, 2 (ragged last Q tile), and short kv
    (8, 8, 4096, 77, 40), (8, 8, 1024, 128, 40), (8, 8, 1024, 20, 40), (6, 8, 1000, 77, 80), (16, 8, 512, 40, 160),
])
def test_attention(ops, b, heads, sq, skv, d, ones_col):
    g = _gen(sq + skv + d)
    d_pad = (d + 63) // 64 * 64
    if ones_col and d == d_pad:
        pytest.skip("no pad column to carry the ones")
    q = _padded_heads(b, sq, heads, d, d_pad, g)
    k = _padded_heads(b, skv, heads, d, d_pad, g)
    v = _padded_heads(b, skv, heads, d, d_pad, g, ones_col)
    out = torch.full((b, sq, heads * d), float("nan"), device="cuda", dtype=torch.float16)
    scale = d ** -0.5
    ops.attention(q, k, v, out, heads, d, d_pad, scale, ones_col)
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, heads, d, d_pad, scale)
    assert_close(f"attention b{b} h{heads} sq{sq} skv{skv} d{d} ones{int(ones_col)}", out, ref, atol=4e-3, rtol=1e-2)


@pytest.mark.parametrize("skv", [129, 192, 257, 321, 384, 385, 448, 520, 832])
def test_attention_ring_lengths(ops, skv):
    """kv longer than the K/V ring (3 .. 13 kv tiles, full and ragged last tiles): every slot is refilled at every ring
    phase, so an off-by-one in a slot or parity shows up as a hang (the bounded waits trap) or as garbage"""
    b, heads, sq, d = 3, 8, 512, 40
    g = _gen(skv)
    d_pad = 64
    q = _padded_heads(b, sq, heads, d, d_pad, g)
    k = _padded_heads(b, skv, heads, d, d_pad, g)
    v = _padded_heads(b, skv, heads, d, d_pad, g, True)
    out = torch.full((b, sq, heads * d), float("nan"), device="cuda", dtype=torch.float16)
    ops.attention(q, k, v, out, heads, d, d_pad, d ** -0.5, True)
    torch.cuda.synchronize()
    assert_close(f"attention ring skv{skv}", out, _attn_ref(q, k, v, heads, d, d_pad, d ** -0.5), atol=4e-3, rtol=1e-2)


@pytest.mark.parametrize("ones_col", [False, True])
def test_attention_growing_logits_forces_rescale(ops, ones_col):
    """Keys ordered so that the row maximum keeps rising tile after tile by far more than 2^8: the running maximum and
    the rescale of the O accumulator change on every tile."""
    g = _gen(99)
    b, heads, s, d, d_pad = 1, 2, 1024, 40, 64
    q = _padded_heads(b, s, heads, d, d_pad, g)
    k = _padded_heads(b, s, heads, d, d_pad, g)
    v = _padded_heads(b, s, heads, d, d_pad, g, ones_col)
    ramp = torch.linspace(0.2, 6.0, s, device="cuda").reshape(1, s, 1, 1)
    kk = k.reshape(b, s, heads, d_pad).float()
    qq = q.reshape(b, s, heads, d_pad).float()
    kk[..., :d] = ramp * qq[:, :1, :, :d].abs().clamp(min=0.3) * torch.sign(qq[:, :1, :, :d] + 1e-3)
    k = kk.half().reshape(b, s, heads * d_pad)
    out = torch.empty((b, s, heads * d), device="cuda", dtype=torch.float16)
    ops.attention(q, k, v, out, heads, d, d_pad, 1.0, ones_col)
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, heads, d, d_pad, 1.0)
    assert_close(f"attention_growing_logits ones{int(ones_col)}", out, ref, atol=6e-3, rtol=2e-2)


def test_attention_fused_qkv_buffer(ops):
    """Q, K, V as column slices of one projection output (pitch 3*heads*d_pad), large logits."""
    g = _gen(21)
    b, heads, s, d, d_pad = 2, 8, 512, 40, 64
    qkv = torch.zeros((b, s, 3, heads, d_pad), device="cuda", dtype=torch.float16)
    qkv[..., :d] = _rand((b, s, 3, heads, d), g, 3.0)
    flat = qkv.reshape(b, s, 3 * heads * d_pad)
    q, k, v = (flat[..., i * heads * d_pad:(i + 1) * heads * d_pad] for i in range(3))
    out = torch.empty((b, s, heads * d), device="cuda", dtype=torch.float16)
    ops.attention(q, k, v, out, heads, d, d_pad, d ** -0.5)
    torch.cuda.synchronize()
    ref = _attn_ref(q, k, v, heads, d, d_pad, d ** -0.5)
    assert_close("attention_fused_qkv", out, ref, atol=1e-2, rtol=1e-2)


# ----------------------------------------------------------------------------------------------- norms
@pytest.mark.timeout(300)
@pytest.mark.parametrize("nb,hw,c,silu,eps", [(2, 4096, 320, True, 1e-5), (3, 64, 1280, True, 1e-5),
                                              (2, 1024, 1920, True, 1e-5), (1, 16384, 128, True, 1e-6),
                                              (2, 256, 2560, False, 1e-6), (2, 1024, 960, True, 1e-5)])
def test_groupnorm(ops, nb, hw, c, silu, eps):
    g = _gen(hw + c)
    x = _rand((nb, hw, c), g, 2.0) + 0.5
    gamma = torch.randn(c, generator=g, device="cuda")
    beta = torch.randn(c, generator=g, device="cuda")
    out = torch.empty_like(x)
    stats = torch.zeros((ops.groupnorm_stats_floats(nb, hw, c, 32),), device="cuda")
    ops.groupnorm(x, out, stats, gamma, beta, 32, eps, silu)
    torch.cuda.synchronize()
    # statistics: exact sums in fp32 order-of-magnitude, and bit-identical on a second run over the same (reused,
    # never re-zeroed) buffer — the cross-CTA reduction is ordered, not atomic
    first = stats[:nb * 64].clone()
    xs = x.float().reshape(nb, hw, 32, c // 32)
    ref_stats = torch.stack([xs.sum(dim=(1, 3)), (xs * xs).sum(dim=(1, 3))], dim=-1).reshape(-1)
    assert torch.allclose(first, ref_stats, rtol=2e-4, atol=1e-2)
    # the arrival tickets behind the results are back at zero
    assert int(stats[nb * 64:nb * 64 + nb].view(torch.int32).abs().sum()) == 0
    out2 = torch.empty_like(x)
    ops.groupnorm(x, out2, stats, gamma, beta, 32, eps, silu)
    torch.cuda.synchronize()
    assert torch.equal(stats[:nb * 64], first) and torch.equal(out, out2)
    ref = F.group_norm(x.float().permute(0, 2, 1), 32, gamma, beta, eps).permute(0, 2, 1)
    if silu:
        ref = F.silu(ref)
    assert_close(f"groupnorm nb{nb} hw{hw} c{c}", out, ref, atol=1e-2, rtol=4e-3)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("nb,hw,c,pitch,dt", [(64, 4096, 320, 320, torch.half), (5, 1024, 640, 1280, torch.half),
                                              (3, 4096, 960, 960, torch.bfloat16), (7, 100, 64, 64, torch.half),
                                              (2, 16384, 320, 320, torch.bfloat16), (33, 64, 1280, 2560, torch.half)])
def test_groupnorm_slices_bf16_batch_invariance(ops, nb, hw, c, pitch, dt):
    """the bench's largest site (64 images x 64x64x320: many CTAs per image), channel slices of a wider tensor (the
    UNet's concat buffers), bf16, a ragged last slab, and: an image's result does not depend on the batch it is in, nor
    on the run"""
    g = _gen(nb * 31 + c)
    xw = (_rand((nb, hw, pitch), g, 1.5) + 0.25).to(dt)
    ow = torch.full((nb, hw, pitch), 3.0, device="cuda", dtype=dt)
    x, out = xw[:, :, pitch - c:], ow[:, :, :c]
    gamma = torch.randn(c, generator=g, device="cuda")
    beta = torch.randn(c, generator=g, device="cuda")
    stats = torch.zeros((ops.groupnorm_stats_floats(nb, hw, c, 32),), device="cuda")
    ops.groupnorm(x, out, stats, gamma, beta, 32, 1e-5, True)
    torch.cuda.synchronize()
    ref = F.silu(F.group_norm(x.float().permute(0, 2, 1), 32, gamma, beta, 1e-5).permute(0, 2, 1))
    tol = dict(atol=1e-2, rtol=4e-3) if dt == torch.half else dict(atol=6e-2, rtol=2e-2)
    assert_close(f"groupnorm nb{nb} hw{hw} c{c}/{pitch}", out, ref, **tol)
    if pitch > c:
        assert float((ow[:, :, c:].float() - 3.0).abs().max()) == 0.0   # nothing written outside the slice
    assert int(stats[nb * 64:nb * 64 + nb].view(torch.int32).abs().sum()) == 0
    # run to run, and image by image (batch of one, fresh scratch): identical bits
    for _ in range(3):
        again = torch.empty((nb, hw, c), device="cuda", dtype=dt)
        ops.groupnorm(x, again, stats, gamma, beta, 32, 1e-5, True)
        assert torch.equal(again, out)
    for k in (0, nb - 1):
        alone = torch.empty((1, hw, c), device="cuda", dtype=dt)
        st1 = torch.zeros((ops.groupnorm_stats_floats(1, hw, c, 32),), device="cuda")
        ops.groupnorm(x[k:k + 1], alone, st1, gamma, beta, 32, 1e-5, True)
        assert torch.equal(alone[0], out[k])


@pytest.mark.timeout(300)
def test_groupnorm_under_graph_replay(ops):
    """the step graphs replay GroupNorms back to back on one shared scratch buffer: a chain of launches of different
    shapes, captured once and replayed, must leave the counters at zero and reproduce itself"""
    g = _gen(77)
    shapes = [(8, 4096, 320), (8, 1024, 640), (8, 256, 2560), (8, 64, 1280), (8, 4096, 320)]
    xs = [_rand(s, g, 2.0) + 0.5 for s in shapes]
    outs = [torch.empty_like(x) for x in xs]
    gam = [torch.randn(s[2], generator=g, device="cuda") for s in shapes]
    bet = [torch.randn(s[2], generator=g, device="cuda") for s in shapes]
    need = max(ops.groupnorm_stats_floats(*s, 32) for s in shapes)
    stats = torch.zeros((need,), device="cuda")

    def chain():
        for x, o, ga, be in zip(xs, outs, gam, bet):
            ops.groupnorm(x, o, stats, ga, be, 32, 1e-5, True)
    chain()
    torch.cuda.synchronize()
    want = [o.clone() for o in outs]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        chain()
    for _ in range(5):
        for o in outs:
            o.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for o, w in zip(outs, want):
            assert torch.equal(o, w)
    for x, w, ga, be in zip(xs, want, gam, bet):
        ref = F.silu(F.group_norm(x.float().permute(0, 2, 1), 32, ga, be, 1e-5).permute(0, 2, 1))
        assert_close("groupnorm chain", w, ref, atol=1e-2, rtol=4e-3)


@pytest.mark.parametrize("rows,c,pitch,dt", [(100003, 320, 320, torch.half), (40000, 640, 704, torch.half),
                                              (20001, 1280, 1280, torch.bfloat16), (5000, 64, 64, torch.half),
                                              (3, 320, 320, torch.half)])
def test_layernorm_staged_ring(ops, rows, c, pitch, dt):
    """many tiles per persistent CTA (the input ring and the output stages wrap), a ragged last tile, rows that are
    channel slices of a wider buffer (per-row bulk copies), bf16"""
    g = _gen(rows + c)
    xw = (_rand((rows, pitch), g, 2.0) + 1.0).to(dt)
    ow = torch.full((rows, pitch), 7.0, device="cuda", dtype=dt)
    x, out = xw[:, :c], ow[:, :c]
    gamma = torch.randn(c, generator=g, device="cuda")
    beta = torch.randn(c, generator=g, device="cuda")
    ops.layernorm(x, out, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    tol = dict(atol=1e-2, rtol=4e-3) if dt == torch.half else dict(atol=6e-2, rtol=2e-2)
    assert_close(f"layernorm staged {rows}x{c}/{pitch}", out, F.layer_norm(x.float(), (c,), gamma, beta, 1e-5), **tol)
    if pitch > c:
        assert float((ow[:, c:].float() - 7.0).abs().max()) == 0.0   # nothing written outside the slice
    out2 = torch.empty_like(ow)[:, :c]
    ops.layernorm(x, out2, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)


@pytest.mark.parametrize("rows,c", [(4096, 320), (1000, 640), (77, 1280), (64, 2048)])
def test_layernorm(ops, rows, c):
    g = _gen(rows + c)
    x = _rand((rows, c), g, 2.0) + 1.0
    gamma = torch.randn(c, generator=g, device="cuda")
    beta = torch.randn(c, generator=g, device="cuda")
    out = torch.empty_like(x)
    ops.layernorm(x, out, gamma, beta, 1e-5)
    torch.cuda.synchronize()
    assert_close(f"layernorm {rows}x{c}", out, F.layer_norm(x.float(), (c,), gamma, beta, 1e-5), atol=1e-2, rtol=4e-3)


# ----------------------------------------------------------------------------------------------- small ops
def test_upsample2x(ops):
    g = _gen(31)
    x = _rand((2, 8, 16, 64), g)
    out = torch.empty((2, 16, 32, 64), device="cuda", dtype=torch.float16)
    ops.upsample2x(x, out)
    torch.cuda.synchronize()
    ref = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    assert torch.equal(out, ref)


def test_softmax_rows(ops):
    g = _gen(32)
    s = _rand((300, 4096), g, 4.0)
    ref = torch.softmax(s.float() * 0.125, dim=-1)
    ops.softmax_rows_(s, 0.125)
    torch.cuda.synchronize()
    assert_close("softmax_rows", s, ref, atol=1e-4, rtol=4e-3)


def test_silu_and_timestep_embedding(ops):
    g = _gen(33)
    x = _rand((20, 1280), g, 3.0)
    out = torch.empty_like(x)
    ops.silu(x, out)
    t = torch.tensor([1.0, 51.0, 501.0, 951.0], device="cuda")
    emb = torch.empty((4, 320), device="cuda", dtype=torch.float16)
    ops.timestep_embedding(t, emb)
    torch.cuda.synchronize()
    assert_close("silu", out, F.silu(x.float()), atol=1e-3, rtol=2e-3)
    freqs = torch.exp(-math.log(10000.0) * torch.arange(160, device="cuda", dtype=torch.float32) / 160)
    args = t[:, None] * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    assert_close("timestep_embedding", emb, ref, atol=2e-3, rtol=0)


def test_fold_and_select_bias(ops):
    g = _gen(34)
    emb = _rand((20, 640), g)
    bias = torch.randn(640, generator=g, device="cuda")
    table = torch.empty((20, 640), device="cuda")
    ops.fold_bias(emb, bias, table)
    step = torch.tensor([7], device="cuda", dtype=torch.int32)
    cur = torch.empty(640, device="cuda")
    ops.select_step(table, step, cur)
    torch.cuda.synchronize()
    assert torch.allclose(table, emb.float() + bias)
    assert torch.equal(cur, table[7])


def test_cfg_ddim_step_and_pack(ops):
    g = _gen(35)
    b, hw = 3, 4096
    x = torch.randn((b, hw, 4), generator=g, device="cuda")
    x0 = x.clone()
    xin = torch.zeros((2 * b, hw, 64), device="cuda", dtype=torch.float16)
    ops.pack_unet_input(x, xin, 1.0)
    eps = torch.zeros((2 * b, hw, 32), device="cuda", dtype=torch.float16)
    eps[..., :4] = _rand((2 * b, hw, 4), g)
    coef = torch.tensor([[0.3, 0.95, 0.4, 0.92], [0.5, 0.87, 0.6, 0.8]], device="cuda")
    step = torch.tensor([1], device="cuda", dtype=torch.int32)
    torch.cuda.synchronize()
    assert torch.equal(xin[:b, :, :4], x0.half()) and torch.equal(xin[b:, :, :4], x0.half())
    assert float(xin[..., 4:].abs().max()) == 0.0
    ops.cfg_ddim_step(eps, x, xin, 7.0, coef, step)
    torch.cuda.synchronize()
    ec, eu = eps[:b, :, :4].float(), eps[b:, :, :4].float()
    e = eu + 7.0 * (ec - eu)
    pred_x0 = (x0 - 0.87 * e) / 0.5
    ref = 0.6 * pred_x0 + 0.8 * e
    assert torch.allclose(x, ref, atol=1e-4, rtol=1e-5)
    assert int(step.item()) == 2
    assert torch.equal(xin[b:, :, :4], x.half())


def test_cfg_euler_a_step(ops):
    g = _gen(36)
    b, hw = 2, 1024
    x = torch.randn((b, hw, 4), generator=g, device="cuda") * 10
    x0 = x.clone()
    noise = torch.randn((3, b, hw, 4), generator=g, device="cuda")
    xin = torch.zeros((2 * b, hw, 64), device="cuda", dtype=torch.float16)
    eps = torch.zeros((2 * b, hw, 32), device="cuda", dtype=torch.float16)
    eps[..., :4] = _rand((2 * b, hw, 4), g)
    coef = torch.tensor([[14.6, 9.0, 5.0, 0.1], [10.3, 7.0, 3.0, 0.12], [7.0, 5.0, 2.0, 0.2]], device="cuda")
    step = torch.tensor([1], device="cuda", dtype=torch.int32)
    ops.cfg_euler_a_step(eps, x, noise, xin, 5.0, coef, step)
    torch.cuda.synchronize()
    ec, eu = eps[:b, :, :4].float(), eps[b:, :, :4].float()
    e = eu + 5.0 * (ec - eu)
    ref = x0 + e * (7.0 - 10.3) + noise[1] * 3.0
    assert torch.allclose(x, ref, atol=1e-4, rtol=1e-5)
    assert torch.allclose(xin[:b, :, :4].float(), ref * 0.12, atol=2e-2, rtol=2e-3)


def test_quantize_u8(ops):
    g = _gen(37)
    img = torch.zeros((2, 1000, 32), device="cuda", dtype=torch.float16)
    img[..., :3] = _rand((2, 1000, 3), g, 0.8)
    out = torch.empty((2, 1000, 3), device="cuda", dtype=torch.uint8)
    ops.quantize_u8(img, out)
    torch.cuda.synchronize()
    ref = (255.0 * ((img[..., :3].float() + 1.0) * 0.5).clamp(0, 1)).to(torch.uint8)
    assert torch.equal(out, ref)



def test_blend_latent(ops):
    """inpainting blend: x = x * latmask + init * (1 - latmask), mask shared by channels and images, in place"""
    g = _gen(5)
    b, hw = 3, 1000
    x = torch.randn((b, hw, 4), generator=g, device="cuda")
    init = torch.randn((b, hw, 4), generator=g, device="cuda")
    m = (torch.rand((hw,), generator=g, device="cuda") > 0.5).float()
    m[::7] = 0.25
    ref = x * m[None, :, None] + init * (1 - m[None, :, None])
    ops.blend_latent(x, init, m)
    torch.cuda.synchronize()
    assert torch.allclose(x, ref, rtol=0, atol=1e-6)
    keep = (m == 0)[None, :, None].expand_as(x)
    assert torch.equal(x[keep], init[keep])


def test_resize_latent_bilinear(ops):
    """F.interpolate(mode="bilinear", antialias=False) on NHWC fp32 latents, integer and fractional scales"""
    g = _gen(77)
    for (b, h, w, ho, wo) in [(2, 8, 8, 16, 16), (3, 16, 12, 24, 18), (1, 64, 64, 96, 128)]:
        x = torch.randn((b, h * w, 4), generator=g, device="cuda")
        y = torch.empty((b, ho * wo, 4), device="cuda")
        ops.resize_latent_bilinear(x, y, h, w, ho, wo)
        ref = F.interpolate(x.reshape(b, h, w, 4).permute(0, 3, 1, 2), size=(ho, wo), mode="bilinear", antialias=False)
        assert torch.allclose(y.reshape(b, ho, wo, 4).permute(0, 3, 1, 2), ref, atol=1e-5, rtol=1e-5)


def test_cfg_eps_and_latent_lincomb(ops):
    """the two generic sampler kernels (b200sd_cfg_eps, b200sd_latent_lincomb): CFG combine, a device-selected coefficient
    row, an indexed noise stack, in-place destination, zero weights that must not read a NaN buffer, the packed UNet input"""
    g = _gen(91)
    b, hw, pitch = 3, 257, 32
    eps = _rand((2 * b, hw, pitch), g)
    e = torch.empty((b, hw, 4), device="cuda")
    ops.cfg_eps(eps, e, 6.5)
    ec, eu = eps[:b, :, :4].float(), eps[b:, :, :4].float()
    assert torch.allclose(e, eu + 6.5 * (ec - eu), atol=1e-6, rtol=1e-6)
    x = torch.randn((b, hw, 4), generator=g, device="cuda")
    h = torch.full((b, hw, 4), float("nan"), device="cuda")
    noise = torch.randn((5, b, hw, 4), generator=g, device="cuda")
    coef = torch.zeros((4, 32), device="cuda")
    coef[2, 3:8] = torch.tensor([0.5, -1.25, 0.0, 2.0, 0.75])    # x, e, h (weight 0), noise, pack scale
    coef[2, 31] = 3.0                                              # noise row
    step = torch.tensor([2], device="cuda", dtype=torch.int32)
    xin = torch.zeros((2 * b, hw, 64), device="cuda", dtype=torch.float16)
    want = 0.5 * x - 1.25 * e + 2.0 * noise[3]
    ops.latent_lincomb(x, [x, e, h, noise], coef, 3, step, xin, idx_col=31)
    assert torch.allclose(x, want, atol=1e-6, rtol=1e-6) and not torch.isnan(x).any()
    assert torch.equal(xin[:b, :, :4], (want * 0.75).half()) and torch.equal(xin[b:, :, :4], (want * 0.75).half())
    assert float(xin[..., 4:].abs().max()) == 0.0
    ops.bump_step(step)
    assert int(step.item()) == 3
    u = torch.empty_like(x)
    coef[3, 0:2] = torch.tensor([1.0, 1.0])
    ops.latent_lincomb(u, [x, e], coef, 0, step)
    assert torch.allclose(u, x + e, atol=1e-6, rtol=1e-6)


@pytest.mark.parametrize("b,heads,sq,skv,d,d_pad", [(2, 8, 4096, 4096, 40, 48), (2, 8, 1024, 1024, 80, 96), (2, 8, 256, 256, 160, 176),
                                                    (3, 8, 1024, 77, 40, 48), (2, 8, 300, 200, 80, 96), (2, 2, 256, 256, 32, 48),
                                                    (1, 8, 64, 64, 160, 176)])
def test_attention_narrow_head_pitch(ops, b, heads, sq, skv, d, d_pad):
    """round 2: heads sit d_pad = round16(d + 1) columns apart (40 -> 48, 80 -> 96, 160 -> 176) inside ONE fused q|k|v
    buffer, so a head's 64-column TMA boxes overlap the next head's data (and, for v's last head, run off the buffer's
    row): those columns must never reach a result.  The ones column of V delivers the softmax denominators."""
    g = _gen(sq * 3 + skv + d_pad)
    w = heads * d_pad
    if sq == skv:
        buf = torch.zeros((b, sq, 3 * w), device="cuda", dtype=torch.float16)
        q, k, v = buf[..., :w], buf[..., w:2 * w], buf[..., 2 * w:]
    else:
        bq = torch.zeros((b, sq, w), device="cuda", dtype=torch.float16)
        bkv = torch.zeros((b, skv, 2 * w), device="cuda", dtype=torch.float16)
        q, k, v = bq, bkv[..., :w], bkv[..., w:]
    for t in (q, k, v):
        t.reshape(t.shape[0], t.shape[1], heads, d_pad)[..., :d] = _rand((t.shape[0], t.shape[1], heads, d), g)
    v.reshape(b, skv, heads, d_pad)[..., d] = 1.0
    out = torch.full((b, sq, heads * d), float("nan"), device="cuda", dtype=torch.float16)
    scale = d ** -0.5
    ops.attention(q, k, v, out, heads, d, d_pad, scale, True)
    torch.cuda.synchronize()
    ref = _attn_ref(q.contiguous(), k.contiguous(), v.contiguous(), heads, d, d_pad, scale)
    assert_close(f"attention narrow pitch d{d}/{d_pad} sq{sq} skv{skv}", out, ref, atol=4e-3, rtol=1e-2)
