"""Attention kernel schedule: 128-key tiles (heads of one 64-column chunk), the K / V ring at every slot and parity,
a math warpgroup with no valid Q rows, and varlen rows bitwise equal to plain calls, in fp16 and bf16 at 1, 2 and 3
chunks.  References are fp32 PyTorch on the unpadded heads."""
import pytest
import torch

from kutil import assert_close

pytestmark = pytest.mark.gpu

TOL = {torch.float16: 4e-3, torch.bfloat16: 1.6e-2}


@pytest.fixture(scope="module")
def ops():
    from b200sd import ops as _ops
    return _ops


def _heads(b, s, heads, d, d_pad, seed, dtype):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    t = torch.zeros((b, s, heads, d_pad), device="cuda", dtype=dtype)
    t[..., :d] = torch.randn((b, s, heads, d), generator=g, device="cuda").to(dtype)
    return t.reshape(b, s, heads * d_pad)


def _ref(q, k, v, heads, d, d_pad, scale):
    b, sq, _ = q.shape
    skv = k.shape[1]
    qh, kh, vh = (x.float().reshape(b, x.shape[1], heads, d_pad)[..., :d].permute(0, 2, 1, 3) for x in (q, k, v))
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    return (p @ vh).permute(0, 2, 1, 3).reshape(b, sq, heads * d)


def _run(ops, b, heads, sq, skv, d, dtype, seed, kv_len=None):
    d_pad = (d + 15) // 16 * 16
    q = _heads(b, sq, heads, d, d_pad, seed, dtype)
    k = _heads(b, skv, heads, d, d_pad, seed + 1, dtype)
    v = _heads(b, skv, heads, d, d_pad, seed + 2, dtype)
    out = torch.empty((b, sq, heads * d), device="cuda", dtype=dtype)
    ops.attention(q, k, v, out, heads, d, d_pad, d ** -0.5, kv_len=kv_len)
    torch.cuda.synchronize()
    return q, k, v, out, d_pad


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("skv", [1, 63, 64, 65, 127, 128, 129, 255, 257, 385, 640, 896, 4096])
def test_kv128_tile_lengths(ops, skv, dtype):
    """d = 40 and 64 (one chunk, 128-key tiles): ragged and whole last tiles, and 5 / 7 / 32 tiles, which wrap the
    three-slot ring through every slot at both parities"""
    for d in (40, 64):
        q, k, v, out, d_pad = _run(ops, 2, 2, 200, skv, d, dtype, skv + d)
        assert_close(f"attention d{d} skv{skv}", out, _ref(q, k, v, 2, d, d_pad, d ** -0.5), atol=TOL[dtype], rtol=1e-2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("d", [40, 80, 160])
@pytest.mark.parametrize("sq", [64, 65, 200, 1000])
def test_q_rows_and_chunks(ops, sq, d, dtype):
    """Sq = 64 leaves warpgroup 1 of the only Q tile without a valid row, 65 / 200 / 1000 leave partial tiles: the
    empty warpgroup keeps taking its turns and stores nothing"""
    for skv in (77, 300):
        q, k, v, out, d_pad = _run(ops, 2, 3, sq, skv, d, dtype, sq + d + skv)
        assert_close(f"attention sq{sq} d{d} skv{skv}", out, _ref(q, k, v, 3, d, d_pad, d ** -0.5), atol=TOL[dtype],
                     rtol=1e-2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("d", [40, 64, 80, 160])
def test_varlen_rows_equal_plain_calls(ops, d, dtype):
    """rows of one varlen call (buffer of 400 keys, finite data past each row's length) equal plain calls on their
    own key counts, bit for bit: 1, 77, 128, 129, 231, 256, 400 keys"""
    lens = [1, 77, 128, 129, 231, 256, 400]
    b, heads, sq, skv = len(lens), 2, 130, 400
    kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    q, k, v, out, d_pad = _run(ops, b, heads, sq, skv, d, dtype, d, kv_len=kv_len)
    for i, n in enumerate(lens):
        one = torch.empty((1, sq, heads * d), device="cuda", dtype=dtype)
        ops.attention(q[i:i + 1], k[i, :n].clone().unsqueeze(0), v[i, :n].clone().unsqueeze(0), one, heads, d, d_pad,
                      d ** -0.5)
        torch.cuda.synchronize()
        assert torch.equal(out[i:i + 1], one), f"varlen row {i} (kv_len {n}) differs from the plain call"
