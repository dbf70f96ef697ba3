"""Attention heads of one 64-column chunk (SD1.5 d = 40, SDXL d = 64) run 192-row Q tiles on three math warpgroups:
Q lengths around the 64-row warpgroup and 192-row tile edges (one, two or three warpgroups with valid rows in the last
tile), key counts that end inside a 128-key tile, on one and that wrap the four-slot K / V ring, and varlen rows bitwise
equal to plain calls.  References are fp32 PyTorch on the unpadded heads."""
import pytest
import torch

from kutil import assert_close

pytestmark = pytest.mark.gpu

TOL = {torch.float16: 4e-3, torch.bfloat16: 1.6e-2}
SQ = [1, 63, 64, 65, 128, 129, 191, 192, 193, 383, 385, 4096]
SKV = [77, 128, 129, 640, 4096]


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


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("sq", SQ)
def test_q_tile_edges(ops, sq, dtype):
    heads = 2
    for d in (40, 64):
        d_pad = (d + 15) // 16 * 16
        for skv in SKV:
            seed = sq * 7 + skv + d
            q = _heads(1, sq, heads, d, d_pad, seed, dtype)
            k = _heads(1, skv, heads, d, d_pad, seed + 1, dtype)
            v = _heads(1, skv, heads, d, d_pad, seed + 2, dtype)
            out = torch.empty((1, sq, heads * d), device="cuda", dtype=dtype)
            ops.attention(q, k, v, out, heads, d, d_pad, d ** -0.5)
            torch.cuda.synchronize()
            assert_close(f"attention sq{sq} d{d} skv{skv}", out, _ref(q, k, v, heads, d, d_pad, d ** -0.5),
                         atol=TOL[dtype], rtol=1e-2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("d", [40, 64])
def test_varlen_rows_equal_plain_calls(ops, d, dtype):
    """one varlen call per Q length over a 4096-key buffer; row i attends to SKV[i] keys"""
    heads, skv = 2, max(SKV)
    d_pad = (d + 15) // 16 * 16
    kv_len = torch.tensor(SKV, dtype=torch.int32, device="cuda")
    k = _heads(len(SKV), skv, heads, d, d_pad, d + 1, dtype)
    v = _heads(len(SKV), skv, heads, d, d_pad, d + 2, dtype)
    for sq in SQ:
        q = _heads(len(SKV), sq, heads, d, d_pad, d + sq, dtype)
        out = torch.empty((len(SKV), sq, heads * d), device="cuda", dtype=dtype)
        ops.attention(q, k, v, out, heads, d, d_pad, d ** -0.5, kv_len=kv_len)
        for i, n in enumerate(SKV):
            one = torch.empty((1, sq, heads * d), device="cuda", dtype=dtype)
            ops.attention(q[i:i + 1], k[i, :n].clone().unsqueeze(0), v[i, :n].clone().unsqueeze(0), one, heads, d,
                          d_pad, d ** -0.5)
            torch.cuda.synchronize()
            assert torch.equal(out[i:i + 1], one), f"sq {sq}: varlen row {i} (kv_len {n}) differs from the plain call"
