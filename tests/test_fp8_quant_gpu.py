"""lmod_quant_rows_e4m3 and lmod_rmsnorm_quant_e4m3 (csrc/quant.cu) against the CPU restatement of the quantiser, bit for bit: every
scale and every byte, except that a NaN byte (0x7F or 0xFF) only has to be a NaN byte and a NaN scale a NaN."""
import pytest
import torch

from tests import fp8_oracle as O

pytestmark = pytest.mark.gpu


def _rows(M, K, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, K, generator=g) * torch.rand(M, 1, generator=g) * 4).to(torch.bfloat16)
    if M > 2:
        x[1] = 0                                            # a zero row: scale 1, zero bytes
        x[2] = -0.3                                         # one repeated value: every byte is -448's
    if M > 4:
        x[3] = torch.where(torch.arange(K) % 2 == 0, 2.0 ** -133, -(2.0 ** -132)).to(torch.bfloat16)     # subnormal amax
        x[4, ::3] = 0
    return x


def _check(got, x_cpu):
    q, s = O.quant_rows(x_cpu)
    gq, gs = got.q.cpu(), got.scale.cpu()
    assert torch.equal(gs.isnan(), s.isnan()), "NaN scales at rows %s, the oracle at %s" % (torch.nonzero(gs.isnan()).flatten().tolist(),
                                                                                           torch.nonzero(s.isnan()).flatten().tolist())
    fin = ~s.isnan()
    assert torch.equal(gs[fin].view(torch.int32), s[fin].view(torch.int32)), "scales differ in bits"
    nan = O.is_nan_byte(q)
    bad = (O.is_nan_byte(gq) != nan) | ((gq != q) & ~nan)
    assert not bad.any(), "%d bytes differ; first at %s: got 0x%02x want 0x%02x" % (
        int(bad.sum()), torch.nonzero(bad)[0].tolist(), gq[bad][0].item(), q[bad][0].item())


@pytest.mark.parametrize("M", [1, 7, 2048])
@pytest.mark.parametrize("K", [896, 1024, 4096, 11008])
def test_quant_rows_bits(M, K):
    from llavamod import kernels as Kk
    x = _rows(M, K, M + K)
    _check(Kk.quant_rows(x.cuda()), x)


def test_quant_rows_strided_input():
    from llavamod import kernels as Kk
    x = _rows(33, 1024 + 64, 5)
    got = Kk.quant_rows(x.cuda()[:, 32:32 + 1024])          # ld = 1088, a 16-byte aligned column offset
    _check(got, x[:, 32:32 + 1024])


@pytest.mark.parametrize("H", [128, 896, 4096, 11008])
@pytest.mark.parametrize("with_res", [False, True])
def test_rmsnorm_quant_equals_quant_of_rmsnorm(H, with_res):
    from llavamod import kernels as Kk
    g = torch.Generator().manual_seed(H)
    rows = 77
    x = torch.randn(rows, H, generator=g).to(torch.bfloat16).cuda()
    res = torch.randn(rows, H, generator=g).to(torch.bfloat16).cuda() if with_res else None
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).cuda()
    x[5] = 0
    if with_res:
        res[5] = 0
    with torch.no_grad():
        y, stream = Kk.rmsnorm(x, w, 1e-6, res=res)
        got, stream_q = Kk.rmsnorm_quant(x, w, 1e-6, res=res)
    want = Kk.quant_rows(y)
    assert torch.equal(got.q, want.q) and torch.equal(got.scale.view(torch.int32), want.scale.view(torch.int32))
    assert torch.equal(stream_q, stream)                    # the updated residual stream is today's
    _check(got, y.cpu())


def test_quant_rows_rounds_every_bf16_value_up_to_448():
    """Every finite bf16 value v with |v| <= 448 (+-0, the bf16 subnormals, every e4m3 tie and subnormal), 255 to a row whose last element is
    448: the scale is exactly 1, so each byte must be torch's round-to-nearest-even conversion of v itself."""
    from llavamod import kernels as Kk
    pos = torch.arange(0, 0x43E1, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)     # +0 ... 448 = 0x43E0
    vals = torch.cat([pos, -pos])                                                               # -0 ... -448
    assert float(pos[-1]) == 448.0 and torch.signbit(vals[len(pos)]) and vals.numel() == 2 * 0x43E1
    rows = -(-vals.numel() // 255)
    flat = torch.zeros(rows * 255, dtype=torch.bfloat16)
    flat[:vals.numel()] = vals
    x = torch.cat([flat.view(rows, 255), torch.full((rows, 1), 448.0, dtype=torch.bfloat16)], dim=1)
    got = Kk.quant_rows(x.cuda())
    assert bool((got.scale == 1.0).all())
    want = x.float().to(torch.float8_e4m3fn).view(torch.uint8)
    bad = got.q.cpu() != want
    assert not bad.any(), "%d bytes differ; first for v = %r: got 0x%02x want 0x%02x" % (
        int(bad.sum()), x[bad][0].item(), got.q.cpu()[bad][0].item(), want[bad][0].item())
    _check(got, x)


def test_negative_underflow_and_negative_zero_give_0x80():
    from llavamod import kernels as Kk
    x = torch.zeros(4, 128, dtype=torch.bfloat16)
    x[0, 0] = 7.0                                           # scale 7 / 448 = 2^-6: x / scale = 64 x
    x[0, 1:40] = -(2.0 ** -17)                              # -> -2^-11: below half the smallest subnormal, -0
    x[0, 40:60] = -(2.0 ** -16)                             # -> -2^-10: a tie between -0 and -2^-9, even is -0
    x[0, 60:80] = -0.0
    x[1, 0] = 448.0                                         # scale 1
    x[1, 1:] = -(2.0 ** -12)
    x[2] = -0.0                                             # all -0: amax 0, scale 1, every byte -0
    x[3, ::2] = -(2.0 ** -133)                              # a subnormal amax with -0 beside it
    x[3, 1::2] = -0.0
    got = Kk.quant_rows(x.cuda())
    q = got.q.cpu()
    assert (q[0, 1:80] == 0x80).all() and (q[1, 1:] == 0x80).all() and (q[2] == 0x80).all() and (q[3, 1::2] == 0x80).all()
    assert q[3, 0].item() == 0xFE and got.scale[2].item() == 1.0
    _check(got, x)


def _non_finite_rows(M, K, seed):
    """Finite rows with a NaN row, a +inf row, a -inf row and a row holding NaN and both infinities among them."""
    x = _rows(M, K, seed)
    x[5, K // 3] = float("nan")
    x[9, K - 1] = float("inf")
    x[10, 0] = float("-inf")
    x[12, 7], x[12, K // 2], x[12, K - 9] = float("-inf"), float("nan"), float("inf")
    return x


@pytest.mark.parametrize("K", [128, 4096, 11008])
def test_quant_rows_non_finite_rows(K):
    from llavamod import kernels as Kk
    x = _non_finite_rows(16, K, K)
    got = Kk.quant_rows(x.cuda())
    _check(got, x)
    s, q = got.scale.cpu(), got.q.cpu()
    assert s[[5, 12]].isnan().all() and O.is_nan_byte(q[[5, 12]]).all()
    assert (s[[9, 10]] == float("inf")).all()
    assert O.is_nan_byte(q[9, K - 1]) and O.is_nan_byte(q[10, 0]) and int(O.is_nan_byte(q[[9, 10]]).sum()) == 2
    assert ((q[[9, 10]] & 0x7F) == 0).sum() == 2 * K - 2                                   # +-0 elsewhere
    fin = [i for i in range(16) if i not in (5, 9, 10, 12)]
    alone = Kk.quant_rows(x[fin].cuda())                                                   # the other rows do not notice
    assert torch.equal(alone.q.cpu(), q[fin]) and torch.equal(alone.scale.cpu().view(torch.int32), s[fin].view(torch.int32))


@pytest.mark.parametrize("H", [128, 4096])
@pytest.mark.parametrize("where", ["x", "res", "x_without_res"])
def test_rmsnorm_quant_non_finite_rows(H, where):
    """NaN / inf in the stream or in the residual: the row's normalised values are all NaN, so its scale and every byte are NaN."""
    from llavamod import kernels as Kk
    g = torch.Generator().manual_seed(H + len(where))
    rows = 16
    x = torch.randn(rows, H, generator=g).to(torch.bfloat16)
    res = torch.randn(rows, H, generator=g).to(torch.bfloat16) if where != "x_without_res" else None
    t = res if where == "res" else x
    t[3, H // 2] = float("nan")
    t[7, 0] = float("inf")
    t[8, H - 1] = float("-inf")
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).cuda()
    xc, rc = x.cuda(), (res.cuda() if res is not None else None)
    with torch.no_grad():
        y, stream = Kk.rmsnorm(xc, w, 1e-6, res=rc)
        got, stream_q = Kk.rmsnorm_quant(xc, w, 1e-6, res=rc)
    _check(got, y.cpu())
    assert torch.equal(stream_q.view(torch.int16), stream.view(torch.int16))
    bad_rows = [3, 7, 8]
    assert got.scale[bad_rows].isnan().all() and O.is_nan_byte(got.q[bad_rows]).all()
    fin = [i for i in range(rows) if i not in bad_rows]
    with torch.no_grad():
        alone, _ = Kk.rmsnorm_quant(xc[fin], w, 1e-6, res=rc[fin] if rc is not None else None)
    assert torch.equal(alone.q, got.q[fin]) and torch.equal(alone.scale.view(torch.int32), got.scale[fin].view(torch.int32))


def test_rmsnorm_quant_refuses_autograd():
    from llavamod import kernels as Kk
    x = torch.randn(4, 128, device="cuda").to(torch.bfloat16).requires_grad_()
    with pytest.raises(RuntimeError, match="forward-only"):
        Kk.rmsnorm_quant(x, torch.ones(128, device="cuda", dtype=torch.bfloat16), 1e-6)
