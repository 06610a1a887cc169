"""lmod_quant_rows_e4m3 and lmod_rmsnorm_quant_e4m3 (csrc/quant.cu) against the CPU restatement of the quantiser, bit for bit."""
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
    assert torch.equal(got.scale.cpu().view(torch.int32), s.view(torch.int32)), "scales differ in bits"
    bad = got.q.cpu() != q
    assert not bad.any(), "%d bytes differ; first at %s" % (int(bad.sum()), torch.nonzero(bad)[0].tolist())


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


def test_rmsnorm_quant_refuses_autograd():
    from llavamod import kernels as Kk
    x = torch.randn(4, 128, device="cuda").to(torch.bfloat16).requires_grad_()
    with pytest.raises(RuntimeError, match="forward-only"):
        Kk.rmsnorm_quant(x, torch.ones(128, device="cuda", dtype=torch.bfloat16), 1e-6)
