"""CPU restatement of the FP8 (e4m3) frozen teacher: the row-wise quantiser of csrc/quant.cu, the dequantised GEMM in float64, and a
fake-quantised dense decoder on top of oracle/restated.py.

The quantiser, in fp32, for one row x (the expression csrc/quant.cu states in its header):
    amax  = max_k |x[k]|, NaN-propagating (any NaN -> NaN; +-inf -> inf)
    scale = amax == 0 ? 1 : amax / 448          (NaN -> NaN, inf -> inf)
    q[k]  = e4m3_rn(clamp(x[k] / scale, +-448)), the clamp passing NaN through
(an fp32 division for the scale and one per element, the clamp after it, round to nearest even).  So a row holding a NaN gets scale NaN
and NaN bytes; a row holding an inf gets scale inf, NaN bytes at its infinite elements and +-0 elsewhere; every e4m3 GEMM output of
such a row is NaN.  torch's amax and clamp propagate NaN already.  e4m3 is torch.float8_e4m3fn (finite values up to 448, smallest
subnormal 2^-9, NaN encoded as 0x7F or 0xFF)."""
import contextlib
import re

import torch
import torch.nn.functional as F

E4M3_MAX = 448.0
DECODER_LINEAR = re.compile(r"\.layers\.\d+\.(self_attn\.(q|k|v|o)_proj|mlp\.(gate|up|down)_proj)\.weight$")


def quant_rows(x):
    """x [..., K] (bf16 or fp32 values) -> (q uint8 [..., K] holding the e4m3 bytes, scale fp32 [...])."""
    x = x.detach().to("cpu", torch.float32)
    amax = x.abs().amax(-1)
    scale = torch.where(amax == 0, torch.ones_like(amax), amax / torch.tensor(E4M3_MAX, dtype=torch.float32))
    q = (x / scale[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8), scale


def is_nan_byte(q):
    """The e4m3 NaN encodings, 0x7F and 0xFF (quantiser outputs are compared by NaN class there and bit for bit elsewhere)."""
    return (q & 0x7F) == 0x7F


def dequant(q, scale, dtype=torch.float64):
    """scale * e4m3(q), exactly, in float64 (or rounded once to `dtype`)."""
    return (q.view(torch.float8_e4m3fn).to(torch.float64) * scale.to(torch.float64)[..., None]).to(dtype)


def fake_quant(x):
    """x -> dequant(quant_rows(x)) in x's dtype: what an e4m3 GEMM sees of x."""
    q, s = quant_rows(x)
    return dequant(q, s, torch.float32).to(x.dtype)


def gemm_dequant_fp64(qa, sa, qw, sw, bias=None):
    """float64 product of the dequantised operands: D[m,n] = sum_k (sa[m] a[m,k]) (sw[n] w[n,k]) (+ bias[n])."""
    d = dequant(qa, sa) @ dequant(qw, sw).t()
    return d if bias is None else d + bias.to(torch.float64)


def fake_quant_state(sd):
    """A copy of a LLaVA-Qwen state dict whose decoder linears (q/k/v/o_proj, gate/up/down_proj of every layer) are fake-quantised per
    output channel.  Per-row scales make the fused q|k|v and gate|up buffers of the model equal to their separately quantised parts."""
    return {k: (fake_quant(v) if DECODER_LINEAR.search(k) else v) for k, v in sd.items()}


class _FakeQuantLinear:
    """torch.nn.functional for oracle/restated.py's attention / mlp bodies, with `linear` quantising the rows of its input first."""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def linear(x, w, b=None):
        return F.linear(fake_quant(x), w, b)


@contextlib.contextmanager
def fp8_decoder(R):
    """Inside, R.lm_forward (and everything built on it) runs the FP8 teacher's decoder: every linear of R.attention and R.mlp sees its
    input rows fake-quantised (q|k|v and gate|up share one quantised input, as in the model).  Feed it fake_quant_state weights.  The CLIP
    tower, the projector and lm_head are untouched."""
    attention, mlp = R.attention, R.mlp

    def with_fq(fn):
        def run(*a, **kw):
            R.F = _FakeQuantLinear()
            try:
                return fn(*a, **kw)
            finally:
                R.F = F
        return run

    R.attention, R.mlp = with_fq(attention), with_fq(mlp)
    try:
        yield
    finally:
        R.attention, R.mlp = attention, mlp
