"""Flash-attention forward (csrc/attn.cu) and backward (csrc/attn_bwd.cu) element by element against the float64 reference of
tests/helpers.py, with the bounds derived there from the kernels' arithmetic.

Random inputs hide masking errors: one leaked or dropped key moves a row with n visible keys by about |v|/n.  So most cases also plant
"needles": half of the head-dim columns of q and k are zeroed, and a needle writes one of them into chosen query rows and one key, which
gives that key a scaled score of +16 to +24 for those rows only, and a distinctive v.  A leaked or dropped needle key moves its rows by
O(1).  Keys the rows must not see: the key just past the causal diagonal (at tile edges and past row 1024), padding keys, and the first
rows of the next sample, which the tail tile of a ragged sample loads.  Keys the rows must see: the first and last key of a key block, the
diagonal, key T-1 and key kv_lo of a left-padded sample."""
import math
import time

import pytest
import torch

from tests.helpers import attn_reference_fp64, attn_visible, check_attn, check_attn_grads

pytestmark = pytest.mark.gpu

REPORT = {}          # test name + output -> largest err / bound seen


@pytest.fixture(scope="module", autouse=True)
def _wall_time_and_memory():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print(f"\ntest_attn_exact_gpu on {torch.cuda.get_device_name()}: {time.time() - t0:.1f} s, "
          f"peak allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    for k in sorted(REPORT):
        print(f"  max err/bound {REPORT[k]:.3g}  {k}")


def _bkv(hd):
    return 128 if hd == 64 else 64          # keys per block of the forward kernel (the backward uses 128-key blocks, 64-query blocks)


class Needles:
    """Plants needles into an fp32 fused QKV buffer x [B*T, (nh + 2 nkv) hd] before it is rounded to bf16."""

    def __init__(self, x, B, T, nh, nkv, hd, scale):
        self.B, self.T, self.nh, self.group, self.hd, self.scale = B, T, nh, nh // nkv, hd, scale
        self.q = x[:, :nh * hd].view(B, T, nh, hd)
        self.k = x[:, nh * hd:(nh + nkv) * hd].view(B, T, nkv, hd)
        self.v = x[:, (nh + nkv) * hd:].view(B, T, nkv, hd)
        self.ncol = hd // 2
        self.q[..., :self.ncol] = 0
        self.k[..., :self.ncol] = 0
        self.used, self.n = set(), 0
        self.d = torch.arange(hd, device=x.device, dtype=torch.float32)

    def add(self, b, rows, key, score=24.0, kb=None):
        """Query rows `rows` of sample b (one head, taken in turn) get a scaled score of about `score` on key `key` of sample kb (b)."""
        kb = b if kb is None else kb
        h = self.n % self.nh
        self.n += 1
        hk = h // self.group
        c = next((c for c in range(self.ncol) if (b, hk, c) not in self.used and (kb, hk, c) not in self.used), None)
        assert c is not None, "out of needle columns"
        self.used |= {(b, hk, c), (kb, hk, c)}
        a = math.sqrt(score / self.scale)
        self.q[b, list(rows), h, c] = a
        self.k[kb, key, hk, c] = a
        self.v[kb, key, hk] = 3.0 * torch.cos(0.7 * (c + 1) * self.d + 0.3 * h)


FORBIDDEN_OFFSETS = (0, 1, 63, 64, 127, 128, 191, 255, 256, 999, 1023, 1024, 1535, 2047, 3071, 4094)


def plant_standard_needles(nd, ranges, causal, bkv):
    """ranges: [(kv_lo, kv_hi)] per sample."""
    T = nd.T
    for b, (lo, hi) in enumerate(ranges):
        if b + 1 < nd.B:                                           # the next sample's first rows, loaded by this sample's tail tile
            nd.add(b, range(max(0, T - 3), T), 0, kb=b + 1)
        if hi <= lo:                                               # all padding: every row sees every key, the future ones too
            nd.add(b, [0], T - 1, score=16.0)
            continue
        if causal:
            for r in sorted({lo + o for o in FORBIDDEN_OFFSETS} | {hi - 2}):
                if lo <= r and r + 1 < hi:
                    nd.add(b, [r], r + 1)                          # just past the diagonal
            if hi < T:                                             # right padding: no row at or after kv_lo sees it
                for key in sorted({hi, T - 1}):
                    nd.add(b, range(lo, T), key)
            if lo > 0:                                             # left padding: the un-masked rows in front see it, the others must not
                for key in sorted({0, lo - 1}):
                    nd.add(b, range(T), key)
            for key in sorted({lo, bkv - 1, bkv, 2 * bkv - 1, 2 * bkv, hi - 1}):
                if lo <= key < hi:                                 # the diagonal (the row maximum in the last visible key block) and a later row
                    nd.add(b, sorted({key, min(T - 1, key + bkv + 5)}), key, score=16.0)
        else:
            for key in sorted({0, bkv - 1, bkv, 2 * bkv - 1, T - 1}):
                if key < T:
                    nd.add(b, sorted({0, T // 2, T - 1}), key, score=16.0)


def ranges_of(B, T, lens=None, side=None):
    if lens is None:
        return [(0, T)] * B, None
    keep = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    ranges = []
    for b, n in enumerate(lens):
        lo = 0 if side == "right" or n == 0 else T - n
        keep[b, lo:lo + n] = True
        ranges.append((lo, lo + n) if n else (0, 0))
    return ranges, keep


def make_case(B, T, nh, nkv, hd, causal, seed, lens=None, side=None, needles=True, qk_mult=1.0, equal_keys=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g)
    dout = torch.randn(B * T, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    scale = hd ** -0.5
    x[:, :(nh + nkv) * hd] *= qk_mult
    if equal_keys:
        k = x[:, nh * hd:(nh + nkv) * hd].view(B, T, nkv, hd)
        k.copy_(k[:, :1].expand(B, T, nkv, hd).clone())
    ranges, keep = ranges_of(B, T, lens, side)
    if needles:
        plant_standard_needles(Needles(x, B, T, nh, nkv, hd, scale), ranges, causal, _bkv(hd))
    return x.to(torch.bfloat16), dout, keep, scale


def assert_single_key_rows_exact(out, qkv, B, T, nh, nkv, hd, causal, keep):
    """A row with exactly one visible key reproduces that key's v bit for bit (P = 1 in bf16, l = 1 +- 2^-23)."""
    vis = attn_visible(B, T, causal, keep, out.device)
    b, t = torch.nonzero(vis.sum(-1) == 1, as_tuple=True)
    if not len(b):
        return 0
    key = vis[b, t].to(torch.int8).argmax(-1)
    o = out.view(B, T, nh, hd)[b, t]                                               # [n, nh, hd]
    hk = torch.arange(nh, device=out.device) // (nh // nkv)
    v = qkv.view(B, T, nh + 2 * nkv, hd)[b, key][:, nh + nkv + hk]                 # [n, nh, hd]
    bad = (o.view(torch.int16) != v.view(torch.int16)).any(-1)
    assert not bad.any(), f"{int(bad.sum())} single-key (row, head) pairs differ from v; first at {torch.nonzero(bad)[0].tolist()}"
    return len(b)


def run_and_check(tag, qkv, dout, B, T, nh, nkv, hd, causal, scale, keep, bwd=True, repeat=False):
    from llavamod import kernels as K
    pad = K.pad_ranges(keep) if keep is not None else None
    out, lse = K.attention_fwd(qkv, B, T, nh, nkv, hd, causal, scale, need_lse=True, pad=pad)
    dqkv = K.attention_bwd(qkv, out, dout, lse, B, T, nh, nkv, hd, causal, scale, pad=pad) if bwd else None
    torch.cuda.synchronize()
    ref = attn_reference_fp64(qkv, B, T, nh, nkv, hd, causal, scale, keep=keep, dout=dout if bwd else None, out_kernel=out, lse_kernel=lse)
    check_attn(f"{tag} o", out, ref["o"], ref["o_tol"], T, hd, REPORT)
    check_attn(f"{tag} lse", lse, ref["lse"], ref["lse_tol"], T, report=REPORT)
    assert_single_key_rows_exact(out, qkv, B, T, nh, nkv, hd, causal, keep)
    if bwd:
        check_attn_grads(tag, dqkv, ref, T, nh, nkv, hd, REPORT)
    if repeat:                                                  # determinism: bytes of the forward, dK|dV of the backward
        out2, lse2 = K.attention_fwd(qkv, B, T, nh, nkv, hd, causal, scale, need_lse=True, pad=pad)
        assert torch.equal(out2, out) and torch.equal(lse2, lse)
        if bwd:
            d2 = K.attention_bwd(qkv, out, dout, lse, B, T, nh, nkv, hd, causal, scale, pad=pad)
            assert torch.equal(d2[:, nh * hd:], dqkv[:, nh * hd:])
    return out, lse, dqkv, ref, pad


TILE_T = (1, 2, 17, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 257, 577, 1000)


@pytest.mark.parametrize("T", TILE_T)
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("hd", [64, 128])
def test_attn_tile_edges(hd, causal, T):
    """T around every tile size (forward 128 query rows with 128 / 64 keys, backward 128 keys with 64 queries), three samples so that the
    ragged tail tiles load the next sample's rows; GQA group 2."""
    B, nh, nkv = 3, 2, 1
    qkv, dout, keep, scale = make_case(B, T, nh, nkv, hd, causal, seed=T * 4 + hd + causal)
    run_and_check("tile_edges", qkv, dout, B, T, nh, nkv, hd, causal, scale, keep)


MODEL_SHAPES = [  # name, B, T, nh, nkv, hd, causal, backward
    ("0.5B student", 2, 2048, 16, 16, 64, True, True),
    ("1.8B student", 1, 4096, 16, 16, 128, True, True),
    ("7B teacher", 1, 2048, 32, 32, 128, True, False),
    ("CLIP-L", 5, 577, 16, 16, 64, False, True),
    ("GQA 14/2", 2, 1100, 14, 2, 64, True, True),
    ("GQA 12/2", 2, 1100, 12, 2, 128, True, True),
    ("GQA 28/4", 1, 1100, 28, 4, 128, True, True),
    ("GQA 8/1", 2, 1100, 8, 1, 64, True, True),
]


@pytest.mark.parametrize("name,B,T,nh,nkv,hd,causal,bwd", MODEL_SHAPES, ids=[m[0].replace(" ", "_") for m in MODEL_SHAPES])
def test_attn_model_shapes(name, B, T, nh, nkv, hd, causal, bwd):
    """The shapes the models run, with needles past row 1024; two launches give identical bytes."""
    qkv, dout, keep, scale = make_case(B, T, nh, nkv, hd, causal, seed=T + nh + hd)
    run_and_check("model_shapes", qkv, dout, B, T, nh, nkv, hd, causal, scale, keep, bwd=bwd, repeat=True)


@pytest.mark.parametrize("kind,hd,causal", [("equal_keys", 64, True), ("equal_keys", 128, False), ("large_scores", 64, True),
                                            ("large_scores", 128, True), ("large_scores", 64, False)])
def test_attn_numeric_edges(kind, hd, causal):
    """All-equal keys (uniform attention: the longest accumulations) and scaled scores spanning about +-100 (peaked rows, P underflow,
    |lse| near 100)."""
    B, T, nh, nkv = 2, 1000, 4, 2
    if kind == "equal_keys":
        qkv, dout, keep, scale = make_case(B, T, nh, nkv, hd, causal, seed=hd, needles=False, equal_keys=True)
    else:
        qkv, dout, keep, scale = make_case(B, T, nh, nkv, hd, causal, seed=hd + 1, needles=False, qk_mult=math.sqrt(30.0))
        s = qkv[:T, :hd].float() @ qkv[:T, nh * hd:nh * hd + hd].float().T * scale
        assert s.abs().max() > 60, float(s.abs().max())
    run_and_check(kind, qkv, dout, B, T, nh, nkv, hd, causal, scale, keep)


PAD_CASES = [(64, "right", 4, 4, 193), (64, "left", 8, 2, 193), (128, "right", 6, 2, 257), (128, "left", 4, 1, 257),
             (128, "left", 12, 2, 600)]


@pytest.mark.parametrize("hd,side,nh,nkv,T", PAD_CASES)
def test_attn_padded_batch_samples_match_alone(hd, side, nh, nkv, T):
    """Eight samples of lengths 0, 1, tile edges +-1 and T, needles on the padding keys.  Every sample equals the same sample launched
    alone with its own key range: out, lse, dK and dV bit for bit, dQ within its bound (the red.add order over key blocks varies)."""
    from llavamod import kernels as K
    B = 8
    lens = [0, 1, 63, 64, 65, 127, 129, T]
    qkv, dout, keep, scale = make_case(B, T, nh, nkv, hd, True, seed=T + hd + nh, lens=lens, side=side)
    out, lse, dqkv, ref, (lo, hi) = run_and_check("padded", qkv, dout, B, T, nh, nkv, hd, True, scale, keep, repeat=True)
    for b in range(B):
        rows = slice(b * T, (b + 1) * T)
        pad_b = (lo[b:b + 1], hi[b:b + 1])
        o1, l1 = K.attention_fwd(qkv[rows], 1, T, nh, nkv, hd, True, scale, need_lse=True, pad=pad_b)
        d1 = K.attention_bwd(qkv[rows], o1, dout[rows], l1, 1, T, nh, nkv, hd, True, scale, pad=pad_b)
        assert torch.equal(o1, out[rows]) and torch.equal(l1, lse[b:b + 1]), b
        assert torch.equal(d1[:, nh * hd:], dqkv[rows, nh * hd:]), b
        qs = slice(0, nh * hd)
        check_attn("padded alone dq", d1[:, qs], ref["dqkv"][rows, qs], ref["dqkv_tol"][rows, qs], T, hd, REPORT)


@pytest.mark.parametrize("hd,causal,side", [(64, True, "left"), (128, True, "right"), (128, False, None)])
def test_attn_autograd_entry_point(hd, causal, side):
    """K.attention with requires_grad runs AttnFn (the student's path): output and dq|dk|dv element-wise, with and without a padded batch."""
    from llavamod import kernels as K
    B, T, nh, nkv = 3, 300, 4, 2
    lens = [T, 150, 1] if side else None
    qkv, dout, keep, scale = make_case(B, T, nh, nkv, hd, causal, seed=hd + 7, lens=lens, side=side)
    pad = K.pad_ranges(keep) if keep is not None else None
    x = qkv.clone().requires_grad_(True)
    out = K.attention(x, B, T, nh, nkv, hd, causal, pad=pad)
    assert out.grad_fn is not None and "AttnFn" in type(out.grad_fn).__name__
    out.backward(dout)
    ref = attn_reference_fp64(qkv, B, T, nh, nkv, hd, causal, scale, keep=keep, dout=dout, out_kernel=out.detach())
    check_attn("autograd o", out, ref["o"], ref["o_tol"], T, hd, REPORT)
    check_attn_grads("autograd", x.grad, ref, T, nh, nkv, hd, REPORT)


def test_attn_key_padding_without_causal_mask_is_rejected_on_device():
    from llavamod import _C, kernels as K
    B, T, nh, hd = 2, 64, 2, 64
    qkv = torch.randn(B * T, 3 * nh * hd, device="cuda").to(torch.bfloat16)
    pad = K.pad_ranges(torch.ones(B, T, dtype=torch.bool, device="cuda"))
    for fn in (lambda: K.attention(qkv, B, T, nh, nh, hd, causal=False, pad=pad),
               lambda: K.attention_fwd(qkv, B, T, nh, nh, hd, False, pad=pad)):
        with pytest.raises(_C.LmodError, match="causal"):
            fn()
    out = torch.empty(B * T, nh * hd, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(_C.LmodError, match="causal"):
        _C.call("lmod_attn_fwd", _C.ptr(qkv), qkv.stride(0), B, T, nh, nh, hd, 0, 0.125, _C.ptr(out), out.stride(0), None,
                _C.ptr(pad[0]), _C.ptr(pad[1]))
