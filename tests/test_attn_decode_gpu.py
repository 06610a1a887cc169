"""lmod_attn_decode (split-KV single-query attention over the KV cache) element by element against float64 attention, and lmod_kv_append
bit for bit.

Cache rows at or past len[b] are NaN in every case: unwritten rows hold whatever the allocator left there, and a kernel that multiplied
them by a zero probability would return NaN.  Planted "needle" keys with scaled scores of +16 to +24 at the first, last and split-edge
positions make an off-by-one in len, a lost split or the wrong KV head move the output by O(1)."""
import json
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from llavamod import kernels as K  # noqa: E402
from tests.decode_exact import decode_reference_fp64  # noqa: E402,F401  (the float64 attention with the kernel's bound)

BK = 64                          # keys per ring stage (csrc/decode.cu)
NST = {64: 4, 128: 3}            # ring stages per head width
REPORT = {}


def split_keys(max_len, nkv):
    """Keys per split, as decode_splits in csrc/decode.cu computes it."""
    blocks = -(-max_len // BK)
    ns = -(-2 * torch.cuda.get_device_properties(0).multi_processor_count // nkv)
    ns = max(1, min(ns, -(-blocks // 4)))
    return -(-blocks // ns) * BK


def make_cache(B, nh, nkv, hd, lens, max_len, seed, needles=()):
    """q [B, nh*hd], k / v [B, nkv, max_len, hp] bf16 with NaN rows from lens[b] on; needles: (b, pos, scaled score) planted for the
    first query head of every KV group."""
    hp = K.attn_head_dim(hd)
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, nh * hd, device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn(B, nkv, max_len, hp, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(B, nkv, max_len, hp, device="cuda", generator=g).to(torch.bfloat16)
    k[..., hd:] = 0
    v[..., hd:] = 0
    G = nh // nkv
    scale = hd ** -0.5
    for b, pos, score in needles:
        for j in range(nkv):
            qh = q[b, (j * G) * hd:(j * G + 1) * hd].double()
            k[b, j, pos, :hd] = (qh * (score / scale) / qh.dot(qh)).to(torch.bfloat16)
            v[b, j, pos, :hd] = 4.0
    for b in range(B):
        k[b, :, lens[b]:] = float("nan")
        v[b, :, lens[b]:] = float("nan")
    return q, k, v


def run_decode(q, k, v, lens, nh, nkv, hd):
    B, max_len = q.shape[0], k.shape[2]
    ws = torch.empty(K.attn_decode_ws_elems(B, nh, nkv, hd, max_len), dtype=torch.float32, device="cuda")
    lt = torch.tensor(lens, dtype=torch.int32, device="cuda")
    return K.attn_decode(q, nh, nkv, hd, k, v, lt, ws, need_lse=True)


def check(name, q, k, v, lens, nh, nkv, hd):
    out, lse = run_decode(q, k, v, lens, nh, nkv, hd)
    B = q.shape[0]
    ref, ref_lse, tol, tol_lse = decode_reference_fp64(q, k, v, lens, nh, nkv, hd, hd ** -0.5)
    o = out.double().view(B, nh, hd)
    assert torch.isfinite(o).all(), name
    r_out = ((o - ref).abs() / tol).max().item()
    r_lse = ((lse.double() - ref_lse).abs() / tol_lse).max().item()
    REPORT[name] = dict(out=round(r_out, 4), lse=round(r_lse, 4))
    assert r_out <= 1.0, (name, r_out)
    assert r_lse <= 1.0, (name, r_lse)
    return out, lse


CASES = [   # hd, nh, nkv
    (64, 4, 4), (128, 4, 2), (64, 12, 2), (128, 14, 2), (128, 16, 2), (32, 4, 2), (80, 7, 1),
    (64, 6, 2), (64, 8, 2), (64, 10, 2), (128, 2, 2), (128, 6, 2), (128, 8, 2), (128, 10, 2), (128, 12, 2), (128, 32, 32),
]


@pytest.mark.parametrize("hd,nh,nkv", CASES)
def test_decode_matches_fp64_at_split_and_ring_edges(hd, nh, nkv):
    max_len = 4096
    sk = split_keys(max_len, nkv)
    ring = NST[K.attn_head_dim(hd)] * BK
    lens = sorted({1, 2, BK - 1, BK, BK + 1, ring - 1, ring, ring + 1, sk - 1, sk, sk + 1, 2 * sk - 1, 2 * sk + 1, 4095, 4096} & set(range(1, max_len + 1)))
    B = len(lens)
    needles = []
    for b, n in enumerate(lens):          # first, last and (when inside the range) split-edge positions
        needles.append((b, n - 1, 24.0))
        if n > 2:
            needles.append((b, 0, 16.0))
        if n > sk + 1:
            needles.append((b, sk - 1, 20.0))
            needles.append((b, sk, 20.0))
    q, k, v = make_cache(B, nh, nkv, hd, lens, max_len, seed=hd * 100 + nh, needles=needles)
    name = "hd%d_g%d" % (hd, nh // nkv) + ("_nkv%d" % nkv if nkv > 4 else "")
    out, lse = check(name, q, k, v, lens, nh, nkv, hd)
    # no needles: the plain softmax average
    q2, k2, v2 = make_cache(B, nh, nkv, hd, lens, max_len, seed=hd * 100 + nh + 1)
    check(name + "_plain", q2, k2, v2, lens, nh, nkv, hd)
    # every sequence alone gives the same bits as inside the unequal-length batch; a second launch gives the same bytes
    for b in range(B):
        o1, l1 = run_decode(q[b:b + 1].contiguous(), k[b:b + 1].contiguous(), v[b:b + 1].contiguous(), lens[b:b + 1], nh, nkv, hd)
        assert torch.equal(o1[0], out[b]) and torch.equal(l1[0], lse[b]), (b, lens[b])
    out2, lse2 = run_decode(q, k, v, lens, nh, nkv, hd)
    assert torch.equal(out, out2) and torch.equal(lse, lse2)


def test_decode_long_context():
    for hd, nh, nkv in [(128, 28, 4), (64, 14, 2)]:
        lens = [32768, 32767, 16385]
        q, k, v = make_cache(len(lens), nh, nkv, hd, lens, 32768, seed=7, needles=[(0, 32767, 20.0), (1, 0, 20.0)])
        check("long_hd%d_g%d" % (hd, nh // nkv), q, k, v, lens, nh, nkv, hd)


@pytest.mark.parametrize("hd,nh,nkv", [(64, 4, 2), (128, 7, 1)])
def test_decode_agrees_with_flash_forward_row(hd, nh, nkv):
    """The last row of lmod_attn_fwd (causal) over T tokens equals decode over the same K / V appended to a cache, within both bounds."""
    T = 777
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = torch.randn(T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
    fwd, fwd_lse = K.attention_fwd(qkv, 1, T, nh, nkv, hd, True, need_lse=True)
    kc = torch.full((1, nkv, 1024, hd), float("nan"), dtype=torch.bfloat16, device="cuda")
    vc = kc.clone()
    K.kv_append(qkv, 1, T, nh, nkv, hd, kc, vc, torch.zeros(1, dtype=torch.int32, device="cuda"))
    out, lse = check("vs_fwd_hd%d" % hd, qkv[T - 1:].contiguous(), kc, vc, [T], nh, nkv, hd)
    ref, _, tol, _ = decode_reference_fp64(qkv[T - 1:].contiguous(), kc, vc, [T], nh, nkv, hd, hd ** -0.5)
    diff = (out.double().view(nh, hd) - fwd[T - 1].double().view(nh, hd)).abs()
    assert (diff <= 2 * tol[0] + 2.0 ** -8 * ref[0].abs()).all()
    assert ((lse[0].double() - fwd_lse[0, :, T - 1].double()).abs() < 1e-3).all()


@pytest.mark.parametrize("hd", [64, 128, 32])
def test_kv_append_is_bit_exact_and_touches_nothing_else(hd):
    B, nh, nkv, max_len = 3, 6, 2, 300
    hp = K.attn_head_dim(hd)
    sentinel = -777.0
    kc = torch.full((B, nkv, max_len, hp), sentinel, dtype=torch.bfloat16, device="cuda")
    vc = kc.clone()
    want_k, want_v = kc.clone(), vc.clone()
    g = torch.Generator(device="cuda").manual_seed(hd)
    for n_new, offs in [(37, [0, 0, 0]), (1, [37, 37, 37]), (5, [0, 100, 295]), (1, [299, 7, 250])]:
        qkv = torch.randn(B * n_new, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
        K.kv_append(qkv, B, n_new, nh, nkv, hd, kc, vc, torch.tensor(offs, dtype=torch.int32, device="cuda"))
        x = qkv.view(B, n_new, nh + 2 * nkv, hd)
        for b in range(B):
            want_k[b, :, offs[b]:offs[b] + n_new, :hd] = x[b, :, nh:nh + nkv].transpose(0, 1)
            want_v[b, :, offs[b]:offs[b] + n_new, :hd] = x[b, :, nh + nkv:].transpose(0, 1)
            if hp != hd:
                want_k[b, :, offs[b]:offs[b] + n_new, hd:] = 0
                want_v[b, :, offs[b]:offs[b] + n_new, hd:] = 0
        assert torch.equal(kc.view(torch.int16), want_k.view(torch.int16))
        assert torch.equal(vc.view(torch.int16), want_v.view(torch.int16))


def teardown_module(module):
    out = os.environ.get("LLAVAMOD_TEST_REPORT")
    if out and REPORT:
        with open(out, "a") as f:
            f.write(json.dumps({"attn_decode_err_over_bound": REPORT}) + "\n")
    print("attn_decode err/bound:", json.dumps(REPORT))
