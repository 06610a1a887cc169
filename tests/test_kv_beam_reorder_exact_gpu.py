"""lmod_kv_beam_reorder bit for bit against torch gathers on clones: every listed buffer's rows below rows[b] of beam j of prompt b take
beam parent[b*n + j]'s bytes in columns [0, hd); rows past rows[b], the padded head columns and buffers not listed keep their sentinel
bytes.  Maps: identity, swaps, 3-cycles, all from one beam, random maps with repeats; rows 0, 1, row-block edges +-1 and cap."""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

BEAM_CHUNK, BEAM_STAGE = 512, 32768          # csrc/decode.cu: rows per CTA and staged bytes, which set the row block R


def _row_block(n, hd):
    return max(1, min(BEAM_CHUNK, BEAM_STAGE // (n * hd * 2)))


def _maps(n, rng):
    maps = [list(range(n)), [0] * n, [n - 1] * n, [rng.randrange(n) for _ in range(n)], [rng.randrange(n) for _ in range(n)]]
    if n >= 2:
        maps.append([1, 0] + list(range(2, n)))                                        # a swap
        maps.append(list(range(n))[::-1])                                              # swaps of every pair
    if n >= 3:
        maps.append([1, 2, 0] + list(range(3, n)))                                     # a 3-cycle
        maps.append([(j + 1) % n for j in range(n)])                                   # an n-cycle
    return maps


def _rows(P, cap, n, hd, rng):
    R = _row_block(n, hd)
    edges = sorted({0, 1, R - 1, R, R + 1, 2 * R + 1, BEAM_CHUNK - 1, BEAM_CHUNK, BEAM_CHUNK + 1, cap - 1, cap})
    edges = [e for e in edges if 0 <= e <= cap]
    return [edges[(rng.randrange(len(edges)) + p) % len(edges)] for p in range(P)]


def _sentinel(shape, hd, g):
    """Random bytes with NaN / Inf patterns in the padded columns, so a write there is seen."""
    t = torch.randn(shape, generator=g).to(torch.bfloat16)
    t[..., hd:] = float("nan")
    return t.cuda()


def _expect(buf, n, hd, rows, parent):
    P = buf.shape[0] // n
    out = buf.clone()
    for b in range(P):
        r = rows[b]
        src = torch.tensor([b * n + p for p in parent[b * n:(b + 1) * n]], device=buf.device)
        out[b * n:(b + 1) * n, :, :r, :hd] = buf.index_select(0, src)[:, :, :r, :hd]
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8, 16])
@pytest.mark.parametrize("hd,hp,nkv", [(32, 64, 2), (64, 64, 3), (128, 128, 1), (128, 128, 4)])
def test_reorder_matches_gather(n, hd, hp, nkv):
    from llavamod import kernels as K
    rng = random.Random(n * 1000 + hd + nkv)
    g = torch.Generator().manual_seed(n * 7 + hd)
    P, cap = 3, 1100 if n <= 4 else 300
    bufs = [_sentinel((P * n, nkv, cap, hp), hd, g) for _ in range(5)]
    spare = _sentinel((P * n, nkv, cap, hp), hd, g)                       # not listed: must not change
    spare0 = spare.clone()
    for m in range(3):
        maps = _maps(n, rng)
        parent = sum((maps[(m + b) % len(maps)] for b in range(P)), [])
        rows = _rows(P, cap, n, hd, rng)
        want = [_expect(t, n, hd, rows, parent) for t in bufs]
        K.kv_beam_reorder(bufs, n, hd, rows, parent)
        torch.cuda.synchronize()
        for i, (t, w) in enumerate(zip(bufs, want)):
            assert torch.equal(t.view(torch.int16), w.view(torch.int16)), (i, rows, parent)
    assert torch.equal(spare.view(torch.int16), spare0.view(torch.int16))


def test_many_buffers_one_launch():
    """All K and V of a 24-layer model: 48 buffers in one launch (one more launch counted), identity prompts untouched."""
    from llavamod import kernels as K
    g = torch.Generator().manual_seed(3)
    n, P, hd = 4, 2, 64
    bufs = [_sentinel((P * n, 2, 200, hd), hd, g) for _ in range(48)]
    parent, rows = [0, 0, 1, 3] + [0, 1, 2, 3], [150, 200]
    want = [_expect(t, n, hd, rows, parent) for t in bufs]
    c0 = K._C.launch_count()
    K.kv_beam_reorder(bufs, n, hd, rows, parent)
    torch.cuda.synchronize()
    assert K._C.launch_count() == c0 + 1
    assert all(torch.equal(t.view(torch.int16), w.view(torch.int16)) for t, w in zip(bufs, want))


def test_single_beam_launches_nothing():
    from llavamod import kernels as K
    t = torch.randn(3, 2, 64, 64, device="cuda").to(torch.bfloat16)
    c0 = K._C.launch_count()
    K.kv_beam_reorder([t], 1, 64, [64, 64, 64], [0, 0, 0])
    assert K._C.launch_count() == c0


def test_bad_operands_are_refused():
    from llavamod import _C, kernels as K
    t = torch.zeros(6, 2, 64, 64, device="cuda", dtype=torch.bfloat16)
    bad = [
        dict(rows=[65, 0, 0]),                          # rows > cap
        dict(rows=[-1, 0, 0]),
        dict(parent=[0, 2, 0, 0, 0, 0]),                # parent outside [0, n)
        dict(parent=[0, -1, 0, 0, 0, 0]),
        dict(parent=[0, 0, 0]),                         # wrong count
        dict(rows=[1, 1]),
        dict(bufs=[t, t[:4].contiguous()]),             # shapes differ
        dict(bufs=[t.float()]),                         # dtype
        dict(bufs=[t.transpose(2, 3)]),                 # not contiguous
        dict(bufs=[t.cpu()]),                           # not on the GPU
        dict(bufs=[]),
        dict(hd=72),                                    # hd > hp
        dict(hd=20),                                    # not a multiple of 8
        dict(n=4),                                      # 6 rows are not prompts of 4 beams
    ]
    for kw in bad:
        args = dict(bufs=[t], n=2, hd=64, rows=[1, 1, 1], parent=[0, 0, 1, 1, 0, 1])
        args.update(kw)
        with pytest.raises(_C.LmodError):
            K.kv_beam_reorder(args["bufs"], args["n"], args["hd"], args["rows"], args["parent"])
