"""Designs that make lmod_attn_decode and lmod_attn_decode_chunk (csrc/decode.cu) exact, their expected bytes, and the float64 attention
reference with the kernel's error bound.  Pure torch: nothing here imports the kernels, so the CPU tests can check the designs.

Exact design, per query row r and query head h (KV head j = h // G):
  * scale:  the kernel folds the softmax scale into scale_log2 = fp32(scale * LOG2E_F); SCALE[1] and SCALE[2] make that exactly 1 and 2,
    so a score s in the cache becomes the exponent mult * s of ex2 with no rounding.
  * q:      one-hot, 1 in column col[r, h] of head h and 0 elsewhere; the heads of one KV group get different columns.  Columns past
    nh * hd of the fused row are NaN (the kernel must not read them).
  * k:      k[b, j, t, c] is the score of key t for every head that reads column c.  Tier 1: scores in {0, -200}; ex2.approx.ftz gives 1 at
    0 and flushes 2^-200 to 0, so every probability, every running sum l and every rescale factor is exactly 0 or 1.  Tier 2: scores in
    {0, -1, -2, -3}; it also needs ex2.approx to be exact at those small negative integers.  Every weight is then 2^(e - m) with
    e - m >= -3 (-6 at mult 2) in whatever frame the kernel holds, so every partial sum is a multiple of 2^-6.
  * v:      integers in [-8, 8], different per key, column and head.  |sum p v| <= 8 len <= 2^18 at len 32768, in steps of at least 2^-6:
    every fp32 sum is exact, whatever order the kernel adds in.
  Expected: out = bf16(fp32(sum w v) / fp32(sum w)) with an IEEE fp32 divide (the build does not use fast math), bit for bit;
  lse = (M + log2 L) fp32(ln 2), within lse_tol (lg2.approx and three fp32 roundings).
Keys with score 0 sit at the first and last key of a 64-key block, of a ring pass and of a split, at each row's last visible key and at
random interior positions, each with probability 1/2 (1/4 at plain block edges) per column; one column in five has no 0 at all, so its
attention is uniform over every key (tier 1).  A lost, doubled or shifted key then changes an integer sum."""
import math

import numpy as np
import torch

BK = 64                          # keys per ring stage (csrc/decode.cu)
NST = {64: 4, 128: 3}            # ring stages per padded head width
MIN_BLOCKS = 4                   # DEC_MIN_BLOCKS
MAX_G = 8                        # DEC_MAX_G
LOG2E_F = np.float32(1.4426950408889634)
LN2_F = float(np.float32(math.log(2.0)))   # the kernel's LN2_F


def _scale_for(target):
    s = np.float32(target * math.log(2.0))
    for _ in range(8):           # the float32 nearest target ln 2, nudged until fp32(s * log2e) is exactly target
        p = np.float32(s * LOG2E_F)
        if p == target:
            return float(s)
        s = np.nextafter(s, np.float32(np.inf) if p < target else np.float32(-np.inf))
    raise AssertionError(target)


SCALE = {1: _scale_for(1.0), 2: _scale_for(2.0)}
assert np.float32(np.float32(SCALE[1]) * LOG2E_F) == 1.0 and np.float32(np.float32(SCALE[2]) * LOG2E_F) == 2.0, SCALE
assert SCALE[1] == 0.6931471824645996 and SCALE[2] == 1.3862943649291992


def head_dim_padded(hd):
    """attn_head_dim in llavamod/kernels.py: 64 / 128, smaller widths zero-padded."""
    return hd if hd in (64, 128) else (64 if hd < 64 else 128)


def decode_splits(max_len, nkv, sms):
    """(nsplit, blocks per split) as decode_splits in csrc/decode.cu computes them for a GPU with `sms` SMs."""
    blocks = -(-max_len // BK)
    ns = -(-2 * sms // nkv)
    ns = max(1, min(ns, -(-blocks // MIN_BLOCKS)))
    sb = -(-blocks // ns)
    return -(-blocks // sb), sb


def ring_regimes(hd, max_len, nkv, sms):
    """The ring and split regimes a launch at full length runs: the blocks per split against the ring's NST stages, one split, and a last
    split shorter than the others."""
    hp = head_dim_padded(hd)
    nst = NST[hp]
    ns, sb = decode_splits(max_len, nkv, sms)
    blocks = -(-max_len // BK)
    reg = set()
    if ns == 1:
        reg.add("one split")
    if sb < nst:
        reg.add("split below one ring pass")
    if sb == nst:
        reg.add("split = NST blocks")
    if sb == nst + 1:
        reg.add("split = NST + 1 blocks")
    if sb >= 2 * nst + 1:
        reg.add("split >= 2 NST + 1 blocks")
    if ns > 1 and blocks - (ns - 1) * sb < sb:
        reg.add("short last split")
    return {(hp, r) for r in reg}


def edge_positions(n, sk, ring):
    """Positions in [0, n) on either side of the split, ring-pass and (separately returned) 64-key block edges of a sequence of n keys."""
    strong = {0, n - 1}
    for s0 in range(0, n, sk):
        strong |= {s0 - 1, s0}
        for r0 in range(s0, min(n, s0 + sk), ring):
            strong |= {r0 - 1, r0}
    block = set()
    for b0 in range(0, n, BK):
        block |= {b0 - 1, b0}
    strong = {p for p in strong if 0 <= p < n}
    return strong, {p for p in block if 0 <= p < n} - strong


def edge_lengths(max_len, sk, ring):
    """Lengths on both sides of every block, ring-pass and split edge the sequence crosses (within the first two splits and the end)."""
    lens = {1, 2, BK - 1, BK, BK + 1, ring - 1, ring, ring + 1, 2 * ring + 1, sk - 1, sk, sk + 1, sk + ring - 1, sk + ring, sk + ring + 1,
            2 * sk - 1, 2 * sk, 2 * sk + 1, max_len - 1, max_len}
    return sorted(n for n in lens if 1 <= n <= max_len)


class Design:
    """One launch's operands.  q [R, ld] bf16 (R = B T rows, row b T + t), k / v [B, nkv, max_len, hp] bf16 with NaN rows from len[b] on,
    col [R, nh] the one-hot column of each query head, lims [R] the keys each row sees."""

    def __init__(self, B, T, nh, nkv, hd, lens, max_len, sk, seed, tier=1, mult=1, device="cpu"):
        assert tier in (1, 2) and mult in (1, 2) and nh % nkv == 0 and nh // nkv <= MAX_G
        self.B, self.T, self.nh, self.nkv, self.hd, self.lens, self.max_len = B, T, nh, nkv, hd, list(lens), max_len
        self.hp, self.G, self.tier, self.mult, self.sk = head_dim_padded(hd), nh // nkv, tier, mult, sk
        self.scale = SCALE[mult]
        ring = NST[self.hp] * BK
        dev = torch.device(device)
        g = torch.Generator(device=dev).manual_seed(seed)
        gc = torch.Generator().manual_seed(seed)
        f32 = torch.float32
        self.k = torch.zeros(B, nkv, max_len, self.hp, dtype=torch.bfloat16, device=dev)
        self.v = torch.zeros_like(self.k)
        for b in range(B):
            n = lens[b]
            assert T <= n <= max_len
            strong, block = edge_positions(n, sk, ring)
            strong |= {n - T + t for t in range(T)}                  # the last key each row of a chunk sees
            prob = torch.full((max_len,), min(0.5, 3.0 / n), dtype=f32)
            prob[sorted(block)] = 0.25
            prob[sorted(strong)] = 0.5
            prob = prob.to(dev)
            if tier == 1:
                s = torch.full((nkv, max_len, hd), -200.0, device=dev)
            else:
                s = -torch.randint(1, 4, (nkv, max_len, hd), generator=g, device=dev).to(f32)
            zero = torch.rand(nkv, max_len, hd, generator=g, device=dev) < prob[None, :, None]
            uniform = (torch.arange(nkv, device=dev)[:, None] + torch.arange(hd, device=dev)[None, :] + b) % 5 == 4
            zero &= ~uniform[:, None, :]
            s[zero] = 0.0
            self.k[b, :, :, :hd] = s.to(torch.bfloat16)
            self.v[b, :, :, :hd] = torch.randint(-8, 9, (nkv, max_len, hd), generator=g, device=dev).to(torch.bfloat16)
            self.k[b, :, n:] = float("nan")
            self.v[b, :, n:] = float("nan")
        R = B * T
        self.col = torch.empty(R, nh, dtype=torch.long)
        for r in range(R):
            for j in range(nkv):
                self.col[r, j * self.G:(j + 1) * self.G] = torch.randperm(hd, generator=gc)[:self.G]
        self.col = self.col.to(dev)
        self.ld = (nh + 2 * nkv) * hd                                # a row of the fused qkv buffer; the k and v columns are NaN here
        q = torch.full((R, self.ld), float("nan"), dtype=torch.bfloat16, device=dev)
        q[:, :nh * hd] = 0
        q.view(R, -1)[torch.arange(R, device=dev)[:, None], torch.arange(nh, device=dev)[None, :] * hd + self.col] = 1
        self.q = q
        self.lims = [lens[r // T] - T + r % T + 1 for r in range(R)]

    def expected(self, defect=None):
        """-> (out [R, nh*hd] bf16, lse [R, nh] float64, lse_tol [R, nh] float64).

        defect plants one kernel defect in the expectation (for the CPU check that the design sees it): ("drop", p) drops key p;
        ("score", p) gives key p the score of key p + 1; ("vrow", p) gives key p the V row of key p + 1; ("kvhead",) makes head h read KV
        head j + 1; ("split", i) loses split i (keys [i sk, (i + 1) sk))."""
        R, nh, G, hd = self.B * self.T, self.nh, self.G, self.hd
        dev = self.k.device
        out = torch.empty(R, nh * hd, dtype=torch.bfloat16, device=dev)
        lse = torch.empty(R, nh, dtype=torch.float64, device=dev)
        tol = torch.empty_like(lse)
        kind = defect[0] if defect else None
        for r in range(R):
            b, lim = r // self.T, self.lims[r]
            jh = torch.arange(nh, device=dev) // G
            if kind == "kvhead":
                jh = (jh + 1) % self.nkv
            pos = torch.arange(lim, device=dev)
            kk = self.k[b]
            vv = self.v[b, :, :lim, :hd].double()
            if kind == "kvhead":
                vv = vv.roll(-1, 0)
            s = kk[jh[:, None], pos[None, :], self.col[r][:, None]].double()        # [nh, lim]
            if kind == "score" and defect[1] + 1 < lim:
                s[:, defect[1]] = kk[jh, defect[1] + 1, self.col[r]].double()
            if kind == "vrow" and defect[1] + 1 < lim:
                vv = vv.clone()
                vv[:, defect[1]] = vv[:, defect[1] + 1]
            e = s * self.mult
            keep = torch.ones(lim, dtype=torch.bool, device=dev)
            if kind == "drop" and defect[1] < lim:
                keep[defect[1]] = False
            if kind == "split":
                keep[defect[1] * self.sk:(defect[1] + 1) * self.sk] = False
            e = torch.where(keep[None, :], e, torch.full_like(e, float("-inf")))
            M = e.amax(1, keepdim=True)
            w = torch.where(e - M > -126, torch.exp2(e - M), torch.zeros_like(e))      # ex2.approx.ftz: below 2^-126 is 0
            num = torch.bmm(w.view(self.nkv, G, lim), vv).view(nh, hd)
            den = w.sum(1)
            if defect is None:                                                         # every sum is exact in fp32
                assert bool((num.abs() <= 2.0 ** 21).all()) and bool(((num * 64).round() == num * 64).all())
            out[r] = (num.float() / den.float()[:, None]).to(torch.bfloat16).view(-1)
            lg = torch.log2(den)
            lse[r] = (M[:, 0] + lg) * LN2_F
            # lg2.approx.ftz: at most 2^-22 (1 + |log2 L|) absolute; M + lg2 L, LN2_F and the product: 2^-24 relative each
            tol[r] = LN2_F * 2.0 ** -22 * (1 + lg.abs()) + 3 * 2.0 ** -24 * (M[:, 0].abs() + lg.abs())
        return out, lse, tol


def decode_reference_fp64(q, k, v, lens, nh, nkv, hd, scale):
    """float64 attention of q [B, nh*hd] over cache rows [0, lens[b]) of k / v [B, nkv, max_len, hp], with the error bound of the kernel.

    Kernel arithmetic and its error, per (b, h):
      * score q.k: bf16 x bf16 products are exact in fp32; the fp32 sum of hd terms (fma chain over 8, then a shuffle tree) errs by at
        most hd * 2^-24 * sum|q_i k_i|; the multiply by scale*log2(e) and the subtraction of the running max add 2^-24 relative each;
      * p = ex2.approx(s - m): 2^-22 relative, plus the rescale factors 2^(m_old - m_new), applied once per block and once per split
        merge (another 2^-22 each, at most len/64 + 2 of them);
      * a relative error d on every weight p_t moves sum p_t v_t / sum p_t by at most 2 d max|v|;
      * fp32 sums of p_t v_t and of p_t over len terms: len * 2^-24 relative to sum p |v| <= max|v| sum p;
      * the output is rounded to bf16: 2^-9 |out|.
    Bound: |out - ref| <= 2^-8 |ref| + max|v| (2 d + len 2^-23 + 2^-20), d = scale hd 2^-23 max_t sum|q k_t| + (len/64 + 4) 2^-21.
    For the LSE (natural log): |lse - ref| <= d + len 2^-23 + 2^-20."""
    B = q.shape[0]
    G = nh // nkv
    q64 = q[:, :nh * hd].double().reshape(B, nh, hd)
    out = torch.zeros(B, nh, hd, dtype=torch.float64, device=q.device)
    lse = torch.zeros(B, nh, dtype=torch.float64, device=q.device)
    tol = torch.zeros(B, nh, hd, dtype=torch.float64, device=q.device)
    tol_lse = torch.zeros(B, nh, dtype=torch.float64, device=q.device)
    for b in range(B):
        n = int(lens[b])
        for h in range(nh):
            kk = k[b, h // G, :n, :hd].double()
            vv = v[b, h // G, :n, :hd].double()
            s = (kk @ q64[b, h]) * scale
            lse[b, h] = torch.logsumexp(s, 0)
            p = torch.softmax(s, 0)
            out[b, h] = p @ vv
            d = scale * hd * 2.0 ** -23 * (kk.abs() @ q64[b, h].abs()).max() + (n / 64 + 4) * 2.0 ** -21
            vmax = vv.abs().max()
            tol[b, h] = 2.0 ** -8 * out[b, h].abs() + vmax * (2 * d + n * 2.0 ** -23 + 2.0 ** -20)
            tol_lse[b, h] = d + n * 2.0 ** -23 + 2.0 ** -20
    return out, lse, tol, tol_lse
