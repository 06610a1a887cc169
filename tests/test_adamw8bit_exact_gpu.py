"""lmod_adamw_8bit (csrc/optim.cu) against its numpy float32 restatement (tests/adamw8_oracle.py::step_fp32): codes and the bf16 weight
byte for byte, scales and master bit for bit, at block and slice edges, from a fresh and from a random state, with clipping, decay and a
gradient scale, on an all-zero block, on gradients spanning 1e-12 .. 1e2, on a NaN gradient, and around element 2^31 of a long slice.
Then TrainState(optim_bits=8) over its optimizer-group slices against a host loop of the restatement."""
import numpy as np
import pytest
import torch

from tests import adamw8_oracle as O

pytestmark = pytest.mark.gpu

HP = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint16)


def assert_bit_equal(got, want, what):
    """Equal bit patterns, except that every NaN matches every NaN (the kernel and numpy write different NaN payloads)."""
    got, want = np.asarray(got), np.asarray(want)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), "%s: NaN at different positions" % what
    bad = np.nonzero(_bits(got[~gn]) != _bits(want[~wn]))[0]
    assert bad.size == 0, "%s: %d elements differ, first %s: kernel %r, restatement %r" % (
        what, bad.size, bad[:5], got[~gn][bad[:5]], want[~wn][bad[:5]])


def run_kernel(master, qm, qv, am, av, grad_bf16, offset=0, with_model=True, gnorm_sq=None, max_norm=0.0, grad_scale=1.0, **hp):
    """Places the slice at element ``offset`` of larger buffers (the scales at their own offset), runs one kernel step, returns numpy."""
    from llavamod import kernels as K
    n, nb = master.shape[0], am.shape[0]
    dev = "cuda"
    P = torch.zeros(offset + n, dtype=torch.float32, device=dev)
    QM = torch.zeros(offset + n, dtype=torch.uint8, device=dev)
    QV = torch.zeros(offset + n, dtype=torch.uint8, device=dev)
    G = torch.zeros(offset + n, dtype=torch.bfloat16, device=dev)
    W = torch.zeros(offset + n, dtype=torch.bfloat16, device=dev)
    S = torch.zeros(3 + 2 * nb, dtype=torch.float32, device=dev)
    P[offset:] = torch.from_numpy(master).to(dev)
    QM[offset:] = torch.from_numpy(qm).to(dev)
    QV[offset:] = torch.from_numpy(qv).to(dev)
    G[offset:] = grad_bf16.to(dev)
    S[3:3 + nb] = torch.from_numpy(am).to(dev)
    S[3 + nb:] = torch.from_numpy(av).to(dev)
    gn = torch.tensor([gnorm_sq], dtype=torch.float32, device=dev) if gnorm_sq is not None else None
    K.adamw_8bit_(P[offset:], QM[offset:], QV[offset:], S[3:3 + nb], S[3 + nb:], G[offset:], W[offset:] if with_model else None,
                  gnorm_sq=gn, max_norm=max_norm, grad_scale=grad_scale, **hp)
    torch.cuda.synchronize()
    assert torch.all(P[:offset] == 0) and torch.all(QM[:offset] == 0) and torch.all(W[:offset] == 0) and torch.all(S[:3] == 0)
    return (P[offset:].cpu().numpy(), W[offset:].cpu(), QM[offset:].cpu().numpy(), QV[offset:].cpu().numpy(),
            S[3:3 + nb].cpu().numpy(), S[3 + nb:].cpu().numpy())


def compare(got, want, with_model=True):
    p, w, qm, qv, am, av = got
    p_r, w_r, qm_r, qv_r, am_r, av_r = want
    assert np.array_equal(qm, qm_r), "m codes: %d differ" % int(np.sum(qm != qm_r))
    assert np.array_equal(qv, qv_r), "v codes: %d differ" % int(np.sum(qv != qv_r))
    assert_bit_equal(am, am_r, "absmax_m")
    assert_bit_equal(av, av_r, "absmax_v")
    assert_bit_equal(p, p_r, "master")
    if with_model:
        assert_bit_equal(w.float().numpy(), w_r.float().numpy(), "bf16 weight")       # bf16 -> fp32 is exact: same bits
        fin = torch.isfinite(w_r)
        assert torch.equal(w.view(torch.int16)[fin], w_r.view(torch.int16)[fin])


def make_case(n, seed, zero, g_lo=None, g_hi=None):
    rng = np.random.default_rng(seed)
    master = (rng.standard_normal(n) * 0.05).astype(np.float32)
    if g_lo is None:
        g = torch.from_numpy((rng.standard_normal(n) * 1e-2).astype(np.float32)).to(torch.bfloat16)
    else:                                             # magnitudes log-uniform over [g_lo, g_hi], random signs
        mag = np.exp(rng.uniform(np.log(g_lo), np.log(g_hi), n)) * rng.choice([-1.0, 1.0], n)
        g = torch.from_numpy(mag.astype(np.float32)).to(torch.bfloat16)
    nb = (n + O.BLOCK - 1) // O.BLOCK
    if zero:
        qm, qv, am, av = O.zero_state(n)
    else:
        qm = rng.integers(0, 256, n).astype(np.uint8)
        qv = rng.integers(0, 256, n).astype(np.uint8)
        am = rng.uniform(1e-3, 2e-2, nb).astype(np.float32)
        av = rng.uniform(1e-6, 1e-4, nb).astype(np.float32)
    return master, qm, qv, am, av, g


def restated(master, qm, qv, am, av, g, **kw):
    return O.step_fp32(master, qm, qv, am, av, g.float().numpy(), **kw)


@pytest.mark.parametrize("n", [128, 1920, 2048, 2176, 6784])
@pytest.mark.parametrize("state", ["fresh-step1", "random-step5"])
@pytest.mark.parametrize("clip,wd,gs", [(False, 0.0, 1.0), (True, 0.1, 0.125)])
def test_kernel_equals_restatement(n, state, clip, wd, gs):
    zero = state.startswith("fresh")
    step = 1 if zero else 5
    master, qm, qv, am, av, g = make_case(n, seed=n + step, zero=zero)
    gnorm_sq = float((g.float() ** 2).sum()) if clip else None          # any fp32 value: the kernel reads it from the device scalar
    kw = dict(HP, wd=wd, step=step, gnorm_sq=gnorm_sq, max_norm=1.0 if clip else 0.0, grad_scale=gs)
    got = run_kernel(master, qm, qv, am, av, g, **kw)
    compare(got, restated(master, qm, qv, am, av, g, **kw))


@pytest.mark.parametrize("offset", [1152, 2048 + 640])
def test_slice_offset_not_a_multiple_of_the_block(offset):
    """Blocks start at the slice, not at the arena: the slice sits at an offset that is not a multiple of 2048."""
    master, qm, qv, am, av, g = make_case(4224, seed=3, zero=False)
    kw = dict(HP, wd=0.01, step=3)
    compare(run_kernel(master, qm, qv, am, av, g, offset=offset, **kw), restated(master, qm, qv, am, av, g, **kw))


def test_without_model_copy():
    master, qm, qv, am, av, g = make_case(2176, seed=4, zero=False)
    kw = dict(HP, wd=0.0, step=2)
    compare(run_kernel(master, qm, qv, am, av, g, with_model=False, **kw), restated(master, qm, qv, am, av, g, **kw), with_model=False)


def test_all_zero_block_and_fresh_state():
    """Block 1 gets zero gradients from a fresh state: scale 0, the code of 0, master only decayed, no NaN."""
    master, qm, qv, am, av, g = make_case(3 * 2048, seed=5, zero=True)
    g[2048:4096] = 0
    kw = dict(HP, wd=0.1, step=1)
    got = run_kernel(master, qm, qv, am, av, g, **kw)
    compare(got, restated(master, qm, qv, am, av, g, **kw))
    p, _, q_m, q_v, a_m, a_v = got
    assert a_m[1] == 0 and a_v[1] == 0 and np.all(q_m[2048:4096] == 127) and np.all(q_v[2048:4096] == 0) and np.all(np.isfinite(p))


@pytest.mark.parametrize("state", ["fresh", "random"])
def test_gradients_spanning_fourteen_decades(state):
    master, qm, qv, am, av, g = make_case(2048 + 1024, seed=6, zero=state == "fresh", g_lo=1e-12, g_hi=1e2)
    kw = dict(HP, wd=0.0, step=1 if state == "fresh" else 4)
    compare(run_kernel(master, qm, qv, am, av, g, **kw), restated(master, qm, qv, am, av, g, **kw))


def test_nan_gradient_poisons_its_own_block_only():
    """Clipping off, one NaN gradient in block 1: that block's scales become NaN, its other codes the code of 0 (a NaN scale is inverted
    to 0) and its other master elements take a normal step; blocks 0 and 2 are untouched by it.  On the next step the whole block is NaN."""
    master, qm, qv, am, av, g = make_case(3 * 2048, seed=7, zero=False)
    g[2048 + 100] = float("nan")
    kw = dict(HP, wd=0.0, step=3)
    got = run_kernel(master, qm, qv, am, av, g, **kw)
    want = restated(master, qm, qv, am, av, g, **kw)
    compare(got, want)
    p, _, q_m, q_v, a_m, a_v = got
    assert np.isnan(a_m[1]) and np.isnan(a_v[1]) and np.all(np.isfinite(a_m[[0, 2]])) and np.all(np.isfinite(a_v[[0, 2]]))
    assert np.isnan(p[2048 + 100]) and np.sum(np.isnan(p)) == 1
    ok = np.ones(3 * 2048, bool)
    ok[2048 + 100] = False
    assert np.all(q_m[2048:4096][ok[2048:4096]] == 127) and np.all(q_v[2048:4096][ok[2048:4096]] == 0)
    g2 = torch.zeros_like(g)
    got2 = run_kernel(p, q_m, q_v, a_m, a_v, g2, **dict(kw, step=4))
    compare(got2, restated(p, q_m, q_v, a_m, a_v, g2, **dict(kw, step=4)))
    assert np.all(np.isnan(got2[0][2048:4096])) and np.all(np.isfinite(got2[0][:2048])) and np.all(np.isfinite(got2[0][4096:]))


def test_blocks_around_element_2_pow_31():
    """64-bit indexing: a slice of 2^31 + 4096 elements (about 17.2 GB of master, codes and gradient, no model copy); the three blocks
    around element 2^31 get random state and gradients, and must equal the restatement run on just those blocks."""
    n = (1 << 31) + 4096
    need = n * (4 + 1 + 1 + 2) + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free (the GPU is shared)" % (need / 2 ** 30, free / 2 ** 30))
    from llavamod import kernels as K
    nb = (n + O.BLOCK - 1) // O.BLOCK
    lo = (1 << 31) - 2048                          # blocks lo/2048 .. +2: the last one below 2^31, the one at 2^31, the one after
    master, qm, qv, am, av, g = make_case(3 * 2048, seed=8, zero=False)
    P = torch.zeros(n, dtype=torch.float32, device="cuda")
    QM = torch.zeros(n, dtype=torch.uint8, device="cuda")
    QV = torch.zeros(n, dtype=torch.uint8, device="cuda")
    G = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    AM = torch.zeros(nb, dtype=torch.float32, device="cuda")
    AV = torch.zeros(nb, dtype=torch.float32, device="cuda")
    sl, bl = slice(lo, lo + 3 * 2048), slice(lo // 2048, lo // 2048 + 3)
    P[sl] = torch.from_numpy(master).cuda()
    QM[sl] = torch.from_numpy(qm).cuda()
    QV[sl] = torch.from_numpy(qv).cuda()
    G[sl] = g.cuda()
    AM[bl] = torch.from_numpy(am).cuda()
    AV[bl] = torch.from_numpy(av).cuda()
    kw = dict(HP, wd=0.01, step=6)
    K.adamw_8bit_(P, QM, QV, AM, AV, G, None, **kw)
    torch.cuda.synchronize()
    got = (P[sl].cpu().numpy(), None, QM[sl].cpu().numpy(), QV[sl].cpu().numpy(), AM[bl].cpu().numpy(), AV[bl].cpu().numpy())
    compare(got, restated(master, qm, qv, am, av, g, **kw), with_model=False)
    assert int(torch.count_nonzero(AM)) <= 3 and float(P[:lo].abs().max()) == 0      # the zero rest of the slice stays zero
    del P, QM, QV, G, AM, AV
    torch.cuda.empty_cache()


def test_trainstate_8bit_equals_a_host_loop_over_its_group_slices():
    """TrainState(optim_bits=8) on the tiny sparse student with decay, no-decay and --mm_projector_lr groups: after several steps the
    master, bf16 weights, codes and scales equal the restatement applied slice by slice with the same gradients, LRs and clip norm."""
    from llavamod.train.engine import TrainState
    from tests.helpers import tiny_pair
    student, _ = tiny_pair()
    for n_, p_ in student.named_parameters():
        p_.requires_grad_("image_tower" not in n_)
    ts = TrainState(student, lr=1e-3, weight_decay=0.1, max_grad_norm=1.0, mm_projector_lr=3e-3, optim_bits=8)
    keys = [k for k, _, _ in ts.segments["16"]]
    assert len(keys) >= 3 and len(set(keys)) == len(keys)
    assert {k[0] for k in keys} == {False, True} and {k[1] for k in keys} == {False, True}
    assert ts.m16 is None and ts.v16 is None and ts.m8.dtype == torch.uint8
    # the state holds exactly the counted bytes
    held = sum(t.numel() * t.element_size() for t in (ts.master, ts.m8, ts.v8, ts.absmax, ts.m32, ts.v32) if t is not None)
    assert held == ts.state_bytes()
    st = {}
    for _, a, b in ts.segments["16"]:
        st[a] = [ts.master[a:b].cpu().numpy().copy(), *O.zero_state(b - a)]
    gen = torch.Generator(device="cuda").manual_seed(0)
    for step in range(1, 5):
        ts.zero_grad()
        ts.g16.copy_((torch.randn(ts.g16.shape, device="cuda", generator=gen) * 1e-2).to(torch.bfloat16))
        if ts.n32:
            ts.g32.copy_(torch.randn(ts.g32.shape, device="cuda", generator=gen) * 1e-2)
        lr = 1e-3 * (0.5 + 0.1 * step)
        ts.step(lr=lr, grad_scale=0.5)
        torch.cuda.synchronize()
        gn = float(ts.gnorm_sq[0])
        g16 = ts.g16.float().cpu().numpy()
        for (is_proj, no_decay), a, b in ts.segments["16"]:
            so, nb = ts.scale_slices[[x[1] for x in ts.segments["16"]].index(a)]
            g_lr = lr * (3e-3 / 1e-3) if is_proj else lr                  # TrainState's projector-LR rule, same Python floats
            p, w, qm, qv, am, av = O.step_fp32(*st[a], g16[a:b], lr=g_lr, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0 if no_decay else 0.1,
                                               step=step, gnorm_sq=gn, max_norm=1.0, grad_scale=0.5)
            st[a] = [p, qm, qv, am, av]
            got = (ts.master[a:b].cpu().numpy(), ts.w16[a:b].cpu(), ts.m8[a:b].cpu().numpy(), ts.v8[a:b].cpu().numpy(),
                   ts.absmax[so:so + nb].cpu().numpy(), ts.absmax[so + nb:so + 2 * nb].cpu().numpy())
            compare(got, (p, w, qm, qv, am, av))
