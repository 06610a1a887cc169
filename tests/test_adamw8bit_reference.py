"""CPU checks of the 8-bit block-wise AdamW restatement (tests/adamw8_oracle.py) that the GPU tests hold lmod_adamw_8bit to: the code
tables, the quantiser's tie rule, the fp32 step against float64, planted defects, the committed kernel tables, the ``--optim`` mapping,
the state byte count and the argument checks of the C entry point."""
import numpy as np
import pytest

from tests import adamw8_oracle as O

HP = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8)


def test_code_tables_follow_the_dynamic_map_definition():
    tm, tv = O.tables()
    assert tm.dtype == tv.dtype == np.float32 and tm.shape == tv.shape == (256,)
    assert np.all(np.diff(tm) > 0) and np.all(np.diff(tv) > 0)              # strictly ascending: every code distinct
    # signed: 127 negatives, 0, 127 positives, 1.0; the positive and negative halves mirror each other
    assert tm[127] == 0 and tm[255] == 1 and -1 < tm[0] < -0.99
    assert np.array_equal(-tm[:127][::-1], tm[128:255])
    # unsigned: 0, 254 positives, 1.0
    assert tv[0] == 0 and tv[255] == 1 and tv[1] > 0
    # decade i (values in (1e-7, 1e-6) * 10^i) holds 2^i codes per sign (signed) or 2^(i+1) (unsigned)
    for i in range(7):
        lo, hi = 10.0 ** (i - 7), 10.0 ** (i - 6)
        assert np.sum((tm > lo) & (tm < hi)) == 2 ** i, i
        assert np.sum((tv > lo) & (tv < hi)) == 2 ** (i + 1), i


def test_committed_kernel_tables_equal_the_restatement():
    tm, tv = O.tables()
    cm, cv = O.committed_tables()
    assert np.array_equal(cm.view(np.uint32), tm.view(np.uint32)), "regenerate csrc/adamw8_tables.cuh with `python -m tests.adamw8_oracle`"
    assert np.array_equal(cv.view(np.uint32), tv.view(np.uint32)), "regenerate csrc/adamw8_tables.cuh with `python -m tests.adamw8_oracle`"


@pytest.mark.parametrize("signed", [True, False])
def test_quantiser_is_nearest_with_ties_to_the_lower_code(signed):
    t = O.tables()[0 if signed else 1]
    mids = O.midpoints(t)
    k = np.arange(255)
    assert np.array_equal(O.quantize(mids, t), k.astype(np.uint8))                                     # on a midpoint: the lower code
    assert np.array_equal(O.quantize(np.nextafter(mids, np.float32(np.inf)), t), (k + 1).astype(np.uint8))
    assert np.array_equal(O.quantize(t, t), np.arange(256).astype(np.uint8))                           # every code is its own nearest
    assert O.quantize(np.float32(np.nan), t) == 0
    assert O.quantize(np.float32(0), t) == (127 if signed else 0)
    assert O.quantize(np.float32(1), t) == 255 and O.quantize(np.float32(-1), t) == 0
    # nearest by brute force on random points
    x = np.random.default_rng(1).uniform(-1 if signed else 0, 1, 20000).astype(np.float32)
    d = np.abs(x[:, None].astype(np.float64) - t[None, :].astype(np.float64))
    q = O.quantize(x, t).astype(np.int64)
    assert np.all(d[np.arange(len(x)), q] <= d.min(axis=1) * (1 + 1e-6) + 1e-30)


def random_state(n, seed, zero=False):
    rng = np.random.default_rng(seed)
    master = rng.standard_normal(n).astype(np.float32) * np.float32(0.05)
    grad = rng.standard_normal(n).astype(np.float32) * np.float32(1e-2)
    import torch
    grad = torch.from_numpy(grad).to(torch.bfloat16).float().numpy()                  # a bf16 gradient
    if zero:
        qm, qv, am, av = O.zero_state(n)
    else:
        nb = (n + O.BLOCK - 1) // O.BLOCK
        qm = rng.integers(0, 256, n).astype(np.uint8)
        qv = rng.integers(0, 256, n).astype(np.uint8)
        am = rng.uniform(1e-3, 2e-2, nb).astype(np.float32)
        av = rng.uniform(1e-6, 1e-4, nb).astype(np.float32)
    return master, qm, qv, am, av, grad


def fp64_mismatches(out, ref, master, qm, qv, am, av, grad):
    """What of the fp32 step ``out`` does not agree with the float64 step ``ref`` up to fp32 rounding: a list of reasons (empty = agrees).
    master: within 16 ulp of fp32 of the larger of |p| and the update; scales: within 16 ulp; codes: the nearest code of the float64
    moment over the float64 scale, allowed to differ by one code on at most 0.5 % of the elements (fp32 rounding near a midpoint)."""
    p32, _, q_m, q_v, a_m, a_v = out
    p64, m64, v64, am64, av64 = ref
    e = float(np.finfo(np.float32).eps)
    bad = []
    upd = np.abs(p64 - master.astype(np.float64))
    if not np.all(np.abs(p32 - p64) <= 16 * e * (np.abs(p64) + upd) + 1e-30):
        bad.append("master")
    for name, a32, a64 in (("absmax_m", a_m, am64), ("absmax_v", a_v, av64)):
        if not np.all(np.abs(a32 - a64) <= 16 * e * np.abs(a64)):
            bad.append(name)
    tm, tv = O.tables()
    blk = np.arange(len(p32)) // O.BLOCK
    for name, q32, mom, sc, t in (("m codes", q_m, m64, am64, tm), ("v codes", q_v, v64, av64, tv)):
        with np.errstate(all="ignore"):
            x = np.where(sc[blk] > 0, mom / sc[blk], 0.0)
        d = np.abs(q32.astype(np.int64) - O.quantize(x.astype(np.float32), t).astype(np.int64))
        if d.max() > 1 or np.mean(d != 0) > 5e-3:
            bad.append(name)
    return bad


CASES = [dict(n=6784, zero=True, step=1, wd=0.0, gnorm_sq=None, max_norm=0.0, grad_scale=1.0),
         dict(n=6784, zero=False, step=7, wd=0.1, gnorm_sq=40.0, max_norm=1.0, grad_scale=0.25),
         dict(n=2176, zero=False, step=2, wd=0.0, gnorm_sq=1e-4, max_norm=1.0, grad_scale=1.0),
         dict(n=128, zero=False, step=3, wd=0.01, gnorm_sq=None, max_norm=0.0, grad_scale=0.5)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "n%d-step%d" % (c["n"], c["step"]))
def test_fp32_step_equals_fp64_step_up_to_fp32_rounding(case):
    st = random_state(case["n"], case["n"] + case["step"], zero=case["zero"])
    kw = dict(HP, wd=case["wd"], step=case["step"], gnorm_sq=case["gnorm_sq"], max_norm=case["max_norm"], grad_scale=case["grad_scale"])
    out = O.step_fp32(*st, **kw)
    ref = O.step_fp64(*st, **kw)
    assert fp64_mismatches(out, ref, *st) == []


@pytest.mark.parametrize("defect", ["no_bias_correction", "absmax_before_update", "floor", "block_off_by_one"])
def test_planted_defects_are_caught(defect):
    """Each defect, planted in the fp32 step, makes it disagree with the float64 step: the comparison the kernel is held to has teeth."""
    st = random_state(6784, 11, zero=False)
    kw = dict(HP, wd=0.0, step=3, gnorm_sq=None, max_norm=0.0, grad_scale=1.0)
    ref = O.step_fp64(*st, **kw)
    assert fp64_mismatches(O.step_fp32(*st, **kw), ref, *st) == []
    assert fp64_mismatches(O.step_fp32(*st, **kw, defect=defect), ref, *st) != []


def test_zero_block_stores_the_code_of_zero_and_no_nan():
    n = 2048 + 256
    master, qm, qv, am, av, grad = random_state(n, 5, zero=True)
    grad[:2048] = 0
    p, model, q_m, q_v, a_m, a_v = O.step_fp32(master, qm, qv, am, av, grad, step=1, wd=0.0, **HP)
    assert a_m[0] == 0 and a_v[0] == 0 and np.all(q_m[:2048] == 127) and np.all(q_v[:2048] == 0)
    assert np.array_equal(p[:2048], master[:2048]) and np.all(np.isfinite(p))


def test_optim_values_map_to_state_bits():
    from llavamod.config.args import TrainingArguments, parse_args_into_dataclasses
    from llavamod.train.engine import optim_bits_of
    assert optim_bits_of("adamw_bnb_8bit") == 8 and optim_bits_of("adamw_8bit") == 8
    for other in ("adamw_torch", "adamw_hf", "adamw_torch_fused", "adafactor", "sgd", "paged_adamw_8bit", "lion_8bit"):
        assert optim_bits_of(other) == 32, other
    (targs,) = parse_args_into_dataclasses((TrainingArguments,), ["--output_dir", "/tmp/x"])
    assert targs.optim == "adamw_torch" and optim_bits_of(targs.optim) == 32
    (targs,) = parse_args_into_dataclasses((TrainingArguments,), ["--output_dir", "/tmp/x", "--optim", "adamw_bnb_8bit"])
    assert optim_bits_of(targs.optim) == 8


def test_state_bytes_count_the_layout():
    from llavamod.train.engine import state_bytes
    # two group slices of 2048 + 128 and 4096 elements: 1 + 1 + 2 blocks of scales, two per block
    assert state_bytes([2176, 4096], 6272, 256, 8) == 6 * 6272 + 4 * 2 * 4 + 8 * 256
    assert state_bytes([2176, 4096], 6272, 256, 32) == 12 * 6272 + 8 * 256
    # 0.5B-4E student (521.2 M trainable, one slice): 16 B/param today, 10 B/param with 8-bit moments (both with bf16 weight + gradient)
    n = 521_200_000
    assert state_bytes([n], n, 0, 32) + 4 * n == 16 * n
    assert 0 < state_bytes([n], n, 0, 8) + 4 * n - 10 * n < 8 * n // 2048 + 8


def test_entry_point_checks_arguments_before_any_launch():
    from llavamod import _C
    L = _C.lib()
    p = 1 << 20                                 # never dereferenced: every call below must return before
    args = lambda count=4096, step=1, master=p: (master, p, p, p, p, p, None, count, 1e-3, 0.9, 0.999, 1e-8, 0.0, step, None, 0.0, 1.0, None)
    assert L.lmod_adamw_8bit(*args(count=4100)) == -1 and b"multiple of 8" in L.lmod_last_error()
    assert L.lmod_adamw_8bit(*args(master=p + 4)) == -1 and b"16B aligned" in L.lmod_last_error()
    assert L.lmod_adamw_8bit(*args(step=0)) == -1
    assert L.lmod_adamw_8bit(*args(count=0)) == -1
