"""The FP8 (e4m3) teacher's CPU side: the restated quantiser (tests/fp8_oracle.py) on hand-computed cases, the fake-quantised decoder
oracle, and the host logic of the mode (--ref_fp8, the refusals of quantize_fp8_).  No GPU."""
import pytest
import torch

from oracle import restated as R
from tests import fp8_oracle as O


def _e4m3(values):
    return torch.tensor(values, dtype=torch.float32).to(torch.float8_e4m3fn).float().tolist()


def test_e4m3_rounds_to_nearest_even_at_the_ties():
    # 3 mantissa bits: between 16 and 32 the step is 2, so 17 lies halfway between 16 (even mantissa) and 18 (odd), 19 between 18 and 20
    assert _e4m3([17.0, 19.0, 21.0, 23.0]) == [16.0, 20.0, 20.0, 24.0]
    assert _e4m3([17.01, 18.99, -17.0, -19.0]) == [18.0, 18.0, -16.0, -20.0]
    # largest finite value 448 = 1.75 * 2^8; step 32 below it: 432 lies halfway between 416 (odd mantissa) and 448 (even)
    assert _e4m3([448.0, -448.0, 432.0, 431.9]) == [448.0, -448.0, 448.0, 416.0]
    # subnormals: multiples of 2^-9 below 2^-6; 1.5 * 2^-9 is a tie between 2^-9 (odd) and 2^-8 (even); 2^-10 a tie between 0 and 2^-9
    assert _e4m3([2.0 ** -9, 1.5 * 2.0 ** -9, 2.0 ** -10, 0.6 * 2.0 ** -9, 2.5 * 2.0 ** -9]) == [2.0 ** -9, 2.0 ** -8, 0.0, 2.0 ** -9, 2.0 ** -8]


def test_quantiser_on_hand_computed_rows():
    # amax 448 -> scale exactly 1, the bytes are the e4m3 encodings of the values: 448 = 0x7E, -448 = 0xFE, 1 = 0x38, 17 -> 16 = 0x58
    x = torch.tensor([[448.0, -448.0, 1.0, 17.0, 0.0, 2.0 ** -9, 2.0 ** -10, -19.0]])
    q, s = O.quant_rows(x)
    assert s.tolist() == [1.0]
    assert q[0].tolist() == [0x7E, 0xFE, 0x38, 0x58, 0x00, 0x01, 0x00, 0xDA]
    # amax 7 -> scale 7/448 = 2^-6 exactly: x / scale = 64 x
    x = torch.tensor([[7.0, -3.5, 0.25, 0.265625]])            # 64 x = 448, -224, 16, 17 (a tie -> 16)
    q, s = O.quant_rows(x)
    assert s.tolist() == [2.0 ** -6]
    assert O.dequant(q, s).tolist() == [[7.0, -3.5, 0.25, 0.25]]
    assert torch.equal(O.fake_quant(x.to(torch.bfloat16)), torch.tensor([[7.0, -3.5, 0.25, 0.25]], dtype=torch.bfloat16))


def test_zero_row_gets_scale_one_and_zero_bytes():
    x = torch.zeros(2, 16)
    x[1, 3] = -2.0
    q, s = O.quant_rows(x)
    assert s[0].item() == 1.0 and not q[0].any()
    assert s[1].item() == float(torch.tensor(2.0) / torch.tensor(448.0)) and q[1, 3].item() == 0xFE and int((q[1] != 0).sum()) == 1


def test_row_of_one_repeated_value_and_a_subnormal_amax():
    q, s = O.quant_rows(torch.full((1, 32), -0.3).to(torch.bfloat16))
    assert (q == 0xFE).all() and s.item() == float(torch.tensor(0.3).to(torch.bfloat16).float() / torch.tensor(448.0))
    # amax = 2^-133, the smallest bf16 subnormal: the scale 2^-133 / 448 is an fp32 subnormal (146 units of 2^-149 after rounding), the
    # quotient 2^16 / 146 = 448.9 is clamped, so the row's largest value still maps to +-448 and half of it to 224.4 -> 224
    tiny = torch.tensor([[2.0 ** -133, -(2.0 ** -133), 2.0 ** -133, 0.0]], dtype=torch.bfloat16)
    assert float(tiny[0, 0]) == 2.0 ** -133
    q, s = O.quant_rows(tiny)
    assert s.item() == 146 * 2.0 ** -149
    assert q[0].tolist() == [0x7E, 0xFE, 0x7E, 0x00]
    q2, s2 = O.quant_rows(torch.tensor([[2.0 ** -132, 2.0 ** -133]], dtype=torch.bfloat16))
    assert s2.item() == 293 * 2.0 ** -149 and q2[0].tolist() == [0x7E, 0x76]     # 2^16 / 293 = 223.7 -> 224 = 0x76


NAN, INF = float("nan"), float("inf")
FINITE_ROW = [448.0, -448.0, 1.0, 17.0, 0.0, 2.0 ** -9, 2.0 ** -10, -19.0]
FINITE_BYTES = [0x7E, 0xFE, 0x38, 0x58, 0x00, 0x01, 0x00, 0xDA]


def test_non_finite_rows_propagate_and_leave_their_neighbours_alone():
    x = torch.tensor([FINITE_ROW,
                      [1.0, NAN, -2.0, 0.0, -0.0, 448.0, 3.0, -3.0],          # NaN: scale NaN, every byte NaN
                      [1.0, INF, -2.0, 0.0, -0.0, 448.0, 3.0, -3.0],          # +inf: scale inf, NaN at the inf, +-0 elsewhere
                      [-INF, 3.0, -3.0, 0.0, -0.0, 1e30, -1e-30, 7.0],        # -inf likewise
                      [NAN, INF, -INF, 1.0, -1.0, 0.0, 2.0, 3.0],             # both: the NaN wins
                      FINITE_ROW]).to(torch.bfloat16)
    q, s = O.quant_rows(x)
    assert q.dtype == torch.uint8 and s.dtype == torch.float32
    assert s[0].item() == 1.0 and s[5].item() == 1.0 and q[0].tolist() == FINITE_BYTES and q[5].tolist() == FINITE_BYTES
    assert torch.isnan(s[1]) and O.is_nan_byte(q[1]).all()
    assert s[2].item() == INF and s[3].item() == INF
    assert q[2].tolist() == [0x00, q[2, 1].item(), 0x80, 0x00, 0x80, 0x00, 0x00, 0x80] and O.is_nan_byte(q[2, 1])
    assert q[3].tolist() == [q[3, 0].item(), 0x00, 0x80, 0x00, 0x80, 0x00, 0x80, 0x00] and O.is_nan_byte(q[3, 0])
    assert torch.isnan(s[4]) and O.is_nan_byte(q[4]).all()
    # a row is quantised on its own: without the non-finite rows the finite ones come out the same
    q2, s2 = O.quant_rows(x[[0, 5]])
    assert torch.equal(q2, q[[0, 5]]) and torch.equal(s2, s[[0, 5]])
    # every product with a non-finite row is NaN in every column (an inf row dequantises to NaN at the inf and inf * 0 = NaN elsewhere);
    # the finite rows keep their values
    w = torch.tensor([[1.0] * 8, [0.0] * 8, [-1.0, 2.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.5]])
    qw, sw = O.quant_rows(w)
    d = O.gemm_dequant_fp64(q, s, qw, sw)
    assert torch.isnan(d[1:5]).all() and torch.isfinite(d[[0, 5]]).all()
    assert torch.equal(d[0], O.gemm_dequant_fp64(q[:1], s[:1], qw, sw)[0])


def test_negative_values_that_underflow_keep_their_sign():
    # amax 448 -> scale 1: -2^-11 rounds to -0 (0x80), -2^-10 (a tie with 0) to -0, -0.0 stays -0, -0.6 * 2^-9 to -2^-9 (0x81)
    x = torch.tensor([[448.0, -(2.0 ** -11), -(2.0 ** -10), -0.0, -0.6 * 2.0 ** -9, 2.0 ** -11]])
    q, s = O.quant_rows(x)
    assert s.item() == 1.0 and q[0].tolist() == [0x7E, 0x80, 0x80, 0x80, 0x81, 0x00]


def test_dequantised_gemm_is_the_float64_product():
    g = torch.Generator().manual_seed(0)
    a, w = torch.randn(5, 64, generator=g).to(torch.bfloat16), torch.randn(7, 64, generator=g).to(torch.bfloat16)
    (qa, sa), (qw, sw) = O.quant_rows(a), O.quant_rows(w)
    d = O.gemm_dequant_fp64(qa, sa, qw, sw)
    want = (qa.view(torch.float8_e4m3fn).double() @ qw.view(torch.float8_e4m3fn).double().t()) * sa.double()[:, None] * sw.double()[None, :]
    assert d.dtype == torch.float64 and torch.allclose(d, want, rtol=1e-12, atol=1e-12)      # exact integer-grid sums, scaled
    # 3 mantissa bits: an element is within 2^-4 of its value relative to the row's amax-scaled grid; the product stays close to the exact one
    assert (d - a.double() @ w.double().t()).abs().max() < 0.08 * 64 ** 0.5 * 3


def test_fake_quantised_decoder_touches_the_decoder_linears_only():
    cfg = R.LMCfg(hidden=64, inter=128, layers=2, heads=2, kv_heads=1, vocab=96)
    sd = R.init_lm(cfg, 32, torch.Generator().manual_seed(1))
    fq = O.fake_quant_state(sd)
    changed = sorted(k for k in sd if not torch.equal(sd[k], fq[k]))
    assert len(changed) == 2 * 7 and all(O.DECODER_LINEAR.search(k) for k in changed), changed
    x = torch.randn(2, 9, 64, generator=torch.Generator().manual_seed(2))
    plain, _ = R.lm_forward(fq, cfg, x, None, None)
    with O.fp8_decoder(R):
        quant, _ = R.lm_forward(fq, cfg, x, None, None)
    again, _ = R.lm_forward(fq, cfg, x, None, None)
    assert torch.equal(plain, again) and R.F is torch.nn.functional          # the patch is gone
    rel = (quant - plain).norm() / plain.norm()
    assert 0 < rel < 0.2, rel                                                # activations are quantised too, and only mildly


def test_ref_fp8_flag_parses():
    from llavamod.config.args import AlignArguments, DPOArguments, parse_args_into_dataclasses
    assert AlignArguments().ref_fp8 is False and DPOArguments().ref_fp8 is False
    (a,) = parse_args_into_dataclasses((AlignArguments,), ["--ref_fp8", "True"])
    (d,) = parse_args_into_dataclasses((DPOArguments,), ["--ref_fp8", "True"])
    (a0,) = parse_args_into_dataclasses((AlignArguments,), ["--loss_type", "kd_lm"])
    assert a.ref_fp8 is True and d.ref_fp8 is True and a0.ref_fp8 is False


def _cpu(kind):
    from llavamod.model import synthetic as S
    if kind == "teacher":
        return S.make_teacher(dict(S.ARCH["tiny"]), "tiny", device="cpu", dtype=torch.float32)
    return S.make_student(dict(S.ARCH["tiny"]), "tiny", device="cpu", dtype=torch.float32, margs=S.moe_args())


def test_quantize_fp8_refuses_trainable_decoder_weights_and_sparse_models():
    t = _cpu("teacher").eval()
    for p in t.parameters():
        p.requires_grad = False
    t.model.layers[1].mlp.down_proj.weight.requires_grad = True
    with pytest.raises(ValueError, match=r"model\.layers\.1\.mlp\.down_proj\.weight requires grad"):
        t.quantize_fp8_()
    t.model.layers[1].mlp.down_proj.weight.requires_grad = False
    t.train()
    with pytest.raises(ValueError, match="eval"):
        t.quantize_fp8_()
    t.eval()
    with pytest.raises(ValueError, match="GPU"):                # every refusal comes before the first kernel
        t.quantize_fp8_()
    assert not t.is_fp8 and t.model.layers[0].self_attn.o_proj.weight is not None
    s = _cpu("student").eval()
    for p in s.parameters():
        p.requires_grad = False
    with pytest.raises(ValueError, match="sparse"):
        s.quantize_fp8_()


def test_trainers_take_ref_fp8_and_the_environment_switch(monkeypatch):
    import inspect
    from llavamod.train import align_trainer as A, trainer_base as B
    from llavamod.train.dpo_trainer import DPOTrainer
    assert inspect.signature(A.AlignTrainer.__init__).parameters["ref_fp8"].default is False
    assert inspect.signature(DPOTrainer.__init__).parameters["ref_fp8"].default is False

    class Ref:
        is_fp8, calls = False, 0

        def quantize_fp8_(self):
            self.calls += 1
            self.is_fp8 = True

    r = Ref()
    monkeypatch.delenv("LLAVAMOD_REF_FP8", raising=False)
    B.quantize_ref_fp8(r, False)
    assert r.calls == 0
    monkeypatch.setenv("LLAVAMOD_REF_FP8", "1")
    B.quantize_ref_fp8(r, False)
    B.quantize_ref_fp8(r, True)                                 # already quantised: not again
    assert r.calls == 1
