"""Pin of the third-party piece behind the reference's ``--optim adamw_bnb_8bit`` / ``adamw_8bit`` (align_trainer.py:409-429: HF's
``Trainer.get_optimizer_cls_and_kwargs`` returns ``bitsandbytes.optim.AdamW`` with ``optim_bits=8``).  bitsandbytes is not installable
in the build container, so the 8-bit AdamW of this project (csrc/optim.cu ``lmod_adamw_8bit``, restated in tests/adamw8_oracle.py) is
"parity unpinned" -- THIS test turns the code tables, the block size and one block-wise step into a pin the moment bitsandbytes is
importable.  Skipped, loudly, while it is absent.

The step is compared with a tolerance, not bit for bit: bitsandbytes applies weight decay after the update and folds the second bias
correction into eps (``eps * sqrt(1 - beta2^t)``), and its block-wise quantiser is its own; DESIGN.md section 5 lists the differences."""
import importlib

import numpy as np
import pytest
import torch

from tests import adamw8_oracle as O


def _bnb_functional():
    try:
        return importlib.import_module("bitsandbytes.functional")
    except Exception as e:                                  # noqa: BLE001 -- any import failure means "no usable bitsandbytes here"
        pytest.skip("bitsandbytes is not importable here (%s: %s): the 8-bit AdamW state stays 'parity unpinned'" % (type(e).__name__, e))


@pytest.mark.parametrize("signed", [True, False])
def test_restated_code_tables_equal_bitsandbytes(signed):
    F = _bnb_functional()
    theirs = F.create_dynamic_map(signed=signed).float().cpu().numpy()
    mine = O.create_dynamic_map(signed=signed).numpy()
    assert np.array_equal(theirs.view(np.uint32), mine.view(np.uint32))


def test_block_size_and_one_blockwise_step_agree_with_bitsandbytes():
    F = _bnb_functional()
    if not torch.cuda.is_available():
        pytest.skip("bitsandbytes' block-wise optimizer update runs on CUDA only")
    n = 3 * O.BLOCK + 256
    rng = np.random.default_rng(0)
    p = torch.from_numpy(rng.standard_normal(n).astype(np.float32) * np.float32(0.05)).cuda()
    g = torch.from_numpy(rng.standard_normal(n).astype(np.float32) * np.float32(1e-2)).cuda()
    tm, tv = (torch.from_numpy(t).cuda() for t in O.tables())
    s1 = torch.zeros(n, dtype=torch.uint8, device="cuda")
    s2 = torch.zeros(n, dtype=torch.uint8, device="cuda")
    nb = (n + O.BLOCK - 1) // O.BLOCK
    a1 = torch.zeros(nb, device="cuda")
    a2 = torch.zeros(nb, device="cuda")
    p_bnb = p.clone()
    F.optimizer_update_8bit_blockwise("adam", g, p_bnb, s1, s2, 0.9, 0.999, 0.0, 0.0, 1e-8, 1, 1e-3, tm, tv, a1, a2, 0.0, 1.0, False)
    torch.cuda.synchronize()
    assert a1.numel() == nb                                                     # one scale per 2048 elements
    qm, qv, am, av = O.zero_state(n)
    mine = O.step_fp32(p.cpu().numpy(), qm, qv, am, av, g.cpu().numpy(), lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0, step=1)
    np.testing.assert_allclose(p_bnb.cpu().numpy(), mine[0], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(a1.cpu().numpy(), mine[4], rtol=1e-5)
    np.testing.assert_allclose(a2.cpu().numpy(), mine[5], rtol=1e-5)
