"""N>1 correctness ON HARDWARE (SURVEY.md section 4: "1/2/4/8-GPU runs asserting identical loss to the 1-GPU run at equal global batch"):
two ranks over NCCL, one sample each per optimizer step (global batch 2), against ONE rank accumulating the same two samples locally.
The loss sequence, the global gradient norm and the trained weights after K steps must agree -- the only difference allowed is the
order in which two bf16 gradients are added (NCCL sum of two rounded buffers vs. in-place accumulation), i.e. ~2^-8 relative.
Needs 2 visible GPUs; skipped on a 1-GPU machine."""
import os
import socket
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 6


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(rank, world, port, q, loss_kind, graphs=False):
    try:
        _run_inner(rank, world, port, q, loss_kind, graphs)
    except BaseException:                                  # noqa: BLE001 -- hand the child's traceback to the parent instead of a bare EOFError
        import traceback
        q.put(("error", "rank %d: %s" % (rank, traceback.format_exc()), None))
        raise


def _run_inner(rank, world, port, q, loss_kind, graphs=False):
    for p in (ROOT, os.path.join(ROOT, "llava-mod_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from tests import helpers as Hh
    dev = "cuda:%d" % rank
    student, teacher = Hh.tiny_pair(device=dev, seed=5)
    GLOBAL = 2
    accum = GLOBAL // world
    kind = "dpo" if loss_kind == "sigmoid" else "align"
    tr = Hh.make_trainer(student, teacher, loss_kind, accum=accum, lr=1e-3, max_steps=STEPS, kind=kind)
    tr.use_cuda_graphs = graphs             # graphs on: micro-batches replay their graphs; the NCCL all-reduce runs eagerly in the optimizer step
    assert tr.world_size == world
    losses, gnorms = [], []
    for step in range(STEPS):
        mine = []
        for j in range(accum):
            idx = step * GLOBAL + rank * accum + j            # sample index in the global batch: the same samples whatever the world size
            batch, noise = Hh.tiny_batch(student, B=1, seed=1000 + idx)
            if kind == "dpo":
                rej, noise_r = Hh.tiny_batch(student, B=1, seed=5000 + idx)
                rej["input_ids"][:, :16] = batch["input_ids"][:, :16]
                rej["labels"][:, :16] = batch["labels"][:, :16]
                inputs = dict(chosen_input_ids=batch["input_ids"], chosen_labels=batch["labels"], chosen_attention_mask=batch["attention_mask"],
                              rejected_input_ids=rej["input_ids"], rejected_labels=rej["labels"], rejected_attention_mask=rej["attention_mask"],
                              images=batch["images"], moe_noise=([n.to(dev) for n in noise], [n.to(dev) for n in noise_r]))
            else:
                inputs = dict(batch, moe_noise=[n.to(dev) for n in noise])
            mine.append(tr.training_step(student, inputs))
        t = torch.stack(mine).float().sum()
        if world > 1:
            dist.all_reduce(t)
        losses.append(float(t) / GLOBAL)
        gnorms.append(tr.optimizer.grad_norm(1.0 / GLOBAL))
    # numpy, not torch tensors: torch.multiprocessing would hand CPU tensors over as shared-memory file descriptors, which die with this process
    sd = {k: v.detach().float().cpu().numpy() for k, v in student.state_dict().items() if "image_tower" not in k}
    if rank == 0:
        q.put((losses, gnorms, sd))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def _launch(world, loss_kind, graphs=False):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_run, args=(r, world, port, q, loss_kind, graphs)) for r in range(world)]
    for p in procs:
        p.start()
    out = q.get(timeout=300)
    assert not (isinstance(out[0], str) and out[0] == "error"), out[1]
    out = (out[0], out[1], {k: torch.from_numpy(v) for k, v in out[2].items()})
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    return out


def _same_weights(sd1, sd2, lr=1e-3):
    """Adam moves every element by ~lr per step whatever the gradient's size, so an element whose gradient is rounding noise may step the
    other way on the two sides: the allowance is 2e-3 of the tensor norm plus 10 % of the distance Adam can travel in STEPS steps.  Ranks
    that had NOT exchanged gradients would differ by about that full distance on most elements."""
    assert len(sd1) > 10
    for k in sd1:
        a, b = sd1[k], sd2[k]
        assert (a - b).norm().item() <= 2e-3 * a.norm().item() + 0.1 * lr * STEPS * a.numel() ** 0.5, k


@pytest.mark.parametrize("loss_kind", ["kd_lm", "sigmoid"])
def test_two_gpus_match_one_gpu_at_equal_global_batch(loss_kind):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    l1, g1, sd1 = _launch(1, loss_kind)
    l2, g2, sd2 = _launch(2, loss_kind)
    for s in range(STEPS):
        assert abs(l1[s] - l2[s]) < 2e-3 * abs(l1[s]) + 1e-4, (s, l1, l2)
        assert abs(g1[s] - g2[s]) < 1e-2 * abs(g1[s]) + 1e-6, (s, g1, g2)
    _same_weights(sd1, sd2)


def test_two_gpus_with_cuda_graphs_match_one_gpu():
    """Same equivalence with CUDA graphs ON (the way bench.py and the entry points run): from the third step on every micro-batch replays a
    captured graph, the all-reduce follows the replay -- the sequence must still equal the single-GPU run (explicit router noise is a
    static graph input, so routing is identical on all sides)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    l1, g1, sd1 = _launch(1, "kd_lm", graphs=True)
    l2, g2, sd2 = _launch(2, "kd_lm", graphs=True)
    for s in range(STEPS):
        assert abs(l1[s] - l2[s]) < 2e-3 * abs(l1[s]) + 1e-4, (s, l1, l2)
        assert abs(g1[s] - g2[s]) < 1e-2 * abs(g1[s]) + 1e-6, (s, g1, g2)
    _same_weights(sd1, sd2)
