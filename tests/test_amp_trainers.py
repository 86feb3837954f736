"""CPU-only (gloo): the trainers' amp_dtype under torch.autocast("cpu", dtype=torch.bfloat16).

1. train_model on a 3-stage pipeline of plain PyTorch layers: with amp_dtype=torch.bfloat16 the receive and gradient
   buffers are bf16 while the parameters, their gradients and the optimizer state stay fp32; amp_dtype=None keeps
   today's dtypes (the parameters' dtype throughout).
2. Every training script with --dtype accepts --dtype bf16-amp, in the same CPU control-flow mode as
   tests/test_benchmark_scripts.py (spatial layers swapped for halo-less PyTorch ops, numerics not checked)."""
import math
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from tests.test_benchmark_scripts import ROOT, RUNS, SPATIAL_RUNS, _run

WORLD, BATCH = 3, 4


def _model():
    torch.manual_seed(7)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), nn.BatchNorm2d(8), nn.ReLU(), nn.Conv2d(8, 8, 3, stride=2, padding=1),
                         nn.ReLU(), nn.Conv2d(8, 4, 3, padding=1), nn.Flatten(), nn.Linear(4 * 8 * 8, 10))


def _worker(rank, amp, port, q):
    import sys
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(WORLD),
                      CUDA_VISIBLE_DEVICES="")
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    torch.set_num_threads(1)
    from mpi4dl_b200.torchgems.mp_pipeline import model_generator, train_model
    gen = model_generator(model=_model(), split_size=WORLD, input_size=(BATCH // 2, 3, 16, 16), balance=[3, 2, 3])
    gen.ready_model(split_rank=rank)
    tm = train_model(gen, rank, BATCH, epochs=1, parts=2, amp_dtype=torch.bfloat16 if amp else None)
    losses, grads = [], []
    for step in range(2):
        g = torch.Generator().manual_seed(10 + step)
        loss, _ = tm.run_step(torch.randn(BATCH, 3, 16, 16, generator=g), torch.randint(0, 10, (BATCH,), generator=g))
        grads.append(sorted({str(p.grad.dtype) for p in tm.models.parameters()}))
        tm.update()
        losses.append(float(loss))
    bufs = [t for b in tm.input_x_list for t in tm._as_list(b)] if rank else []
    if rank != WORLD - 1:
        bufs += tm._as_list(tm.grad_overhead)
    opt_state = {str(v.dtype) for s in tm.optimizer.state.values() for v in s.values() if torch.is_tensor(v)}
    bn = [m for m in tm.models.modules() if isinstance(m, nn.BatchNorm2d)]
    q.put((rank, dict(bufs=sorted({str(t.dtype) for t in bufs}), params=sorted({str(p.dtype) for p in tm.models.parameters()}),
                      grads=grads, opt=sorted(opt_state), bn=sorted({str(t.dtype) for m in bn for t in m.buffers()
                                                                   if t.is_floating_point()}),
                      losses=losses)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("amp", [True, False], ids=["bf16_amp", "none"])
def test_train_model_amp_dtypes(amp):
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    ps = [ctx.Process(target=_worker, args=(r, amp, 29610 + int(amp), q)) for r in range(WORLD)]
    for p in ps:
        p.start()
    got = dict(q.get() for _ in ps)
    for p in ps:
        p.join(60)
        assert p.exitcode == 0
    want_buf = "torch.bfloat16" if amp else "torch.float32"
    for r in range(WORLD):
        assert got[r]["bufs"] == [want_buf], (r, got[r])
        assert got[r]["params"] == ["torch.float32"], (r, got[r])
        assert got[r]["grads"] == [["torch.float32"]] * 2, (r, got[r])
        assert got[r]["opt"] in ([], ["torch.float32"]), (r, got[r])
    assert got[0]["bn"] == ["torch.float32"]
    assert all(math.isfinite(v) for v in got[WORLD - 1]["losses"])


AMP_RUNS = [r for r in RUNS if r[0] in ("lp_resnet_2", "gems_resnet_2")]
AMP_SPATIAL_RUNS = [r for r in SPATIAL_RUNS if r[0] in ("sp_amoebanet_d2_4tiles", "gems_sp_resnet")]


@pytest.mark.parametrize("idx,name,nproc,script,flags", [(90 + i,) + r for i, r in enumerate(AMP_RUNS)],
                         ids=[r[0] for r in AMP_RUNS])
def test_benchmark_script_runs_bf16_amp(idx, name, nproc, script, flags):
    _run(idx, nproc, script, flags + " --dtype bf16-amp", {})


@pytest.mark.parametrize("idx,name,nproc,script,flags", [(100 + i,) + r for i, r in enumerate(AMP_SPATIAL_RUNS)],
                         ids=[r[0] for r in AMP_SPATIAL_RUNS])
def test_spatial_benchmark_script_control_flow_bf16_amp(idx, name, nproc, script, flags):
    hooks = os.path.join(ROOT, "tests", "cpu_smoke_hooks")
    _run(idx, nproc, script, flags + " --dtype bf16-amp",
         {"SPCONV_TEST_CPU_SMOKE": "1", "PYTHONPATH": os.pathsep.join([hooks, ROOT, os.environ.get("PYTHONPATH", "")])})
