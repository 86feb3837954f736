"""CPU-only (gloo): recompute of the spatial cells (torchgems.recompute) in the trainers.

The spatial layers here are a test-only halo convolution on CPU: a _SpatialTopology layer that exchanges its
edge columns through the same choke point as conv_spatial / Pool (_SpatialTopology._exchange) with a CPU
transport (torch slicing + exchange_strips over gloo), then convolves the padded tile with F.conv2d.  The
product's kernels are CUDA-only; tests/test_gpu_recompute.py checks them.

1. train_model_spatial on 2 tiles + a join rank, and train_model on a 2-stage pipeline: recompute=True gives the
   same loss sequence, BatchNorm running buffers and parameters as recompute=False, bit for bit, and the same
   state_dict keys.  The recompute calls no transport: the transport raises when called during backward.
2. The SP and GEMS+SP scripts accept --recompute, in the CPU control-flow mode of tests/test_benchmark_scripts.py."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F

from tests.test_benchmark_scripts import ROOT, SPATIAL_RUNS, _run

P, IMG, BATCH, STEPS = 2, 16, 4, 3


def _make_layers():
    from mpi4dl_b200.torchgems import spatial

    class HaloConv(nn.Conv2d, spatial._SpatialTopology):
        """3x3 convolution of a vertical tile whose left / right padding columns come from the neighbours."""

        def __init__(self, rank, parts, cin, cout):
            nn.Conv2d.__init__(self, cin, cout, 3, bias=False)
            self._init_topology(rank, 1, parts, "vertical")
            self.get_neighbours()
            self.rank_neighbours = [-1] * 9
            if self.neighbours is not None:
                self.get_neighbours_rank()

        def forward(self, x):
            with torch.no_grad():
                s = self._exchange(x, 1, 1)
            edge = torch.zeros(x.shape[0], x.shape[1], x.shape[2], 1)
            xp = torch.cat([s[3] if s[3] is not None else edge, x, s[5] if s[5] is not None else edge], dim=3)
            return F.conv2d(xp, self.weight, padding=(1, 0))

    return HaloConv


class CpuTransport:
    """Strips cut with torch slicing, moved with exchange_strips.  Raises while `forbid` is set."""

    def __init__(self):
        self.calls = 0
        self.forbid = False

    def exchange(self, layer, x, hh, hw, mask, ranks):
        from mpi4dl_b200.torchgems import halo_transport as ht
        if self.forbid:
            raise RuntimeError("halo exchange during backward")
        self.calls += 1
        H, W = x.shape[2], x.shape[3]
        send, recv = [None] * 9, [None] * 9
        for i in range(9):
            if i != 4 and mask[i]:
                dr, dc = ht._DIRS[i]
                rs = {-1: slice(0, hh), 0: slice(0, H), 1: slice(H - hh, H)}[dr]
                cs = {-1: slice(0, hw), 0: slice(0, W), 1: slice(W - hw, W)}[dc]
                send[i] = x[:, :, rs, cs].contiguous()
                recv[i] = torch.empty(ht.strip_shape(i, *x.shape, hh, hw), dtype=x.dtype)
        ht.exchange_strips(send, recv, ranks)
        return recv


def _model(HaloConv, rank, parts):
    torch.manual_seed(5)
    cell = lambda ci, co: nn.Sequential(HaloConv(rank % parts, parts, ci, co), nn.BatchNorm2d(co), nn.ReLU())  # noqa: E731
    return nn.Sequential(cell(3, 8), cell(8, 8), nn.AdaptiveAvgPool2d(2), nn.Flatten(), nn.Linear(32, 10))


def _batch(step):
    g = torch.Generator().manual_seed(40 + step)
    return torch.randn(BATCH, 3, IMG, IMG, generator=g), torch.randint(0, 10, (BATCH,), generator=g)


def _steps(tm, tr, data):
    losses = []
    backward = tm.backward_pass

    def guarded(*a, **k):                       # the recompute in backward must not exchange
        tr.forbid = True
        try:
            backward(*a, **k)
        finally:
            tr.forbid = False

    tm.backward_pass = guarded
    for step in range(STEPS):
        x, y = _batch(step)
        loss, _ = tm.run_step(data(x), y)
        tm.update()
        losses.append(float(loss))
    # numpy arrays: tensors sent through a multiprocessing queue would need the sender alive
    bn = {k: v.numpy().copy() for k, v in tm.models.state_dict().items() if "running" in k or "num_batches" in k}
    params = [p.detach().numpy().copy() for p in tm.models.parameters()]
    return losses, bn, params, sorted(tm.models.state_dict().keys())


def _worker(rank, world, kind, port, q):
    import sys
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      CUDA_VISIBLE_DEVICES="")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    from mpi4dl_b200.torchgems import halo_transport
    from mpi4dl_b200.torchgems.mp_pipeline import model_generator, train_model
    from mpi4dl_b200.torchgems.train_spatial import split_input, train_model_spatial
    tr = CpuTransport()
    halo_transport.set_transport(tr)
    HaloConv = _make_layers()
    out = {}
    for recompute in (False, True):
        if kind == "spatial":
            model = _model(HaloConv, rank, P)
            shapes = [(BATCH, 8, IMG, IMG // P), (BATCH, 10)]
            gen = model_generator(model=model, split_size=2, input_size=(BATCH, 3, IMG, IMG), balance=[2, 3],
                                  shape_list=shapes)
            gen.ready_model(split_rank=0 if rank < P else 1)
            tm = train_model_spatial(gen, rank, BATCH, 1, spatial_size=1, num_spatial_parts=P, slice_method="vertical",
                                     recompute=recompute)
            data = (lambda x: split_input(x, IMG, "vertical", rank, [P])) if rank < P else (lambda x: x)
        else:
            model = _model(HaloConv, 0, 1)
            gen = model_generator(model=model, split_size=2, input_size=(BATCH, 3, IMG, IMG), balance=[2, 3],
                                  shape_list=[(BATCH, 8, IMG, IMG), (BATCH, 10)])
            gen.ready_model(split_rank=rank)
            tm = train_model(gen, rank, BATCH, 1, recompute=recompute)
            data = lambda x: x  # noqa: E731
        calls0 = tr.calls
        wrapped = sorted(n for n, c in tm.models.named_children() if "forward" in c.__dict__)
        out[recompute] = _steps(tm, tr, data) + (tr.calls - calls0, wrapped)
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def _spawn(world, kind, port):
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    ps = [ctx.Process(target=_worker, args=(r, world, kind, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    got = dict(q.get() for _ in ps)
    for p in ps:
        p.join(120)
        assert p.exitcode == 0
    return got


@pytest.mark.parametrize("kind,world,port", [("spatial", P + 1, 29640), ("pipeline", 2, 29641)])
def test_trainer_recompute_matches_plain(kind, world, port):
    got = _spawn(world, kind, port)
    for r in range(world):
        plain, rec = got[r][False], got[r][True]
        assert rec[0] == plain[0], (r, rec[0], plain[0])                   # loss sequence
        assert rec[1].keys() == plain[1].keys() and all(np.array_equal(rec[1][k], plain[1][k]) for k in plain[1]), r
        assert len(rec[2]) == len(plain[2]) and all(np.array_equal(a, b) for a, b in zip(rec[2], plain[2])), r
        assert rec[3] == plain[3], r                                       # state_dict keys
        assert rec[4] == plain[4], r                                       # exchanges: forward only, same count
        assert plain[5] == [], r
        first_stage = r < P if kind == "spatial" else r == 0
        assert rec[5] == (["0", "1"] if first_stage else []), (r, rec[5])
    if kind == "spatial":                                                  # one exchange per cell and step
        assert all(got[r][True][4] == 2 * STEPS for r in range(P))
    assert any(abs(b).sum() > 0 for b in got[0][True][1].values())


RECOMPUTE_RUNS = [r for r in SPATIAL_RUNS if r[0] in ("sp_amoebanet_d2_4tiles", "gems_sp_resnet")]


@pytest.mark.parametrize("idx,name,nproc,script,flags", [(110 + i,) + r for i, r in enumerate(RECOMPUTE_RUNS)],
                         ids=[r[0] for r in RECOMPUTE_RUNS])
def test_spatial_benchmark_script_control_flow_recompute(idx, name, nproc, script, flags):
    hooks = os.path.join(ROOT, "tests", "cpu_smoke_hooks")
    _run(idx, nproc, script, flags + " --recompute",
         {"SPCONV_TEST_CPU_SMOKE": "1", "PYTHONPATH": os.pathsep.join([hooks, ROOT, os.environ.get("PYTHONPATH", "")])})
