"""-m gpu: spatial layers of an fp32 model under torch.autocast("cuda", dtype=torch.bfloat16).

The contract is nn.Conv2d's under autocast: activations and the rounded weights are bf16, the parameters, their .grad
and the BatchNorm buffers stay fp32.  conv_spatial / local_conv2d round the weight and bias inside _ConvSpatialFn and
return the wgrad kernel's fp32 dW unrounded.

1. One layer on one tile (the middle tile of a 3x3 grid, halo strips injected in place of the exchange), for 1x1 s1 /
   s2, 3x3 s1 / s2 (C = 3 too), 1x7 and 7x1, with and without bias, and local_conv2d(padding=0): against a bf16 layer
   holding W.to(bf16), y and dx are bit-identical, after the bf16 layer's y and dx were seen to be bit-reproducible
   run to run.  The weight and bias gradients need not be: every wgrad kernel (pw_wgrad_kernel, wgrad_tap_kernel,
   wgrad_direct_kernel, bias_grad_kernel) adds partial sums into dW / db with fp32 atomics, in no fixed order.  So
   dW / db are checked to be fp32, within tests/test_gpu_tc_coverage.py's per-element fp64 bound for the bf16 wgrad
   kernels, and not bf16-representable (they were not rounded on the way back).  The same holds with
   exact_backward on, through the 4-process peer-transport harness of tests/test_gpu_exact_backward.py, where the
   fp32 layer's halo slots are bf16-sized and a second run without autocast gets its own fp32 slots.
2. fp32 master weights keep updates below half a bf16 ulp that a .to(bf16) copy loses.
3. The first cells of amoebanetd_spatial and resnet_spatial: no fp32 direct-conv kernel runs, the fused BatchNorm
   (AmoebaNet-D) runs on bf16, every .grad and BN buffer is fp32 and finite.
4. A 4-tile chain's autocast forward + backward replays from a CUDA graph to the eager step.
5. train_model_spatial(amp_dtype=torch.bfloat16) on 2 tiles + join + tail tracks the fp32 single-process model.
6. Under fp16 autocast the layers warn once and compute exactly what they compute without autocast."""
import math
import os
import warnings

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from oracle import spatial_oracle as so
from tests import test_gpu_tc_coverage as cov

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
BF16 = torch.bfloat16
N, H, W = 2, 32, 64

# (C, K, R, S, stride, bias)
LAYER_CASES = [(64, 96, 1, 1, 1, True), (64, 96, 1, 1, 2, False), (32, 48, 3, 3, 1, True), (32, 48, 3, 3, 2, False),
               (3, 32, 3, 3, 2, True), (3, 16, 3, 3, 1, False), (32, 32, 1, 7, 1, True), (32, 32, 7, 1, 1, False)]


def _master(K, Cc, R, S, bias, seed):
    """fp32 weights and bias that bf16 cannot represent"""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(K, Cc, R, S, generator=g) / math.sqrt(Cc * R * S), (torch.randn(K, generator=g) if bias else None)


def _conv_layer(Cc, K, R, S, st, w, b, dtype, mask=None, strips=None):
    """conv_spatial on one tile; with `strips`, they stand in for what the neighbours in `mask` would send"""
    from mpi4dl_b200.torchgems.spatial import conv_spatial
    m = conv_spatial(local_rank=0, spatial_size=1, num_spatial_parts=1, in_channels=Cc, out_channels=K, kernel_size=(R, S),
                     stride=st, padding=((R - 1) // 2, (S - 1) // 2), bias=b is not None, slice_method="square")
    with torch.no_grad():
        m.weight.copy_(w)
        if b is not None:
            m.bias.copy_(b)
    m = m.to(DEV).to(dtype)
    m.exact_backward = False
    if strips is not None and any(s is not None for s in strips):
        m.neighbours = list(mask)
        dev_strips = [s.to(DEV) if s is not None else None for s in strips]
        m._exchange = lambda x, hh, hw: dev_strips
    return m


def _step(m, x, dy, amp):
    xx = x.to("cuda").requires_grad_(True)              # the current device (the transport workers set theirs)
    with torch.autocast("cuda", dtype=BF16, enabled=amp):
        y = m(xx)
    y.backward(dy.to("cuda"))
    return [y.detach(), xx.grad, m.weight.grad, m.bias.grad if m.bias is not None else None]


def _zero(m):
    for p in m.parameters():
        p.grad = None


def _compare(amp_m, bf_m, x, dy, what):
    """the fp32 layer under autocast against the bf16 layer; returns (dw, db) of the fp32 layer"""
    runs = []
    for _ in range(2):
        _zero(bf_m)
        runs.append(_step(bf_m, x.to(BF16), dy, False))
    for name, a, b in zip(("y", "dx"), *runs):
        assert torch.equal(a, b), "%s: bf16 %s is not bit-reproducible run to run" % (what, name)
    y_ref, dx_ref, dw_ref, db_ref = runs[0]
    _zero(amp_m)
    y, dx, dw, db = _step(amp_m, x.float(), dy, True)
    assert y.dtype == BF16 and torch.equal(y, y_ref), what
    assert dx.dtype == torch.float32 and torch.equal(dx, dx_ref.float()), what
    assert all(p.dtype == torch.float32 for p in amp_m.parameters()), what
    for name, g, ref in (("dw", dw, dw_ref), ("db", db, db_ref)):
        if ref is None:
            continue
        assert g.dtype == torch.float32, (what, name)
        assert not torch.equal(g, g.to(BF16).float()), "%s: %s came back rounded to bf16" % (what, name)
    return dw, db


@pytest.mark.parametrize("Cc,K,R,S,st,bias", LAYER_CASES, ids=["C%dK%d_%dx%ds%d_%s" % (c[:5] + ("b" if c[5] else "nob",))
                                                                for c in LAYER_CASES])
def test_conv_spatial_tile_matches_bf16_layer(Cc, K, R, S, st, bias):
    c = cov.Case(Cc, K, R, S, st, N, H, W, bias, frozenset(), "")
    mask = so.neighbour_mask("square", 9, 4, R, S)
    x, _, _, dy, strips = cov.make_inputs(c, mask)
    w32, b32 = _master(K, Cc, R, S, bias, Cc * 1000 + K * 10 + R * S + st)
    amp_m = _conv_layer(Cc, K, R, S, st, w32, b32, torch.float32, mask, strips)
    bf_m = _conv_layer(Cc, K, R, S, st, w32.to(BF16), b32.to(BF16) if bias else None, BF16, mask, strips)
    dw, db = _compare(amp_m, bf_m, x, dy, "conv %s" % (c[:5],))
    ref, A = cov.reference(x, w32.to(BF16), b32.to(BF16) if bias else None, dy, strips, st)
    cov.check_grad(dw, ref["dw"], A["dw"], "dw")
    if bias:
        cov.check_grad(db, ref["db"], A["db"], "db")


def test_local_conv2d_valid_matches_bf16_layer():
    from mpi4dl_b200.torchgems.spatial import local_conv2d
    Cc, K = 16, 32
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, Cc, H, W, generator=g).to(BF16)
    dy = torch.randn(N, K, H - 2, W - 2, generator=g).to(BF16)
    w32, b32 = _master(K, Cc, 3, 3, True, 4)
    mods = []
    for dtype, w, b in ((torch.float32, w32, b32), (BF16, w32.to(BF16), b32.to(BF16))):
        m = local_conv2d(Cc, K, 3, padding=0)
        with torch.no_grad():
            m.weight.copy_(w)
            m.bias.copy_(b)
        mods.append(m.to(DEV).to(dtype))
    dw, db = _compare(mods[0], mods[1], x, dy, "local_conv2d")
    xd, dyd = x.double(), dy.double()
    for got, ref, A in ((dw, torch.nn.grad.conv2d_weight(xd, w32.shape, dyd), torch.nn.grad.conv2d_weight(xd.abs(), w32.shape,
                                                                                                          dyd.abs())),
                        (db, dyd.sum((0, 2, 3)), dyd.abs().sum((0, 2, 3)))):
        cov.check_grad(got, ref, A, "local_conv2d grad")


# ---- 1b. exact backward through the peer transport, 4 square tiles ---------------------------------------------------
def _exact_worker(rank, P, port, ngpu, q):
    from tests.test_gpu_exact_backward import _init
    dev = _init(rank, P, "peer", port, ngpu)
    from mpi4dl_b200.torchgems import spatial
    errs = []
    try:
        g = torch.Generator().manual_seed(21)
        full = torch.randn(1, 16, 24, 32, generator=g).to(BF16).float()
        hs, ws = so.tile_slices("square", P, rank, 24, 32)
        x = full[:, :, hs, ws].contiguous()
        for (K, R, S, st) in [(16, 3, 3, 1), (8, 1, 7, 1), (8, 7, 1, 1), (16, 3, 3, 2)]:
            w32, b32 = _master(K, 16, R, S, True, K + R * 10 + S + st)
            mods = []
            for dtype, w, b in ((torch.float32, w32, b32), (BF16, w32.to(BF16), b32.to(BF16))):
                m = spatial.conv_spatial(rank, 1, P, 16, K, (R, S), stride=st, padding=((R - 1) // 2, (S - 1) // 2),
                                         slice_method="square")
                with torch.no_grad():
                    m.weight.copy_(w)
                    m.bias.copy_(b)
                mods.append(m.to(dev).to(dtype))
                assert m.exact_backward
            Ho, Wo = (x.shape[2] - 1) // st + 1, (x.shape[3] - 1) // st + 1
            dy = torch.randn(1, K, Ho, Wo, generator=torch.Generator().manual_seed(rank + 7 * K)).to(BF16)
            what = "rank %d %dx%d s%d" % (rank, R, S, st)
            try:
                dw, db = _compare(mods[0], mods[1], x, dy, what)
                # fp64 reference: the tile with its halo is the zero-padded full image's window around the tile
                ph, pw = (R - 1) // 2, (S - 1) // 2
                xp = torch.nn.functional.pad(full.double(), (pw, pw, ph, ph))[:, :, hs.start:hs.stop + 2 * ph,
                                                                             ws.start:ws.stop + 2 * pw]
                dyd, wsh = dy.double(), (K, 16, R, S)
                cov.check_grad(dw, torch.nn.grad.conv2d_weight(xp, wsh, dyd, st),
                               torch.nn.grad.conv2d_weight(xp.abs(), wsh, dyd.abs(), st), what + " dw")
                cov.check_grad(db, dyd.sum((0, 2, 3)), dyd.abs().sum((0, 2, 3)), what + " db")
            except AssertionError as e:
                errs.append(str(e))
            # halo slots: bf16-sized for the autocast run; a run without autocast gets its own fp32 slots
            fwd = {k[1]: v for k, v in mods[0].__dict__.get("_halo_slots", {}).items() if k[0] != "reverse"}
            if list(fwd) != [BF16]:
                errs.append((what, "slots after the autocast runs", list(fwd)))
            _zero(mods[0])
            _step(mods[0], x, dy.float(), False)
            fwd = {k[1]: v for k, v in mods[0].__dict__.get("_halo_slots", {}).items() if k[0] != "reverse"}
            if set(fwd) != {BF16, torch.float32} or fwd[BF16]["data"] == fwd[torch.float32]["data"] or \
                    not fwd[BF16]["slot_bytes"] < fwd[torch.float32]["slot_bytes"]:
                errs.append((what, "slots with and without autocast", {str(k): v["slot_bytes"] for k, v in fwd.items()}))
        torch.cuda.synchronize()
    except Exception as ex:  # report instead of hanging the peers
        import traceback
        errs.append(("exception", repr(ex), traceback.format_exc()[-1500:]))
    q.put((rank, errs))
    try:
        dist.barrier()
        dist.destroy_process_group()
    except Exception:
        pass


def test_exact_backward_through_peer_transport():
    from tests.test_gpu_exact_backward import _spawn
    res = _spawn(_exact_worker, 4, (29861, torch.cuda.device_count()))
    bad = [(r, e) for r, e in res if e]
    assert not bad, bad


# ---- 2. master weights --------------------------------------------------------------------------------------------
def test_master_weights_keep_updates_below_half_a_bf16_ulp():
    """dW does not depend on W for loss = sum(y * G), so every step applies the same lr * g; lr is chosen so that
    |lr * g| is below half a bf16 ulp of every weight"""
    Cc, K = 8, 16
    g = torch.Generator().manual_seed(8)
    x = torch.randn(N, Cc, H, W, generator=g).to(BF16)
    G = torch.randn(N, K, H, W, generator=g).to(BF16)
    w0 = (torch.rand(K, Cc, 3, 3, generator=g) * 0.04 + 0.03) * torch.sign(torch.randn(K, Cc, 3, 3, generator=g))
    w0 = w0.to(BF16).float()                             # both copies start from the same values
    amp_m = _conv_layer(Cc, K, 3, 3, 1, w0, None, torch.float32)
    bf_m = _conv_layer(Cc, K, 3, 3, 1, w0, None, BF16)
    _step(amp_m, x.float(), G, True)
    grad = amp_m.weight.grad.detach().clone()
    half_ulp = 2.0 ** (torch.floor(torch.log2(w0.abs())) - 8)
    lr = 0.25 * float((half_ulp.to(DEV) / grad.abs().clamp_min(1e-30)).min())
    opts = [torch.optim.SGD(m.parameters(), lr=lr) for m in (amp_m, bf_m)]
    for _ in range(10):
        for m, opt, amp in ((amp_m, opts[0], True), (bf_m, opts[1], False)):
            opt.zero_grad(set_to_none=True)
            _step(m, x.float() if amp else x, G, amp)
            opt.step()
    assert torch.equal(bf_m.weight.detach().float().cpu(), w0), "the bf16 copy moved"
    moved = (amp_m.weight.detach() - w0.to(DEV)).double()
    want = -10 * lr * grad.double()
    tol = 10 * 2.0 ** -24 * w0.abs().double().to(DEV) * 2
    assert (want.abs() > 0).all()
    assert ((moved - want).abs() <= tol).all(), float(((moved - want).abs() / tol).max())


# ---- 3. model level -----------------------------------------------------------------------------------------------
def _amoebanet_cells():
    from mpi4dl_b200.models import amoebanet
    m = amoebanet.amoebanetd_spatial(0, 1, 1, mp_size=2, slice_method="square", num_classes=10, num_layers=6,
                                     num_filters=64)
    return nn.Sequential(*list(m.children())[:6]), 128


def _resnet_cells():
    from mpi4dl_b200.models import resnet_spatial
    m = resnet_spatial.get_resnet_v2((1, 3, 64, 64), 29, local_rank=0, mp_size=2, num_spatial_parts=1)
    return nn.Sequential(*list(m.children())[:4]), 64


def _cells_worker(which, q):
    import sys
    sys.path.insert(0, ROOT)
    errs = []
    try:
        from mpi4dl_b200.torchgems.spatial import conv_spatial, local_conv2d
        torch.manual_seed(0)
        model, img = (_amoebanet_cells if which == "amoebanet" else _resnet_cells)()
        model = model.to(DEV).train()
        x = torch.randn(2, 3, img, img, device=DEV)

        def run():
            with torch.autocast("cuda", dtype=BF16):
                y = model(x)
            y = y[0] if isinstance(y, tuple) else y
            y.float().square().mean().backward()
            torch.cuda.synchronize()
            return y

        y, kernels = cov.traced(run)
        if y.dtype != BF16:
            errs.append(("output dtype", str(y.dtype)))
        direct32 = sorted(k for k in kernels if "direct" in k[0] and k[1][:1] == ("float",))
        if direct32:
            errs.append(("fp32 direct kernels ran", direct32))
        if which == "amoebanet" and not any(k[0] == "bn_stats_kernel" and k[1][:1] == ("__nv_bfloat16",) for k in kernels):
            errs.append(("fused BatchNorm did not run on bf16", sorted(kernels)))
        convs = [m for m in model.modules() if isinstance(m, (conv_spatial, local_conv2d))]
        if not convs or any(m.weight.grad is None for m in convs):
            errs.append("a conv layer got no weight gradient")
        for n, p in model.named_parameters():
            # (resnet_layer keeps a BatchNorm for the conv order it does not run: no .grad)
            if p.dtype != torch.float32 or (p.grad is not None and (p.grad.dtype != torch.float32 or
                                                                    not torch.isfinite(p.grad).all())):
                errs.append((n, str(p.dtype), None if p.grad is None else str(p.grad.dtype)))
        for n, b in model.named_buffers():
            if b.is_floating_point() and (b.dtype != torch.float32 or not torch.isfinite(b).all()):
                errs.append((n, str(b.dtype)))
    except Exception as ex:
        import traceback
        errs.append(("exception", repr(ex), traceback.format_exc()[-1500:]))
    q.put(errs)


@pytest.mark.parametrize("which", ["amoebanet", "resnet"])
def test_model_cells_run_bf16_with_fp32_state(which):
    """in a child process: run in the pytest process, this trace was followed by lost launch records in the
    kernel-coverage tests' traces (tests/test_gpu_direct_pool_coverage.py)"""
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    p = ctx.Process(target=_cells_worker, args=(which, q))
    p.start()
    errs = q.get()
    p.join(60)
    assert not errs, errs


# ---- 4. CUDA graph ------------------------------------------------------------------------------------------------
def _graph_worker(rank, P, port, ngpu, q):
    from tests.test_gpu_exact_backward import _chain, _init
    dev = _init(rank, P, "peer", port, ngpu)
    from mpi4dl_b200.torchgems import spatial
    errs = []
    try:
        g = torch.Generator().manual_seed(5)
        full, G = torch.randn(1, 4, 32, 32, generator=g), torch.randn(1, 8, 16, 16, generator=g)
        hs, ws = so.tile_slices("square", P, rank, 32, 32)
        ohs, ows = so.tile_slices("square", P, rank, 16, 16)
        x, gt = full[:, :, hs, ws].contiguous().to(dev), G[:, :, ohs, ows].contiguous().to(dev)
        torch.manual_seed(0)
        model = _chain(spatial, rank, P, True).to(dev)

        def close(a, b):
            """the weight gradients are summed with atomics (see the module docstring)"""
            return bool(((a - b).abs() <= 1e-5 * b.abs().max()).all())

        def step(xx):
            with torch.autocast("cuda", dtype=BF16, cache_enabled=False):
                y = model(xx)
            (y.float() * gt).sum().backward()

        xx = x.clone().requires_grad_(True)
        step(xx)
        eager_dx, eager_dw = xx.grad.clone(), [p.grad.clone() for p in model.parameters()]
        if not all(p.grad.dtype == torch.float32 for p in model.parameters()):
            errs.append("grads not fp32")
        for p in model.parameters():
            p.grad = None
        sx = x.clone().requires_grad_(True)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step(sx)
        for rep in range(3):
            graph.replay()
            torch.cuda.synchronize()
            if not torch.equal(sx.grad, eager_dx) or not all(close(p.grad, e) for p, e in zip(model.parameters(), eager_dw)):
                errs.append(("graph replay", rep, float((sx.grad - eager_dx).abs().max())))
        del graph
        torch.cuda.synchronize()
    except Exception as ex:  # report instead of hanging the peers
        import traceback
        errs.append(("exception", repr(ex), traceback.format_exc()[-1500:]))
    q.put((rank, errs))
    try:
        dist.barrier()
        dist.destroy_process_group()
    except Exception:
        pass


def test_chain_replays_in_a_cuda_graph():
    from tests.test_gpu_exact_backward import _spawn
    res = _spawn(_graph_worker, 4, (29862, torch.cuda.device_count()))
    bad = [(r, e) for r, e in res if e]
    assert not bad, bad


# ---- 5. trainer ---------------------------------------------------------------------------------------------------
def _trainer_worker(rank, method, width, port, ngpu, q):
    import sys
    sys.path.insert(0, ROOT)
    from tests import test_gpu_sp_trainer as spt
    world = spt.P + spt.SPLIT - 1
    multi = ngpu >= world
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank if multi else 0), SPCONV_DIST_BACKEND="nccl" if multi else "gloo",
                      SPCONV_ARENA_MB="64")
    from mpi4dl_b200 import _lib
    from mpi4dl_b200.torchgems import comm as gems_comm
    from mpi4dl_b200.torchgems.mp_pipeline import model_generator
    from mpi4dl_b200.torchgems.spatial import Pool, conv_spatial
    from mpi4dl_b200.torchgems.train_spatial import get_shapes_spatial, split_input, train_model_spatial
    gems_comm.initialize_cuda()
    P = spt.P
    mpi_comm = gems_comm.MPIComm(split_size=spt.SPLIT, ENABLE_MASTER=False, ENABLE_SPATIAL=True, num_spatial_parts=P,
                                 spatial_size=1)
    sync = gems_comm.SyncAllreduce(mpi_comm)
    local_rank, split_rank = mpi_comm.rank, mpi_comm.split_rank
    sp = dict(local_rank=local_rank % P, spatial_size=1, num_spatial_parts=P, slice_method=method)
    model = nn.Sequential(*spt._layers(
        lambda ci, co, k, s: conv_spatial(in_channels=ci, out_channels=co, kernel_size=k, stride=s, padding=k // 2, **sp),
        lambda: Pool(operation="AvgPool2d", kernel_size=3, stride=1, padding=1, **sp), width))
    B, IMG = spt.BATCH, spt.IMG
    full = [(B, width, IMG // 2, IMG // 2), (B, 4, IMG // 2, IMG // 2), (B, 10)]
    gen = model_generator(model=model, split_size=spt.SPLIT, input_size=(B, 3, IMG, IMG), balance=spt.BALANCE,
                          shape_list=get_shapes_spatial(full, method, 1, [P], 1))
    gen.ready_model(split_rank=split_rank)
    opt = torch.optim.SGD(gen.models.parameters(), lr=0.005, momentum=0.9)
    tm = train_model_spatial(gen, local_rank, B, epochs=1, spatial_size=1, num_spatial_parts=P, optimizer=opt, parts=1,
                             slice_method=method, mpi_comm=mpi_comm, amp_dtype=BF16)
    sync.sync_model_spatial(gen)
    bufs = [t for b in tm.input_x_list for t in (b if isinstance(b, list) else [b]) for t in tm._as_list(t)]
    losses = []
    for step in range(spt.STEPS):
        x, y = spt._batch(step)
        if local_rank < P:
            x = split_input(x, IMG, method, local_rank, [P])
        loss, _ = tm.run_step(x, y)
        if local_rank < P:
            sync.apply_allreduce(gen, mpi_comm.spatial_allreduce_grp)
        tm.update()
        losses.append(float(loss))
    dtypes = sorted({str(p.dtype) for p in gen.models.parameters()} | {str(p.grad.dtype) for p in gen.models.parameters()})
    q.put((local_rank, losses, int(_lib.lib().spc_launch_count(0)), dtypes, sorted({str(t.dtype) for t in bufs})))
    dist.barrier()
    dist.destroy_process_group()


def test_sp_trainer_amp_tracks_fp32_model():
    import queue
    import time
    from tests import test_gpu_sp_trainer as spt
    width, tol = 64, 5e-2
    want = spt._sequential_losses(width)
    world = spt.P + spt.SPLIT - 1
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_trainer_worker, args=(r, "vertical", width, 29863, torch.cuda.device_count(), q))
          for r in range(world)]
    for p in ps:
        p.start()
    got = {}
    deadline = time.time() + 240
    while len(got) < world and time.time() < deadline:
        try:
            r, losses, launches, dtypes, bufs = q.get(timeout=1)
            got[r] = (losses, launches, dtypes, bufs)
        except queue.Empty:
            if any(p.exitcode not in (None, 0) for p in ps):
                break
    ok = len(got) == world
    for p in ps:
        p.join(30 if ok else 1)
        if p.is_alive():
            p.kill()
    assert ok, "worker exit codes: %s" % [p.exitcode for p in ps]
    assert got[0][1] > 0 and got[1][1] > 0, "tile ranks did not run libspconv kernels"
    for r in range(world):
        assert got[r][2] == ["torch.float32"], (r, got[r][2])
        assert got[r][3] in ([], ["torch.bfloat16"]), (r, got[r][3])
    assert got[2][3] == ["torch.bfloat16"]              # the join rank's tile buffers
    assert got[world - 1][0] == pytest.approx(want, rel=tol, abs=tol)


# ---- 6. fp16 autocast ---------------------------------------------------------------------------------------------
def test_fp16_autocast_warns_once_and_changes_nothing():
    from mpi4dl_b200.torchgems import spatial
    torch.manual_seed(6)
    m = _conv_layer(16, 16, 3, 3, 1, torch.randn(16, 16, 3, 3) / 12, torch.randn(16), torch.float32)
    x = torch.randn(N, 16, H, W)
    dy = torch.randn(N, 16, H, W)
    _zero(m)
    plain = _step(m, x, dy, False)
    spatial._fp16_autocast_warned = False
    outs = []
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        for _ in range(2):
            _zero(m)
            xx = x.to(DEV).requires_grad_(True)
            with torch.autocast("cuda", dtype=torch.float16):
                y = m(xx)
            y.backward(dy.to(DEV))
            outs.append([y.detach(), xx.grad, m.weight.grad, m.bias.grad])
    msgs = [w for w in rec if "float16" in str(w.message)]
    assert len(msgs) == 1, [str(w.message) for w in rec]
    for got in outs:
        for name, a, b in zip(("y", "dx", "dw", "db"), got, plain):
            assert a.dtype == torch.float32, name
            if name in ("y", "dx"):
                assert torch.equal(a, b), name
            else:                                         # summed with atomics (see the module docstring)
                torch.testing.assert_close(a, b, rtol=0, atol=1e-5 * float(b.abs().max()))
