"""-m gpu: spatial stages run from captured CUDA graphs (torchgems.graphs) against the eager stage.

Every comparison runs a graphed copy and an eager copy built from one seed, under
torch.use_deterministic_algorithms(True), so it is bit for bit:

1. one tile, no neighbours: the first six AmoebaNet-D cells and a ResNet-v2 spatial stage, 3 steps with SGD between
   them, in fp32, fp32 with SPCONV_ALLOW_TF32=strided and bf16 autocast, recompute off and on.  After each step the
   output, every .grad (input included) and every BatchNorm buffer are identical.  Without deterministic mode the
   parameter gradients agree within the recompute tests' 1e-5 * max|g| (the atomic wgrad), the rest is identical.
2. four tiles sharing one GPU (square-4, peer transport): a conv / pool / halo-exchange chain and the same cells,
   exact backward off and on, SPCONV_HALO_OVERLAP off and on; every tile identical.
3. train_model_spatial(..., cuda_graph=True), 2 tiles + join + tail, parts 1 and 2: loss sequence and parameters
   after 3 steps identical to cuda_graph=False, and spc_launch_count does not grow on the tile ranks during graphed
   steps 2-3.  The same for train_spatial_model_master (two mirrored replicas), 2 steps.
4. refusals: a changed input shape, a no-grad call and a stage exchanging through DistTransport raise.

All CUDA work runs in spawned processes (as in test_gpu_recompute.py); the multi-process tests use gloo for
torch.distributed and a small mailbox arena."""
import os
import queue
import time

import pytest
import torch
import torch.multiprocessing as mp
import torch.nn as nn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spawn(target, world, args, timeout=600):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=target, args=(r, world) + tuple(args) + (q,)) for r in range(world)]
    for p in ps:
        p.start()
    got = {}
    deadline = time.time() + timeout
    while len(got) < world and time.time() < deadline:
        try:
            r, res = q.get(timeout=1)
            got[r] = res
        except queue.Empty:
            if any(p.exitcode not in (None, 0) for p in ps):
                break
    ok = len(got) == world
    for p in ps:
        p.join(60 if ok else 1)
        if p.is_alive():
            p.kill()
    assert ok, "worker exit codes: %s" % [p.exitcode for p in ps]
    return got


def _env(port, deterministic=True, **kw):
    import sys
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), SPCONV_HALO_TRANSPORT="peer", SPCONV_ARENA_MB="64",
                      CUBLAS_WORKSPACE_CONFIG=":4096:8", **kw)
    torch.cuda.set_device(0)
    torch.use_deterministic_algorithms(deterministic)


def _stage(kind, rank, parts, img):
    from mpi4dl_b200.models import amoebanet, resnet_spatial
    from mpi4dl_b200.torchgems import spatial
    torch.manual_seed(0)
    if kind == "amoebanet":
        m = amoebanet.amoebanetd_spatial(rank, 1, parts, mp_size=2, slice_method="square", num_classes=10, num_layers=18,
                                         num_filters=416)
        m = nn.Sequential(*list(m.children())[:6])
    elif kind == "resnet":
        m = resnet_spatial.get_resnet_v2((1, 3, img, img), 20, rank, 2, spatial_size=1, num_spatial_parts=parts,
                                         slice_method="square")
        m = nn.Sequential(*list(m.children())[:4])
    else:                                  # conv / pool / halo-exchange chain
        sp = dict(local_rank=rank, spatial_size=1, num_spatial_parts=parts, slice_method="square")
        m = nn.Sequential(spatial.conv_spatial(in_channels=3, out_channels=16, kernel_size=3, padding=1, **sp), nn.ReLU(),
                          spatial.Pool(kernel_size=3, stride=1, padding=1, operation="MaxPool2d", **sp),
                          spatial.halo_exchange_layer(halo_len=1, **sp), spatial.local_conv2d(16, 16, 3, padding=0),
                          nn.BatchNorm2d(16),
                          spatial.conv_spatial(in_channels=16, out_channels=32, kernel_size=3, stride=2, padding=1, **sp),
                          spatial.Pool(kernel_size=3, stride=1, padding=1, operation="AvgPool2d", **sp))
    return m.cuda().train()


def _out(y):
    return y[0] if isinstance(y, tuple) else y


def _steps(m, x, gy, amp, nsteps, graphed=False, exact=False):
    """nsteps of forward + backward + SGD; the state after each step."""
    from mpi4dl_b200.torchgems import graphs, spatial
    for mod in m.modules():
        if isinstance(mod, spatial._SpatialTopology):
            mod.exact_backward = exact
    opt = torch.optim.SGD(m.parameters(), lr=1e-2, momentum=0.9)
    g = graphs.graph_stage(m, [x.clone().requires_grad_(True)], amp_dtype=torch.bfloat16 if amp else None) if graphed else None
    states = []
    for _ in range(nsteps):
        xx = x.clone().requires_grad_(True)
        if graphed:
            y = _out(g(xx))
        else:
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                y = _out(m(xx))
        y.backward(gy.to(y.dtype))
        torch.cuda.synchronize()
        states.append(dict(y=y.detach().clone(), dx=xx.grad.clone(),
                           grads=[p.grad.clone() if p.grad is not None else None for p in m.parameters()],
                           bufs=[b.clone() for b in m.buffers()]))
        if graphed:
            static = {t.data_ptr() for s in g.slots for t in s.static_grads if t is not None}
            if any(p.grad is not None and p.grad.data_ptr() in static for p in m.parameters()):
                states[-1]["alias"] = True
        opt.step()
        opt.zero_grad(set_to_none=False)
    return states


def _compare(tag, a, b, errs, grad_tol=0.0):
    for step, (sa, sb) in enumerate(zip(a, b)):
        t = tag + (step,)
        if sb.get("alias"):
            errs.append((t, ".grad aliases a static graph buffer"))
        for k in ("y", "dx"):
            if not torch.equal(sa[k], sb[k]):
                errs.append((t, k, float((sa[k].float() - sb[k].float()).abs().max())))
        for i, (ga, gb) in enumerate(zip(sa["grads"], sb["grads"])):
            if (ga is None) != (gb is None):
                errs.append((t, "grad", i, "None"))
            elif ga is not None and not (torch.equal(ga, gb) if grad_tol == 0 else
                                         torch.allclose(gb, ga, rtol=0, atol=grad_tol * float(ga.abs().max()))):
                errs.append((t, "grad", i, float((ga - gb).abs().max())))
        for i, (ba, bb) in enumerate(zip(sa["bufs"], sb["bufs"])):
            if not torch.equal(ba, bb):
                errs.append((t, "buffer", i))


def _report(q, rank, fn):
    try:
        errs = fn()
    except Exception as ex:  # report instead of hanging the peers
        import traceback
        errs = [("exception", repr(ex), traceback.format_exc()[-2000:])]
    q.put((rank, errs))


# ---- 1. one tile -------------------------------------------------------------------------------------------------
def _one_tile_worker(rank, world, port, q):
    def run():
        _env(port)
        from mpi4dl_b200.torchgems import recompute
        errs = []
        img = 128
        g = torch.Generator().manual_seed(7)
        x = torch.randn(1, 3, img, img, generator=g).cuda()
        for tf32 in ("0", "strided"):
            os.environ["SPCONV_ALLOW_TF32"] = tf32                 # read by the conv layers' constructors
            for amp in ((False, True) if tf32 == "0" else (False,)):
                for rc in (False, True):
                    for kind in ("amoebanet", "resnet"):
                        def build():
                            m = _stage(kind, 0, 1, img)
                            return recompute.checkpoint_spatial_cells(m) if rc else m
                        with torch.no_grad():
                            shape = _out(build()(x)).shape
                        gy = torch.randn(shape, generator=g).cuda()
                        a = _steps(build(), x, gy, amp, 3)
                        b = _steps(build(), x, gy, amp, 3, graphed=True)
                        _compare((kind, tf32, amp, rc), a, b, errs)
        # without deterministic mode: the atomic wgrad orders its sums differently from run to run
        torch.use_deterministic_algorithms(False)
        os.environ["SPCONV_ALLOW_TF32"] = "0"
        gy = torch.randn(_out(_stage("amoebanet", 0, 1, img)(x)).shape, generator=g).cuda()
        a = _steps(_stage("amoebanet", 0, 1, img), x, gy, False, 1)
        b = _steps(_stage("amoebanet", 0, 1, img), x, gy, False, 1, graphed=True)
        _compare(("nondeterministic",), a, b, errs, grad_tol=1e-5)
        return errs

    _report(q, rank, run)


def test_graphed_stage_one_tile_matches_eager():
    got = _spawn(_one_tile_worker, 1, (29881,))
    assert not got[0], got[0]


# ---- 2. four tiles -----------------------------------------------------------------------------------------------
def _four_tile_worker(rank, world, overlap, port, q):
    def run():
        import torch.distributed as dist
        _env(port, SPCONV_HALO_OVERLAP=overlap)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        errs = []
        img = 256
        g = torch.Generator().manual_seed(11 + rank)
        x = torch.randn(1, 3, img // 2, img // 2, generator=g).cuda()
        for kind in ("chain", "amoebanet"):
            with torch.no_grad():
                shape = _out(_stage(kind, rank, world, img)(x)).shape
            gy = torch.randn(shape, generator=g).cuda()
            for exact in (False, True):
                a = _steps(_stage(kind, rank, world, img), x, gy, False, 2, exact=exact)
                b = _steps(_stage(kind, rank, world, img), x, gy, False, 2, graphed=True, exact=exact)
                _compare((kind, overlap, exact), a, b, errs)
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()
        return errs

    _report(q, rank, run)


@pytest.mark.parametrize("overlap,port", [("1", 29882), ("0", 29883)], ids=["overlap", "serial"])
def test_graphed_stage_four_tiles_matches_eager(overlap, port):
    got = _spawn(_four_tile_worker, 4, (overlap, port))
    bad = {r: e for r, e in got.items() if e}
    assert not bad, bad


# ---- 3. trainers -------------------------------------------------------------------------------------------------
P, SPLIT, IMG, BATCH = 2, 3, 64, 2


def _layers(sp, width=8):
    from mpi4dl_b200.torchgems.spatial import Pool, conv_spatial
    torch.manual_seed(99)
    return [conv_spatial(in_channels=3, out_channels=width, kernel_size=3, padding=1, **sp), nn.BatchNorm2d(width),
            nn.ReLU(), conv_spatial(in_channels=width, out_channels=width, kernel_size=3, stride=2, padding=1, **sp),
            Pool(operation="AvgPool2d", kernel_size=3, stride=1, padding=1, **sp),           # spatial stage
            nn.Conv2d(width, 4, 3, padding=1), nn.ReLU(),                                   # join rank
            nn.Flatten(), nn.Linear(4 * (IMG // 2) ** 2, 10)]                              # tail


def _batch(step, n=BATCH):
    g = torch.Generator().manual_seed(500 + step)
    return torch.randn(n, 3, IMG, IMG, generator=g), torch.randint(0, 10, (n,), generator=g)


def _trainer_worker(rank, world, master, parts, port, q):
    def run():
        import torch.distributed as dist
        _env(port)
        os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0", SPCONV_DIST_BACKEND="gloo")
        from mpi4dl_b200 import _lib
        from mpi4dl_b200.torchgems import comm as gems_comm
        from mpi4dl_b200.torchgems.mp_pipeline import model_generator
        from mpi4dl_b200.torchgems.train_spatial import get_shapes_spatial, split_input, train_model_spatial
        from mpi4dl_b200.torchgems.train_spatial_master import train_spatial_model_master
        gems_comm.initialize_cuda()
        full = [(BATCH // parts, 8, IMG // 2, IMG // 2), (BATCH // parts, 4, IMG // 2, IMG // 2), (BATCH // parts, 10)]
        shapes = get_shapes_spatial(full, "vertical", 1, [P], 1)
        L = _lib.lib()
        comm1 = gems_comm.MPIComm(split_size=SPLIT, ENABLE_MASTER=False, ENABLE_SPATIAL=True, num_spatial_parts=P,
                                  spatial_size=1)
        comms = [comm1]
        if master:
            comm2 = gems_comm.MPIComm(split_size=SPLIT, ENABLE_MASTER=True, ENABLE_SPATIAL=True, num_spatial_parts=P,
                                      spatial_size=1, LOCAL_DP_LP=1, DISABLE_INIT=True)
            gems_comm.sync_comms_for_master(comm1, comm2)
            comms.append(comm2)

        def gen(comm):
            sp = dict(local_rank=comm.local_rank % P, spatial_size=1, num_spatial_parts=P, slice_method="vertical")
            g = model_generator(model=nn.Sequential(*_layers(sp)), split_size=SPLIT,
                                input_size=(BATCH // parts, 3, IMG, IMG), balance=[5, 2, 2], shape_list=shapes)
            g.ready_model(split_rank=comm.split_rank)
            return g

        def train(cuda_graph):
            gens = [gen(c) for c in comms]
            if master:
                tm = train_spatial_model_master(gens[0], gens[1], BATCH, 1, P, "vertical", comm1, comms[1], 1, parts=parts,
                                                cuda_graph=cuda_graph)
                tiles = [tm.train_model1, tm.train_model2]
            else:
                tm = train_model_spatial(gens[0], comm1.local_rank, BATCH, epochs=1, spatial_size=1, num_spatial_parts=P,
                                         parts=parts, slice_method="vertical", mpi_comm=comm1, cuda_graph=cuda_graph)
                tiles = [tm]
            is_tile = any(t.local_rank < P for t in tiles)
            losses, launches = [], []
            for step in range(2 if master else 3):
                x, y = _batch(step, 2 * BATCH if master else BATCH)
                tile = [c.local_rank for c in comms if c.local_rank < P]
                if tile:
                    x = split_input(x, IMG, "vertical", tile[0], [P])
                L.spc_launch_count(1)
                loss, _ = tm.run_step(x, y)
                torch.cuda.synchronize()
                launches.append(int(L.spc_launch_count(0)))
                for t in tiles:
                    t.update()
                losses.append(float(loss))
            params = [p.detach().clone() for g in gens for p in g.models.parameters()]
            return losses, params, launches, is_tile

        la, pa, _, _ = train(False)
        lb, pb, launches, is_tile = train(True)
        errs = []
        if la != lb:
            errs.append(("losses", la, lb))
        if len(pa) != len(pb) or not all(torch.equal(a, b) for a, b in zip(pa, pb)):
            errs.append(("parameters differ",))
        if is_tile and (launches[0] == 0 or any(launches[1:])):
            errs.append(("libspconv launches per step on a tile rank", launches))
        dist.barrier()
        dist.destroy_process_group()
        return errs

    _report(q, rank, run)


@pytest.mark.parametrize("master,parts,port", [(False, 1, 29884), (False, 2, 29885), (True, 1, 29886)],
                         ids=["sp-parts1", "sp-parts2", "gems-master"])
def test_trainer_cuda_graph_matches_eager(master, parts, port):
    got = _spawn(_trainer_worker, P + SPLIT - 1, (master, parts, port))
    bad = {r: e for r, e in got.items() if e}
    assert not bad, bad


# ---- 4. refusals -------------------------------------------------------------------------------------------------
def _refusal_worker(rank, world, port, q):
    def run():
        _env(port)
        from mpi4dl_b200.torchgems import graphs, halo_transport
        errs = []
        x = torch.randn(1, 3, 64, 64, device="cuda")
        g = graphs.graph_stage(_stage("chain", 0, 1, 64), [x.clone().requires_grad_(True)])
        for name, call, words in (
                ("shape", lambda: g(torch.randn(1, 3, 32, 32, device="cuda", requires_grad=True)), "differs from the capture"),
                ("no_grad", lambda: torch.no_grad()(g)(x.clone().requires_grad_(True)), "without grad mode")):
            try:
                call()
                errs.append((name, "did not raise"))
            except graphs.GraphCaptureError as e:
                if words not in str(e):
                    errs.append((name, str(e)))
        halo_transport.set_transport(halo_transport.DistTransport())
        try:
            graphs.graph_stage(_stage("chain", 0, 4, 64), [x.clone().requires_grad_(True)])
            errs.append(("dist", "did not raise"))
        except graphs.GraphCaptureError as e:
            if "DistTransport" not in str(e):
                errs.append(("dist", str(e)))
        return errs

    _report(q, rank, run)


def test_graphed_stage_refusals():
    got = _spawn(_refusal_worker, 1, (29887,))
    assert not got[0], got[0]
