"""-m gpu: recompute of the spatial cells (torchgems.recompute.checkpoint_spatial_cells) against the plain stage.

Four processes share one GPU (or get one each), one tile of a 2x2 grid each, with the peer-memory transport, halo
overlap on and off.  Each builds, from the same seed, two copies of a spatial stage -- the first six AmoebaNet-D
cells (stem1-3, cell1_normal1-3 of amoebanetd_spatial) and a ResNet-v2 spatial stage -- and runs one
forward + backward through the plain copy and one through the checkpointed copy, in three arms: fp32, bf16
autocast, and fp32 with exact_backward.  Per tile:

* the output and the input gradient are bit-identical;
* every parameter gradient is within 1e-5 * max|g| of the plain one (the wgrad kernels add with fp32 atomics in no
  fixed order, so two plain runs differ too);
* the BatchNorm running buffers are identical (one update per step, not two);
* the recompute exchanges no halo: the transport's forward exchange raises during the checkpointed backward (the
  exact backward's reverse exchange is allowed);
* under torch.no_grad() the checkpointed copy records no strips and gives the plain copy's output.

All CUDA work runs in the spawned processes, none in the test process.

Memory (AmoebaNet-D, fp32): the bytes autograd saves, summed with saved_tensors_hooks over unique storages, are
exactly the region inputs for the checkpointed stage; with the recorded strips they are less than the plain
stage's, and torch.cuda.max_memory_allocated of the checkpointed step is below the plain one."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, IMG = 4, 256


def _stage(kind, rank, parts=P):
    from mpi4dl_b200.models import amoebanet, resnet_spatial
    torch.manual_seed(0)
    if kind == "amoebanet":
        m = amoebanet.amoebanetd_spatial(rank, 1, parts, mp_size=2, slice_method="square", num_classes=10, num_layers=18,
                                         num_filters=416)
        m = nn.Sequential(*list(m.children())[:6])
    else:
        m = resnet_spatial.get_resnet_v2((1, 3, IMG, IMG), 20, rank, 2, spatial_size=1, num_spatial_parts=parts,
                                         slice_method="square")
        m = nn.Sequential(*list(m.children())[:4])
    return m.cuda().train()


def _out(y):
    return y[0] if isinstance(y, tuple) else y


def _storage(t):
    return t.untyped_storage().data_ptr(), t.untyped_storage().nbytes()


def _unique_bytes(storages):
    return sum(dict(storages).values())


def _run(m, x, dy, amp, exact, tr=None, saved=None):
    from mpi4dl_b200.torchgems import spatial
    for mod in m.modules():
        if isinstance(mod, spatial._SpatialTopology):
            mod.exact_backward = exact
    for p in m.parameters():
        p.grad = None
    xx = x.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    with torch.autograd.graph.saved_tensors_hooks(lambda t: (saved.append(_storage(t)), t)[1] if saved is not None else t,
                                                  lambda t: t):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            y = _out(m(xx))
    if tr is not None:
        tr.forbid = True
    try:
        y.backward(dy.to(y.dtype))
    finally:
        if tr is not None:
            tr.forbid = False
    torch.cuda.synchronize()
    bufs = [b.clone() for n, b in m.named_buffers()]
    return dict(y=y.detach(), dx=xx.grad, grads=[p.grad.clone() if p.grad is not None else None for p in m.parameters()], bufs=bufs,
                peak=torch.cuda.max_memory_allocated())


def _compare(tag, a, b, errs):
    if not torch.equal(a["y"], b["y"]):
        errs.append((tag, "y", float((a["y"].float() - b["y"].float()).abs().max())))
    if not torch.equal(a["dx"], b["dx"]):
        errs.append((tag, "dx", float((a["dx"].float() - b["dx"].float()).abs().max())))
    for i, (ga, gb) in enumerate(zip(a["grads"], b["grads"])):
        if ga is None or gb is None:                   # ResNet's unused BatchNorm of each unit
            if (ga is None) != (gb is None):
                errs.append((tag, "grad", i, "None"))
            continue
        tol = 1e-5 * float(ga.abs().max())
        if not torch.allclose(gb, ga, rtol=0, atol=tol):
            errs.append((tag, "grad", i, float((ga - gb).abs().max()), tol))
    for i, (ba, bb) in enumerate(zip(a["bufs"], b["bufs"])):
        if not torch.equal(ba, bb):
            errs.append((tag, "buffer", i))


def _worker(rank, overlap, port, ngpu, q):
    import sys
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), SPCONV_HALO_TRANSPORT="peer", SPCONV_ARENA_MB="64",
                      SPCONV_HALO_OVERLAP=overlap)
    multi = ngpu >= P
    dev = torch.device("cuda", rank if multi else 0)
    torch.cuda.set_device(dev)
    if multi:
        dist.init_process_group("nccl", rank=rank, world_size=P, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=P)
    from mpi4dl_b200.torchgems import halo_transport, recompute

    errs = []
    try:
        tr = halo_transport.get_transport(dev)
        exchange = tr.exchange

        def guarded(*a, **k):
            if tr.forbid:
                raise RuntimeError("halo exchange during the recompute")
            return exchange(*a, **k)

        tr.forbid = False
        tr.exchange = guarded
        recorders = []
        init = recompute._HaloRecorder.__init__

        def track(self, module):
            init(self, module)
            recorders.append(self)

        recompute._HaloRecorder.__init__ = track
        g = torch.Generator().manual_seed(11 + rank)
        x = torch.randn(1, 3, IMG // 2, IMG // 2, generator=g).cuda()
        for kind in ("amoebanet", "resnet"):
            plain, ckpt = _stage(kind, rank), recompute.checkpoint_spatial_cells(_stage(kind, rank))
            if sorted(plain.state_dict().keys()) != sorted(ckpt.state_dict().keys()):
                errs.append((kind, "state_dict keys"))
            del recorders[:]
            with torch.no_grad():                      # both copies: one BatchNorm update each
                y0 = _out(plain(x))
                shape = y0.shape
                if not torch.equal(_out(ckpt(x)), y0) or recorders:
                    errs.append((kind, "no_grad forward", len(recorders)))
            gy = torch.randn(shape, generator=g).cuda()
            for arm, amp, exact in (("fp32", False, False), ("bf16_amp", True, False), ("exact", False, True)):
                sp, sc = [], []
                del recorders[:]
                a = _run(plain, x, gy, amp, exact, saved=sp)
                b = _run(ckpt, x, gy, amp, exact, tr=tr, saved=sc)
                _compare((kind, arm), a, b, errs)
                if kind == "amoebanet" and arm == "fp32":
                    inputs = []
                    hooks = [c.register_forward_pre_hook(lambda mod, args: inputs.extend(recompute._flatten(args)[0]))
                             for c in ckpt.children()]
                    sp, sc = [], []
                    del recorders[:]
                    a = _run(plain, x, gy, amp, exact, saved=sp)
                    b = _run(ckpt, x, gy, amp, exact, tr=tr, saved=sc)
                    for h in hooks:
                        h.remove()
                    strips = sum(r.nbytes() for r in recorders)
                    region = _unique_bytes([_storage(t) for t in inputs if torch.is_tensor(t)])
                    if _unique_bytes(sc) != region or strips == 0 or region + strips >= _unique_bytes(sp):
                        errs.append(("saved bytes", _unique_bytes(sc), region, strips, _unique_bytes(sp)))
                    if not b["peak"] < a["peak"]:
                        errs.append(("peak", b["peak"], a["peak"]))
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


@pytest.mark.parametrize("overlap,port", [("1", 29871), ("0", 29872)], ids=["overlap", "serial"])
def test_recompute_four_tiles_matches_plain(overlap, port):
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    procs = [ctx.Process(target=_worker, args=(r, overlap, port, torch.cuda.device_count(), q)) for r in range(P)]
    for p in procs:
        p.start()
    res = [q.get() for _ in range(P)]
    for p in procs:
        p.join(120)
        if p.is_alive():
            p.kill()
    bad = [(r, e) for r, e in res if e]
    assert not bad, bad
