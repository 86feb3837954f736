"""-m gpu: the exact backward (SPCONV_EXACT_BACKWARD=1 / layer.exact_backward).

1. The new kernels, one process, through the C ABI: strip gradients of conv (any R x S, stride 1/2, C = 3), pool
   (avg / max) and the halo ring under every neighbour mask of a 3x3 grid and of 3-way vertical / horizontal
   slicing, against float64 (|err| <= 2^-12 A, A = the same op on absolute values); the accumulate kernel against
   float64 and bit-identical across two runs.
2. The transports, 2 / 4 processes: conv_spatial, Pool and halo_exchange_layer forward + backward with the switch
   on, 4 iterations interleaved with extra forward exchanges, dx against the float64 full-image gradient, sliced.
3. A chain on 4 square tiles in fp32: the input gradient and the rank-summed dw equal the same modules run once on
   the whole image (num_spatial_parts=1); with the switch off the input gradient misses that bound.
4. The chain's forward + backward captured in a CUDA graph (peer transport) and replayed."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import spatial_oracle as so
from tests import exact_oracle as xo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def _masks():
    out = [("square9", r, "square", 9) for r in range(9)]
    out += [("vertical3", r, "vertical", 3) for r in range(3)]
    out += [("horizontal3", r, "horizontal", 3) for r in range(3)]
    return out


def _ptrs(ts):
    return (C.c_void_p * 9)(*[C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None) for t in ts])


def _strip_bufs(mask, N, Cc, H, W, hh, hw):
    from mpi4dl_b200.torchgems.halo_transport import strip_shape
    return [torch.full(strip_shape(i, N, Cc, H, W, hh, hw), float("nan"), device=DEV) if (i != 4 and mask[i]) else None
            for i in range(9)]


def _check_strips(got, ref_pad, A_pad, hh, hw, what, bound=2.0 ** -12):
    Hp, Wp = ref_pad.shape[2:]
    for i, g in enumerate(got):
        if g is None:
            continue
        (r0, r1), (c0, c1) = so._recv_region(i, hh, hw, Hp, Wp)
        ref, A = ref_pad[:, :, r0:r1, c0:c1], A_pad[:, :, r0:r1, c0:c1]
        err = (g.double().cpu() - ref).abs()
        assert torch.isfinite(g).all(), "%s strip %d: not written" % (what, i)
        assert (err <= bound * A).all(), "%s strip %d: max err/bound %.3g" % (
            what, i, float((err / (bound * A).clamp_min(1e-300)).max()))


CONV_CASES = [(20, 24, 3, 3, 1), (20, 24, 3, 3, 2), (20, 16, 1, 7, 1), (20, 16, 7, 1, 1), (20, 24, 5, 5, 1),
              (3, 16, 3, 3, 2), (3, 16, 7, 7, 2)]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("Cc,K,R,S,st", CONV_CASES, ids=["C%dK%d_%dx%ds%d" % c for c in CONV_CASES])
def test_conv_strip_gradient(Cc, K, R, S, st, dtype):
    from mpi4dl_b200 import _lib
    L = _lib.lib()
    torch.manual_seed(0)
    N, H, W = 2, 12, 20
    hh, hw = (R - 1) // 2, (S - 1) // 2
    Ho, Wo = (H + 2 * hh - R) // st + 1, (W + 2 * hw - S) // st + 1
    w = torch.randn(K, Cc, R, S).to(dtype)
    dy = torch.randn(N, K, Ho, Wo).to(dtype)
    shape = (N, Cc, H + 2 * hh, W + 2 * hw)
    ref = torch.nn.grad.conv2d_input(shape, w.double(), dy.double(), (st, st))
    A = torch.nn.grad.conv2d_input(shape, w.double().abs(), dy.double().abs(), (st, st))
    wd, dyd = w.to(DEV), dy.to(DEV)
    d = _lib.ConvDesc(N, Cc, H, W, K, R, S, st, st, hh, hw, _lib.dtype_code(dtype), 0)
    for name, rank, method, P in _masks():
        mask = so.neighbour_mask(method, P, rank, R, S)
        g = _strip_bufs(mask, N, Cc, H, W, hh, hw)
        _lib.check(L.spc_conv2d_dgrad_halo(C.byref(d), C.c_void_p(dyd.data_ptr()), C.c_void_p(wd.data_ptr()),
                                           C.byref(_ptrs(g)), None), "spc_conv2d_dgrad_halo")
        torch.cuda.synchronize()
        _check_strips(g, ref, A, hh, hw, "%s rank %d" % (name, rank))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("mode,st", [("avg", 1), ("avg", 2), ("max", 1), ("max", 2)])
def test_pool_strip_gradient(mode, st, dtype):
    from mpi4dl_b200 import _lib
    from tests.gpu_util import strips_from_padded
    L = _lib.lib()
    rng = np.random.default_rng(1)
    k, h = 3, 1

    def aten_bwd(xp, gy):
        """ATen's pool backward on the padded tile in float64 (max: first maximum, NaN wins, the last of two NaNs)"""
        xd = torch.tensor(xp, dtype=torch.float64, requires_grad=True)
        y = torch.nn.functional.max_pool2d(xd, k, st) if mode == "max" else torch.nn.functional.avg_pool2d(xd, k, st)
        return torch.autograd.grad(y, xd, gy)[0]

    # random data; integers in {-2..2} (tied maxima, also with the zero pad); 4 % NaN, received strips included
    for regime, (name, rank, method, P) in [(r, m) for r in ("normal", "ties", "nan") for m in _masks()]:
        H0, W0 = {"square": (36, 48), "vertical": (12, 48), "horizontal": (36, 16)}[method]
        if regime == "ties":
            full = rng.integers(-2, 3, (2, 8, H0, W0)).astype(np.float32)
        else:
            full = rng.standard_normal((2, 8, H0, W0)).astype(np.float32)
            if regime == "nan":
                full[rng.random(full.shape) < 0.04] = np.nan
        full = torch.tensor(full).to(dtype).float().numpy()
        tiles = so.split(full, method, P)
        xp = so.exchange_halos(tiles, method, h, h)[rank]
        mask = so.neighbour_mask(method, P, rank)
        N, Cc, H, W = tiles[rank].shape
        Ho, Wo = (H + 2 * h - k) // st + 1, (W + 2 * h - k) // st + 1
        gy = torch.randn(N, Cc, Ho, Wo).to(dtype)
        ref = aten_bwd(xp, gy.double())
        A = aten_bwd(xp, gy.double().abs())
        name = "%s %s" % (regime, name)
        x = torch.tensor(tiles[rank], dtype=dtype, device=DEV)
        strips = strips_from_padded(xp, mask, h, h, dtype)
        gyd = gy.to(DEV)
        g = _strip_bufs(mask, N, Cc, H, W, h, h)
        d = _lib.PoolDesc(N, Cc, H, W, k, st, h, _lib.SPC_POOL_MAX if mode == "max" else _lib.SPC_POOL_AVG,
                          _lib.dtype_code(dtype))
        halo = _lib.make_halo(strips)
        _lib.check(L.spc_pool2d_bwd_halo(C.byref(d), C.c_void_p(x.data_ptr()), C.byref(halo), C.c_void_p(gyd.data_ptr()),
                                         C.byref(_ptrs(g)), None), "spc_pool2d_bwd_halo")
        torch.cuda.synchronize()
        _check_strips(g, ref, A, h, h, "%s rank %d" % (name, rank))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("hh,hw", [(1, 1), (2, 2), (3, 3), (0, 3), (3, 0)])
def test_ring_and_accumulate(hh, hw, dtype):
    from mpi4dl_b200 import _lib
    L = _lib.lib()
    torch.manual_seed(2)
    N, Cc, H, W = 2, 5, 9, 14
    dc = _lib.dtype_code(dtype)
    for name, rank, method, P in _masks():
        mask = so.neighbour_mask(method, P, rank, 2 * hh + 1, 2 * hw + 1)
        # ring: the pad strips of a padded gradient, exactly (a copy to fp32)
        gy = torch.randn(N, Cc, H + 2 * hh, W + 2 * hw).to(dtype).to(DEV)
        g = _strip_bufs(mask, N, Cc, H, W, hh, hw)
        _lib.check(L.spc_halo_ring(N, Cc, H, W, hh, hw, dc, C.c_void_p(gy.data_ptr()), C.byref(_ptrs(g)), None),
                   "spc_halo_ring")
        torch.cuda.synchronize()
        ref = gy.double().cpu()
        _check_strips(g, ref, torch.zeros_like(ref), hh, hw, "ring %s rank %d" % (name, rank), bound=0.0)
        # accumulate: dx[band e] += g[e], summed in fp32 and rounded once; bit-identical run to run
        recv = [torch.randn(t.shape, device=DEV) if t is not None else None for t in g]
        dx0 = torch.randn(N, Cc, H, W).to(dtype).to(DEV)
        outs = []
        for _ in range(2):
            dx = dx0.clone()
            _lib.check(L.spc_halo_accumulate(N, Cc, H, W, hh, hw, dc, C.c_void_p(dx.data_ptr()), C.byref(_ptrs(recv)),
                                             None), "spc_halo_accumulate")
            outs.append(dx)
        torch.cuda.synchronize()
        assert torch.equal(outs[0], outs[1]), "accumulate is not bit-reproducible"
        exp = dx0.double().cpu().clone()
        mag = dx0.double().cpu().abs()
        for e, t in enumerate(recv):
            if t is None:
                continue
            dr, dcol = so.DIRS[e]
            rs = {-1: slice(0, hh), 0: slice(0, H), 1: slice(H - hh, H)}[dr]
            cs = {-1: slice(0, hw), 0: slice(0, W), 1: slice(W - hw, W)}[dcol]
            exp[:, :, rs, cs] += t.double().cpu()
            mag[:, :, rs, cs] += t.double().cpu().abs()
        rnd = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -24
        err = (outs[0].double().cpu() - exp).abs()
        assert (err <= rnd * exp.abs() + 2.0 ** -21 * mag).all(), "accumulate %s rank %d" % (name, rank)


# ---- 2. transports ----------------------------------------------------------------------------------------------

def _init(rank, P, transport, port, ngpu):
    import sys
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["SPCONV_HALO_TRANSPORT"] = transport
    os.environ["SPCONV_ARENA_MB"] = "64"
    os.environ["SPCONV_EXACT_BACKWARD"] = "1"
    multi = ngpu >= P
    dev = torch.device("cuda", rank if multi else 0)
    torch.cuda.set_device(dev)
    if multi:
        dist.init_process_group("nccl", rank=rank, world_size=P, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=P)
    return dev


def _bound_err(dx, ref, own, A, dtype):
    """max err / bound (<= 1 passes)"""
    if dtype == torch.bfloat16:
        b = 2.0 ** -8 * (np.abs(ref) + np.abs(own)) + 2.0 ** -12 * A
    else:
        b = 2.0 ** -16 * (np.abs(ref) + A)
    return float((np.abs(dx - ref) / np.maximum(b, 1e-300)).max())


def _transport_worker(rank, P, method, transport, port, ngpu, q):
    dev = _init(rank, P, transport, port, ngpu)
    from mpi4dl_b200.torchgems import spatial

    errs = []
    try:
        rng = np.random.default_rng(11)
        full = rng.standard_normal((1, 16, 24, 32)).astype(np.float32)
        for dtype in (torch.bfloat16, torch.float32):
            fullq = torch.tensor(full).to(dtype).float().numpy()
            tiles = so.split(fullq, method, P)
            for (K, R, S, st) in [(16, 3, 3, 1), (8, 1, 7, 1), (8, 7, 1, 1), (16, 3, 3, 2), (8, 5, 5, 1)]:
                w = torch.tensor(rng.standard_normal((K, 16, R, S)).astype(np.float32) / np.sqrt(16 * R * S)).to(dtype)
                w = w.float().numpy()
                m = spatial.conv_spatial(rank, 1, P, 16, K, (R, S), stride=st, padding=((R - 1) // 2, (S - 1) // 2),
                                         bias=False, slice_method=method).to(dev).to(dtype)
                assert m.exact_backward and "exact_backward" not in dict(m.named_buffers())
                with torch.no_grad():
                    m.weight.copy_(torch.tensor(w))
                ys = so.conv_spatial(tiles, w, None, method, (st, st))
                gys = [torch.tensor(rng.standard_normal(y["y"].shape).astype(np.float32)).to(dtype).float().numpy()
                       for y in ys]
                res = xo.conv_spatial(tiles, w, method, (st, st), gys)
                ref, A = xo.full_reference("conv", fullq, gys, method, P, w=w, stride=(st, st))
                for it in range(4):
                    x = torch.tensor(tiles[rank], dtype=dtype, device=dev, requires_grad=True)
                    if it % 2 == 1:
                        with torch.no_grad():
                            m(x)          # an extra forward exchange: forward and reverse slots at different parity
                    y = m(x)
                    y.backward(torch.tensor(gys[rank], dtype=dtype, device=dev))
                    e = _bound_err(x.grad.float().cpu().numpy(), ref[rank], res[rank]["n2"], A[rank], dtype)
                    if e > 1:
                        errs.append(("conv", str(dtype), K, R, S, st, it, e))
                    m.weight.grad = None
            for mode, st in [("avg", 1), ("avg", 2), ("max", 1), ("max", 2)]:
                pm = spatial.Pool(rank, 1, P, 3, st, 1, slice_method=method,
                                  operation="AvgPool2d" if mode == "avg" else "MaxPool2d")
                ys = so.pool_spatial(tiles, method, mode, 3, st, 1)
                gys = [torch.tensor(rng.standard_normal(y["y"].shape).astype(np.float32)).to(dtype).float().numpy()
                       for y in ys]
                res = xo.pool_spatial(tiles, method, mode, 3, st, gys)
                ref, A = xo.full_reference("pool", fullq, gys, method, P, mode=mode, k=3, stride=st)
                for it in range(4):
                    x = torch.tensor(tiles[rank], dtype=dtype, device=dev, requires_grad=True)
                    if it % 2 == 1:
                        with torch.no_grad():
                            pm(x)
                    pm(x).backward(torch.tensor(gys[rank], dtype=dtype, device=dev))
                    e = _bound_err(x.grad.float().cpu().numpy(), ref[rank], res[rank]["n2"], A[rank], dtype)
                    if e > 1:
                        errs.append(("pool", str(dtype), mode, st, it, e))
            for h in (1, 2, 3):
                hl = spatial.halo_exchange_layer(rank, 1, P, h, slice_method=method)
                gys = [torch.tensor(rng.standard_normal((1, 16, t.shape[2] + 2 * h, t.shape[3] + 2 * h))
                                    .astype(np.float32)).to(dtype).float().numpy() for t in tiles]
                res = xo.halo_exchange_layer(tiles, method, h, gys)
                ref, A = xo.full_reference("halo", fullq, gys, method, P, halo_len=h)
                for it in range(4):
                    x = torch.tensor(tiles[rank], dtype=dtype, device=dev, requires_grad=True)
                    if it % 2 == 1:
                        with torch.no_grad():
                            hl(x)
                    hl(x).backward(torch.tensor(gys[rank], dtype=dtype, device=dev))
                    e = _bound_err(x.grad.float().cpu().numpy(), ref[rank], res[rank]["n2"], A[rank], dtype)
                    if e > 1:
                        errs.append(("halo", str(dtype), h, it, e))
        # switch off: no reverse slot is ever allocated
        m = spatial.conv_spatial(rank, 1, P, 16, 8, 3, padding=1, bias=False, slice_method=method).to(dev)
        m.exact_backward = False
        x = torch.tensor(so.split(full, method, P)[rank], device=dev, requires_grad=True)
        m(x).sum().backward()
        if any(k[0] == "reverse" for k in m.__dict__.get("_halo_slots", {})):
            errs.append(("reverse slot allocated with the switch off",))
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


def _spawn(target, P, args):
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    procs = [ctx.Process(target=target, args=(r, P) + args + (q,)) for r in range(P)]
    for p in procs:
        p.start()
    res = [q.get() for _ in range(P)]
    for p in procs:
        p.join(120)
        if p.is_alive():
            p.kill()
    return res


@pytest.mark.parametrize("P,method,transport,port", [
    (2, "vertical", "peer", 29831), (2, "horizontal", "peer", 29832), (4, "square", "peer", 29833),
    (2, "vertical", "dist", 29834), (4, "square", "dist", 29835)])
def test_exact_backward_transports(P, method, transport, port):
    ngpu = torch.cuda.device_count()
    if transport == "dist" and ngpu < P:
        pytest.skip("torch.distributed transport on GPUs needs NCCL with one GPU per rank")
    res = _spawn(_transport_worker, P, (method, transport, port, ngpu))
    bad = [(r, e) for r, e in res if e]
    assert not bad, bad


# ---- 3 + 4. the chain on 4 square tiles, eager and in a CUDA graph ---------------------------------------------------

def _chain(spatial, rank, P, exact):
    import torch.nn as nn
    layers = [spatial.conv_spatial(rank, 1, P, 4, 8, 3, padding=1, slice_method="square"),
              spatial.Pool(rank, 1, P, 3, 1, 1, slice_method="square", operation="AvgPool2d"),
              spatial.conv_spatial(rank, 1, P, 8, 8, (1, 7), padding=(0, 3), slice_method="square"),
              spatial.conv_spatial(rank, 1, P, 8, 8, (7, 1), padding=(3, 0), slice_method="square"),
              spatial.conv_spatial(rank, 1, P, 8, 8, 3, stride=2, padding=1, slice_method="square"),
              spatial.halo_exchange_layer(rank, 1, P, 2, slice_method="square"),
              spatial.local_conv2d(8, 8, 3, padding=0),
              spatial.local_conv2d(8, 8, 3, padding=0)]
    for m in layers:
        m.exact_backward = exact
    return nn.Sequential(*layers)


def _chain_worker(rank, P, port, ngpu, q):
    dev = _init(rank, P, "peer", port, ngpu)
    from mpi4dl_b200.torchgems import spatial

    errs = []
    try:
        g = torch.Generator().manual_seed(5)
        full = torch.randn(1, 4, 32, 32, generator=g)
        G = torch.randn(1, 8, 16, 16, generator=g)           # dL/dy of the full-image output
        torch.manual_seed(0)
        ref_model = _chain(spatial, 0, 1, False).to(dev)
        xf = full.to(dev).requires_grad_(True)
        (ref_model(xf) * G.to(dev)).sum().backward()
        hs, ws = so.tile_slices("square", P, rank, 32, 32)
        ohs, ows = so.tile_slices("square", P, rank, 16, 16)
        ref_dx = xf.grad[:, :, hs, ws].cpu()
        ref_dw = [p.grad.cpu() for p in ref_model.parameters()]
        sd = ref_model.state_dict()
        x = full[:, :, hs, ws].contiguous().to(dev)
        gt = G[:, :, ohs, ows].contiguous().to(dev)

        def step(model):
            xx = x.clone().requires_grad_(True)
            (model(xx) * gt).sum().backward()
            return xx

        def close(a, b):
            return bool(((a - b).abs() <= 1e-5 * b.abs().max()).all())

        def rank_sum(t):
            """sum over the ranks (NCCL on device tensors, gloo on host ones)"""
            t = t.detach().clone() if dist.get_backend() == "nccl" else t.detach().cpu().clone()
            dist.all_reduce(t)
            return t.cpu()

        for exact in (True, False):
            model = _chain(spatial, rank, P, exact).to(dev)
            model.load_state_dict(sd)
            xx = step(model)
            dws = [rank_sum(p.grad) for p in model.parameters()]
            ok_dx = close(xx.grad.cpu(), ref_dx)
            ok_dw = all(close(a, b) for a, b in zip(dws, ref_dw))
            if exact and not (ok_dx and ok_dw):
                errs.append(("chain exact", ok_dx, ok_dw, float((xx.grad.cpu() - ref_dx).abs().max()),
                             float(ref_dx.abs().max())))
            if not exact:
                # the test has teeth: with the reference's backward some rank's input gradient misses the bound
                misses = rank_sum(torch.tensor([0.0 if ok_dx else 1.0], device=dev)).item()
                if misses == 0:
                    errs.append(("chain with the switch off matches the full image: the check has no teeth",))
            if exact:
                # 4. CUDA graph: after the eager step, capture forward + backward and replay
                eager_dx = xx.grad.clone()
                eager_dw = [p.grad.clone() for p in model.parameters()]
                for p in model.parameters():
                    p.grad = None
                sx = x.clone().requires_grad_(True)
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    (model(sx) * gt).sum().backward()
                for rep in range(3):
                    graph.replay()
                    torch.cuda.synchronize()
                    if not close(sx.grad, eager_dx) or not all(close(p.grad, e) for p, e in zip(model.parameters(), eager_dw)):
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


def test_chain_matches_single_gpu_and_replays_in_a_graph():
    ngpu = torch.cuda.device_count()
    res = _spawn(_chain_worker, 4, (29836, ngpu))
    bad = [(r, e) for r, e in res if e]
    assert not bad, bad
