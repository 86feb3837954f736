"""CPU-only, world_size 2 and 4 over gloo: the reverse halo exchange of the exact backward routes fp32 strip
gradients through `exchange_strips` (DistTransport.reverse) with the forward pairing -- the gradient of received
strip d goes to neighbour d, which gets it as its strip 8-d and adds it into its edge band 8-d.  The strips are cut
from the oracle's padded input gradient HERE, and added with numpy: the product's kernels are CUDA-only."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, P, method, port, q):
    import sys
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=P)
    from mpi4dl_b200.torchgems import halo_transport as ht
    from mpi4dl_b200.torchgems import spatial
    from oracle import spatial_oracle as so
    from tests import exact_oracle as xo

    errs = []
    rng = np.random.default_rng(3)
    full = rng.standard_normal((2, 3, 16, 16)).astype(np.float32)
    tiles = so.split(full, method, P)
    for R, S in [(3, 3), (5, 5), (1, 7), (7, 1)]:
        w = rng.standard_normal((4, 3, R, S)).astype(np.float32)
        gys = [rng.standard_normal((2, 4, t.shape[2], t.shape[3])).astype(np.float32) for t in tiles]
        hh, hw = (R - 1) // 2, (S - 1) // 2
        layer = spatial.conv_spatial(rank, 1, P, 3, 4, (R, S), padding=(hh, hw), bias=False, slice_method=method)
        padded = so.exchange_halos(tiles, method, hh, hw, kh=R, kw=S)
        dxp = xo.conv_dgrad64(padded[rank].shape, w, gys[rank], (1, 1)).astype(np.float32)
        Hp, Wp = dxp.shape[2:]
        grads = [None] * 9
        for i in range(9):
            if i != 4 and layer.neighbours[i]:
                (r0, r1), (c0, c1) = so._recv_region(i, hh, hw, Hp, Wp)
                grads[i] = torch.tensor(np.ascontiguousarray(dxp[:, :, r0:r1, c0:c1]))
        shape = tiles[rank].shape
        recv = ht.DistTransport().reverse(layer, grads, shape, hh, hw, layer.neighbours, layer.rank_neighbours)
        dx = so.crop(dxp, hh, hw).astype(np.float64)
        H, W = shape[2:]
        for e in range(9):
            if recv[e] is None:
                continue
            if tuple(recv[e].shape) != ht.strip_shape(e, *shape, hh, hw) or recv[e].dtype != torch.float32:
                errs.append(("strip", R, S, e, tuple(recv[e].shape), str(recv[e].dtype)))
                continue
            dr, dc = so.DIRS[e]
            rs = {-1: slice(0, hh), 0: slice(0, H), 1: slice(H - hh, H)}[dr]
            cs = {-1: slice(0, hw), 0: slice(0, W), 1: slice(W - hw, W)}[dc]
            dx[:, :, rs, cs] += recv[e].numpy()
        ref = xo.conv_spatial(tiles, w, method, (1, 1), gys)[rank]["exact64"]
        if not np.allclose(dx, ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max()):
            errs.append((R, S, float(np.abs(dx - ref).max())))
    q.put((rank, errs))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("P,method,port", [(2, "vertical", 29721), (2, "horizontal", 29722), (4, "square", 29723),
                                           (4, "vertical", 29724)])
def test_reverse_strips_over_gloo(P, method, port):
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    procs = [ctx.Process(target=_worker, args=(r, P, method, port, q)) for r in range(P)]
    for p in procs:
        p.start()
    res = [q.get() for _ in range(P)]
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert all(not e for _, e in res), res
