"""Halo-exchange sweep (BASELINE.json config 5): one neighbour exchange of a 3x3 convolution's halo
(halo_len 1) between tiles of 2048..16384 pixels on P in {2, 4, 8} GPUs, through the SAME layer the models use
(torchgems.spatial.halo_exchange_layer / the transport under conv_spatial), one process per GPU:

    torchrun --nproc-per-node P benchmarks/communication/halo/halo_sweep.py [--tiles 2048 4096 ...] [--channels 16 64]
                                                                             [--halo-len 1] [--dtype bf16|fp32]

Per configuration it reports, as one JSON line on rank 0 (and appended to --out):
  us_exchange      device time of ONE exchange (post + collect kernels, no pad), CUDA events, max over ranks
  us_layer         halo_exchange_layer.forward (exchange + materialised padded tile, what the reference times)
  recv_bytes       bytes this rank receives per exchange (max over ranks)
  GBps             recv_bytes / us_exchange   -- against 900 GB/s (the frac_of_900GBps field; H100 NVLink 4 is 450 GB/s per direction)
The reference's number for this path (benchmarks/communication/halo/README.md:24-43): 0.334 ms per exchange of
a 1024^2 image in 4 vertical parts, halo_len 3, C = 1 -- `--reference-point` runs exactly that shape.
Messages are small (a 2048-px edge of 64 bf16 channels is 256 KB), so the exchange is LATENCY-bound: us_exchange
is the number to read, GB/s shows how far below link bandwidth that leaves it."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", "..", "..")]

from mpi4dl_b200.torchgems import comm as gems_comm  # noqa: E402
from mpi4dl_b200.torchgems import halo_transport  # noqa: E402
from mpi4dl_b200.torchgems.spatial import halo_exchange_layer  # noqa: E402


def timed(fn, iters, warmup, dev):
    for _ in range(warmup):
        fn()
    dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters * 1e3], device=dev)     # microseconds
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, nargs="+", default=[2048, 4096, 8192, 16384], help="tile edge in pixels")
    ap.add_argument("--channels", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--halo-len", type=int, default=1)
    ap.add_argument("--dtype", choices=["bf16", "fp32"], default="bf16")
    ap.add_argument("--slice-methods", nargs="+", default=None)
    ap.add_argument("--iterations", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reference-point", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gems_comm.initialize_cuda()
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("nccl", device_id=dev)
    rank, P = dist.get_rank(), dist.get_world_size()
    tr = halo_transport.negotiate(dev)
    dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float32
    methods = args.slice_methods or (["square", "vertical"] if int(P ** 0.5) ** 2 == P else ["vertical", "horizontal"])
    cases = [(m, t, c, args.halo_len, dtype) for m in methods for t in args.tiles for c in args.channels]
    if args.reference_point:      # README.md:24-43: 1024^2 image, 4 vertical parts, halo 3, C = 1, fp32
        cases = [("vertical", None, 1, 3, torch.float32)] + cases
    rows = []
    for method, tile, C_, halo, dt in cases:
        if tile is None:
            th, tw = 1024, 1024 // P
        else:
            th, tw = tile, tile
        # memory bound: a 16384^2 tile of 64 bf16 channels is 34 GB (+ the padded copy)
        if th * tw * C_ * (2 if dt == torch.bfloat16 else 4) > 40e9:
            continue
        x = torch.randn(1, C_, th, tw, device=dev).to(dt)
        layer = halo_exchange_layer(local_rank=rank, spatial_size=1, num_spatial_parts=P, halo_len=halo, slice_method=method)
        recv = sum(t.numel() * t.element_size() for t in layer._exchange(x, halo, halo) if t is not None)
        with torch.no_grad():
            us_x = timed(lambda: layer._exchange(x, halo, halo), args.iterations, args.warmup, dev)
            us_l = timed(lambda: layer(x), max(5, args.iterations // 5), 2, dev)
        rb = torch.tensor([recv], device=dev, dtype=torch.int64)
        dist.all_reduce(rb, op=dist.ReduceOp.MAX)
        row = dict(P=P, slice_method=method, tile=[th, tw], channels=C_, halo_len=halo, dtype=str(dt).replace("torch.", ""),
                   transport=tr.name, us_exchange=round(us_x, 2), us_layer=round(us_l, 2), recv_bytes=int(rb.item()),
                   GBps=round(int(rb.item()) / us_x / 1e3, 2), frac_of_900GBps=round(int(rb.item()) / us_x / 1e3 / 900, 4))
        rows.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
        del x, layer
        torch.cuda.empty_cache()
    if rank == 0 and args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
