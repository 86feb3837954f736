"""Self-checking halo-exchange (+ convolution) benchmark, one process per tile -- the reference's own
validation tool for this path (benchmarks/communication/halo/benchmark_sp_halo_exchange_conv.py and
benchmark_sp_halo_exchange.py), same flags, launched with torchrun:

    torchrun --nproc-per-node 4 benchmarks/communication/halo/benchmark_sp_halo_exchange_conv.py \\
        --image-size 1024 --halo-len 3 --num-spatial-parts 4 --slice-method vertical \\
        --enable-val-recv-tensors --enable-val-conv

Input = arange image, weights = bias = 1 (known answers, exact for small images).  Prints per rank
"Rank:r Time taken (ms):t" for the timed op (exchange + conv through conv_spatial; exchange only with
--exchange-only) and "Validation passed Rank:r" / "Validation failed Rank:r" for each enabled check.
"""
import argparse
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", "..", ".."), HERE]

import halo_common as hc  # noqa: E402
from mpi4dl_b200.torchgems import comm as gems_comm  # noqa: E402
from mpi4dl_b200.torchgems.spatial import conv_spatial, halo_exchange_layer  # noqa: E402


def get_parser(exchange_only_default=False):
    p = argparse.ArgumentParser(description="Halo exchange benchmark", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--fp16-allreduce", action="store_true", default=False, help="accepted for compatibility, unused")
    p.add_argument("--image-size", type=int, default=8, help="Full image size")
    p.add_argument("--batch-size", type=int, default=1, help="input batch size")
    p.add_argument("--halo-len", type=int, default=1, help="halo length")
    p.add_argument("--warmup", type=int, default=10, help="warmups")
    p.add_argument("--iterations", type=int, default=100, help="Iterations")
    p.add_argument("--in-channels", type=int, default=1, help="number of input channels")
    p.add_argument("--out-channels", type=int, default=256, help="number of output channels")
    p.add_argument("--enable-val-recv-tensors", action="store_true", default=False, help="Enable validation of recv tensors")
    p.add_argument("--enable-val-conv", action="store_true", default=False, help="Enable validation of convolution")
    p.add_argument("--enable-val-small-conv", action="store_true", default=False,
                   help="accepted for compatibility: the convolution here is deterministic, --enable-val-conv covers it")
    p.add_argument("--enable-deterministic", action="store_true", default=False,
                   help="torch.use_deterministic_algorithms(True): bit-reproducible weight gradients")
    p.add_argument("--enable-one-h-dim-kernel", action="store_true", default=False, help="Set dimension (height) of kernel to 1")
    p.add_argument("--enable-one-w-dim-kernel", action="store_true", default=False, help="Set dimension (width) of kernel to 1")
    p.add_argument("--num-spatial-parts", type=int, default=4, help="Number of partitions in spatial parallelism")
    p.add_argument("--slice-method", type=str, default="square", help="Slice method (square, vertical, and horizontal)")
    p.add_argument("--exchange-only", action="store_true", default=exchange_only_default,
                   help="time and validate the halo exchange alone (benchmark_sp_halo_exchange.py)")
    p.add_argument("--dtype", choices=["fp32", "bf16"], default="fp32")
    return p


def main(exchange_only_default=False):
    args = get_parser(exchange_only_default).parse_args()
    if args.enable_deterministic:
        torch.use_deterministic_algorithms(True)
    gems_comm.initialize_cuda()
    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        dist.init_process_group(os.environ.get("SPCONV_DIST_BACKEND", "nccl"))
    rank, size = dist.get_rank(), dist.get_world_size()
    P, method, halo = args.num_spatial_parts, args.slice_method, args.halo_len
    assert size == P, "launch one process per spatial part (world %d, --num-spatial-parts %d)" % (size, P)
    print("rank : %d size:  %d" % (rank, size), flush=True)
    kh = 1 if args.enable_one_h_dim_kernel else 2 * halo + 1
    kw = 1 if args.enable_one_w_dim_kernel else 2 * halo + 1
    dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float32
    dev = torch.device("cuda", torch.cuda.current_device())

    full = hc.full_image(args.batch_size, args.in_channels, args.image_size)
    x = torch.from_numpy(hc.tile(full, method, P, rank)).to(dev).to(dtype)
    exchange = halo_exchange_layer(local_rank=rank, spatial_size=1, num_spatial_parts=P, halo_len=halo, slice_method=method)
    conv = conv_spatial(local_rank=rank, spatial_size=1, num_spatial_parts=P, in_channels=args.in_channels,
                        out_channels=args.out_channels, kernel_size=(kh, kw), stride=1, padding=((kh - 1) // 2, (kw - 1) // 2),
                        slice_method=method).to(dev).to(dtype)
    with torch.no_grad():
        conv.weight.fill_(1.0)
        conv.bias.fill_(1.0)
    op = (lambda: exchange(x)) if args.exchange_only else (lambda: conv(x))

    with torch.no_grad():
        for _ in range(args.warmup):
            op()
        dist.barrier()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iterations):
            op()
        t1.record()
        torch.cuda.synchronize()
        print("Rank:%d Time taken (ms):%s" % (rank, t0.elapsed_time(t1) / max(1, args.iterations)), flush=True)

        ok = True
        if args.enable_val_recv_tensors or args.exchange_only:
            got = exchange(x).float().cpu().numpy()
            want = hc.expected_padded_tile(full, method, P, rank, halo)
            ok = ok and got.shape == want.shape and bool(np.equal(got.astype(np.int64), want.astype(np.int64)).all())
        if args.enable_val_conv and not args.exchange_only:
            got = conv(x).float().cpu().numpy()
            want = hc.expected_conv_tile(full, method, P, rank, kh, kw, args.out_channels)
            ok = ok and got.shape == want.shape and bool(np.equal(got.astype(np.int64), want.astype(np.int64)).all())
        if args.enable_val_recv_tensors or args.enable_val_conv or args.exchange_only:
            print(("Validation passed Rank:%d" if ok else "Validation failed Rank:%d") % rank, flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
