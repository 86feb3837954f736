"""Time the fused BatchNorm2d + ReLU (csrc/bnrelu.cu) at the BatchNorm shapes of the AmoebaNet-D spatial stage at the
N = 4 tile (tests/test_bnrelu_bounds.py STAGE: 104 channels at 2048^2, 208 and 52 channels at 2048^2 and 1024^2), bf16,
with CUDA events after a warm-up: each of the four entry points through the C ABI, and bn_relu forward + backward
(what a training step runs per BatchNorm).  Every measurement is repeated in `--rounds` rounds and the table gives the
fastest and the slowest round, next to the GPU name and power limit.

    python benchmarks/bn_relu.py [--iters 20] [--warmup 3] [--rounds 2] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from benchmarks.tf32_pointwise import gpu_info  # noqa: E402
from mpi4dl_b200 import _lib  # noqa: E402
from mpi4dl_b200.torchgems.fused import bn_relu  # noqa: E402
from tests.test_bnrelu_bounds import STAGE, run_apply, run_bwd_apply, run_bwd_reduce, run_stats  # noqa: E402

OPS = ("stats", "apply", "bwd_reduce", "bwd_apply", "bn_relu_fwd_bwd")


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_shape(s, iters, warmup):
    g = torch.Generator(device="cuda").manual_seed(0)
    shape = (s.N, s.C, s.H, s.W)
    y = torch.randn(shape, device="cuda", generator=g).add_(0.3).to(torch.bfloat16)
    dz = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    gamma = torch.rand(s.C, device="cuda", generator=g) + 0.5
    beta = torch.rand(s.C, device="cuda", generator=g) - 0.5
    mean, var = run_stats(y)
    rstd = torch.rsqrt(var + 1e-5)
    dsum, dsumx = run_bwd_reduce(dz, y, mean, rstd, gamma, beta, True)
    bn = torch.nn.BatchNorm2d(s.C).cuda().to(torch.bfloat16)
    x = y.clone().requires_grad_(True)

    def fwd_bwd():
        bn_relu(x, bn, relu=True).backward(dz)
        x.grad = None
        bn.weight.grad = bn.bias.grad = None

    fns = {
        "stats": lambda: run_stats(y),
        "apply": lambda: run_apply(y, mean, rstd, gamma, beta, True),
        "bwd_reduce": lambda: run_bwd_reduce(dz, y, mean, rstd, gamma, beta, True),
        "bwd_apply": lambda: run_bwd_apply(dz, y, mean, rstd, gamma, beta, True, dsum, dsumx),
        "bn_relu_fwd_bwd": fwd_bwd,
    }
    return {op: time_ms(fns[op], iters, warmup) for op in OPS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = gpu_info()
    print("%s  (power.limit, clocks.max.sm: %s)  libspconv %d" % (name, power, _lib.lib().spc_version()))
    rounds = [{}]
    for r in range(args.rounds):
        rounds.append({})
        for s in STAGE:
            key = "%dx%dx%d" % (s.C, s.H, s.W)
            rounds[-1][key] = bench_shape(s, args.iters, args.warmup)
            torch.cuda.empty_cache()
    rounds = rounds[1:]
    print("%-16s" % "shape" + "".join("%22s" % op for op in OPS) + "   (ms: fastest / slowest round)")
    out = {"gpu": name, "power": power, "shapes": {}}
    for key in rounds[0]:
        row = {op: [min(rd[key][op] for rd in rounds), max(rd[key][op] for rd in rounds)] for op in OPS}
        out["shapes"][key] = row
        print("%-16s" % key + "".join("%22s" % ("%.4f / %.4f" % tuple(row[op])) for op in OPS))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
