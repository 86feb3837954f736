"""Time the stride-2 3x3 convolutions of the two BASELINE spatial stages (tests/golden/layers_amoebanetd_sp4.json,
tests/golden/layers_resnet101_sp2.json) in four arms:

    fp32_direct    libspconv, fp32, SPC_ALGO_AUTO (the CUDA-core direct kernels)
    fp32_strided   libspconv, fp32, SPC_ALGO_TF32_STRIDED (conv_tap_s2_tf32.cu)
    bf16           libspconv, bf16, SPC_ALGO_AUTO
    cudnn_tf32     PyTorch / cuDNN fp32 with torch.backends.cudnn.allow_tf32 = True

at the N=1 tile (one GPU holds the whole stage extent) and the N=4 tile (half of it), fprop / dgrad / wgrad, with CUDA
events after a warm-up, the arms alternated in each of two rounds (the table gives the faster round): ms per call and
TFLOP/s per shape and the sums over the layers, next to the GPU name and power limit.  Shapes that do not fit the GPU in
fp32 with all arms' buffers are reported as such.  Then the sum over ALL convolutions of each stage list in fp32 under
SPC_ALGO_TF32_STRIDED (no fp32 convolution of either list is left on the direct kernels) against cuDNN with allow_tf32.

    python benchmarks/tf32_strided.py [--iters 5] [--warmup 2] [--tiles 1,4] [--stage-tiles 4] [--json out.json]
"""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import torch  # noqa: E402

from mpi4dl_b200 import _lib  # noqa: E402
from tf32_pointwise import gpu_info, time_ms  # noqa: E402
from tf32_tap import LISTS, OPS, CudnnConv, LibConv, tap_layers  # noqa: E402

ARMS = ("fp32_direct", "fp32_strided", "bf16", "cudnn_tf32")
STAGE_ARMS = ("fp32_strided", "cudnn_tf32")


def all_convs(tag, fn):
    """{(list, C, K, R, S, stride, H, W): count} of every convolution of one list"""
    count = collections.Counter()
    for l in json.load(open(os.path.join(ROOT, "tests", "golden", fn)))["layers"]:
        if l["op"] == "conv":
            assert l["stride_h"] == l["stride_w"], l
            count[(tag, l["C"], l["K"], l["R"], l["S"], l["stride_h"], l["H"], l["W"])] += 1
    return sorted(count.items())


def measure_shape(Cc, K, R, S, s, H, W, arms, iters, warmup, rounds):
    """{arm: {op: best ms}} for one shape; the arms alternate inside each round"""
    best = {a: {} for a in arms}
    gen = torch.Generator(device="cuda").manual_seed(Cc + K + H + R)
    pad = ((R - 1) // 2, (S - 1) // 2)
    x = torch.randn((1, Cc, H, W), device="cuda", generator=gen)
    w = torch.randn((K, Cc, R, S), device="cuda", generator=gen) / (Cc * R * S) ** 0.5
    Ho, Wo = (H + 2 * pad[0] - R) // s + 1, (W + 2 * pad[1] - S) // s + 1
    dy = torch.randn((1, K, Ho, Wo), device="cuda", generator=gen)
    f32 = torch.float32
    impl = {"fp32_direct": lambda: LibConv(Cc, K, R, S, s, H, W, f32, _lib.SPC_ALGO_AUTO, x, w, dy),
            "fp32_strided": lambda: LibConv(Cc, K, R, S, s, H, W, f32, _lib.SPC_ALGO_TF32_STRIDED, x, w, dy),
            "bf16": lambda: LibConv(Cc, K, R, S, s, H, W, torch.bfloat16, _lib.SPC_ALGO_AUTO, x.bfloat16(),
                                    w.bfloat16(), dy.bfloat16()),
            "cudnn_tf32": lambda: CudnnConv(s, pad, x, w, dy)}
    impl = {a: impl[a]() for a in arms}
    assert impl["fp32_strided"].tc == [1, 1, 1], "%d->%d %dx%d s%d left the tensor cores" % (Cc, K, R, S, s)
    for _ in range(rounds):
        for arm in arms:
            for op in OPS:
                with torch.backends.cudnn.flags(enabled=True, allow_tf32=True):
                    t = time_ms(lambda: impl[arm].run(op), iters, warmup)
                best[arm][op] = min(best[arm].get(op, float("inf")), t)
    del impl, x, w, dy
    torch.cuda.empty_cache()
    return best


def table(title, layers, arms, n, args, results, per_shape=True):
    div = {1: 1, 4: 2}[n]
    totals = {a: collections.Counter() for a in arms}
    print("\n## %s, N=%d tile" % (title, n))
    if per_shape:
        print("%-30s %5s %-6s " % ("list C->K RxS stride HxW", "count", "op") + " ".join("%20s" % a for a in arms) +
              "   (ms | TFLOP/s)")
    for (tag, Cc, K, R, S, s, H, W), cnt in layers:
        H, W = H // div, W // div
        label = "%s %d->%d %dx%d s%d %dx%d" % (tag, Cc, K, R, S, s, H, W)
        rec = {"table": title, "tile": n, "list": tag, "C": Cc, "K": K, "R": R, "S": S, "stride": s, "H": H, "W": W,
               "count": cnt}
        try:
            best = measure_shape(Cc, K, R, S, s, H, W, arms, args.iters, args.warmup, args.rounds)
        except torch.cuda.OutOfMemoryError:
            torch.cuda.empty_cache()
            print("%-30s %5d  does not fit the GPU in fp32 with all arms' buffers: not in the sums" % (label, cnt))
            results.append(dict(rec, oom=True))
            continue
        flops = 2.0 * Cc * K * R * S * (H // s) * (W // s)
        for op in OPS:
            cells = []
            for a in arms:
                ms = best[a][op]
                totals[a][op] += ms * cnt
                cells.append("%9.3f | %6.1f" % (ms, flops / ms / 1e9))
            if per_shape:
                print("%-30s %5d %-6s " % (label, cnt, op) + " ".join(cells))
        results.append(dict(rec, ms=best))
    print("sum over the layers (ms x count)" + ("" if per_shape else ":  " + " ".join("%20s" % a for a in arms)))
    for op in OPS + ("all",):
        print("%-37s %-6s " % ("", op) + " ".join(
            "%20.2f" % (sum(totals[a].values()) if op == "all" else totals[a][op]) for a in arms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--tiles", default="1,4", help="N of the square tiles: 1 (whole extent) and/or 4 (half)")
    ap.add_argument("--stage-tiles", default="4", help="tiles of the whole-stage sums ('' skips them)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tf32_strided.py: no CUDA device")
    name, power = gpu_info()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power))
    print("# %d warm-up + %d timed calls per (arm, op), arms alternated, best of %d rounds" %
          (args.warmup, args.iters, args.rounds))
    results = []
    for n in [int(v) for v in args.tiles.split(",") if v]:
        table("stride-2 3x3 layers", tap_layers(2), ARMS, n, args, results)
    for n in [int(v) for v in args.stage_tiles.split(",") if v]:
        for tag, fn in LISTS:
            table("all %d convolutions of %s, fp32" % (sum(c for _, c in all_convs(tag, fn)), fn), all_convs(tag, fn),
                  STAGE_ARMS, n, args, results, per_shape=False)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit_max_sm_clock": power, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
