"""Time the 1x1 convolutions of the AmoebaNet-D spatial stage (tests/golden/layers_amoebanetd_sp4.json) in four arms:

    fp32_direct  libspconv, fp32, SPC_ALGO_AUTO (the CUDA-core direct kernels)
    fp32_tf32    libspconv, fp32, SPC_ALGO_TF32 (gemm_tf32.cu)
    bf16         libspconv, bf16, SPC_ALGO_AUTO (gemm_tc.cu)
    cudnn_tf32   PyTorch / cuDNN fp32 with torch.backends.cudnn.allow_tf32 = True (how PyTorch runs the reference)

at the N=1 tile (one GPU holds the whole stage extent) and the N=4 tile (half of it), fprop / dgrad / wgrad, with CUDA
events after a warm-up.  The arms run alternated, in two rounds; the table gives the faster round.  Prints ms per call
and TFLOP/s per distinct shape, then the sums over every 1x1 layer of the stage (shape time x count), next to the GPU
name and power limit.  Shapes that do not fit the GPU in fp32 are reported as such.

    python benchmarks/tf32_pointwise.py [--iters 5] [--warmup 2] [--json out.json]
"""
import argparse
import collections
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from mpi4dl_b200 import _lib  # noqa: E402

ARMS = ("fp32_direct", "fp32_tf32", "bf16", "cudnn_tf32")
OPS = ("fprop", "dgrad", "wgrad")


def pointwise_layers():
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "layers_amoebanetd_sp4.json")))
    count = collections.Counter()
    for l in d["layers"]:
        if l["op"] == "conv" and (l["R"], l["S"]) == (1, 1):
            count[(l["C"], l["K"], l["stride_h"], l["H"], l["W"])] += 1
    return sorted(count.items())


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = "nvidia-smi unavailable"
    return name, q


class LibConv:
    """one 1x1 convolution through the C ABI, buffers allocated once"""

    def __init__(self, Cc, K, s, H, W, dtype, algo, x, w, dy):
        self.d = _lib.ConvDesc(1, Cc, H, W, K, 1, 1, s, s, 0, 0, _lib.dtype_code(dtype), algo)
        self.x, self.w, self.dy = x, w, dy
        self.y = torch.empty((1, K, H // s, W // s), dtype=dtype, device="cuda")
        self.dx = torch.empty_like(x)
        self.dw = torch.empty(w.shape, dtype=torch.float32, device="cuda")
        L = _lib.lib()
        n = max(L.spc_conv_workspace_bytes(C.byref(self.d), op) for op in range(3))
        self.ws = torch.empty(max(n, 16), dtype=torch.uint8, device="cuda")
        self.halo = _lib.make_halo([None] * 9)
        self.tc = [L.spc_conv_uses_tcgen05(C.byref(self.d), op) for op in range(3)]

    def run(self, op):
        L, p = _lib.lib(), lambda t: C.c_void_p(t.data_ptr())
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        nws = self.ws.numel()
        if op == "fprop":
            rc = L.spc_conv2d_fwd(C.byref(self.d), p(self.x), C.byref(self.halo), p(self.w), None, p(self.y), p(self.ws),
                                  nws, st)
        elif op == "dgrad":
            rc = L.spc_conv2d_dgrad(C.byref(self.d), p(self.dy), p(self.w), p(self.dx), p(self.ws), nws, st)
        else:
            rc = L.spc_conv2d_wgrad(C.byref(self.d), p(self.x), C.byref(self.halo), p(self.dy), p(self.dw), None, 0,
                                    p(self.ws), nws, st)
        _lib.check(rc, op)


class CudnnConv:
    def __init__(self, s, x, w, dy):
        self.s, self.x, self.w, self.dy = s, x, w, dy

    def run(self, op):
        if op == "fprop":
            F.conv2d(self.x, self.w, None, self.s)
        elif op == "dgrad":
            torch.nn.grad.conv2d_input(self.x.shape, self.w, self.dy, self.s)
        else:
            torch.nn.grad.conv2d_weight(self.x, self.w.shape, self.dy, self.s)


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


def measure_shape(Cc, K, s, H, W, iters, warmup, rounds):
    """{arm: {op: best ms}} for one shape; the arms alternate inside each round"""
    best = {a: {} for a in ARMS}
    gen = torch.Generator(device="cuda").manual_seed(Cc + K + H)
    x = torch.randn((1, Cc, H, W), device="cuda", generator=gen)
    w = torch.randn((K, Cc, 1, 1), device="cuda", generator=gen) / Cc ** 0.5
    dy = torch.randn((1, K, H // s, W // s), device="cuda", generator=gen)
    xb, wb, dyb = x.bfloat16(), w.bfloat16(), dy.bfloat16()
    impl = {"fp32_direct": LibConv(Cc, K, s, H, W, torch.float32, _lib.SPC_ALGO_AUTO, x, w, dy),
            "fp32_tf32": LibConv(Cc, K, s, H, W, torch.float32, _lib.SPC_ALGO_TF32, x, w, dy),
            "bf16": LibConv(Cc, K, s, H, W, torch.bfloat16, _lib.SPC_ALGO_AUTO, xb, wb, dyb),
            "cudnn_tf32": CudnnConv(s, x, w, dy)}
    assert impl["fp32_tf32"].tc == [1, 1, 1] and impl["fp32_direct"].tc == [0, 0, 0], (Cc, K, s, H)
    for _ in range(rounds):
        for arm in ARMS:
            for op in OPS:
                with torch.backends.cudnn.flags(enabled=True, allow_tf32=True):
                    t = time_ms(lambda: impl[arm].run(op), iters, warmup)
                best[arm][op] = min(best[arm].get(op, float("inf")), t)
    del impl, x, w, dy, xb, wb, dyb
    torch.cuda.empty_cache()
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--tiles", default="1,4", help="N of the square tiles: 1 (whole extent) and/or 4 (half)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tf32_pointwise.py: no CUDA device")
    name, power = gpu_info()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power))
    print("# %d warm-up + %d timed calls per (arm, op), arms alternated, best of %d rounds" %
          (args.warmup, args.iters, args.rounds))
    layers = pointwise_layers()
    results = []
    for n in [int(v) for v in args.tiles.split(",")]:
        div = {1: 1, 4: 2}[n]
        totals = {a: collections.Counter() for a in ARMS}
        print("\n## N=%d tile" % n)
        print("%-24s %5s %-6s " % ("C->K stride HxW", "count", "op") +
              " ".join("%20s" % a for a in ARMS) + "   (ms | TFLOP/s)")
        for (Cc, K, s, H, W), cnt in layers:
            H, W = H // div, W // div
            try:
                best = measure_shape(Cc, K, s, H, W, args.iters, args.warmup, args.rounds)
            except torch.cuda.OutOfMemoryError:
                torch.cuda.empty_cache()
                print("%-24s %5d  does not fit the GPU in fp32" % ("%d->%d s%d %dx%d" % (Cc, K, s, H, W), cnt))
                results.append({"tile": n, "C": Cc, "K": K, "stride": s, "H": H, "W": W, "count": cnt, "oom": True})
                continue
            flops = 2.0 * Cc * K * (H // s) * (W // s)
            for op in OPS:
                cells = []
                for a in ARMS:
                    ms = best[a][op]
                    totals[a][op] += ms * cnt
                    cells.append("%9.3f | %6.1f" % (ms, flops / ms / 1e9))
                print("%-24s %5d %-6s " % ("%d->%d s%d %dx%d" % (Cc, K, s, H, W), cnt, op) + " ".join(cells))
            results.append({"tile": n, "C": Cc, "K": K, "stride": s, "H": H, "W": W, "count": cnt, "ms": best})
        print("%-37s " % ("sum over the stage's 1x1 layers") +
              " ".join("%20s" % "" for _ in ARMS))
        for op in OPS + ("all",):
            print("%-30s %-6s " % ("", op) + " ".join(
                "%20.2f" % (sum(totals[a].values()) if op == "all" else totals[a][op]) for a in ARMS))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit_max_sm_clock": power, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
