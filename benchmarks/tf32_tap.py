"""Time the stride-1 multi-tap convolutions of the two BASELINE spatial stages (tests/golden/layers_amoebanetd_sp4.json:
1x7 / 7x1, tests/golden/layers_resnet101_sp2.json: 3x3) in four arms:

    fp32_direct    libspconv, fp32, SPC_ALGO_AUTO (the CUDA-core direct kernels)
    fp32_tf32_all  libspconv, fp32, SPC_ALGO_TF32_ALL (conv_tap_tf32.cu)
    bf16           libspconv, bf16, SPC_ALGO_AUTO (conv_tap.cu / wgrad_tap.cu)
    cudnn_tf32     PyTorch / cuDNN fp32 with torch.backends.cudnn.allow_tf32 = True (how PyTorch runs the reference)

at the N=1 tile (one GPU holds the whole stage extent) and the N=4 tile (half of it), fprop / dgrad / wgrad, with CUDA
events after a warm-up, the arms alternated in each of two rounds (the table gives the faster round).  Prints ms per
call and TFLOP/s per distinct shape and the sums over the stage's layers (shape time x count), then the fp32 layers that
SPC_ALGO_TF32_ALL leaves on the direct kernels (the stride-2 3x3 ones), next to the GPU name and power limit.  Shapes
that do not fit the GPU in fp32 are reported as such.

    python benchmarks/tf32_tap.py [--iters 5] [--warmup 2] [--json out.json]
"""
import argparse
import collections
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from mpi4dl_b200 import _lib  # noqa: E402
from tf32_pointwise import gpu_info, time_ms  # noqa: E402

ARMS = ("fp32_direct", "fp32_tf32_all", "bf16", "cudnn_tf32")
OPS = ("fprop", "dgrad", "wgrad")
LISTS = (("amoeba", "layers_amoebanetd_sp4.json"), ("resnet", "layers_resnet101_sp2.json"))


def tap_layers(stride):
    """{(list, C, K, R, S, stride, H, W): count} of the multi-tap convolutions with this stride"""
    count = collections.Counter()
    for tag, fn in LISTS:
        for l in json.load(open(os.path.join(ROOT, "tests", "golden", fn)))["layers"]:
            if l["op"] == "conv" and l["R"] * l["S"] > 1 and l["stride_h"] == stride:
                count[(tag, l["C"], l["K"], l["R"], l["S"], stride, l["H"], l["W"])] += 1
    return sorted(count.items())


class LibConv:
    """one convolution through the C ABI, buffers allocated once"""

    def __init__(self, Cc, K, R, S, s, H, W, dtype, algo, x, w, dy):
        self.d = _lib.ConvDesc(1, Cc, H, W, K, R, S, s, s, (R - 1) // 2, (S - 1) // 2, _lib.dtype_code(dtype), algo)
        L = _lib.lib()
        Ho, Wo = C.c_int(), C.c_int()
        L.spc_conv_out_shape(C.byref(self.d), C.byref(Ho), C.byref(Wo))
        self.x, self.w, self.dy = x, w, dy
        self.y = torch.empty((1, K, Ho.value, Wo.value), dtype=dtype, device="cuda")
        self.dx = torch.empty_like(x)
        self.dw = torch.empty(w.shape, dtype=torch.float32, device="cuda")
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
    def __init__(self, s, pad, x, w, dy):
        self.s, self.pad, self.x, self.w, self.dy = s, pad, x, w, dy

    def run(self, op):
        if op == "fprop":
            F.conv2d(self.x, self.w, None, self.s, self.pad)
        elif op == "dgrad":
            torch.nn.grad.conv2d_input(self.x.shape, self.w, self.dy, self.s, self.pad)
        else:
            torch.nn.grad.conv2d_weight(self.x, self.w.shape, self.dy, self.s, self.pad)


def measure_shape(Cc, K, R, S, s, H, W, arms, iters, warmup, rounds):
    """{arm: {op: best ms}} for one shape; the arms alternate inside each round"""
    best = {a: {} for a in arms}
    gen = torch.Generator(device="cuda").manual_seed(Cc + K + H + R)
    pad = ((R - 1) // 2, (S - 1) // 2)
    x = torch.randn((1, Cc, H, W), device="cuda", generator=gen)
    w = torch.randn((K, Cc, R, S), device="cuda", generator=gen) / (Cc * R * S) ** 0.5
    Ho, Wo = (H + 2 * pad[0] - R) // s + 1, (W + 2 * pad[1] - S) // s + 1
    dy = torch.randn((1, K, Ho, Wo), device="cuda", generator=gen)
    impl = {"fp32_direct": lambda: LibConv(Cc, K, R, S, s, H, W, torch.float32, _lib.SPC_ALGO_AUTO, x, w, dy),
            "fp32_tf32_all": lambda: LibConv(Cc, K, R, S, s, H, W, torch.float32, _lib.SPC_ALGO_TF32_ALL, x, w, dy),
            "bf16": lambda: LibConv(Cc, K, R, S, s, H, W, torch.bfloat16, _lib.SPC_ALGO_AUTO, x.bfloat16(),
                                    w.bfloat16(), dy.bfloat16()),
            "cudnn_tf32": lambda: CudnnConv(s, pad, x, w, dy)}
    impl = {a: impl[a]() for a in arms}
    if "fp32_tf32_all" in impl:
        assert impl["fp32_tf32_all"].tc == [1, 1, 1] and impl["fp32_direct"].tc == [0, 0, 0], (Cc, K, R, S)
    for _ in range(rounds):
        for arm in arms:
            for op in OPS:
                with torch.backends.cudnn.flags(enabled=True, allow_tf32=True):
                    t = time_ms(lambda: impl[arm].run(op), iters, warmup)
                best[arm][op] = min(best[arm].get(op, float("inf")), t)
    del impl, x, w, dy
    torch.cuda.empty_cache()
    return best


def table(title, layers, arms, n, args, results):
    div = {1: 1, 4: 2}[n]
    totals = {a: collections.Counter() for a in arms}
    print("\n## %s, N=%d tile" % (title, n))
    print("%-30s %5s %-6s " % ("list C->K RxS stride HxW", "count", "op") + " ".join("%20s" % a for a in arms) +
          "   (ms | TFLOP/s)")
    for (tag, Cc, K, R, S, s, H, W), cnt in layers:
        H, W = H // div, W // div
        label = "%s %d->%d %dx%d s%d %dx%d" % (tag, Cc, K, R, S, s, H, W)
        rec = {"tile": n, "list": tag, "C": Cc, "K": K, "R": R, "S": S, "stride": s, "H": H, "W": W, "count": cnt}
        try:
            best = measure_shape(Cc, K, R, S, s, H, W, arms, args.iters, args.warmup, args.rounds)
        except torch.cuda.OutOfMemoryError:
            torch.cuda.empty_cache()
            print("%-30s %5d  does not fit the GPU in fp32" % (label, cnt))
            results.append(dict(rec, oom=True))
            continue
        flops = 2.0 * Cc * K * R * S * (H // s) * (W // s)
        for op in OPS:
            cells = []
            for a in arms:
                ms = best[a][op]
                totals[a][op] += ms * cnt
                cells.append("%9.3f | %6.1f" % (ms, flops / ms / 1e9))
            print("%-30s %5d %-6s " % (label, cnt, op) + " ".join(cells))
        results.append(dict(rec, ms=best))
    print("sum over the layers (ms x count)")
    for op in OPS + ("all",):
        print("%-37s %-6s " % ("", op) + " ".join(
            "%20.2f" % (sum(totals[a].values()) if op == "all" else totals[a][op]) for a in arms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--tiles", default="1,4", help="N of the square tiles: 1 (whole extent) and/or 4 (half)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tf32_tap.py: no CUDA device")
    name, power = gpu_info()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power))
    print("# %d warm-up + %d timed calls per (arm, op), arms alternated, best of %d rounds" %
          (args.warmup, args.iters, args.rounds))
    results = []
    for n in [int(v) for v in args.tiles.split(",")]:
        table("stride-1 multi-tap layers", tap_layers(1), ARMS, n, args, results)
        table("fp32 layers left on the direct kernels (stride 2)", tap_layers(2), ("fp32_direct",), n, args, results)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit_max_sm_clock": power, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
