"""What the exact backward (SPCONV_EXACT_BACKWARD=1) adds to a training step, per halo layer of the AmoebaNet-D
spatial stage (tests/golden/layers_amoebanetd_sp4.json), at the tile shapes of a 4-GPU square split with all
neighbours present (an interior tile; 1-D kernels exchange along one axis only), bf16, on one GPU:

    python benchmarks/communication/halo/exact_backward_cost.py [--image 8192] [--reps 10] [--step-ms X]

Per layer it times, with CUDA events, the two kernels the exact backward adds on the tile's own GPU -- the strip
gradient (spc_conv2d_dgrad_halo / spc_pool2d_bwd_halo) and the accumulate (spc_halo_accumulate) -- next to the
layer's existing input-gradient kernel (spc_conv2d_dgrad / spc_pool2d_bwd).  The strips' trip to the neighbours
(one more post + collect per layer, the size of the forward exchange in fp32) needs several ranks and is not
included.  It also prints the mailbox arena the peer transport hands out for the layer list at that split: the
forward slots and, with the switch on, the reverse (fp32) slots.  --step-ms: a measured step time to relate the
added time to.  The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", "..", ".."))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from mpi4dl_b200 import _lib  # noqa: E402
from mpi4dl_b200.torchgems import halo_transport as ht  # noqa: E402

GR, GC = 2, 2    # 4 GPUs, square split


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "power limit unavailable"
    return "%s (%s)" % (name, out)


def halo_layers(image):
    """Distinct exchanging layers (one module per distinct shape, as bench.py builds them) at the N=4 tile, with
    the number of times the step runs each."""
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "layers_amoebanetd_sp4.json")))
    shrink = d["image"] // image
    uniq = {}
    for l in d["layers"]:
        l = dict(l, H=l["H"] // shrink, W=l["W"] // shrink)
        key = json.dumps({k: v for k, v in l.items() if k != "kind"}, sort_keys=True)
        h = (l["R"] // 2, l["S"] // 2) if l["op"] == "conv" else ((l["k"] - 1) // 2,) * 2
        if h != (0, 0):
            uniq.setdefault(key, [l, l["H"] // GR, l["W"] // GC, h, 0])[4] += 1
    return [tuple(v) for v in uniq.values()]


def mask_for(l):
    m = [1, 1, 1, 1, 0, 1, 1, 1, 1]
    if l["op"] == "conv":
        if l["R"] == 1:
            for i in (0, 1, 2, 6, 7, 8):
                m[i] = 0
        if l["S"] == 1:
            for i in (0, 3, 6, 2, 5, 8):
                m[i] = 0
    return m


def arena_bytes(layers, esize):
    """Forward and reverse slot bytes the peer transport allocates for these layers (its own sizing code)."""
    tr = ht.PeerTransport.__new__(ht.PeerTransport)
    tr.arena_bytes, tr.nflags, tr.data_top, tr.flag_top = 1 << 62, 1 << 30, 0, 0

    class Layer:
        pass

    fwd = rev = 0
    for l, th, tw, (hh, hw), _ in layers:
        shape = (1, l["C"], th, tw)
        top = tr.data_top
        tr._slot_for(Layer(), ("fwd",), shape, esize, hh, hw)
        fwd += tr.data_top - top
        top = tr.data_top
        tr._slot_for(Layer(), ("reverse",), shape, 4, hh, hw)
        rev += tr.data_top - top
    return fwd, rev


def ev(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--image", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--step-ms", type=float, default=0.0)
    args = ap.parse_args()
    layers = halo_layers(args.image)
    fwd, rev = arena_bytes(layers, 2)
    print("mailbox arena at N=4 (square), bf16, %d exchanging layers: forward slots %.1f MB, reverse slots %.1f MB, "
          "high-water %.1f MB with SPCONV_EXACT_BACKWARD=1 (default arena %d MB)"
          % (len(layers), fwd / 2**20, rev / 2**20, (fwd + rev) / 2**20, int(os.environ.get("SPCONV_ARENA_MB", "256"))))
    if not torch.cuda.is_available():
        raise SystemExit("timing needs a CUDA device")
    L = _lib.lib()
    dev = "cuda:0"
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P9 = C.c_void_p * 9
    dt = torch.bfloat16
    print("card: %s" % card())
    print("%-46s %5s %9s %9s %9s %9s" % ("layer (N=4 tile)", "runs", "strip ms", "accum ms", "added ms", "dgrad ms"))
    tot_add = tot_base = 0.0
    for l, th, tw, (hh, hw), runs in layers:
        mask = mask_for(l)
        C_ = l["C"]
        x = torch.randn(1, C_, th, tw, device=dev).to(dt)
        strips = [torch.randn(ht.strip_shape(i, 1, C_, th, tw, hh, hw), device=dev).to(dt) if mask[i] else None
                  for i in range(9)]
        g = [torch.empty(ht.strip_shape(i, 1, C_, th, tw, hh, hw), device=dev) if mask[i] else None for i in range(9)]
        gp = P9(*[C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None) for t in g])
        dx = torch.empty_like(x)
        if l["op"] == "conv":
            d = _lib.ConvDesc(1, C_, th, tw, l["K"], l["R"], l["S"], l["stride_h"], l["stride_w"], hh, hw,
                              _lib.SPC_BF16, 0)
            Ho, Wo = C.c_int(), C.c_int()
            L.spc_conv_out_shape(C.byref(d), C.byref(Ho), C.byref(Wo))
            w = (torch.randn(l["K"], C_, l["R"], l["S"], device=dev) * 0.05).to(dt)
            gy = torch.randn(1, l["K"], Ho.value, Wo.value, device=dev).to(dt)
            nws = L.spc_conv_workspace_bytes(C.byref(d), 1)
            ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=dev)
            strip = lambda: _lib.check(L.spc_conv2d_dgrad_halo(C.byref(d), C.c_void_p(gy.data_ptr()),  # noqa: E731
                                                               C.c_void_p(w.data_ptr()), C.byref(gp), st), "dgrad_halo")
            base = lambda: _lib.check(L.spc_conv2d_dgrad(C.byref(d), C.c_void_p(gy.data_ptr()),  # noqa: E731
                                                         C.c_void_p(w.data_ptr()), C.c_void_p(dx.data_ptr()),
                                                         C.c_void_p(ws.data_ptr()), nws, st), "dgrad")
            name = "conv %dx%d s%d %d->%d @%dx%d" % (l["R"], l["S"], l["stride_h"], C_, l["K"], th, tw)
        else:
            mode = _lib.SPC_POOL_MAX if l["mode"] == "max" else _lib.SPC_POOL_AVG
            d = _lib.PoolDesc(1, C_, th, tw, l["k"], l["stride"], l["pad"], mode, _lib.SPC_BF16)
            Ho, Wo = (th + 2 * l["pad"] - l["k"]) // l["stride"] + 1, (tw + 2 * l["pad"] - l["k"]) // l["stride"] + 1
            gy = torch.randn(1, C_, Ho, Wo, device=dev).to(dt)
            halo = _lib.make_halo(strips)
            strip = lambda: _lib.check(L.spc_pool2d_bwd_halo(C.byref(d), C.c_void_p(x.data_ptr()), C.byref(halo),  # noqa: E731
                                                             C.c_void_p(gy.data_ptr()), C.byref(gp), st), "pool_bwd_halo")
            base = lambda: _lib.check(L.spc_pool2d_bwd(C.byref(d), C.c_void_p(x.data_ptr()), C.byref(halo),  # noqa: E731
                                                       C.c_void_p(gy.data_ptr()), C.c_void_p(dx.data_ptr()), st),
                                      "pool_bwd")
            name = "%s pool %d s%d %d ch @%dx%d" % (l["mode"], l["k"], l["stride"], C_, th, tw)
        acc = lambda: _lib.check(L.spc_halo_accumulate(1, C_, th, tw, hh, hw, _lib.SPC_BF16,  # noqa: E731
                                                       C.c_void_p(dx.data_ptr()), C.byref(gp), st), "accumulate")
        t_s, t_a, t_b = ev(strip, args.reps), ev(acc, args.reps), ev(base, args.reps)
        tot_add += runs * (t_s + t_a)
        tot_base += runs * t_b
        print("%-46s %5d %9.3f %9.3f %9.3f %9.3f" % (name, runs, t_s, t_a, t_s + t_a, t_b))
        del x, strips, g, dx, gy
    print("per step (each layer times its runs): added %.3f ms (the same layers' existing input-gradient kernels: %.3f ms)"
          % (tot_add, tot_base))
    if args.step_ms:
        print("against a step of %.1f ms: +%.1f %%" % (args.step_ms, 100.0 * tot_add / args.step_ms))


if __name__ == "__main__":
    main()
