"""Cost of the deterministic weight gradient (spc_conv2d_wgrad_deterministic, torch.use_deterministic_algorithms(True)).

Per unique conv layer of both bench layer lists (AmoebaNet-D(18, 416) at 8192^2, ResNet-v2-101 at 4096^2), on the tile
of 4 GPUs (a quarter of the image) and of 1 GPU (the whole image), in bf16 and in fp32 with SPC_ALGO_TF32_STRIDED:
spc_conv2d_wgrad and spc_conv2d_wgrad_deterministic in ms (CUDA events, median of --reps calls after a warm-up), and
the slice-buffer MB (workspace op 3 - op 2).  Shapes whose tensors do not fit the GPU are "not measured".  Then the
six-cell step of benchmarks/amp_stage.py (bf16_amp and fp32_strided arms) with the mode off, on, and on with
torch.utils.deterministic.fill_uninitialized_memory = False, which separates PyTorch's NaN fill of new tensors from
this library's cost.  The GPU name and power limit are read in the same run.

    python benchmarks/deterministic_wgrad.py [--tiles 4,1] [--reps 5] [--image 4096] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import torch  # noqa: E402

from mpi4dl_b200 import _lib  # noqa: E402
from tf32_pointwise import gpu_info  # noqa: E402

LISTS = ("layers_amoebanetd_sp4.json", "layers_resnet101_sp2.json")
PATHS = (("bf16", torch.bfloat16, _lib.SPC_BF16, _lib.SPC_ALGO_AUTO),
         ("fp32_strided", torch.float32, _lib.SPC_F32, _lib.SPC_ALGO_TF32_STRIDED))


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def time_layer(l, edge_div, dtype, spc_dtype, algo, reps):
    L = _lib.lib()
    H, W = l["H"] // edge_div, l["W"] // edge_div
    d = _lib.ConvDesc(1, l["C"], H, W, l["K"], l["R"], l["S"], l["stride_h"], l["stride_w"], l["pad_h"], l["pad_w"],
                      spc_dtype, algo)
    Ho, Wo = C.c_int(), C.c_int()
    L.spc_conv_out_shape(C.byref(d), C.byref(Ho), C.byref(Wo))
    w2, w3 = L.spc_conv_workspace_bytes(C.byref(d), 2), L.spc_conv_workspace_bytes(C.byref(d), 3)
    res = dict(slice_MB=(w3 - w2) / 2 ** 20)
    try:
        x = torch.randn(1, l["C"], H, W, device="cuda").to(dtype)
        dy = torch.randn(1, l["K"], Ho.value, Wo.value, device="cuda").to(dtype)
        dw = torch.empty(l["K"], l["C"], l["R"], l["S"], device="cuda")
        db = torch.empty(l["K"], device="cuda") if l.get("bias") else None
        ws = torch.empty(max(w3, 16), dtype=torch.uint8, device="cuda")
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        return dict(res, default_ms="not measured", deterministic_ms="not measured")
    halo = _lib.Halo()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for name, fn, n in (("default_ms", L.spc_conv2d_wgrad, w2), ("deterministic_ms", L.spc_conv2d_wgrad_deterministic, w3)):
        ts = []
        for i in range(reps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(fn(C.byref(d), _ptr(x), C.byref(halo), _ptr(dy), _ptr(dw), _ptr(db), 0, _ptr(ws), n, st), name)
            e1.record()
            torch.cuda.synchronize()
            if i:
                ts.append(e0.elapsed_time(e1))
        res[name] = round(statistics.median(ts), 3)
    del x, dy, dw, db, ws
    torch.cuda.empty_cache()
    return res


def stage_arms(image, steps, warmup):
    import amp_stage
    import torch.utils.deterministic as tud
    out = {}
    for arm in ("bf16_amp", "fp32_strided"):
        for mode in ("off", "on", "on_no_fill"):
            torch.use_deterministic_algorithms(mode != "off")
            tud.fill_uninitialized_memory = mode != "on_no_fill"
            try:
                out["%s/%s" % (arm, mode)] = amp_stage.measure(arm, image, steps, warmup)["ms"]
            except torch.cuda.OutOfMemoryError:
                torch.cuda.empty_cache()
                out["%s/%s" % (arm, mode)] = "not measured"
            print("stage %-13s %-10s %s" % (arm, mode, out["%s/%s" % (arm, mode)]), flush=True)
    torch.use_deterministic_algorithms(False)
    tud.fill_uninitialized_memory = True
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", default="4,1", help="GPU counts whose square tiles to time (4: a quarter, 1: the image)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--image", type=int, default=4096, help="tile edge of the six-cell step")
    ap.add_argument("--stage-steps", type=int, default=3)
    ap.add_argument("--no-stage", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("deterministic_wgrad.py: no CUDA device")
    name, power = gpu_info()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power), flush=True)
    rows = []
    for tiles in (int(t) for t in args.tiles.split(",")):
        div = int(round(tiles ** 0.5))
        for fn in LISTS:
            seen = set()
            for l in json.load(open(os.path.join(ROOT, "tests", "golden", fn)))["layers"]:
                if l["op"] != "conv":
                    continue
                key = tuple(l[k] for k in ("C", "K", "R", "S", "stride_h", "H", "W")) + (bool(l.get("bias")),)
                if key in seen:
                    continue
                seen.add(key)
                for path, dtype, spc_dtype, algo in PATHS:
                    r = dict(list=fn, tiles=tiles, path=path, C=l["C"], K=l["K"], R=l["R"], S=l["S"], stride=l["stride_h"],
                             H=l["H"] // div, W=l["W"] // div)
                    r.update(time_layer(l, div, dtype, spc_dtype, algo, args.reps))
                    if isinstance(r["default_ms"], float) and r["default_ms"] > 0:
                        r["ratio"] = round(r["deterministic_ms"] / r["default_ms"], 2)
                    print(json.dumps(r), flush=True)
                    rows.append(r)
    stage = {} if args.no_stage else stage_arms(args.image, args.stage_steps, 2)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit_max_sm_clock": power, "layers": rows, "stage_ms": stage}, f, indent=1)


if __name__ == "__main__":
    main()
