"""Time the spatial stage's first six AmoebaNet-D cells (stem1-3 + cell1_normal1-3 of amoebanetd_spatial(18, 416), the
cells of bench.py's model_stage arm) on one tile, forward + backward + an SGD step, in three arms:

    bf16          the model cast with .to(torch.bfloat16): bf16 parameters, gradients and SGD update
    bf16_amp      fp32 model under torch.autocast("cuda", dtype=torch.bfloat16): bf16 kernels, fp32 master weights,
                  weight gradients and SGD update
    fp32_strided  fp32 model with SPCONV_ALLOW_TF32=strided (every convolution on the TF32 tensor cores)

Each round builds every arm's model afresh (same seed), warms it up and times --steps steps with CUDA events; the arms
alternate inside a round and the best round is reported.  Per arm: ms per step, peak memory allocated during the timed
steps, and libspconv launches per step (spc_launch_count over one step).  The GPU name and power limit are read in the
same run.  An arm that does not fit the GPU is reported as such.

    python benchmarks/amp_stage.py [--image 4096] [--steps 3] [--warmup 2] [--rounds 2] [--json out.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from mpi4dl_b200 import _lib  # noqa: E402
from tf32_pointwise import gpu_info  # noqa: E402

ARMS = ("bf16", "bf16_amp", "fp32_strided")


def build(arm):
    from mpi4dl_b200.models import amoebanet
    if arm == "fp32_strided":
        os.environ["SPCONV_ALLOW_TF32"] = "strided"       # read by each conv layer's constructor
    else:
        os.environ.pop("SPCONV_ALLOW_TF32", None)
    torch.manual_seed(0)
    m = amoebanet.amoebanetd_spatial(0, 1, 1, mp_size=2, slice_method="square", num_classes=10, num_layers=18,
                                     num_filters=416)
    m = nn.Sequential(*list(m.children())[:6]).cuda().train()
    return m.to(torch.bfloat16) if arm == "bf16" else m


def measure(arm, image, steps, warmup, recompute=False):
    m = build(arm)
    if recompute:
        from mpi4dl_b200.torchgems.recompute import checkpoint_spatial_cells
        checkpoint_spatial_cells(m)
    opt = torch.optim.SGD(m.parameters(), lr=1e-3, momentum=0.9)
    x = torch.randn(1, 3, image, image, device="cuda", dtype=torch.bfloat16 if arm == "bf16" else torch.float32)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=arm == "bf16_amp"):
            y, _ = m(x)
        y.backward(torch.ones_like(y))
        opt.step()
        opt.zero_grad(set_to_none=False)

    L = _lib.lib()
    for _ in range(max(1, warmup)):
        step()
    torch.cuda.synchronize()
    L.spc_launch_count(1)
    step()
    torch.cuda.synchronize()
    launches = int(L.spc_launch_count(0))
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    res = dict(ms=e0.elapsed_time(e1) / steps, peak_GB=torch.cuda.max_memory_allocated() / 1e9, launches=launches,
               param_dtype=str(next(m.parameters()).dtype).replace("torch.", ""),
               grad_dtype=str(next(m.parameters()).grad.dtype).replace("torch.", ""))
    del m, opt, x
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--image", type=int, default=4096, help="tile edge (4096 = the N=4 tile of the 8192^2 stage)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("amp_stage.py: no CUDA device")
    name, power = gpu_info()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power))
    print("# first six AmoebaNet-D cells (18, 416) on a %d^2 tile, fwd + bwd + SGD step; %d warm-up + %d timed steps "
          "per arm, arms alternated, best of %d rounds" % (args.image, args.warmup, args.steps, args.rounds))
    best = {}
    for r in range(args.rounds):
        for arm in ARMS:
            try:
                res = measure(arm, args.image, args.steps, args.warmup)
            except torch.cuda.OutOfMemoryError:
                torch.cuda.empty_cache()
                res = dict(oom=True)
            print("round %d %-13s %s" % (r, arm, json.dumps(res)), flush=True)
            if arm not in best or res.get("ms", float("inf")) < best[arm].get("ms", float("inf")):
                best[arm] = res
    print("\n%-13s %10s %9s %9s %7s %6s" % ("arm", "ms/step", "peak GB", "launches", "params", "grads"))
    for arm in ARMS:
        b = best[arm]
        if b.get("oom"):
            print("%-13s does not fit the GPU" % arm)
        else:
            print("%-13s %10.1f %9.1f %9d %7s %6s" % (arm, b["ms"], b["peak_GB"], b["launches"], b["param_dtype"],
                                                     b["grad_dtype"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit_max_sm_clock": power, "image": args.image, "best": best}, f, indent=1)


if __name__ == "__main__":
    main()
