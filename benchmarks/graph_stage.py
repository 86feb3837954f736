"""Eager against CUDA-graphed spatial stage (torchgems.graphs.graph_stage): the first six AmoebaNet-D cells of
benchmarks/amp_stage.py on one tile, forward + backward + an SGD step, eager and graphed, each plain and with recompute,
in two arms:

    bf16_amp      fp32 model under torch.autocast("cuda", dtype=torch.bfloat16)
    fp32_strided  fp32 model with SPCONV_ALLOW_TF32=strided

plus one ResNet-v2 spatial stage (the first four children of resnet_spatial.get_resnet_v2, depth 20) at the 1024^2
tile, bf16 autocast.  Method as in amp_stage.py / recompute_stage.py: every run builds its model afresh from one seed,
warms up (the graphed run captures after its warm-up) and times --steps steps; the runs alternate inside a round and
the best round is reported.  Per run:

    wall ms     host clock around the timed steps, ending in a device synchronise, per step
    GPU ms      CUDA events around the device work of one step, enqueued behind a sleep kernel that outlasts the
                enqueue, so the device runs the step back to back.  An eager step of more launches than the launch
                queue holds blocks the host before the sleep ends, and its GPU ms then still contains host gaps: on
                small tiles it is an upper bound, and the graphed run's GPU ms is the device time of the same work
    host ms     host clock around the enqueue of one step, without synchronising
    peak GB     torch.cuda.max_memory_allocated during the timed steps.  It does not count the graphed run's private
                graph pools (allocated at capture, before the timed steps), so it compares eager runs only
    launches    libspconv launches per step, counted on an eager step (a replayed graph launches nothing from the
                host, so the graphed run reports the eager count of the same stage)

The GPU name and power limit are read in the same run.

    python benchmarks/graph_stage.py [--image 512 1024 2048 4096] [--steps 5] [--warmup 2] [--rounds 2] [--json out]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from mpi4dl_b200 import _lib  # noqa: E402
from tf32_pointwise import gpu_info  # noqa: E402

CLOCK_HZ = 2.0e9          # >= the H100's SM clock: the sleep lasts at least twice the slowest enqueue
RUNS = [(arm, rc, gr) for arm in ("bf16_amp", "fp32_strided") for rc in (False, True) for gr in (False, True)]


def _name(model, arm, rc, gr):
    return "%s %s %s %s" % (model, arm, "recompute" if rc else "plain", "graphed" if gr else "eager")


def build(model, arm, image):
    if arm == "fp32_strided":
        os.environ["SPCONV_ALLOW_TF32"] = "strided"       # read by each conv layer's constructor
    else:
        os.environ.pop("SPCONV_ALLOW_TF32", None)
    torch.manual_seed(0)
    if model == "amoebanet":
        from mpi4dl_b200.models import amoebanet
        m = amoebanet.amoebanetd_spatial(0, 1, 1, mp_size=2, slice_method="square", num_classes=10, num_layers=18,
                                         num_filters=416)
        m = nn.Sequential(*list(m.children())[:6])
    else:
        from mpi4dl_b200.models import resnet_spatial
        m = resnet_spatial.get_resnet_v2((1, 3, image, image), 20, 0, 2, spatial_size=1, num_spatial_parts=1,
                                         slice_method="square")
        m = nn.Sequential(*list(m.children())[:4])
    return m.cuda().train()


def measure(model, arm, image, steps, warmup, recompute=False, graphed=False):
    from mpi4dl_b200.torchgems import graphs
    from mpi4dl_b200.torchgems.recompute import checkpoint_spatial_cells
    m = build(model, arm, image)
    if recompute:
        checkpoint_spatial_cells(m)
    amp = arm == "bf16_amp"
    opt = torch.optim.SGD(m.parameters(), lr=1e-3, momentum=0.9)
    x = torch.randn(1, 3, image, image, device="cuda")

    def out(y):
        return y[0] if isinstance(y, tuple) else y

    def eager_fwd():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            return out(m(x))

    L = _lib.lib()
    # launches of one eager step (warms the eager path up too)
    for _ in range(2):
        L.spc_launch_count(1)
        y = eager_fwd()
        y.backward(torch.ones_like(y))
        opt.zero_grad(set_to_none=False)
        torch.cuda.synchronize()
        launches = int(L.spc_launch_count(0))
    del y
    fwd = eager_fwd
    if graphed:
        g = graphs.graph_stage(m, [x], amp_dtype=torch.bfloat16 if amp else None)

        def fwd():
            return out(g(x))

    def step():
        y = fwd()
        y.backward(torch.ones_like(y))
        opt.step()
        opt.zero_grad(set_to_none=False)

    for _ in range(max(1, warmup)):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    host = []
    t0 = time.perf_counter()
    for _ in range(steps):
        h0 = time.perf_counter()
        step()
        host.append(time.perf_counter() - h0)
        torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / steps
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    gpu = []
    for _ in range(steps):
        torch.cuda._sleep(int(max(host) * 2 * CLOCK_HZ) + 1000)    # holds the stream while the host enqueues
        e0.record()
        step()
        e1.record()
        torch.cuda.synchronize()
        gpu.append(e0.elapsed_time(e1))
    res = dict(wall_ms=wall * 1e3, gpu_ms=min(gpu), host_ms=min(host) * 1e3,
               peak_GB=torch.cuda.max_memory_allocated() / 1e9, launches=launches)
    del m, opt, x
    if graphed:
        del g
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--image", type=int, nargs="+", default=[512, 1024, 2048, 4096], help="tile edges")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("graph_stage.py: no CUDA device")
    name, power = gpu_info()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power))
    print("# fwd + bwd + SGD step; %d warm-up + %d timed steps per run, runs alternated, best of %d rounds; each timed "
          "step synchronises, so wall time = host enqueue + the GPU work it does not overlap" % (args.warmup, args.steps,
                                                                                               args.rounds))
    plan = [(image, [("amoebanet",) + r for r in RUNS]) for image in args.image]
    if 1024 in args.image:
        plan.append((1024, [("resnet", "bf16_amp", False, gr) for gr in (False, True)]))
    results = {}
    for image, runs in plan:
        best = {}
        for r in range(args.rounds):
            for run in runs:
                try:
                    res = measure(run[0], run[1], image, args.steps, args.warmup, recompute=run[2], graphed=run[3])
                except torch.cuda.OutOfMemoryError:
                    torch.cuda.empty_cache()
                    res = dict(oom=True)
                key = _name(*run)
                print("%d^2 round %d %-40s %s" % (image, r, key, json.dumps(res)), flush=True)
                if key not in best or res.get("wall_ms", float("inf")) < best[key].get("wall_ms", float("inf")):
                    best[key] = res
        print("\n%d^2 tile\n%-40s %9s %9s %9s %8s %9s" % (image, "run", "wall ms", "GPU ms", "host ms", "peak GB",
                                                       "launches"))
        for run in runs:
            b = best[_name(*run)]
            if b.get("oom"):
                print("%-40s does not fit the GPU" % _name(*run))
            else:
                print("%-40s %9.1f %9.1f %9.1f %8.1f %9d" % (_name(*run), b["wall_ms"], b["gpu_ms"], b["host_ms"],
                                                            b["peak_GB"], b["launches"]))
        print(flush=True)
        results.setdefault(str(image), {}).update(best)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit_max_sm_clock": power, "best": results}, f, indent=1)


if __name__ == "__main__":
    main()
