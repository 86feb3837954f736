"""Cost and saving of recomputing the spatial cells in backward (torchgems.recompute.checkpoint_spatial_cells): the
first six AmoebaNet-D cells of benchmarks/amp_stage.py on one tile, forward + backward + an SGD step, plain against
recompute, in two arms:

    bf16_amp      fp32 model under torch.autocast("cuda", dtype=torch.bfloat16)
    fp32_strided  fp32 model with SPCONV_ALLOW_TF32=strided

Method as in amp_stage.py: every (arm, mode) builds its model afresh from one seed, warms up and times --steps steps
with CUDA events; the four runs alternate inside a round and the best round is reported.  Per run: ms per step, peak
memory allocated during the timed steps, and libspconv launches per step.  A run that does not fit the GPU is reported
as such.  The GPU name and power limit are read in the same run.

    python benchmarks/recompute_stage.py [--image 2048 4096] [--steps 3] [--warmup 2] [--rounds 2] [--json out.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import torch  # noqa: E402

from amp_stage import measure  # noqa: E402
from tf32_pointwise import gpu_info  # noqa: E402

RUNS = [(arm, rc) for arm in ("bf16_amp", "fp32_strided") for rc in (False, True)]


def _name(arm, rc):
    return "%s %s" % (arm, "recompute" if rc else "plain")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--image", type=int, nargs="+", default=[2048, 4096], help="tile edges")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("recompute_stage.py: no CUDA device")
    name, power = gpu_info()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power))
    print("# first six AmoebaNet-D cells (18, 416), fwd + bwd + SGD step; %d warm-up + %d timed steps per run, runs "
          "alternated, best of %d rounds" % (args.warmup, args.steps, args.rounds))
    results = {}
    for image in args.image:
        best = {}
        for r in range(args.rounds):
            for arm, rc in RUNS:
                try:
                    res = measure(arm, image, args.steps, args.warmup, recompute=rc)
                except torch.cuda.OutOfMemoryError:
                    torch.cuda.empty_cache()
                    res = dict(oom=True)
                key = _name(arm, rc)
                print("%d^2 round %d %-23s %s" % (image, r, key, json.dumps(res)), flush=True)
                if key not in best or res.get("ms", float("inf")) < best[key].get("ms", float("inf")):
                    best[key] = res
        print("\n%d^2 tile\n%-23s %10s %9s %9s" % (image, "run", "ms/step", "peak GB", "launches"))
        for arm, rc in RUNS:
            b = best[_name(arm, rc)]
            if b.get("oom"):
                print("%-23s does not fit the GPU" % _name(arm, rc))
            else:
                print("%-23s %10.1f %9.1f %9d" % (_name(arm, rc), b["ms"], b["peak_GB"], b["launches"]))
        print()
        results[image] = best
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit_max_sm_clock": power, "best": results}, f, indent=1)


if __name__ == "__main__":
    main()
