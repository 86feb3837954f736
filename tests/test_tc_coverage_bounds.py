"""CPU: the case table of test_gpu_tc_coverage.py names every kernel instance libspconv.so contains, and its per-element
bounds are tight enough to catch the errors a wrong tap index, a dropped k-chunk tail or a lost pixel row would make."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from tests import test_gpu_tc_coverage as cov

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mpi4dl_b200", "csrc")
LIB = os.path.join(ROOT, "mpi4dl_b200", "libspconv.so")
# the halo fix-up kernels of halo.cu (the rest of halo.cu is the exchange transport)
HALO_FIXUP = re.compile(r"^(halo_im2col|boundary_\w+)_kernel$")


def _kernel_names(fname):
    src = open(os.path.join(CSRC, fname)).read()
    return set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", src))


def test_instance_table_matches_library():
    if shutil.which("nm") is None:
        pytest.skip("nm (binutils) is not installed")
    assert os.path.exists(LIB), "build libspconv.so first"
    names = set()
    for f in ("gemm_tc.cu", "conv_tap.cu", "wgrad_tap.cu"):
        names |= _kernel_names(f)
    names |= {n for n in _kernel_names("halo.cu") if HALO_FIXUP.match(n)}
    assert {"conv_tap_kernel", "wgrad_tap_kernel", "pw_gemm_kernel", "pw_wgrad_kernel", "halo_im2col_kernel"} <= names
    out = subprocess.run(["nm", "-C", "--defined-only", LIB], capture_output=True, text=True, check=True).stdout
    built = set()
    for line in out.splitlines():
        parts = line.split(None, 2)
        if len(parts) == 3 and "spc::" in parts[2]:
            k = cov.parse_kernel(parts[2])
            if k[0] in names:
                built.add(k)
    covered = cov.table_instances()
    assert not built - covered, "instances without a case in test_gpu_tc_coverage.CASES: %s" % sorted(built - covered)
    assert not covered - built, "table names instances the library does not contain: %s" % sorted(covered - built)


# shapes of the table: 7x1, 1x3 / 1x7 over 64-channel k-chunks, 3x3 with 200 outputs, 5x5, 1x1, 3x3 stride 2
SENS_CASES = [cov._find(13, 29, 7, 1), cov._find(45, 61, 1, 3), cov._find(128, 128, 1, 7), cov._find(13, 200, 3, 3),
              cov._find(29, 45, 5, 5), cov._find(104, 100, 1, 1), cov._find(29, 45, 3, 3, 2),
              cov._find(45, 61, 1, 7, 2)]


def _tap_only(w, r, s):
    m = torch.zeros_like(w)
    m[:, :, r, s] = w[:, :, r, s]
    return m


@pytest.mark.parametrize("c", SENS_CASES, ids=cov.case_id)
def test_bound_detects_planted_errors(c):
    torch.manual_seed(0)
    mask = [1, 1, 1, 1, 0, 1, 1, 1, 1] if c.stride == 1 else [0] * 9
    x, w, b, dy, strips = cov.make_inputs(c, cov.so.neighbour_mask("square", 9, 4, c.R, c.S) if any(mask) else mask)
    ref, A = cov.reference(x, w, b, dy, strips, c.stride)
    st = (c.stride, c.stride)
    ph, pw = (c.R - 1) // 2, (c.S - 1) // 2
    xp = cov.padded(x, strips, ph, pw)
    wd, gd = w.double(), dy.double()
    # the exact results, rounded the way the product stores them, pass
    cov.check_act(ref["y"].to(torch.bfloat16), ref["y"], A["y"], "y bf16")
    cov.check_act(ref["dx"].to(torch.bfloat16), ref["dx"], A["dx"], "dx bf16")
    cov.check_grad(ref["dw"].float(), ref["dw"], A["dw"], "dw fp32")
    cov.check_grad(ref["db"].float(), ref["db"], A["db"], "db fp32")
    # y without the (c, r, s) term of the last channel of the last k-chunk (the middle tap)
    r, s = c.R // 2, c.S // 2
    cl = c.C - 1
    term = torch.nn.functional.conv2d(xp[:, cl:cl + 1], _tap_only(wd, r, s)[:, cl:cl + 1], None, st)
    with pytest.raises(AssertionError):
        cov.check_act((ref["y"] - term).to(torch.bfloat16), ref["y"], A["y"], "y missing (c, r, s)")
    # dx without one tap (the last one: a k-step or tap-index error at the end of the loop)
    H, W = c.H, c.W
    t = torch.nn.grad.conv2d_input(xp.shape, _tap_only(wd, c.R - 1, c.S - 1), gd, st)[:, :, ph:ph + H, pw:pw + W]
    with pytest.raises(AssertionError):
        cov.check_act((ref["dx"] - t).to(torch.bfloat16), ref["dx"], A["dx"], "dx missing a tap")
    # dw without one 64-pixel row segment of the last image (a dropped wgrad chunk or row split)
    g1 = torch.zeros_like(gd)
    Ho, Wo = gd.shape[2:]
    g1[-1, :, Ho - 1, max(0, Wo - 64):] = gd[-1, :, Ho - 1, max(0, Wo - 64):]
    t = torch.nn.grad.conv2d_weight(xp, wd.shape, g1, st)
    with pytest.raises(AssertionError):
        cov.check_grad((ref["dw"] - t).float(), ref["dw"], A["dw"], "dw missing a pixel row")
