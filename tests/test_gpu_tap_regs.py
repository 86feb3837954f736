"""-m gpu: conv_tap_kernel and wgrad_tap_kernel at the shapes their register split and tap passes depend on, against the
fp64 reference and the per-element bounds of test_gpu_tc_coverage.py.

conv_tap (fprop and dgrad, C = K = M so that both ops have M output channels): M from 8 to 128, across the 64-row
boundary of the two consumer warpgroups, at 1x7, 7x1 and 3x3; W = 128 and 192; odd H (the last tile has one row);
resident weights (few channels) and streamed ones (128 channels at 1x7 and 3x3).

wgrad_tap (1x7): every QC, which gives 1, 2 and 3-4 passes of up to 256 / QC taps; row splits > 1; accumulate = 1;
and every call is exactly one kernel launch (the library's launch counter), whatever the number of passes.
conv_tap results are also checked to be bit-identical between two calls.
"""
import pytest
import torch

from mpi4dl_b200 import _lib
from tests.test_gpu_tc_coverage import (DEV, Case, _names, _to_dev, check_act, check_grad, desc, make_inputs, reference,
                                        run_dgrad, run_fwd, run_wgrad, traced)

pytestmark = pytest.mark.gpu

NO_HALO = [0] * 9


def conv_cases():
    out = []
    for m in (8, 52, 64, 65, 104, 128):
        for (r, s) in ((1, 7), (7, 1), (3, 3)):
            for w in (128, 192):
                out.append(Case(m, m, r, s, 1, 1, 9, w, m == 65, frozenset(), ""))
    return out


# (C, K): QC = round_up(min(C, K), 16) = 16 .. 128, mode A (K >= C) and mode B; H = 40 gives row splits > 1
WGRAD_CASES = [Case(c, k, 1, 7, 1, n, 40, w, False, frozenset(), "") for (c, k, n, w) in (
    (13, 40, 1, 128), (40, 29, 2, 64), (45, 64, 1, 128), (64, 52, 1, 192), (77, 93, 1, 64), (96, 128, 1, 128),
    (104, 104, 2, 128), (128, 128, 1, 64))]


def cid(c):
    return "%dto%d-%dx%d-n%d-%dx%d" % (c.C, c.K, c.R, c.S, c.N, c.H, c.W)


def traced_until(fn, name):
    """fn() under the CUDA profiler; returns (result of the first call, kernel base names seen).  The profiler can lose
    single records (see test_gpu_tc_coverage.traced), so while `name` is missing fn runs and is traced again (up to
    twice more) and the names are added; a kernel that was never launched stays missing."""
    out, kernels = traced(fn)
    names = _names(kernels)
    for _ in range(2):
        if name in names:
            break
        names |= _names(traced(fn)[1])
    return out, names


def library_launches(fn):
    """the exact number of kernels libspconv launched during fn() (its own counter, not the profiler)"""
    L = _lib.lib()
    L.spc_launch_count(1)
    fn()
    torch.cuda.synchronize()
    return int(L.spc_launch_count(0))


@pytest.mark.parametrize("c", conv_cases(), ids=cid)
def test_conv_tap(c):
    x, w, b, dy, strips = make_inputs(c, NO_HALO)
    x, w, b, dy = _to_dev(x, w, b, dy)
    strips = _to_dev(*strips)
    ref, A = reference(x, w, b, dy, strips, 1)
    d = desc(c)
    y, kf = traced_until(lambda: run_fwd(d, x, strips, w, b), "conv_tap_kernel")
    check_act(y, ref["y"], A["y"], cid(c) + " y")
    dx, kd = traced_until(lambda: run_dgrad(d, dy, w), "conv_tap_kernel")
    check_act(dx, ref["dx"], A["dx"], cid(c) + " dx")
    assert "conv_tap_kernel" in kf and "conv_tap_kernel" in kd, (sorted(kf), sorted(kd))
    # every output element has one owner and a fixed summation order: a repeated call is bit-identical
    assert torch.equal(run_fwd(d, x, strips, w, b), y), cid(c) + ": y differs between two calls"
    assert torch.equal(run_dgrad(d, dy, w), dx), cid(c) + ": dx differs between two calls"


@pytest.mark.parametrize("c", WGRAD_CASES, ids=cid)
def test_wgrad_tap_one_launch(c):
    x, w, b, dy, strips = make_inputs(c, NO_HALO)
    x, w, dy = _to_dev(x, w, dy)
    strips = _to_dev(*strips)
    ref, A = reference(x, w, None, dy, strips, 1)
    d = desc(c)
    dw = torch.full(w.shape, float("nan"), dtype=torch.float32, device=DEV)
    _, names = traced_until(lambda: run_wgrad(d, x, strips, dy, dw, None, 0), "wgrad_tap_kernel")
    check_grad(dw, ref["dw"], A["dw"], cid(c) + " dw")
    assert "wgrad_tap_kernel" in names, sorted(names)
    # all tap passes in one launch (dw is zeroed by a memset, which the library does not count)
    dw = torch.empty_like(dw)
    assert library_launches(lambda: run_wgrad(d, x, strips, dy, dw, None, 0)) == 1
    # accumulate = 1 adds onto what dw holds
    g = torch.Generator(device=DEV).manual_seed(11)
    dw0 = torch.randn(w.shape, generator=g, device=DEV) * float(ref["dw"].abs().mean())
    dw = dw0.clone()
    assert library_launches(lambda: run_wgrad(d, x, strips, dy, dw, None, 1)) == 1
    check_grad(dw, dw0.double() + ref["dw"], A["dw"], cid(c) + " dw accumulate")
