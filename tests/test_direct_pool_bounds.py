"""CPU: the case tables of test_gpu_direct_pool_coverage.py name every instance of conv_direct.cu and pool.cu that
libspconv.so contains, and the per-element bounds of that module accept the exact result rounded the way the kernels
store it but reject the errors a dropped channel chunk, strip column, parity class, tile, tap pass, bias chunk or ring
element, a tie routed to the wrong maximum, or a dropped NaN would make -- at the tables' own shapes."""
import math
import os
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

from tests import test_gpu_direct_pool_coverage as dp
from tests.test_tc_coverage_bounds import LIB, _kernel_names


def test_instance_table_matches_library():
    if shutil.which("nm") is None:
        pytest.skip("nm (binutils) is not installed")
    assert os.path.exists(LIB), "build libspconv.so first"
    names = _kernel_names("conv_direct.cu") | _kernel_names("pool.cu")
    assert {"conv_direct_kernel", "wgrad_direct_kernel", "bias_grad_kernel", "pool3_s1_tma_kernel"} <= names
    out = subprocess.run(["nm", "-C", "--defined-only", LIB], capture_output=True, text=True, check=True).stdout
    built = set()
    for line in out.splitlines():
        parts = line.split(None, 2)
        if len(parts) == 3 and "spc::" in parts[2]:
            k = dp.parse_kernel(parts[2])
            if k[0] in names:
                built.add(k)
    covered = dp.direct_table_instances() | dp.pool_table_instances()
    assert not built - covered, "instances without a case in the tables: %s" % sorted(built - covered)
    assert not covered - built, "tables name instances the library does not contain: %s" % sorted(covered - built)
    assert len(built) == 28


def _case(**kw):
    return next(c for c in dp.DCASES if all(getattr(c, k) == v for k, v in kw.items()))


def _fails(fn):
    with pytest.raises(AssertionError):
        fn()


def _conv(c):
    x, w, b, dy, strips = dp.make_conv_inputs(c)
    ref, A = dp.reference(x, w, b, dy, strips, c.stride)
    return x, w, b, dy, strips, ref, A


def _stored(v, dtype):
    return v.to(dtype)


def test_y_missing_one_term_of_a_partial_channel_chunk():
    # 3x3 s2, C = 13: CB = 4, chunks 4 + 4 + 4 + 1; the last chunk holds channel 12 alone
    c = _case(C=13, K=16, R=3, S=3, stride=2, N=2)
    x, w, b, dy, strips, ref, A = _conv(c)
    rel, ab = dp.conv_bounds(c)["y"]
    dp.check(_stored(ref["y"], c.dtype), ref["y"], A["y"], rel, ab, "exact")
    w2 = w.double().clone()
    w2[:, 12, 2, 1] = 0
    xp = dp.padded(x, strips, 1, 1)
    bad = F.conv2d(xp, w2, b.double(), (2, 2))
    _fails(lambda: dp.check(_stored(bad, c.dtype), ref["y"], A["y"], rel, ab, "planted"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_vert_strip_missing_its_last_column(dtype):
    # 1x7 s1 with left / right neighbours: the boundary rectangles are 3 columns wide (VERT); the bf16 twin of the
    # 3x3 thin tile has 1-column rectangles on VERT KB=16
    c = _case(R=1, S=7, stride=1, mask="lr") if dtype == torch.float32 else _case(C=2, K=4, dtype=dtype)
    x, w, b, dy, strips, ref, A = _conv(c)
    rel, ab = dp.conv_bounds(c)["y"]
    dp.check(_stored(ref["y"], c.dtype), ref["y"], A["y"], rel, ab, "exact")
    ph, pw = (c.R - 1) // 2, (c.S - 1) // 2
    interior = F.conv2d(dp.padded(x, [None] * 9, ph, pw), w.double(), b.double() if b is not None else None)
    bad = ref["y"].clone()
    bad[..., pw - 1] = interior[..., pw - 1]            # the left rectangle's last column keeps its zero-padded value
    _fails(lambda: dp.check(_stored(bad, c.dtype), ref["y"], A["y"], rel, ab, "planted"))


@pytest.mark.parametrize("H", [17, 16])
def test_dx_missing_one_parity_class(H):
    c = _case(C=13, K=16, R=3, S=3, stride=2, H=H)
    x, w, b, dy, strips, ref, A = _conv(c)
    rel, ab = dp.conv_bounds(c)["dx"]
    dp.check(_stored(ref["dx"], c.dtype), ref["dx"], A["dx"], rel, ab, "exact")
    for a, bb in ((0, 0), (0, 1), (1, 0), (1, 1)):
        bad = ref["dx"].clone()
        bad[:, :, a::2, bb::2] = 0
        _fails(lambda: dp.check(_stored(bad, c.dtype), ref["dx"], A["dx"], rel, ab, "planted %d%d" % (a, bb)))


def test_dx_missing_a_1x1_parity_class():
    c = _case(C=6, K=20, R=1, S=1, stride=2)
    x, w, b, dy, strips, ref, A = _conv(c)
    rel, ab = dp.conv_bounds(c)["dx"]
    bad = ref["dx"].clone()
    bad[:, :, 0::2, 0::2] = 0
    _fails(lambda: dp.check(_stored(bad, c.dtype), ref["dx"], A["dx"], rel, ab, "planted"))


def _dw_without(c, x, w, dy, strips, drop):
    ph, pw = (c.R - 1) // 2, (c.S - 1) // 2
    g = dy.double().clone()
    g[drop] = 0
    return torch.nn.grad.conv2d_weight(dp.padded(x, strips, ph, pw), w.shape, g, (c.stride, c.stride))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_dw_missing_one_tile_of_the_last_image(dtype):
    c = _case(C=3, K=8, H=130, dtype=dtype)
    x, w, b, dy, strips, ref, A = _conv(c)
    rel, ab = dp.conv_bounds(c)["dw"]
    dp.check(ref["dw"].float(), ref["dw"], A["dw"], rel, ab, "exact")
    Ho, Wo = dp.conv_out_hw(c)
    for ty, tx in ((5, 3), (Ho // 4, Wo // 32)):   # a whole tile and the ragged last one
        bad = _dw_without(c, x, w, dy, strips, (c.N - 1, slice(None), slice(4 * ty, 4 * ty + 4), slice(32 * tx, 32 * tx + 32)))
        _fails(lambda: dp.check(bad.float(), ref["dw"], A["dw"], rel, ab, "planted tile %d,%d" % (ty, tx)))


def test_dw_missing_one_tap_pass():
    c = _case(C=29, K=13, R=5, S=5, stride=1)
    x, w, b, dy, strips, ref, A = _conv(c)
    rel, ab = dp.conv_bounds(c)["dw"]
    dp.check(ref["dw"].float(), ref["dw"], A["dw"], rel, ab, "exact")
    bad = ref["dw"].clone().reshape(c.K, c.C, 25)
    bad[:, :, 9:18] = 0
    _fails(lambda: dp.check(bad.reshape(ref["dw"].shape).float(), ref["dw"], A["dw"], rel, ab, "planted"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_db_missing_one_chunk(dtype):
    c = _case(C=2, K=4, dtype=dtype)      # Ho Wo = 264000: 5 chunks of 52800
    x, w, b, dy, strips, ref, A = _conv(c)
    rel, ab = dp.conv_bounds(c)["db"]
    dp.check(ref["db"].float(), ref["db"], A["db"], rel, ab, "exact")
    flat = dy.double().reshape(c.N, c.K, -1)
    for ch in (0, 4):
        bad = flat.sum((0, 2)) - flat[:, :, ch * 52800:(ch + 1) * 52800].sum((0, 2))
        _fails(lambda: dp.check(bad.float(), ref["db"], A["db"], rel, ab, "planted chunk %d" % ch))


def _pcase(mode, k, stride, H, W):
    return next(c for c in dp.PCASES if (c.mode, c.k, c.stride, c.H, c.W) == (mode, k, stride, H, W))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_avg_pool_missing_one_ring_element(dtype):
    c = _pcase("avg", 3, 1, 70, 136)
    mask = dp.pool_masks(c)[0]
    x, strips, dy = dp.make_pool_inputs(c, dtype, mask, "normal")
    y, ya, dx, dxa = dp.pool_reference(c, x, strips, dy)
    bnd = dp.pool_bounds(c, dtype)["y"]
    dp.check_pool(y.to(dtype), y, ya, bnd, "exact")
    no_halo, _, _, _ = dp.pool_reference(c, x, [None] * 9, dy)
    for (h, w) in ((0, 0), (0, 77), (35, 135), (69, 3)):
        bad = y.clone()
        bad[1, 4, h, w] = no_halo[1, 4, h, w]      # the TMA kernel's zero-padded value, not redone by the ring
        _fails(lambda: dp.check_pool(bad.to(dtype), y, ya, bnd, "planted %d,%d" % (h, w)))


def _route_to_last(c, x, strips, dy):
    """max pool dx with ties routed to the LAST maximum: ATen on the tile flipped in H and W"""
    pad = (c.k - 1) // 2
    xp = dp.padded(x, strips, pad, pad).flip(2, 3).requires_grad_(True)
    y = F.max_pool2d(xp, c.k, c.stride, 0)
    g, = torch.autograd.grad(y, xp, dy.double().flip(2, 3))
    return g.flip(2, 3)[:, :, pad:pad + c.H, pad:pad + c.W]


@pytest.mark.parametrize("shape", [("max", 2, 2, 16, 32), ("max", 3, 1, 9, 11), ("max", 3, 1, 130, 264)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_max_dx_routed_to_the_second_tie(shape, dtype):
    c = _pcase(*shape)
    x, strips, dy = dp.make_pool_inputs(c, dtype, [0] * 9, "ties")
    y, ya, dx, dxa = dp.pool_reference(c, x, strips, dy)
    bnd = dp.pool_bounds(c, dtype)["dx"]
    dp.check_pool(dx.to(dtype), dx, dxa, bnd, "exact")
    bad = _route_to_last(c, x, strips, dy)
    assert not torch.equal(bad, dx)
    _fails(lambda: dp.check_pool(bad.to(dtype), dx, dxa, bnd, "planted"))


@pytest.mark.parametrize("shape", [("max", 2, 2, 16, 32), ("max", 3, 1, 33, 512), ("max", 3, 2, 11, 32)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_max_pool_dropping_nan(shape, dtype):
    c = _pcase(*shape)
    mask = dp.pool_masks(c)[0]
    x, strips, dy = dp.make_pool_inputs(c, dtype, mask, "nan")
    y, ya, dx, dxa = dp.pool_reference(c, x, strips, dy)
    assert torch.isnan(y).any()
    dp.check_pool(y.to(dtype), y, ya, None, "exact")
    # fmaxf: the largest non-NaN value of the window
    nonan = [s.masked_fill(torch.isnan(s), -math.inf) if s is not None else None for s in strips]
    dropped, _, ddx, _ = dp.pool_reference(c, x.masked_fill(torch.isnan(x), -math.inf), nonan, dy)
    _fails(lambda: dp.check_pool(dropped.to(dtype), y, ya, None, "planted y"))
    _fails(lambda: dp.check_pool(ddx.to(dtype), dx, dxa, dp.pool_bounds(c, dtype)["dx"], "planted dx"))


def test_aten_max_pool_nan_rule():
    """the oracle's rule: NaN wins, and of two NaNs in a window the later one takes the gradient"""
    x = torch.tensor([[[[1.0, math.nan, 3.0, math.nan]]]], dtype=torch.float64, requires_grad=True)
    y = F.max_pool2d(x, (1, 4), 1, 0)
    assert torch.isnan(y).all()
    g, = torch.autograd.grad(y, x, torch.ones_like(y))
    assert g.tolist() == [[[[0.0, 0.0, 0.0, 1.0]]]]
    x = torch.tensor([[[[2.0, 1.0, 2.0, 2.0]]]], dtype=torch.float64, requires_grad=True)
    g, = torch.autograd.grad(F.max_pool2d(x, (1, 4), 1, 0), x, torch.ones(1, 1, 1, 1, dtype=torch.float64))
    assert g.tolist() == [[[[1.0, 0.0, 0.0, 0.0]]]]
