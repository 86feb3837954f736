"""fp32 1x1 convolutions on the TF32 tensor cores (SPC_ALGO_TF32, gemm_tf32.cu).

CPU: dispatch (which shapes take the tf32 path), the sensitivity of the tight bound, and that CASES names every kernel
instance of gemm_tf32.cu in libspconv.so.
GPU (-m gpu): every case of CASES through the C ABI against an fp64 reference per element, under both bounds of
include/spconv.h, with A = the same operation on |x|, |w|, |dy| (|b|) in fp64:
    inputs rounded to tf32 beforehand (products exact):  |got - ref| <= 2^-12 A
    arbitrary fp32 inputs (two operands rounded or truncated to tf32):  |got - ref| <= (2^-9 + 2^-12) A
then every distinct 1x1 shape of the two BASELINE layer lists at the N=4 tile against cuDNN fp32 (TF32 off), and an
AmoebaNet-D cell with SPCONV_ALLOW_TF32=1 against the same cell on the direct kernels.
Run with -s to see the worst err / bound of every case.
"""
import collections
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import zlib

import pytest
import torch
import torch.nn.functional as F

from mpi4dl_b200 import _lib
from tests import test_gpu_tc_coverage as cov

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mpi4dl_b200", "csrc")
LIB = os.path.join(ROOT, "mpi4dl_b200", "libspconv.so")
DEV = "cuda:0"
TIGHT, LOOSE = 2.0 ** -12, 2.0 ** -9 + 2.0 ** -12
K = cov.K

# ---- the case table --------------------------------------------------------------------------------------------------
# fprop reduces over C into K outputs, dgrad over K into C: tf32_pw_gemm_kernel<NT> with NT = 64 (<= 64 outputs),
# 128 (<= 128) or 256 (groups of 256 outputs).  wgrad: tf32_pw_wgrad_kernel<NBLK, MG>, NBLK = C split evenly over
# blocks of <= 128 channels rounded up to 32 / 64 / 128, MG = 128-row blocks of dY per item (<= 256 / NBLK, <= 4).
# Weights stay resident in smem for one group of outputs when kchunks x NT x 128 B <= 128 KB, else they stream.
Case = collections.namedtuple("Case", "C K N H W stride bias launches note")
CASES = [
    Case(8, 8, 2, 24, 64, 1, True, K("tf32_pw_gemm_kernel<64>", "tf32_pw_wgrad_kernel<32, 1>",
                                     "tf32_repack_weights_kernel"),
         "M = 8 of 64; one partial k-chunk; wgrad 96 pixel chunks over several splits"),
    Case(8, 200, 1, 8, 16, 1, False, K("tf32_pw_gemm_kernel<256>", "tf32_pw_gemm_kernel<64>",
                                       "tf32_pw_wgrad_kernel<32, 2>"),
         "fprop 200 of 256 outputs; dgrad 7 k-chunks, the last 8 of 32 channels"),
    Case(8, 416, 2, 8, 24, 1, True, K("tf32_pw_gemm_kernel<256>", "tf32_pw_gemm_kernel<64>",
                                      "tf32_pw_wgrad_kernel<32, 4>"),
         "fprop 2 output groups (streamed weights), the second 160 of 256; wgrad 4 blocks of 104 rows"),
    Case(52, 104, 2, 10, 20, 1, False, K("tf32_pw_gemm_kernel<128>", "tf32_pw_gemm_kernel<64>",
                                         "tf32_pw_wgrad_kernel<64, 1>"),
         "P = 200 (second 128-pixel tile partial); resident weights, 2 k-chunks, the last 20 of 32"),
    Case(52, 200, 1, 12, 32, 2, True, K("tf32_subsample2_kernel", "tf32_upsample2_zero_kernel",
                                        "tf32_pw_gemm_kernel<256>", "tf32_pw_gemm_kernel<64>",
                                        "tf32_pw_wgrad_kernel<64, 2>"),
         "stride 2, P = 96"),
    Case(52, 1664, 1, 8, 16, 1, False, K("tf32_pw_gemm_kernel<256>", "tf32_pw_gemm_kernel<64>",
                                         "tf32_pw_wgrad_kernel<64, 4>"),
         "fprop 7 output groups, the last 128 of 256; dgrad 52 k-chunks of streamed weights; wgrad 13 blocks"),
    Case(104, 52, 2, 8, 16, 1, True, K("tf32_pw_gemm_kernel<64>", "tf32_pw_gemm_kernel<128>",
                                       "tf32_pw_wgrad_kernel<128, 1>"), ""),
    Case(200, 416, 1, 8, 16, 1, False, K("tf32_pw_gemm_kernel<256>", "tf32_pw_wgrad_kernel<128, 2>"),
         "dgrad 200 of 256 outputs over 13 k-chunks; wgrad 2 channel blocks of 100"),
    Case(1664, 416, 1, 4, 32, 1, False, K("tf32_pw_gemm_kernel<256>", "tf32_pw_wgrad_kernel<128, 2>"),
         "fprop 52 k-chunks; dgrad 7 output groups; wgrad 13 channel blocks"),
    Case(416, 104, 2, 16, 64, 2, True, K("tf32_subsample2_kernel", "tf32_upsample2_zero_kernel",
                                         "tf32_pw_gemm_kernel<128>", "tf32_pw_gemm_kernel<256>",
                                         "tf32_pw_wgrad_kernel<128, 1>"),
         "stride 2; fprop 13 k-chunks of streamed weights (208 KB); dgrad 2 output groups"),
]
TF32_KERNELS = ("tf32_pw_gemm_kernel", "tf32_pw_wgrad_kernel")


def case_id(c):
    return "%dto%d-s%d-n%d-%dx%d%s" % (c.C, c.K, c.stride, c.N, c.H, c.W, "-b" if c.bias else "")


def desc(c, N=None, dtype=_lib.SPC_F32, algo=_lib.SPC_ALGO_TF32, R=1, S=1):
    return _lib.ConvDesc(c.N if N is None else N, c.C, c.H, c.W, c.K, R, S, c.stride, c.stride, (R - 1) // 2,
                         (S - 1) // 2, dtype, algo)


def uses(d, op):
    return _lib.lib().spc_conv_uses_tcgen05(C.byref(d), op)


def round_tf32(t):
    """round fp32 to the nearest tf32 (10 fraction bits), ties away from zero, as cvt.rna.tf32.f32"""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def make_inputs(c, tf32, N=None):
    g = torch.Generator().manual_seed(zlib.crc32(repr((tuple(c[:7]), tf32)).encode()))
    N = c.N if N is None else N
    Ho, Wo = c.H // c.stride, c.W // c.stride
    x = torch.randn((N, c.C, c.H, c.W), generator=g)
    w = torch.randn((c.K, c.C, 1, 1), generator=g) / c.C ** 0.5
    b = torch.randn((c.K,), generator=g) if c.bias else None
    dy = torch.randn((N, c.K, Ho, Wo), generator=g)
    if tf32:
        x, w, dy = round_tf32(x), round_tf32(w), round_tf32(dy)
    return x, w, b, dy


# ---- CPU ---------------------------------------------------------------------------------------------------------
def test_dispatch():
    for c in CASES:
        for op in range(3):
            assert uses(desc(c), op) == 1, (case_id(c), op)
            assert _lib.lib().spc_conv_workspace_bytes(C.byref(desc(c)), op) > 0, (case_id(c), op)
            for algo in (_lib.SPC_ALGO_AUTO, _lib.SPC_ALGO_DIRECT, _lib.SPC_ALGO_TCGEN05):
                assert uses(desc(c, algo=algo), op) == 0, (case_id(c), op, algo)
                assert _lib.lib().spc_conv_workspace_bytes(C.byref(desc(c, algo=algo)), op) == 0
    c = CASES[3]
    for R, S in ((3, 3), (1, 7), (7, 1)):
        for op in range(3):
            assert uses(desc(c, R=R, S=S), op) == 0, (R, S, op)
    for H, W, s in ((5, 5, 1), (3, 12, 1), (8, 16, 2), (9, 64, 2)):   # P % 8, W % 32, odd H
        assert uses(desc(c._replace(H=H, W=W, stride=s)), 0) == 0, (H, W, s)
    # bf16: SPC_ALGO_TF32 is SPC_ALGO_AUTO
    shapes = [(c.C, c.K, c.H, c.W, 1, 1, c.stride) for c in CASES]
    shapes += [(c.C, c.K, c.H, c.W, c.R, c.S, c.stride) for c in cov.CASES]
    for C_, K_, H, W, R, S, st in shapes:
        for op in range(3):
            a, t = (_lib.ConvDesc(2, C_, H, W, K_, R, S, st, st, (R - 1) // 2, (S - 1) // 2, _lib.SPC_BF16, algo)
                    for algo in (_lib.SPC_ALGO_AUTO, _lib.SPC_ALGO_TF32))
            assert uses(a, op) == uses(t, op), (C_, K_, H, W, R, S, st, op)
            assert (_lib.lib().spc_conv_workspace_bytes(C.byref(a), op)
                    == _lib.lib().spc_conv_workspace_bytes(C.byref(t), op))


def test_tight_bound_detects_planted_errors():
    """At C = 2048 the tight bound rejects y without one input channel, y without one k8 step (8 channels), dx without
    one output channel's term and dw without one 32-pixel segment of the reduction"""
    c = Case(2048, 16, 1, 4, 16, 1, False, frozenset(), "")
    x, w, b, dy = make_inputs(c, True)
    ref, A = cov.reference(x, w, b, dy, [None] * 9, 1)
    xd, wd, gd = x.double(), w.double(), dy.double()
    cov.check(ref["y"].float(), ref["y"], A["y"], 0.0, TIGHT, "y fp32")
    cov.check(ref["dx"].float(), ref["dx"], A["dx"], 0.0, TIGHT, "dx fp32")
    cov.check(ref["dw"].float(), ref["dw"], A["dw"], 0.0, TIGHT, "dw fp32")
    for lo, hi, what in ((c.C - 1, c.C, "a channel"), (c.C - 8, c.C, "a k8 step")):
        term = F.conv2d(xd[:, lo:hi], wd[:, lo:hi])
        with pytest.raises(AssertionError):
            cov.check((ref["y"] - term).float(), ref["y"], A["y"], 0.0, TIGHT, "y missing " + what)
    term = torch.nn.grad.conv2d_input(xd.shape, wd[-1:], gd[:, -1:])
    with pytest.raises(AssertionError):
        cov.check((ref["dx"] - term).float(), ref["dx"], A["dx"], 0.0, TIGHT, "dx missing an output channel")
    g1 = torch.zeros_like(gd)
    g1[:, :, -2:, :] = gd[:, :, -2:, :]   # the last 32 pixels (two rows of 16)
    term = torch.nn.grad.conv2d_weight(xd, wd.shape, g1)
    with pytest.raises(AssertionError):
        cov.check((ref["dw"] - term).float(), ref["dw"], A["dw"], 0.0, TIGHT, "dw missing 32 pixels")


def test_instance_table_matches_library():
    if shutil.which("nm") is None:
        pytest.skip("nm (binutils) is not installed")
    assert os.path.exists(LIB), "build libspconv.so first"
    src = open(os.path.join(CSRC, "gemm_tf32.cu")).read()
    names = set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", src))
    assert set(TF32_KERNELS) <= names
    out = subprocess.run(["nm", "-C", "--defined-only", LIB], capture_output=True, text=True, check=True).stdout
    built = set()
    for line in out.splitlines():
        parts = line.split(None, 2)
        if len(parts) == 3 and "spc::" in parts[2]:
            k = cov.parse_kernel(parts[2])
            if k[0] in names:
                built.add(k)
    covered = set().union(*(c.launches for c in CASES))
    assert not built - covered, "instances without a case in CASES: %s" % sorted(built - covered)
    assert not covered - built, "CASES names instances the library does not contain: %s" % sorted(covered - built)


# ---- GPU: the case table -------------------------------------------------------------------------------------------
def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ws(d, op):
    n = _lib.lib().spc_conv_workspace_bytes(C.byref(d), op)
    return torch.empty(max(n, 16), dtype=torch.uint8, device=DEV), n


def run_fwd(d, x, w, b):
    y = torch.empty((d.N, d.K, d.H // d.stride_h, d.W // d.stride_w), dtype=torch.float32, device=DEV)
    ws, n = _ws(d, 0)
    halo = _lib.make_halo([None] * 9)
    _lib.check(_lib.lib().spc_conv2d_fwd(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), _ptr(ws), n,
                                         _st()), "fwd")
    return y


def run_dgrad(d, dy, w):
    dx = torch.empty((d.N, d.C, d.H, d.W), dtype=torch.float32, device=DEV)
    ws, n = _ws(d, 1)
    _lib.check(_lib.lib().spc_conv2d_dgrad(C.byref(d), _ptr(dy), _ptr(w), _ptr(dx), _ptr(ws), n, _st()), "dgrad")
    return dx


def run_wgrad(d, x, dy, dw, db, accumulate):
    ws, n = _ws(d, 2)
    halo = _lib.make_halo([None] * 9)
    _lib.check(_lib.lib().spc_conv2d_wgrad(C.byref(d), _ptr(x), C.byref(halo), _ptr(dy), C.c_void_p(dw.data_ptr()),
                                           _ptr(db), accumulate, _ptr(ws), n, _st()), "wgrad")
    return dw, db


def _names(kernels):
    return {n for n, _ in kernels}


@pytest.mark.gpu
@pytest.mark.parametrize("tf32_inputs", [True, False], ids=["tight", "loose"])
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_case_against_fp64(c, tf32_inputs):
    bound = TIGHT if tf32_inputs else LOOSE
    tag = "%s %s" % (case_id(c), "tight" if tf32_inputs else "loose")
    x, w, b, dy = [t.to(DEV) if t is not None else None for t in make_inputs(c, tf32_inputs)]
    ref, A = cov.reference(x, w, b, dy, [None] * 9, c.stride)
    d = desc(c)
    y, kf = cov.traced(lambda: run_fwd(d, x, w, b))
    print("[tf32] %-32s y  err/bound %.3f" % (tag, cov.check(y, ref["y"], A["y"], 0.0, bound, tag + " y")))
    dx, kd = cov.traced(lambda: run_dgrad(d, dy, w))
    print("[tf32] %-32s dx err/bound %.3f" % (tag, cov.check(dx, ref["dx"], A["dx"], 0.0, bound, tag + " dx")))
    dw = torch.full(w.shape, float("nan"), device=DEV)
    db = torch.full((c.K,), float("nan"), device=DEV) if c.bias else None
    _, kw = cov.traced(lambda: run_wgrad(d, x, dy, dw, db, 0))
    print("[tf32] %-32s dw err/bound %.3f" % (tag, cov.check(dw, ref["dw"], A["dw"], 0.0, bound, tag + " dw")))
    if c.bias:
        cov.check(db, ref["db"], A["db"], 0.0, TIGHT, tag + " db")
    # accumulate = 1 adds onto what dw / db hold
    g = torch.Generator(device=DEV).manual_seed(7)
    dw0 = torch.randn(w.shape, generator=g, device=DEV) * float(ref["dw"].abs().mean())
    db0 = torch.randn((c.K,), generator=g, device=DEV) if c.bias else None
    dw1, db1 = run_wgrad(d, x, dy, dw0.clone(), db0.clone() if c.bias else None, 1)
    cov.check(dw1, dw0.double() + ref["dw"], A["dw"] + dw0.double().abs(), 0.0, bound, tag + " dw accumulate")
    if c.bias:
        cov.check(db1, db0.double() + ref["db"], A["db"] + db0.double().abs(), 0.0, TIGHT, tag + " db accumulate")
    # fprop / dgrad have no atomics: a repeated call is bit-identical
    assert torch.equal(run_fwd(d, x, w, b), y), tag + ": fprop not reproducible"
    assert torch.equal(run_dgrad(d, dy, w), dx), tag + ": dgrad not reproducible"

    def retrace():
        return cov.traced(lambda: (run_fwd(d, x, w, b), run_dgrad(d, dy, w),
                                   run_wgrad(d, x, dy, torch.empty_like(dw), torch.empty_like(db) if c.bias else None, 0)))[1]
    k = kf | kd | kw
    assert cov.launched(k, lambda k: c.launches <= k, retrace), \
        "%s did not launch %s (launched: %s)" % (tag, sorted(c.launches - k), sorted(k))
    assert not {"conv_direct_kernel", "wgrad_direct_kernel"} & _names(k), (tag, sorted(k))
    for kk in (kf, kd, kw):
        assert _names(kk) & set(TF32_KERNELS), (tag, sorted(kk))


@pytest.mark.gpu
def test_empty_batch():
    """N == 0: nothing to compute; wgrad with accumulate = 1 leaves dw / db as they are, accumulate = 0 zeroes them"""
    c = CASES[0]
    d = desc(c, N=0)
    assert uses(d, 0) and uses(d, 2)
    x, w, b, dy = [t.to(DEV) if t is not None else None for t in make_inputs(c, True, N=0)]
    assert run_fwd(d, x, w, b).numel() == 0 and run_dgrad(d, dy, w).numel() == 0
    dw0, db0 = torch.randn(w.shape, device=DEV), torch.randn((c.K,), device=DEV)
    dw, db = run_wgrad(d, None, None, dw0.clone(), db0.clone(), 1)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw0) and torch.equal(db, db0)
    dw, db = run_wgrad(d, None, None, dw, db, 0)
    torch.cuda.synchronize()
    assert not dw.any() and not db.any()


# ---- GPU: full-size BASELINE 1x1 shapes --------------------------------------------------------------------------
def _pointwise_layers():
    out, seen = [], set()
    for fn, tag in (("layers_amoebanetd_sp4.json", "amoeba"), ("layers_resnet101_sp2.json", "resnet")):
        for l in json.load(open(os.path.join(ROOT, "tests", "golden", fn)))["layers"]:
            if l["op"] != "conv" or (l["R"], l["S"]) != (1, 1):
                continue
            key = (l["C"], l["K"], l["stride_h"], l["H"], bool(l.get("bias")))
            if key not in seen:
                seen.add(key)
                out.append((tag,) + key)
    return out


def _check_sliced(got, ref, A, bound, name):
    """per element |got - ref| <= bound * A, in slices of dim 1 so that the temporaries stay small"""
    step = max(1, (1 << 26) // max(1, ref[:, :1].numel()))
    worst = 0.0
    for i in range(0, ref.shape[1], step):
        err = (got[:, i:i + step] - ref[:, i:i + step]).abs_()
        lim = A[:, i:i + step] * bound
        worst = max(worst, float((err - lim).max()))
        bad = int((err > lim).sum())
        assert bad == 0, "%s: %d elements out of bound in channels %d.., worst excess %.3g" % (name, bad, i, worst)
        del err, lim


@pytest.mark.gpu
@pytest.mark.parametrize("layer", _pointwise_layers(), ids=lambda l: "%s-%dto%d-s%d-%d" % l[:5])
def test_fullsize_vs_cudnn_fp32(layer):
    """N=4 tile (half the stage's extent) of every distinct BASELINE 1x1 shape, arbitrary fp32 inputs, against cuDNN
    fp32 with TF32 off (its own rounding error is far below the loose bound); A from |x|, |w|, |dy| the same way"""
    _, Cc, K_, s, H, bias = layer
    H = W = H // 2
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        gen = torch.Generator(device=DEV).manual_seed(Cc * 7 + K_ * 3 + s + H)
        x = torch.randn((1, Cc, H, W), device=DEV, generator=gen)
        w = torch.randn((K_, Cc, 1, 1), device=DEV, generator=gen) / Cc ** 0.5
        b = torch.randn(K_, device=DEV, generator=gen) if bias else None
        c = Case(Cc, K_, 1, H, W, s, bias, frozenset(), "")
        d = desc(c)
        assert uses(d, 0) and uses(d, 1) and uses(d, 2), layer
        y = run_fwd(d, x, w, b)
        _check_sliced(y, F.conv2d(x, w, b, s), F.conv2d(x.abs(), w.abs(), b.abs() if bias else None, s), LOOSE, "y")
        del y
        dy = torch.randn((1, K_, H // s, W // s), device=DEV, generator=gen)
        dx = run_dgrad(d, dy, w)
        _check_sliced(dx, torch.nn.grad.conv2d_input(x.shape, w, dy, s),
                      torch.nn.grad.conv2d_input(x.shape, w.abs(), dy.abs(), s), LOOSE, "dx")
        del dx
        dw, _ = run_wgrad(d, x, dy, torch.empty(w.shape, device=DEV), None, 0)
        _check_sliced(dw, torch.nn.grad.conv2d_weight(x, w.shape, dy, s),
                      torch.nn.grad.conv2d_weight(x.abs(), w.shape, dy.abs(), s), LOOSE, "dw")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        torch.cuda.empty_cache()


# ---- GPU: the layers ---------------------------------------------------------------------------------------------
def _cell(monkeypatch, allow):
    from mpi4dl_b200.models.amoebanet import Cell
    if allow:
        monkeypatch.setenv("SPCONV_ALLOW_TF32", "1")
    else:
        monkeypatch.delenv("SPCONV_ALLOW_TF32", raising=False)
    torch.manual_seed(11)
    sp = dict(local_rank=0, spatial_size=1, num_spatial_parts=1, slice_method="square")
    return Cell(sp, 64, 64, 64, reduction=False, reduction_prev=False).to(DEV).train()


def _run_cell(cell, x):
    """forward, then backward of a fixed random projection of the output (sum(y^2) would give gradients of almost
    zero through the cell's last batch norms, which normalise every channel)"""
    for p in cell.parameters():
        p.grad = None
    xg = x.clone().requires_grad_(True)
    y, _ = cell(xg)
    r = torch.randn(y.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    (y * r).sum().backward()
    return y.detach(), xg.grad, [p.grad for p in cell.parameters()]


@pytest.mark.gpu
def test_amoebanet_cell_with_tf32(monkeypatch):
    """SPCONV_ALLOW_TF32=1: the cell's 1x1 conv_spatial / local_conv2d layers take SPC_ALGO_TF32 and launch the tf32
    kernels; the forward output stays within the loose bound of the direct run per element, scaled by the depth of the
    cell (several convolutions and batch norms in a row), and the input and weight gradients within 10 % in the 2-norm"""
    from mpi4dl_b200.torchgems.spatial import conv_spatial, local_conv2d
    ref_cell = _cell(monkeypatch, False)
    tf_cell = _cell(monkeypatch, True)
    tf_cell.load_state_dict(ref_cell.state_dict())
    convs = [m for m in tf_cell.modules() if isinstance(m, (conv_spatial, local_conv2d))]
    assert convs and all(m.algo == _lib.SPC_ALGO_TF32 for m in convs)
    assert all(m.algo == _lib.SPC_ALGO_AUTO for m in ref_cell.modules() if isinstance(m, (conv_spatial, local_conv2d)))
    x = torch.randn(2, 64, 32, 32, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    ref, kr = cov.traced(lambda: _run_cell(ref_cell, x))
    got, kt = cov.traced(lambda: _run_cell(tf_cell, x))
    assert not set(TF32_KERNELS) & _names(kr), sorted(kr)
    assert set(TF32_KERNELS) <= _names(kt), sorted(kt)
    # the forward output per element; the gradients as a whole: a ReLU kink that the two runs place on different sides
    # (inputs within the tf32 rounding of zero, a fraction f of about 1e-3) moves a gradient element by its full size,
    # which gives a 2-norm difference of about sqrt(f) = 3 %: the gradients are compared in the 2-norm, to 10 %
    tol = 16 * LOOSE
    err = float((got[0] - ref[0]).abs().max())
    print("[tf32] cell y     max err / max |ref| %.3g" % (err / float(ref[0].abs().max())))
    assert err <= tol * float(ref[0].abs().max()), "y: max err %.3g vs max |ref| %.3g" % (err, float(ref[0].abs().max()))
    for name, a, r in [("dx", got[1], ref[1])] + [("dw%d" % i, a, r) for i, (a, r) in enumerate(zip(got[2], ref[2]))]:
        rel = float((a - r).norm() / r.norm())
        print("[tf32] cell %-5s |err| / |ref| %.3g" % (name, rel))
        assert rel <= 0.1, "%s: |err| / |ref| = %.3g" % (name, rel)


@pytest.mark.gpu
def test_amoebanet_cell_default_launches_no_tf32(monkeypatch):
    cell = _cell(monkeypatch, False)
    x = torch.randn(2, 64, 32, 32, device=DEV)
    _, k = cov.traced(lambda: _run_cell(cell, x))
    assert not set(TF32_KERNELS) & _names(k), sorted(k)
    assert "conv_direct_kernel" in _names(k), sorted(k)
