"""fp32 stride-1 multi-tap convolutions on the TF32 tensor cores (SPC_ALGO_TF32_ALL, conv_tap_tf32.cu).

CPU: dispatch (which shapes take the tap kernels, that SPC_ALGO_TF32_ALL leaves everything else as SPC_ALGO_TF32 /
SPC_ALGO_AUTO have it), the sensitivity of the tight bound to planted errors, that CASES names every kernel instance of
conv_tap_tf32.cu in libspconv.so, and conv_algo_default().
GPU (-m gpu): every case of CASES through the C ABI against an fp64 reference per element, under both bounds of
include/spconv.h with A = the same operation on |x|, |w|, |dy| (|b|), summed over all taps:
    inputs rounded to tf32 beforehand (products exact):  |got - ref| <= 2^-12 A
    arbitrary fp32 inputs:                              |got - ref| <= (2^-9 + 2^-12) A
The tight bound holds because no fp32 chain is long: fprop / dgrad add R*S*ceil(Cin/8) k8 partial sums per output,
wgrad at most 512 row segments x 4 k8 steps per work item plus one atomic per item, and L fp32 additions add at most
about L 2^-24 A (<= 2^-12 A for L <= 4096).  Then the cases under halo-strip masks (spc_conv2d_fwd and the split
interior + boundary calls, wgrad with the strips' share), every stride-1 multi-tap shape of the two BASELINE layer lists at the N=4 tile against cuDNN fp32
(TF32 off), an AmoebaNet-D cell and a ResNet-v2 bottleneck with SPCONV_ALLOW_TF32=all against the direct run, and a
CUDA-graph capture of a tap layer.
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
from oracle import spatial_oracle as so
from tests import test_gpu_tc_coverage as cov
from tests import test_tf32_pointwise as pw

ROOT = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(ROOT), "mpi4dl_b200", "libspconv.so")
SRC = os.path.join(os.path.dirname(ROOT), "mpi4dl_b200", "csrc", "conv_tap_tf32.cu")
DEV = "cuda:0"
TIGHT, LOOSE = pw.TIGHT, pw.LOOSE
K = cov.K
ALL = _lib.SPC_ALGO_TF32_ALL
TAP_KERNEL, TAP_WGRAD = "tf32_tap_gemm_kernel", "tf32_tap_wgrad_kernel"
DIRECT = {"conv_direct_kernel", "wgrad_direct_kernel"}

# ---- the case table --------------------------------------------------------------------------------------------------
# fprop reduces over C into K outputs, dgrad over K into C: tf32_tap_gemm_kernel<NT>, NT = the smallest of 16, 32, 64,
# 128 that holds the outputs, else groups of 256; the second parameter is 1 in the small-Cin mode (Cin <= 8).  Weights stay resident in smem for one group of outputs when
# blocks x NT x 128 B <= 128 KB (blocks = R*S x ceil(Cin / 32), or ceil(R*S / 4) in the small-Cin mode of Cin <= 8),
# else they stream with the activations.  wgrad: tf32_tap_wgrad_kernel<NT>, NT from K the same way, 128-channel blocks
# of C.  W % 32 != 0 leaves the last row segment partial.
Case = collections.namedtuple("Case", "C K R S N H W bias launches note")
GEMM, SMALL, WGRAD = "tf32_tap_gemm_kernel<%d, 0>", "tf32_tap_gemm_kernel<%d, 1>", "tf32_tap_wgrad_kernel<%d>"
CASES = [
    Case(3, 16, 3, 3, 2, 12, 36, True, K(SMALL % 16, GEMM % 16, WGRAD % 16, "tf32_tap_repack_kernel"),
         "the C=3 stem: fprop in the small-Cin mode (3 stages of 4 taps, the last 1 of 4); dgrad M = 3; W = 36: a "
         "4-pixel last segment"),
    Case(16, 16, 3, 3, 2, 10, 64, True, K(GEMM % 16, WGRAD % 16), ""),
    Case(64, 16, 3, 3, 1, 9, 40, True, K(GEMM % 16, GEMM % 64, WGRAD % 16), "dgrad M = 64 of 2 k-chunks"),
    Case(52, 52, 1, 7, 2, 6, 64, False, K(GEMM % 64, WGRAD % 64),
         "resident weights (7 taps x 2 k-chunks, the last 20 of 32)"),
    Case(52, 52, 7, 1, 2, 20, 32, False, K(GEMM % 64, WGRAD % 64), ""),
    Case(104, 104, 1, 7, 1, 5, 128, False, K(GEMM % 128, WGRAD % 128), "streamed weights"),
    Case(128, 64, 3, 3, 1, 8, 64, True, K(GEMM % 64, GEMM % 128, WGRAD % 64), "fprop 36 streamed weight chunks"),
    Case(24, 200, 3, 3, 1, 6, 32, False, K(GEMM % 256, GEMM % 32, WGRAD % 256),
         "fprop 200 of 256 outputs; dgrad 7 k-chunks"),
    Case(40, 300, 3, 3, 1, 5, 20, False, K(GEMM % 256, GEMM % 64, WGRAD % 256),
         "2 output groups in fprop and wgrad; W = 20 (one partial segment per row)"),
    Case(20, 416, 3, 1, 1, 6, 16, False, K(GEMM % 256, GEMM % 32, WGRAD % 256), "3x1; dgrad 13 k-chunks"),
    Case(60, 520, 1, 3, 1, 4, 16, True, K(GEMM % 256, GEMM % 64, WGRAD % 256), "3 output groups"),
    Case(200, 136, 5, 5, 1, 6, 24, False, K(GEMM % 256, WGRAD % 256), "5x5; wgrad 2 channel blocks"),
    Case(40, 24, 3, 3, 1, 6, 32, True, K(GEMM % 32, GEMM % 64, WGRAD % 32), ""),
    Case(8, 40, 1, 7, 2, 4, 64, False, K(SMALL % 64, GEMM % 16, WGRAD % 64),
         "fprop small-Cin mode, 2 stages (the last 3 of 4 taps), resident weights"),
    Case(5, 200, 5, 5, 1, 6, 24, False, K(SMALL % 256, GEMM % 16, WGRAD % 256),
         "fprop small-Cin mode, 7 stages of streamed weights"),
    Case(24, 6, 3, 3, 1, 8, 32, False, K(GEMM % 16, SMALL % 32, WGRAD % 16), "dgrad small-Cin mode (K = 6)"),
    Case(6, 100, 3, 3, 1, 6, 32, False, K(SMALL % 128, GEMM % 16, WGRAD % 128), "fprop small-Cin mode, M = 100"),
]


def case_id(c):
    return "%dto%d-%dx%d-n%d-%dx%d%s" % (c.C, c.K, c.R, c.S, c.N, c.H, c.W, "-b" if c.bias else "")


def desc(c, N=None, dtype=_lib.SPC_F32, algo=ALL):
    return _lib.ConvDesc(c.N if N is None else N, c.C, c.H, c.W, c.K, c.R, c.S, 1, 1, (c.R - 1) // 2, (c.S - 1) // 2,
                         dtype, algo)


def uses(d, op):
    return _lib.lib().spc_conv_uses_tcgen05(C.byref(d), op)


def wsb(d, op):
    return _lib.lib().spc_conv_workspace_bytes(C.byref(d), op)


def make_inputs(c, tf32, mask=(0,) * 9, N=None):
    g = torch.Generator().manual_seed(zlib.crc32(repr((tuple(c[:8]), tf32, tuple(mask))).encode()))
    N = c.N if N is None else N
    ph, pw_ = (c.R - 1) // 2, (c.S - 1) // 2
    rnd = pw.round_tf32 if tf32 else (lambda t: t)
    x = rnd(torch.randn((N, c.C, c.H, c.W), generator=g))
    w = rnd(torch.randn((c.K, c.C, c.R, c.S), generator=g) / (c.C * c.R * c.S) ** 0.5)
    b = torch.randn((c.K,), generator=g) if c.bias else None
    dy = rnd(torch.randn((N, c.K, c.H, c.W), generator=g))
    strips = [None] * 9
    for i, (dr, dc) in enumerate(so.DIRS):
        rows, cols = (ph if dr else c.H), (pw_ if dc else c.W)
        if i != 4 and mask[i] and rows and cols:
            strips[i] = rnd(torch.randn((N, c.C, rows, cols), generator=g))
    return x, w, b, dy, strips


def layer_shapes():
    """every distinct stride-1 multi-tap conv of the two BASELINE layer lists: (list, C, K, R, S, H, bias)"""
    out = []
    for fn, tag in (("layers_amoebanetd_sp4.json", "amoeba"), ("layers_resnet101_sp2.json", "resnet")):
        for l in json.load(open(os.path.join(ROOT, "golden", fn)))["layers"]:
            if l["op"] != "conv" or l["R"] * l["S"] == 1 or l["stride_h"] != 1:
                continue
            key = (tag, l["C"], l["K"], l["R"], l["S"], l["H"], bool(l.get("bias")))
            if key not in out:
                out.append(key)
    return out


# ---- CPU ---------------------------------------------------------------------------------------------------------
def test_dispatch():
    for c in CASES:
        for op in range(3):
            assert uses(desc(c), op) == 1, (case_id(c), op)
            assert (wsb(desc(c), op) == 0) if op == 2 else (wsb(desc(c), op) > 0), (case_id(c), op)   # wgrad: none
            for algo in (_lib.SPC_ALGO_AUTO, _lib.SPC_ALGO_DIRECT, _lib.SPC_ALGO_TCGEN05, _lib.SPC_ALGO_TF32):
                assert uses(desc(c, algo=algo), op) == 0, (case_id(c), op, algo)
    # every stride-1 tap shape of both lists, at the N=1 and the N=4 tile
    for _, Cc, K_, R, S, H, bias in layer_shapes():
        for h in (H, H // 2):
            c = Case(Cc, K_, R, S, 1, h, h, bias, frozenset(), "")
            assert all(uses(desc(c), op) for op in range(3)), c
    # stride 2, W % 4 != 0, even or wider than 7 x 7 filters: the direct kernels, as with SPC_ALGO_TF32
    for R, S, st, W in ((3, 3, 2, 64), (1, 7, 2, 64), (7, 1, 2, 64), (3, 3, 1, 18), (1, 7, 1, 30), (9, 9, 1, 64),
                        (2, 2, 1, 64)):
        for op in range(3):
            a, t = (_lib.ConvDesc(2, 16, 16, W, 16, R, S, st, st, (R - 1) // 2, (S - 1) // 2, _lib.SPC_F32, algo)
                    for algo in (ALL, _lib.SPC_ALGO_TF32))
            assert uses(a, op) == uses(t, op) == 0 and wsb(a, op) == wsb(t, op) == 0, (R, S, st, W, op)
    # fp32 1x1: the same kernels and workspace as SPC_ALGO_TF32
    for c in pw.CASES:
        for op in range(3):
            a, t = pw.desc(c, algo=ALL), pw.desc(c)
            assert uses(a, op) == uses(t, op) == 1 and wsb(a, op) == wsb(t, op), (pw.case_id(c), op)
    # bf16: SPC_ALGO_TF32_ALL is SPC_ALGO_AUTO
    shapes = [(c.C, c.K, c.H, c.W, c.R, c.S, 1) for c in CASES]
    shapes += [(c.C, c.K, c.H, c.W, c.R, c.S, c.stride) for c in cov.CASES]
    for C_, K_, H, W, R, S, st in shapes:
        for op in range(3):
            a, t = (_lib.ConvDesc(2, C_, H, W, K_, R, S, st, st, (R - 1) // 2, (S - 1) // 2, _lib.SPC_BF16, algo)
                    for algo in (_lib.SPC_ALGO_AUTO, ALL))
            assert uses(a, op) == uses(t, op) and wsb(a, op) == wsb(t, op), (C_, K_, H, W, R, S, st, op)


def test_tight_bound_detects_planted_errors():
    """At C = 256, 3x3, the tight bound rejects y without one tap, with one tap shifted by a pixel, without the last
    input column, and without one k8 step (8 channels of one tap)"""
    c = Case(256, 8, 3, 3, 1, 6, 16, False, frozenset(), "")
    x, w, b, dy, strips = make_inputs(c, True)
    ref, A = cov.reference(x, w, b, dy, strips, 1)
    xd, wd = x.double(), w.double()
    cov.check(ref["y"].float(), ref["y"], A["y"], 0.0, TIGHT, "y fp32")

    def tap_term(xx, r, s, c0=0, c1=None):
        wt = torch.zeros_like(wd)
        wt[:, c0:c1, r, s] = wd[:, c0:c1, r, s]
        return F.conv2d(xx, wt, padding=1)

    shifted = torch.roll(xd, 1, dims=3)
    shifted[..., 0] = 0
    x_nocol = xd.clone()
    x_nocol[..., -1] = 0
    planted = {
        "a missing tap": ref["y"] - tap_term(xd, 1, 2),
        "a tap shifted by one pixel": ref["y"] - tap_term(xd, 0, 1) + tap_term(shifted, 0, 1),
        "a missing edge column": F.conv2d(x_nocol, wd, padding=1),
        "a missing k8 step": ref["y"] - tap_term(xd, 2, 0, c.C - 8, c.C),
    }
    for what, y in planted.items():
        with pytest.raises(AssertionError):
            cov.check(y.float(), ref["y"], A["y"], 0.0, TIGHT, "y with " + what)


def test_instance_table_matches_library():
    if shutil.which("nm") is None:
        pytest.skip("nm (binutils) is not installed")
    assert os.path.exists(LIB), "build libspconv.so first"
    names = set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", open(SRC).read()))
    assert {TAP_KERNEL, TAP_WGRAD} <= names
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


def test_conv_algo_default(monkeypatch):
    from mpi4dl_b200.torchgems.spatial import conv_algo_default
    monkeypatch.delenv("SPCONV_ALLOW_TF32", raising=False)
    assert conv_algo_default() == _lib.SPC_ALGO_AUTO
    monkeypatch.setenv("SPCONV_ALLOW_TF32", "1")
    assert conv_algo_default() == _lib.SPC_ALGO_TF32
    monkeypatch.setenv("SPCONV_ALLOW_TF32", "all")
    assert conv_algo_default() == _lib.SPC_ALGO_TF32_ALL
    monkeypatch.setenv("SPCONV_ALLOW_TF32", "0")
    assert conv_algo_default() == _lib.SPC_ALGO_AUTO


# ---- GPU: the case table -------------------------------------------------------------------------------------------
def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def run_fwd(d, x, strips, w, b, split=False):
    L = _lib.lib()
    y = torch.empty((d.N, d.K, d.H, d.W), dtype=torch.float32, device=DEV)
    ws, n = cov._ws(d, 0)
    halo = _lib.make_halo(strips)
    if split:
        _lib.check(L.spc_conv2d_fwd_interior(C.byref(d), _ptr(x), _ptr(w), _ptr(b), _ptr(y), _ptr(ws), n, cov._st()),
                   "fwd_interior")
        _lib.check(L.spc_conv2d_fwd_boundary(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), cov._st()),
                   "fwd_boundary")
    else:
        _lib.check(L.spc_conv2d_fwd(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), _ptr(ws), n,
                                    cov._st()), "fwd")
    return y


def _dev(*ts):
    return [t.to(DEV) if t is not None else None for t in ts]


def _names(k):
    return {n for n, _ in k}


@pytest.mark.gpu
@pytest.mark.parametrize("tf32_inputs", [True, False], ids=["tight", "loose"])
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_case_against_fp64(c, tf32_inputs):
    bound = TIGHT if tf32_inputs else LOOSE
    tag = "%s %s" % (case_id(c), "tight" if tf32_inputs else "loose")
    x, w, b, dy, strips = make_inputs(c, tf32_inputs)
    x, w, b, dy = _dev(x, w, b, dy)
    ref, A = cov.reference(x, w, b, dy, strips, 1)
    d = desc(c)
    y, kf = cov.traced(lambda: run_fwd(d, x, strips, w, b))
    print("[tf32-tap] %-34s y  err/bound %.3f" % (tag, cov.check(y, ref["y"], A["y"], 0.0, bound, tag + " y")))
    dx, kd = cov.traced(lambda: pw.run_dgrad(d, dy, w))
    print("[tf32-tap] %-34s dx err/bound %.3f" % (tag, cov.check(dx, ref["dx"], A["dx"], 0.0, bound, tag + " dx")))
    dw = torch.full(w.shape, float("nan"), device=DEV)
    db = torch.full((c.K,), float("nan"), device=DEV) if c.bias else None
    _, kw = cov.traced(lambda: pw.run_wgrad(d, x, dy, dw, db, 0))
    print("[tf32-tap] %-34s dw err/bound %.3f" % (tag, cov.check(dw, ref["dw"], A["dw"], 0.0, bound, tag + " dw")))
    if c.bias:
        cov.check(db, ref["db"], A["db"], 0.0, TIGHT, tag + " db")
    # accumulate = 1 adds onto what dw / db hold
    g = torch.Generator(device=DEV).manual_seed(7)
    dw0 = torch.randn(w.shape, generator=g, device=DEV) * float(ref["dw"].abs().mean())
    db0 = torch.randn((c.K,), generator=g, device=DEV) if c.bias else None
    dw1, db1 = pw.run_wgrad(d, x, dy, dw0.clone(), db0.clone() if c.bias else None, 1)
    cov.check(dw1, dw0.double() + ref["dw"], A["dw"] + dw0.double().abs(), 0.0, bound, tag + " dw accumulate")
    if c.bias:
        cov.check(db1, db0.double() + ref["db"], A["db"] + db0.double().abs(), 0.0, TIGHT, tag + " db accumulate")
    # fprop / dgrad have no atomics: a repeated call is bit-identical
    assert torch.equal(run_fwd(d, x, strips, w, b), y), tag + ": fprop not reproducible"
    assert torch.equal(pw.run_dgrad(d, dy, w), dx), tag + ": dgrad not reproducible"

    def retrace():
        return cov.traced(lambda: (run_fwd(d, x, strips, w, b), pw.run_dgrad(d, dy, w),
                                   pw.run_wgrad(d, x, dy, torch.empty_like(dw), None, 0)))[1]
    k = kf | kd | kw
    assert cov.launched(k, lambda k: c.launches <= k, retrace), \
        "%s did not launch %s (launched: %s)" % (tag, sorted(c.launches - k), sorted(k))
    assert not DIRECT & _names(k), (tag, sorted(k))
    for kk, name in ((kf, TAP_KERNEL), (kd, TAP_KERNEL), (kw, TAP_WGRAD)):
        assert cov.launched(kk, lambda k: name in _names(k), retrace), (tag, name, sorted(kk))


def _masks(c, method, P):
    out = []
    for r in range(P):
        m = so.neighbour_mask(method, P, r, c.R, c.S)
        if m not in out and any(m[i] for i in range(9) if i != 4):
            out.append(m)
    return out


MASK_CASES = [CASES[1], CASES[3], CASES[4]]   # 3x3, 1x7, 7x1


@pytest.mark.gpu
@pytest.mark.parametrize("grid", cov.GRIDS, ids=[g[0] for g in cov.GRIDS])
@pytest.mark.parametrize("c", MASK_CASES, ids=case_id)
def test_halo_masks(c, grid):
    """corner, edge and middle tiles: the interior on the tap kernels, the forward's boundary on the direct kernel
    (through spc_conv2d_fwd and the split interior + boundary calls), wgrad with the strips' share added on the direct
    kernel; dx keeps the reference semantics (no halo)"""
    method, P = grid
    for mask in _masks(c, method, P):
        tag = "%s %s%s" % (case_id(c), method, "".join(map(str, mask)))
        x, w, b, dy, strips = make_inputs(c, True, mask)
        x, w, b, dy = _dev(x, w, b, dy)
        strips = _dev(*strips)
        ref, A = cov.reference(x, w, b, dy, strips, 1)
        d = desc(c)
        y, kf = cov.traced(lambda: run_fwd(d, x, strips, w, b))
        r = cov.check(y, ref["y"], A["y"], 0.0, TIGHT, tag + " y")
        y2 = run_fwd(d, x, strips, w, b, split=True)
        cov.check(y2, ref["y"], A["y"], 0.0, TIGHT, tag + " y split")
        assert torch.equal(y2, y), tag + ": interior + boundary differs from fwd"
        dx = pw.run_dgrad(d, dy, w)
        cov.check(dx, ref["dx"], A["dx"], 0.0, TIGHT, tag + " dx")
        dw = torch.full(w.shape, float("nan"), device=DEV)
        db = torch.full((c.K,), float("nan"), device=DEV) if c.bias else None
        halo = _lib.make_halo(strips)
        ws, n = cov._ws(d, 2)

        def wgrad():
            _lib.check(_lib.lib().spc_conv2d_wgrad(C.byref(d), _ptr(x), C.byref(halo), _ptr(dy),
                                                   C.c_void_p(dw.data_ptr()), _ptr(db), 0, _ptr(ws), n, cov._st()),
                       "wgrad")
        _, kw = cov.traced(wgrad)
        rw = cov.check(dw, ref["dw"], A["dw"], 0.0, TIGHT, tag + " dw")
        if c.bias:
            cov.check(db, ref["db"], A["db"], 0.0, TIGHT, tag + " db")
        print("[tf32-tap] %-40s y err/bound %.3f  dw %.3f" % (tag, r, rw))
        assert cov.launched(kf, lambda k: TAP_KERNEL in _names(k),
                            lambda: cov.traced(lambda: run_fwd(d, x, strips, w, b))[1]), (tag, sorted(kf))
        assert cov.launched(kw, lambda k: TAP_WGRAD in _names(k), lambda: cov.traced(wgrad)[1]), (tag, sorted(kw))
        assert cov.launched(kf, lambda k: "conv_direct_kernel" in _names(k),
                            lambda: cov.traced(lambda: run_fwd(d, x, strips, w, b))[1]), (tag, sorted(kf))


@pytest.mark.gpu
def test_empty_batch():
    c = CASES[1]
    d = desc(c, N=0)
    assert uses(d, 0) and uses(d, 1) and uses(d, 2)
    x, w, b, dy, _ = _dev(*make_inputs(c, True, N=0)[:4], None)
    assert run_fwd(d, x, [None] * 9, w, b).numel() == 0 and pw.run_dgrad(d, dy, w).numel() == 0
    dw0, db0 = torch.randn(w.shape, device=DEV), torch.randn((c.K,), device=DEV)
    dw, db = pw.run_wgrad(d, None, None, dw0.clone(), db0.clone(), 1)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw0) and torch.equal(db, db0)
    dw, db = pw.run_wgrad(d, None, None, dw, db, 0)
    torch.cuda.synchronize()
    assert not dw.any() and not db.any()


@pytest.mark.gpu
def test_pointwise_bit_identical_to_tf32():
    """SPC_ALGO_TF32_ALL runs the 1x1 layers on gemm_tf32.cu exactly as SPC_ALGO_TF32"""
    c = pw.CASES[3]
    x, w, b, dy = [t.to(DEV) if t is not None else None for t in pw.make_inputs(c, False)]
    a, t = pw.desc(c, algo=ALL), pw.desc(c)
    assert torch.equal(pw.run_fwd(a, x, w, b), pw.run_fwd(t, x, w, b))
    assert torch.equal(pw.run_dgrad(a, dy, w), pw.run_dgrad(t, dy, w))


# ---- GPU: full-size BASELINE tap shapes --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("layer", layer_shapes(), ids=lambda l: "%s-%dto%d-%dx%d-%d" % l[:6])
def test_fullsize_vs_cudnn_fp32(layer):
    """N=4 tile (half the stage's extent) of every stride-1 multi-tap BASELINE shape, arbitrary fp32 inputs, against
    cuDNN fp32 with TF32 off under the loose bound"""
    _, Cc, K_, R, S, H, bias = layer
    H = W = H // 2
    pad = ((R - 1) // 2, (S - 1) // 2)
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        gen = torch.Generator(device=DEV).manual_seed(Cc * 7 + K_ * 3 + R + H)
        x = torch.randn((1, Cc, H, W), device=DEV, generator=gen)
        w = torch.randn((K_, Cc, R, S), device=DEV, generator=gen) / (Cc * R * S) ** 0.5
        b = torch.randn(K_, device=DEV, generator=gen) if bias else None
        d = desc(Case(Cc, K_, R, S, 1, H, W, bias, frozenset(), ""))
        assert uses(d, 0) and uses(d, 1) and uses(d, 2), layer
        y = run_fwd(d, x, [None] * 9, w, b)
        pw._check_sliced(y, F.conv2d(x, w, b, padding=pad),
                         F.conv2d(x.abs(), w.abs(), b.abs() if bias else None, padding=pad), LOOSE, "y")
        del y
        dy = torch.randn((1, K_, H, W), device=DEV, generator=gen)
        dx = pw.run_dgrad(d, dy, w)
        pw._check_sliced(dx, torch.nn.grad.conv2d_input(x.shape, w, dy, padding=pad),
                         torch.nn.grad.conv2d_input(x.shape, w.abs(), dy.abs(), padding=pad), LOOSE, "dx")
        del dx
        dw, _ = pw.run_wgrad(d, x, dy, torch.empty(w.shape, device=DEV), None, 0)
        pw._check_sliced(dw, torch.nn.grad.conv2d_weight(x, w.shape, dy, padding=pad),
                         torch.nn.grad.conv2d_weight(x.abs(), w.shape, dy.abs(), padding=pad), LOOSE, "dw")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        torch.cuda.empty_cache()


# ---- GPU: the layers ---------------------------------------------------------------------------------------------
def _set_env(monkeypatch, allow):
    if allow:
        monkeypatch.setenv("SPCONV_ALLOW_TF32", "all")
    else:
        monkeypatch.delenv("SPCONV_ALLOW_TF32", raising=False)


def _amoeba_cell(monkeypatch, allow):
    from mpi4dl_b200.models.amoebanet import Cell
    _set_env(monkeypatch, allow)
    torch.manual_seed(11)
    sp = dict(local_rank=0, spatial_size=1, num_spatial_parts=1, slice_method="square")
    return Cell(sp, 64, 64, 64, reduction=False, reduction_prev=False).to(DEV).train()


def _resnet_cell(monkeypatch, allow):
    from mpi4dl_b200.models.resnet import _SpatialCtx, make_cell_v2
    _set_env(monkeypatch, allow)
    torch.manual_seed(12)
    ctx = _SpatialCtx(0, 1, 1, "square")
    return make_cell_v2(0, 1, 16, 16, 64, "relu", True, ctx=ctx).to(DEV).train()


def _run(cell, x):
    for p in cell.parameters():
        p.grad = None
    xg = x.clone().requires_grad_(True)
    y = cell(xg)
    y = y[0] if isinstance(y, tuple) else y
    r = torch.randn(y.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    (y * r).sum().backward()
    return y.detach(), xg.grad, [p.grad for p in cell.parameters()]


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["amoebanet", "resnet"])
def test_cell_with_tf32_all(monkeypatch, which):
    """SPCONV_ALLOW_TF32=all: every conv of the cell takes SPC_ALGO_TF32_ALL, no direct convolution kernel runs, and
    the results stay within test_amoebanet_cell_with_tf32's tolerances of the direct run"""
    from mpi4dl_b200.torchgems.spatial import conv_spatial, local_conv2d
    make, cin = (_amoeba_cell, 64) if which == "amoebanet" else (_resnet_cell, 16)
    ref_cell = make(monkeypatch, False)
    tf_cell = make(monkeypatch, True)
    tf_cell.load_state_dict(ref_cell.state_dict())
    convs = [m for m in tf_cell.modules() if isinstance(m, (conv_spatial, local_conv2d))]
    assert convs and all(m.algo == ALL for m in convs)
    assert any(tuple(m.kernel_size) != (1, 1) for m in convs)
    x = torch.randn(2, cin, 32, 32, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    ref, kr = cov.traced(lambda: _run(ref_cell, x))
    got, kt = cov.traced(lambda: _run(tf_cell, x))
    assert {TAP_KERNEL, TAP_WGRAD} <= _names(kt), sorted(kt)
    assert not DIRECT & _names(kt), sorted(kt)
    tol = 16 * LOOSE
    err = float((got[0] - ref[0]).abs().max())
    print("[tf32-tap] %s cell y max err / max |ref| %.3g" % (which, err / float(ref[0].abs().max())))
    assert err <= tol * float(ref[0].abs().max()), "y: max err %.3g vs max |ref| %.3g" % (err, float(ref[0].abs().max()))
    # the bias of a convolution that feeds a training-mode BatchNorm has a gradient of zero up to rounding (the
    # normalisation removes any per-channel offset): its relative error says nothing, so gradients below 1e-3 of the
    # largest one are only printed
    grads = [("dx", got[1], ref[1])] + [("d" + n, a, r) for (n, _), a, r in
                                         zip(tf_cell.named_parameters(), got[2], ref[2]) if r is not None]
    floor = 1e-3 * max(float(r.norm()) for _, _, r in grads)
    for name, a, r in grads:
        rel = float((a - r).norm() / r.norm()) if float(r.norm()) > 0 else float(a.norm())
        print("[tf32-tap] %s cell %-24s |ref| %.3g |err| / |ref| %.3g" % (which, name, float(r.norm()), rel))
        assert rel <= 0.1 or float(r.norm()) < floor, "%s: |err| / |ref| = %.3g" % (name, rel)


@pytest.mark.gpu
def test_cuda_graph_replay(monkeypatch):
    """one CUDA-graph capture of a 3x3 conv_spatial layer's forward and backward replays to the eager result"""
    from mpi4dl_b200.torchgems.spatial import conv_spatial
    monkeypatch.setenv("SPCONV_ALLOW_TF32", "all")
    torch.manual_seed(5)
    layer = conv_spatial(in_channels=16, out_channels=32, kernel_size=3, stride=1, padding=1, local_rank=0,
                         spatial_size=1, num_spatial_parts=1, slice_method="square").to(DEV)
    assert layer.algo == ALL
    x = torch.randn(2, 16, 32, 32, device=DEV)
    g = torch.randn(2, 32, 32, 32, device=DEV)

    def step(xs):
        layer.zero_grad(set_to_none=False)
        xg = xs.detach().requires_grad_(True)
        y = layer(xg)
        y.backward(g)
        return y.detach(), xg.grad

    y0, dx0 = [t.clone() for t in step(x)]
    dw0 = layer.weight.grad.clone()
    xs = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(xs)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg, dxg = step(xs)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y0) and torch.equal(dxg, dx0)
    torch.testing.assert_close(layer.weight.grad, dw0, rtol=0, atol=1e-5 * float(dw0.abs().max()))
