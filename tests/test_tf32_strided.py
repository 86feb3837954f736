"""fp32 stride-2 multi-tap convolutions on the TF32 tensor cores (SPC_ALGO_TF32_STRIDED, conv_tap_s2_tf32.cu).

CPU: dispatch (which shapes take the stride-2 kernels, that SPC_ALGO_TF32_STRIDED answers everything else as
SPC_ALGO_TF32_ALL does and that no other algorithm value takes them), the sensitivity of the tight bound to planted
stride-2 errors, that CASES names every kernel instance of conv_tap_s2_tf32.cu in libspconv.so, and conv_algo_default().
GPU (-m gpu): every case of CASES through the C ABI against an fp64 reference per element under both bounds of
include/spconv.h (see tests/test_tf32_tap.py), the cases under halo-strip masks, bit-identity with SPC_ALGO_TF32_ALL on
the shapes that takes, every stride-2 multi-tap shape of the two BASELINE layer lists at the N=4 tile against cuDNN fp32
(TF32 off), an AmoebaNet-D reduction cell and a stride-2 ResNet-v2 bottleneck with SPCONV_ALLOW_TF32=strided against
the direct run, and a CUDA-graph capture of a stride-2 layer.
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
from tests import test_tf32_tap as tap

ROOT = os.path.dirname(os.path.abspath(__file__))
LIB = tap.LIB
SRC = os.path.join(os.path.dirname(ROOT), "mpi4dl_b200", "csrc", "conv_tap_s2_tf32.cu")
DEV = "cuda:0"
TIGHT, LOOSE = pw.TIGHT, pw.LOOSE
K = cov.K
STRIDED, ALL = _lib.SPC_ALGO_TF32_STRIDED, _lib.SPC_ALGO_TF32_ALL
S2_KERNEL, S2_WGRAD = "tf32_s2_gemm_kernel", "tf32_s2_wgrad_kernel"
DIRECT = tap.DIRECT

# ---- the case table --------------------------------------------------------------------------------------------------
# tf32_s2_gemm_kernel<NT, mode>: mode 0 = fprop (NT from K as in test_tf32_tap), 1 = fprop in the small-Cin mode
# (C <= 8), 2 = dgrad (NT from C; always the general mode).  tf32_s2_wgrad_kernel<NT>: NT from K, 128-channel blocks of
# C.  Weights stay resident in smem for one group of outputs when taps x ceil(Cin / 32) x NT x 128 B <= 128 KB.
# W / 2 % 32 != 0 leaves the last row segment partial on the output and on the input side.
Case = collections.namedtuple("Case", "C K R S N H W bias launches note")
GEMM, SMALL, DGRAD = "tf32_s2_gemm_kernel<%d, 0>", "tf32_s2_gemm_kernel<%d, 1>", "tf32_s2_gemm_kernel<%d, 2>"
WGRAD = "tf32_s2_wgrad_kernel<%d>"
CASES = [
    Case(3, 104, 3, 3, 2, 12, 40, False, K(SMALL % 128, DGRAD % 16, WGRAD % 128, "tf32_s2_repack_kernel"),
         "the C=3 stem without bias: fprop in the small-Cin mode (3 stages of 4 taps, the last 1 of 4); W = 40: a "
         "20-pixel segment"),
    Case(52, 52, 3, 3, 2, 8, 64, True, K(GEMM % 64, DGRAD % 64, WGRAD % 64), "streamed weights (18 chunks of 8 KB)"),
    Case(104, 104, 3, 3, 1, 6, 72, True, K(GEMM % 128, DGRAD % 128, WGRAD % 128),
         "streamed weights; W = 72: a full and a 4-pixel output segment per row"),
    Case(64, 64, 3, 3, 2, 8, 32, True, K(GEMM % 64, DGRAD % 64, WGRAD % 64), "the ResNet-v2 layer's channels"),
    Case(16, 16, 3, 3, 2, 10, 64, True, K(GEMM % 16, DGRAD % 16, WGRAD % 16), "resident weights"),
    Case(24, 32, 5, 5, 1, 8, 32, False, K(GEMM % 32, DGRAD % 32, WGRAD % 32),
         "5x5, resident weights (25 taps); dgrad classes of 9, 6, 6 and 4 taps"),
    Case(40, 300, 3, 3, 1, 6, 16, False, K(GEMM % 256, DGRAD % 64, WGRAD % 256),
         "2 output groups in fprop and wgrad; dgrad 10 k-chunks"),
    Case(200, 24, 7, 7, 1, 4, 16, False, K(GEMM % 32, DGRAD % 256, WGRAD % 32),
         "7x7 on a tile shorter than the filter's reach; wgrad 2 channel blocks; fprop 7 k-chunks x 49 taps"),
    Case(8, 40, 3, 5, 2, 4, 64, True, K(SMALL % 64, DGRAD % 16, WGRAD % 64), "3x5; small-Cin mode, 4 stages"),
    Case(5, 200, 5, 5, 1, 6, 24, False, K(SMALL % 256, DGRAD % 16, WGRAD % 256), "small-Cin mode, streamed weights"),
    Case(6, 24, 3, 3, 1, 2, 32, False, K(SMALL % 32, DGRAD % 16, WGRAD % 32), "H = 2: one output row"),
    Case(4, 16, 7, 7, 1, 6, 16, False, K(SMALL % 16, DGRAD % 16, WGRAD % 16),
         "small-Cin mode, 13 stages (the last 1 of 4 taps)"),
]


def case_id(c):
    return "%dto%d-%dx%d-n%d-%dx%d%s" % (c.C, c.K, c.R, c.S, c.N, c.H, c.W, "-b" if c.bias else "")


def desc(c, N=None, dtype=_lib.SPC_F32, algo=STRIDED, stride=(2, 2)):
    return _lib.ConvDesc(c.N if N is None else N, c.C, c.H, c.W, c.K, c.R, c.S, stride[0], stride[1],
                         (c.R - 1) // 2, (c.S - 1) // 2, dtype, algo)


uses, wsb = tap.uses, tap.wsb


def make_inputs(c, tf32, mask=(0,) * 9, N=None):
    g = torch.Generator().manual_seed(zlib.crc32(repr((tuple(c[:8]), tf32, tuple(mask), "s2")).encode()))
    N = c.N if N is None else N
    ph, pw_ = (c.R - 1) // 2, (c.S - 1) // 2
    rnd = pw.round_tf32 if tf32 else (lambda t: t)
    x = rnd(torch.randn((N, c.C, c.H, c.W), generator=g))
    w = rnd(torch.randn((c.K, c.C, c.R, c.S), generator=g) / (c.C * c.R * c.S) ** 0.5)
    b = torch.randn((c.K,), generator=g) if c.bias else None
    dy = rnd(torch.randn((N, c.K, c.H // 2, c.W // 2), generator=g))
    strips = [None] * 9
    for i, (dr, dc) in enumerate(so.DIRS):
        rows, cols = (ph if dr else c.H), (pw_ if dc else c.W)
        if i != 4 and mask[i] and rows and cols:
            strips[i] = rnd(torch.randn((N, c.C, rows, cols), generator=g))
    return x, w, b, dy, strips


def layer_shapes():
    """every distinct stride-2 multi-tap conv of the two BASELINE layer lists: (list, C, K, R, S, H, bias)"""
    out = []
    for fn, tag in (("layers_amoebanetd_sp4.json", "amoeba"), ("layers_resnet101_sp2.json", "resnet")):
        for l in json.load(open(os.path.join(ROOT, "golden", fn)))["layers"]:
            if l["op"] != "conv" or l["R"] * l["S"] == 1 or l["stride_h"] != 2:
                continue
            key = (tag, l["C"], l["K"], l["R"], l["S"], l["H"], bool(l.get("bias")))
            if key not in out:
                out.append(key)
    return out


# ---- CPU ---------------------------------------------------------------------------------------------------------
def test_dispatch():
    others = (_lib.SPC_ALGO_AUTO, _lib.SPC_ALGO_DIRECT, _lib.SPC_ALGO_TF32, ALL)
    for c in CASES:
        for op in range(3):
            assert uses(desc(c), op) == 1, (case_id(c), op)
            assert (wsb(desc(c), op) == 0) if op == 2 else (wsb(desc(c), op) > 0), (case_id(c), op)   # wgrad: none
            for algo in others + (_lib.SPC_ALGO_TCGEN05,):
                assert uses(desc(c, algo=algo), op) == 0 and wsb(desc(c, algo=algo), op) == 0, (case_id(c), op, algo)
    # every stride-2 multi-tap shape of both lists, at the N=1 and the N=4 tile
    shapes = layer_shapes()
    assert len(shapes) == 4 and all(l[3:5] == (3, 3) for l in shapes), shapes
    for _, Cc, K_, R, S, H, bias in shapes:
        for h in (H, H // 2):
            c = Case(Cc, K_, R, S, 1, h, h, bias, frozenset(), "")
            for op in range(3):
                assert uses(desc(c), op) == 1 and (wsb(desc(c), op) > 0) == (op < 2), (c, op)
                for algo in others:
                    assert uses(desc(c, algo=algo), op) == 0 and wsb(desc(c, algo=algo), op) == 0, (c, op, algo)
    # 1x7 / 7x1 at stride 2, mixed strides, odd H, W % 8 != 0, filters wider than 7x7 or even: the direct kernels
    for R, S, st, H, W in ((1, 7, (2, 2), 16, 64), (7, 1, (2, 2), 16, 64), (3, 3, (2, 1), 16, 64),
                           (3, 3, (1, 2), 16, 64), (3, 3, (2, 2), 15, 64), (3, 3, (2, 2), 16, 36),
                           (3, 3, (2, 2), 16, 20), (9, 9, (2, 2), 16, 64), (2, 2, (2, 2), 16, 64)):
        d = desc(Case(16, 16, R, S, 2, H, W, False, frozenset(), ""), stride=st)
        for op in range(3):
            assert uses(d, op) == 0 and wsb(d, op) == 0, (R, S, st, H, W, op)
    # the shapes SPC_ALGO_TF32_ALL takes: the same answers
    for c in tap.CASES:
        for op in range(3):
            a, t = tap.desc(c, algo=STRIDED), tap.desc(c)
            assert uses(a, op) == uses(t, op) == 1 and wsb(a, op) == wsb(t, op), (tap.case_id(c), op)
    for c in pw.CASES:
        for op in range(3):
            a, t = pw.desc(c, algo=STRIDED), pw.desc(c, algo=ALL)
            assert uses(a, op) == uses(t, op) == 1 and wsb(a, op) == wsb(t, op), (pw.case_id(c), op)
    # bf16: SPC_ALGO_TF32_STRIDED is SPC_ALGO_AUTO
    shapes = [(c.C, c.K, c.H, c.W, c.R, c.S, 2) for c in CASES]
    shapes += [(c.C, c.K, c.H, c.W, c.R, c.S, c.stride) for c in cov.CASES]
    for C_, K_, H, W, R, S, st in shapes:
        for op in range(3):
            a, t = (_lib.ConvDesc(2, C_, H, W, K_, R, S, st, st, (R - 1) // 2, (S - 1) // 2, _lib.SPC_BF16, algo)
                    for algo in (_lib.SPC_ALGO_AUTO, STRIDED))
            assert uses(a, op) == uses(t, op) and wsb(a, op) == wsb(t, op), (C_, K_, H, W, R, S, st, op)


def test_tight_bound_detects_planted_errors():
    """At C = 256, 3x3 stride 2, the tight bound rejects y without one tap, with one tap read at stride 1, with the
    two column phases of x swapped, and dx with one parity class left zero"""
    c = Case(256, 8, 3, 3, 1, 8, 16, False, frozenset(), "")
    x, w, b, dy, strips = make_inputs(c, True)
    ref, A = cov.reference(x, w, b, dy, strips, 2)
    xd, wd = x.double(), w.double()
    cov.check(ref["y"].float(), ref["y"], A["y"], 0.0, TIGHT, "y fp32")
    cov.check(ref["dx"].float(), ref["dx"], A["dx"], 0.0, TIGHT, "dx fp32")
    Ho, Wo = ref["y"].shape[2:]

    def tap_term(xx, r, s, stride):
        wt = torch.zeros_like(wd)
        wt[:, :, r, s] = wd[:, :, r, s]
        return F.conv2d(xx, wt, stride=stride, padding=1)[..., :Ho, :Wo]

    swapped = xd.reshape(*xd.shape[:3], -1, 2).flip(-1).reshape(xd.shape)
    planted = {
        "a missing tap": ref["y"] - tap_term(xd, 1, 2, 2),
        "a tap read at stride 1": ref["y"] - tap_term(xd, 0, 1, 2) + tap_term(xd, 0, 1, 1),
        "the column phases swapped": F.conv2d(swapped, wd, stride=2, padding=1),
    }
    for what, y in planted.items():
        with pytest.raises(AssertionError):
            cov.check(y.float(), ref["y"], A["y"], 0.0, TIGHT, "y with " + what)
    for a, b_ in ((0, 0), (0, 1), (1, 0), (1, 1)):
        dx = ref["dx"].clone()
        dx[..., a::2, b_::2] = 0
        with pytest.raises(AssertionError):
            cov.check(dx.float(), ref["dx"], A["dx"], 0.0, TIGHT, "dx without class (%d, %d)" % (a, b_))


def test_instance_table_matches_library():
    if shutil.which("nm") is None:
        pytest.skip("nm (binutils) is not installed")
    assert os.path.exists(LIB), "build libspconv.so first"
    names = set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", open(SRC).read()))
    assert names == {S2_KERNEL, S2_WGRAD, "tf32_s2_repack_kernel"}
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
    monkeypatch.setenv("SPCONV_ALLOW_TF32", "strided")
    assert conv_algo_default() == STRIDED == 5
    for v, algo in (("0", _lib.SPC_ALGO_AUTO), ("1", _lib.SPC_ALGO_TF32), ("all", ALL), ("", _lib.SPC_ALGO_AUTO)):
        monkeypatch.setenv("SPCONV_ALLOW_TF32", v)
        assert conv_algo_default() == algo, v
    monkeypatch.delenv("SPCONV_ALLOW_TF32")
    assert conv_algo_default() == _lib.SPC_ALGO_AUTO


# ---- GPU: the case table -------------------------------------------------------------------------------------------
_ptr, _dev, _names = tap._ptr, tap._dev, tap._names


def _run_fwd(d, x, strips, w, b, split=False):
    y = torch.empty((d.N, d.K, d.H // 2, d.W // 2), dtype=torch.float32, device=DEV)
    L, halo = _lib.lib(), _lib.make_halo(strips)
    ws, n = cov._ws(d, 0)
    if split:
        _lib.check(L.spc_conv2d_fwd_interior(C.byref(d), _ptr(x), _ptr(w), _ptr(b), _ptr(y), _ptr(ws), n, cov._st()),
                   "fwd_interior")
        _lib.check(L.spc_conv2d_fwd_boundary(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), cov._st()),
                   "fwd_boundary")
    else:
        _lib.check(L.spc_conv2d_fwd(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), _ptr(ws), n,
                                    cov._st()), "fwd")
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("tf32_inputs", [True, False], ids=["tight", "loose"])
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_case_against_fp64(c, tf32_inputs):
    bound = TIGHT if tf32_inputs else LOOSE
    tag = "%s %s" % (case_id(c), "tight" if tf32_inputs else "loose")
    x, w, b, dy, strips = make_inputs(c, tf32_inputs)
    x, w, b, dy = _dev(x, w, b, dy)
    ref, A = cov.reference(x, w, b, dy, strips, 2)
    d = desc(c)
    y, kf = cov.traced(lambda: _run_fwd(d, x, strips, w, b))
    print("[tf32-s2] %-34s y  err/bound %.3f" % (tag, cov.check(y, ref["y"], A["y"], 0.0, bound, tag + " y")))
    if c.bias:   # and without bias
        y0 = _run_fwd(d, x, strips, w, None)
        cov.check(y0, ref["y"] - b.double()[None, :, None, None], A["y"] - b.double().abs()[None, :, None, None], 0.0,
                  bound, tag + " y without bias")
    dx = torch.full(x.shape, float("nan"), device=DEV)   # dgrad writes all of dx
    ws, n = cov._ws(d, 1)

    def dgrad():
        _lib.check(_lib.lib().spc_conv2d_dgrad(C.byref(d), _ptr(dy), _ptr(w), _ptr(dx), _ptr(ws), n, cov._st()),
                   "dgrad")
    _, kd = cov.traced(dgrad)
    print("[tf32-s2] %-34s dx err/bound %.3f" % (tag, cov.check(dx, ref["dx"], A["dx"], 0.0, bound, tag + " dx")))
    dw = torch.full(w.shape, float("nan"), device=DEV)
    db = torch.full((c.K,), float("nan"), device=DEV) if c.bias else None
    _, kw = cov.traced(lambda: pw.run_wgrad(d, x, dy, dw, db, 0))
    print("[tf32-s2] %-34s dw err/bound %.3f" % (tag, cov.check(dw, ref["dw"], A["dw"], 0.0, bound, tag + " dw")))
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
    assert torch.equal(_run_fwd(d, x, strips, w, b), y), tag + ": fprop not reproducible"
    assert torch.equal(pw.run_dgrad(d, dy, w), dx), tag + ": dgrad not reproducible"

    def retrace():
        return cov.traced(lambda: (_run_fwd(d, x, strips, w, b), pw.run_dgrad(d, dy, w),
                                   pw.run_wgrad(d, x, dy, torch.empty_like(dw), None, 0)))[1]
    k = kf | kd | kw
    assert cov.launched(k, lambda k: c.launches <= k, retrace), \
        "%s did not launch %s (launched: %s)" % (tag, sorted(c.launches - k), sorted(k))
    assert not DIRECT & _names(k), (tag, sorted(k))
    assert not {tap.TAP_KERNEL, tap.TAP_WGRAD} & _names(k), (tag, sorted(k))


MASK_CASES = [CASES[4], CASES[1], CASES[5], CASES[8]]   # 3x3 (resident, streamed), 5x5, 3x5 small-Cin


def _reaches_strip(c, mask):
    """whether an output window reaches a strip of the mask: at stride 2 the last window ends (R - 1) / 2 - 1 rows past
    the tile, so a 3-tap filter reads the top / left strips only"""
    ph, pw_ = (c.R - 1) // 2, (c.S - 1) // 2
    return bool((ph >= 1 and any(mask[0:3])) or (ph >= 2 and any(mask[6:9])) or
                (pw_ >= 1 and any(mask[0::3])) or (pw_ >= 2 and any(mask[2::3])))


@pytest.mark.gpu
@pytest.mark.parametrize("grid", cov.GRIDS, ids=[g[0] for g in cov.GRIDS])
@pytest.mark.parametrize("c", MASK_CASES, ids=case_id)
def test_halo_masks(c, grid):
    """corner, edge and middle tiles: the interior on the stride-2 kernels, the forward's boundary on the direct kernel
    (through spc_conv2d_fwd and the split interior + boundary calls), wgrad with the strips' share added on the direct
    kernel; dx keeps the reference semantics (no halo)"""
    method, P = grid
    for mask in tap._masks(c, method, P):
        tag = "%s %s%s" % (case_id(c), method, "".join(map(str, mask)))
        x, w, b, dy, strips = make_inputs(c, True, mask)
        x, w, b, dy = _dev(x, w, b, dy)
        strips = _dev(*strips)
        ref, A = cov.reference(x, w, b, dy, strips, 2)
        d = desc(c)
        y, kf = cov.traced(lambda: _run_fwd(d, x, strips, w, b))
        r = cov.check(y, ref["y"], A["y"], 0.0, TIGHT, tag + " y")
        y2 = _run_fwd(d, x, strips, w, b, split=True)
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
        print("[tf32-s2] %-40s y err/bound %.3f  dw %.3f" % (tag, r, rw))

        def refwd():
            return cov.traced(lambda: _run_fwd(d, x, strips, w, b))[1]
        direct = _reaches_strip(c, mask)
        want_f = {S2_KERNEL, "conv_direct_kernel"} if direct else {S2_KERNEL}
        want_w = {S2_WGRAD, "wgrad_direct_kernel"} if direct else {S2_WGRAD}
        assert cov.launched(kf, lambda k: want_f <= _names(k), refwd), (tag, sorted(kf))
        assert cov.launched(kw, lambda k: want_w <= _names(k), lambda: cov.traced(wgrad)[1]), (tag, sorted(kw))
        assert direct or not DIRECT & _names(kf | kw), (tag, sorted(kf | kw))


@pytest.mark.gpu
def test_empty_batch():
    c = CASES[4]
    d = desc(c, N=0)
    assert uses(d, 0) and uses(d, 1) and uses(d, 2)
    x, w, b, dy, _ = _dev(*make_inputs(c, True, N=0)[:4], None)
    assert _run_fwd(d, x, [None] * 9, w, b).numel() == 0 and pw.run_dgrad(d, dy, w).numel() == 0
    dw0, db0 = torch.randn(w.shape, device=DEV), torch.randn((c.K,), device=DEV)
    dw, db = pw.run_wgrad(d, None, None, dw0.clone(), db0.clone(), 1)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw0) and torch.equal(db, db0)
    dw, db = pw.run_wgrad(d, None, None, dw, db, 0)
    torch.cuda.synchronize()
    assert not dw.any() and not db.any()


@pytest.mark.gpu
def test_bit_identical_to_tf32_all():
    """SPC_ALGO_TF32_STRIDED runs the stride-1 tap layers and the 1x1 layers on the kernels SPC_ALGO_TF32_ALL runs"""
    c = tap.CASES[1]
    x, w, b, dy = _dev(*tap.make_inputs(c, False)[:4])
    a, t = tap.desc(c, algo=STRIDED), tap.desc(c)
    assert torch.equal(tap.run_fwd(a, x, [None] * 9, w, b), tap.run_fwd(t, x, [None] * 9, w, b))
    assert torch.equal(pw.run_dgrad(a, dy, w), pw.run_dgrad(t, dy, w))
    c = pw.CASES[3]
    x, w, b, dy = _dev(*pw.make_inputs(c, False))
    a, t = pw.desc(c, algo=STRIDED), pw.desc(c, algo=ALL)
    assert torch.equal(pw.run_fwd(a, x, w, b), pw.run_fwd(t, x, w, b))
    assert torch.equal(pw.run_dgrad(a, dy, w), pw.run_dgrad(t, dy, w))


# ---- GPU: full-size BASELINE stride-2 shapes ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("layer", layer_shapes(), ids=lambda l: "%s-%dto%d-%dx%d-%d" % l[:6])
def test_fullsize_vs_cudnn_fp32(layer):
    """N=4 tile (half the stage's extent) of every stride-2 multi-tap BASELINE shape, arbitrary fp32 inputs, against
    cuDNN fp32 with TF32 off under the loose bound"""
    _, Cc, K_, R, S, H, bias = layer
    H = W = H // 2
    kw = dict(stride=2, padding=((R - 1) // 2, (S - 1) // 2))
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        gen = torch.Generator(device=DEV).manual_seed(Cc * 7 + K_ * 3 + R + H)
        x = torch.randn((1, Cc, H, W), device=DEV, generator=gen)
        w = torch.randn((K_, Cc, R, S), device=DEV, generator=gen) / (Cc * R * S) ** 0.5
        b = torch.randn(K_, device=DEV, generator=gen) if bias else None
        d = desc(Case(Cc, K_, R, S, 1, H, W, bias, frozenset(), ""))
        assert uses(d, 0) and uses(d, 1) and uses(d, 2), layer
        y = _run_fwd(d, x, [None] * 9, w, b)
        pw._check_sliced(y, F.conv2d(x, w, b, **kw), F.conv2d(x.abs(), w.abs(), b.abs() if bias else None, **kw),
                         LOOSE, "y")
        del y
        dy = torch.randn((1, K_, H // 2, W // 2), device=DEV, generator=gen)
        dx = pw.run_dgrad(d, dy, w)
        pw._check_sliced(dx, torch.nn.grad.conv2d_input(x.shape, w, dy, **kw),
                         torch.nn.grad.conv2d_input(x.shape, w.abs(), dy.abs(), **kw), LOOSE, "dx")
        del dx
        dw, _ = pw.run_wgrad(d, x, dy, torch.empty(w.shape, device=DEV), None, 0)
        pw._check_sliced(dw, torch.nn.grad.conv2d_weight(x, w.shape, dy, **kw),
                         torch.nn.grad.conv2d_weight(x.abs(), w.shape, dy.abs(), **kw), LOOSE, "dw")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        torch.cuda.empty_cache()


# ---- GPU: the layers ---------------------------------------------------------------------------------------------
def _set_env(monkeypatch, allow):
    if allow:
        monkeypatch.setenv("SPCONV_ALLOW_TF32", "strided")
    else:
        monkeypatch.delenv("SPCONV_ALLOW_TF32", raising=False)


def _amoeba_cell(monkeypatch, allow):
    from mpi4dl_b200.models.amoebanet import Cell
    _set_env(monkeypatch, allow)
    torch.manual_seed(11)
    sp = dict(local_rank=0, spatial_size=1, num_spatial_parts=1, slice_method="square")
    return Cell(sp, 64, 64, 64, reduction=True, reduction_prev=False).to(DEV).train()


def _resnet_cell(monkeypatch, allow):
    from mpi4dl_b200.models.resnet import _SpatialCtx, make_cell_v2
    _set_env(monkeypatch, allow)
    torch.manual_seed(12)
    ctx = _SpatialCtx(0, 1, 1, "square")
    return make_cell_v2(0, 2, 16, 16, 64, "relu", True, ctx=ctx).to(DEV).train()


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["amoebanet", "resnet"])
def test_cell_with_tf32_strided(monkeypatch, which):
    """SPCONV_ALLOW_TF32=strided: every conv of a reduction cell (AmoebaNet-D) / a stride-2 bottleneck (ResNet-v2) takes
    SPC_ALGO_TF32_STRIDED, no direct convolution kernel runs, and the results stay within test_cell_with_tf32_all's
    tolerances of the direct run"""
    from mpi4dl_b200.torchgems.spatial import conv_spatial, local_conv2d
    make, cin = (_amoeba_cell, 64) if which == "amoebanet" else (_resnet_cell, 16)
    ref_cell = make(monkeypatch, False)
    tf_cell = make(monkeypatch, True)
    tf_cell.load_state_dict(ref_cell.state_dict())
    convs = [m for m in tf_cell.modules() if isinstance(m, (conv_spatial, local_conv2d))]
    assert convs and all(m.algo == STRIDED for m in convs)
    assert any(tuple(m.kernel_size) == (3, 3) and tuple(m.stride) == (2, 2) for m in convs)
    x = torch.randn(2, cin, 32, 32, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    ref, kr = cov.traced(lambda: tap._run(ref_cell, x))
    got, kt = cov.traced(lambda: tap._run(tf_cell, x))
    assert {S2_KERNEL, S2_WGRAD} <= _names(kt), sorted(kt)
    assert not DIRECT & _names(kt), sorted(kt)
    assert DIRECT & _names(kr), sorted(kr)
    tol = 16 * LOOSE
    err = float((got[0] - ref[0]).abs().max())
    print("[tf32-s2] %s cell y max err / max |ref| %.3g" % (which, err / float(ref[0].abs().max())))
    assert err <= tol * float(ref[0].abs().max()), "y: max err %.3g vs max |ref| %.3g" % (err, float(ref[0].abs().max()))
    # gradients below 1e-3 of the largest one are only printed (see test_cell_with_tf32_all)
    grads = [("dx", got[1], ref[1])] + [("d" + n, a, r) for (n, _), a, r in
                                         zip(tf_cell.named_parameters(), got[2], ref[2]) if r is not None]
    floor = 1e-3 * max(float(r.norm()) for _, _, r in grads)
    for name, a, r in grads:
        rel = float((a - r).norm() / r.norm()) if float(r.norm()) > 0 else float(a.norm())
        print("[tf32-s2] %s cell %-24s |ref| %.3g |err| / |ref| %.3g" % (which, name, float(r.norm()), rel))
        assert rel <= 0.1 or float(r.norm()) < floor, "%s: |err| / |ref| = %.3g" % (name, rel)


@pytest.mark.gpu
def test_cuda_graph_replay(monkeypatch):
    """one CUDA-graph capture of a 3x3 stride-2 conv_spatial layer's forward and backward replays to the eager result"""
    from mpi4dl_b200.torchgems.spatial import conv_spatial
    monkeypatch.setenv("SPCONV_ALLOW_TF32", "strided")
    torch.manual_seed(5)
    layer = conv_spatial(in_channels=16, out_channels=32, kernel_size=3, stride=2, padding=1, local_rank=0,
                         spatial_size=1, num_spatial_parts=1, slice_method="square").to(DEV)
    assert layer.algo == STRIDED
    x = torch.randn(2, 16, 32, 32, device=DEV)
    g = torch.randn(2, 32, 16, 16, device=DEV)

    def step(xs):
        layer.zero_grad(set_to_none=False)
        xg = xs.detach().requires_grad_(True)
        y = layer(xg)
        y.backward(g)
        return y.detach(), xg.grad

    (y0, dx0), k = cov.traced(lambda: [t.clone() for t in step(x)])
    assert {S2_KERNEL, S2_WGRAD} <= _names(k) and not DIRECT & _names(k), sorted(k)
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
