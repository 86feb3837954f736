"""-m gpu: every instance of the direct convolution (conv_direct.cu) and of the pools (pool.cu) against a high-precision
reference per element.

The direct kernels run every fp32 convolution (TF32 is opt-in and 1x1 only), the fp32 / SPC_ALGO_DIRECT forward fix-up
of the boundary rectangles, and the bf16 stride-2 dgrad of filters other than 3x3.  The pools run every pool in every
dtype.  DCASES and PCASES are case tables in the layout of test_gpu_tc_coverage.CASES: each case names the instances it
must launch (asserted under torch.profiler) and, in its note, the host-plan branch it reaches.  Together they launch all
12 instances of conv_direct.cu and all 16 of pool.cu; tests/test_direct_pool_bounds.py checks on the CPU that the
tables name exactly the instances libspconv.so contains, and that the bounds below reject planted errors.

References: the convolutions against F.conv2d / torch.nn.grad.* in float64 on the padded tile (test_gpu_tc_coverage.
reference), with A the same operation on absolute values.  The pools against ATen itself: F.max_pool2d / F.avg_pool2d
in float64 on the CPU on the padded tile, with autograd for dx.  ATen's max rule is `v > max || isnan(v)`, so NaN
propagates and the gradient goes to the first maximum in row-major window order (to the last NaN if there are several);
numpy's argmax (oracle.spatial_oracle.pool_bwd) differs on NaN, hence not used here.

Bounds, per element.  u = 2^-24, gamma(n) = n u / (1 - n u) (Higham, Accuracy and Stability, 3.1).  The inputs are
exactly representable in the kernel's fp32 arithmetic, so the only errors are fp32 roundings and the final store.
  * Direct y: one fma chain per output over n = C R S terms in c -> r -> s order, then + bias: n + 1 roundings of
    partial sums, |err| <= gamma(n+1) A.  Direct dx: each stride parity class is a stride-1 direct convolution of dy
    with a sub-filter of Ta x Tb = ceil(R/s) x ceil(S/s) taps, n = K Ta Tb.
  * bf16 y / dx are then rounded once to bf16 (8 significant bits, unit roundoff 2^-8):
    |fl(v) - v| <= 2^-8 |v| <= 2^-8 (|ref| + gamma A), so |err| <= 2^-8 |ref| + (1 + 2^-8) gamma A.  One rounding
    can nearly fill this bound: bf16 cases reach err / bound ~ 1.
  * Direct dw and db: fp32 sums of exact products (inside fma) plus, with accumulate, the old value, so |err| <=
    gamma(n) A with n the longest rounding path of the summation.  dw: a thread's fma chain over tiles_per_cta 4x32
    tiles (tiles_per_cta * 128 terms), then ctas_x atomic adds in any order and the old value: n = tiles_per_cta * 128
    + ctas_x + 1 (wgrad_direct_terms, from launch_wgrad_direct's plan; never more than the always-valid N Ho Wo + 1,
    which at 67600 outputs would be too loose to see a missing tile).  db: bias_grad's per-thread loop over N images
    of ceil(Ho Wo / chunks / 256) terms, two 5-level warp trees, `chunks` atomics and the old value (bias_grad_terms).
  * Max y: a comparison, no arithmetic: bit-exact, NaN included.
  * Max dx: one window per element when k == stride, a copy of dy: bit-exact.  Overlapping windows sum up to 9
    routed dy values in fp32: gamma(9) A (A = the routed |dy|), plus the bf16 rounding as above.
  * Avg y, dx: at most 9 terms summed (8 roundings), times 1/9 (rounded) and one product rounding: <= 10u + O(u^2)
    relative to A; 12u A, plus the bf16 rounding as above.
Non-finite reference values (the inf / NaN data regimes) must be matched exactly: NaN where ATen gives NaN, the same
infinity where it gives one; the bounds apply to the finite ones.

Reproducibility: the pools and direct fprop / dgrad use no atomics, so three calls give bit-identical results.
fwd_interior + fwd_boundary is bit-identical to the one-pass forward: the boundary rectangles are recomputed from the
tile and the strips with the same per-output fma chain (the CTA shape, VERT and KB change which thread computes an
output, not the order of its terms).  Run with -s to see the worst err / bound per case and per kernel family.
"""
import collections
import ctypes as C
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from mpi4dl_b200 import _lib
from oracle import spatial_oracle as so
from tests import test_gpu_tc_coverage as cov
from tests.test_gpu_tc_coverage import K, check, launched, padded, parse_kernel, reference, traced

pytestmark = pytest.mark.gpu

DEV = cov.DEV
U = 2.0 ** -24
BF16_REL = 2.0 ** -8


def gamma(n):
    return n * U / (1 - n * U)


# ---- direct convolution case table -------------------------------------------------------------------------------
# launch_conv_direct: KB = 16 when N Ho Wo > 65536, else 4; CB = min(C, 8) halved while the patch + weights exceed
# 96 KB; VERT only for boundary rectangles with Wo <= 16 < Ho (fwd_rect).  launch_wgrad_direct: 4x32 output tiles,
# tiles_per_cta = max(8, ...), tap passes of 9.  launch_bias_grad: ceil(Ho Wo / 65536) chunks (at most 64).
# mask: "all" = an interior tile of a 3x3 grid (8 strips), "lr" = the middle tile of vertical slicing (left and
# right strips only), "none" = no neighbours.
DCase = collections.namedtuple("DCase", "C K R S stride N H W bias dtype mask launches note")
F32, BF16 = torch.float32, torch.bfloat16


def _dk(dtype, *names):
    t = "float" if dtype == F32 else "__nv_bfloat16"
    return K(*[n.replace("T", t, 1) if "<T" in n else n for n in names])


def _dcase(Cc, Kk, R, S, st, N, H, W, bias, dtype, mask, launches, note):
    return DCase(Cc, Kk, R, S, st, N, H, W, bias, dtype, mask, _dk(dtype, *launches), note)


DCASES = []
for _t in (F32, BF16):
    DCASES += [
        _dcase(3, 8, 3, 3, 1, 2, 130, 260, True, _t, "all",
               ("conv_direct_kernel<T, false, 16>", "conv_direct_kernel<T, false, 4>", "conv_direct_kernel<T, true, 4>",
                "wgrad_direct_kernel<T>", "bias_grad_kernel<T>"),
               "whole tile N Ho Wo = 67600 > 65536: KB=16 (fprop, dgrad); boundary rows KB=4, side columns VERT KB=4; "
               "wgrad 594 tiles in 75 CTAs, ragged last 4x32 tile; one bias chunk"),
        _dcase(2, 4, 3, 3, 1, 2, 33000, 8, True, _t, "lr",
               ("conv_direct_kernel<T, false, 16>", "conv_direct_kernel<T, true, 16>", "wgrad_direct_kernel<T>",
                "bias_grad_kernel<T>"),
               "thin tall tile: side columns 2 x 33000 x 1 > 65536 outputs: VERT KB=16; bias grad 5 chunks"),
    ]
DCASES += [
    _dcase(5, 7, 3, 3, 1, 2, 9, 20, True, F32, "all",
           ("conv_direct_kernel<T, false, 4>", "wgrad_direct_kernel<T>", "bias_grad_kernel<T>"),
           "small: KB=4, C < CB; wgrad one CTA"),
    _dcase(13, 16, 3, 3, 2, 2, 17, 40, True, F32, "all",
           ("conv_direct_kernel<T, false, 4>", "wgrad_direct_kernel<T>"),
           "3x3 s2: CB=4, chunks 4+4+4+1 (last partial); odd H; dgrad 4 parity classes of 2x2, 2x1, 1x2, 1x1 taps"),
    _dcase(13, 16, 3, 3, 2, 1, 16, 41, False, F32, "all", ("conv_direct_kernel<T, false, 4>",),
           "3x3 s2 even H, odd W"),
    _dcase(5, 6, 5, 5, 2, 2, 13, 22, False, F32, "all",
           ("conv_direct_kernel<T, false, 4>", "wgrad_direct_kernel<T>"),
           "5x5 s2: CB=4 (5 = 4 + 1); wgrad 3 tap passes (9 + 9 + 7)"),
    _dcase(5, 8, 7, 7, 2, 1, 12, 19, True, F32, "all", ("conv_direct_kernel<T, false, 4>",),
           "7x7 s2: CB=4, chunks 4+1; wgrad 6 tap passes"),
    _dcase(29, 13, 5, 5, 1, 2, 33, 70, True, F32, "all",
           ("conv_direct_kernel<T, false, 4>", "wgrad_direct_kernel<T>"),
           "5x5 s1: C = 29 = 8+8+8+5; wgrad 3 tap passes, 54 tiles in 7 CTAs, 2 channel blocks"),
    _dcase(6, 20, 1, 1, 2, 2, 16, 20, True, F32, "all", ("conv_direct_kernel<T, false, 4>",),
           "1x1 s2 even: dgrad 1 of 4 parity classes, the rest by the memset; K = 20: 2 k-blocks of wgrad"),
    _dcase(6, 5, 1, 1, 2, 2, 9, 11, False, F32, "none", ("conv_direct_kernel<T, false, 4>",), "1x1 s2 odd H, W"),
    _dcase(7, 9, 1, 7, 2, 2, 10, 23, False, F32, "all", ("conv_direct_kernel<T, false, 4>", "wgrad_direct_kernel<T>"),
           "1x7 s2: dgrad column classes of 4 and 3 taps; wgrad R S = 7"),
    _dcase(7, 9, 7, 1, 2, 2, 23, 10, True, F32, "all", ("conv_direct_kernel<T, false, 4>",),
           "7x1 s2, odd H"),
    _dcase(7, 9, 7, 1, 2, 2, 13, 16, False, BF16, "all", ("conv_direct_kernel<T, false, 4>",),
           "bf16 7x1 s2 on the direct path (dgrad of non-3x3 stride-2 filters runs here under AUTO too)"),
    _dcase(9, 11, 1, 7, 1, 2, 12, 40, True, F32, "lr", ("conv_direct_kernel<T, false, 4>", "conv_direct_kernel<T, true, 4>"),
           "1x7 s1: side rectangles 3 columns wide, VERT"),
]


def dcase_id(c):
    return "%dto%d-%dx%d-s%d-n%d-%dx%d%s-%s-%s" % (c.C, c.K, c.R, c.S, c.stride, c.N, c.H, c.W, "-b" if c.bias else "",
                                                  "fp32" if c.dtype == F32 else "bf16", c.mask)


MASKS = {"all": [1, 1, 1, 1, 0, 1, 1, 1, 1], "lr": [0, 0, 0, 1, 0, 1, 0, 0, 0], "none": [0] * 9}


def conv_out_hw(c):
    return cov.out_hw(c)


def make_conv_inputs(c):
    """fp32-random tensors (CPU) rounded to the case's dtype: x, w, b, dy and the strips of its mask"""
    g = torch.Generator().manual_seed(zlib.crc32(repr((tuple(c[:8]), str(c.dtype), c.mask)).encode()))
    ph, pw = (c.R - 1) // 2, (c.S - 1) // 2
    x = torch.randn((c.N, c.C, c.H, c.W), generator=g).to(c.dtype)
    w = (torch.randn((c.K, c.C, c.R, c.S), generator=g) / math.sqrt(c.C * c.R * c.S)).to(c.dtype)
    b = torch.randn((c.K,), generator=g).to(c.dtype) if c.bias else None
    strips = [None] * 9
    for i, (dr, dc) in enumerate(so.DIRS):
        rows, cols = (ph if dr else c.H), (pw if dc else c.W)
        if i != 4 and MASKS[c.mask][i] and rows and cols:
            strips[i] = torch.randn((c.N, c.C, rows, cols), generator=g).to(c.dtype)
    dy = torch.randn((c.N, c.K) + conv_out_hw(c), generator=g).to(c.dtype)
    return x, w, b, dy, strips


def conv_bounds(c):
    """{op: (rel, abs coefficient of A)} of the module docstring"""
    Ho, Wo = conv_out_hw(c)
    carry = 1.0 + BF16_REL if c.dtype == BF16 else 1.0
    rel = BF16_REL if c.dtype == BF16 else 0.0
    ta, tb = -(-c.R // c.stride), -(-c.S // c.stride)
    return {"y": (rel, carry * gamma(c.C * c.R * c.S + 1)), "dx": (rel, carry * gamma(c.K * ta * tb + 1)),
            "dw": (0.0, gamma(wgrad_direct_terms(c))), "db": (0.0, gamma(bias_grad_terms(c.N, Ho * Wo)))}


def wgrad_direct_terms(c):
    """the longest rounding path of wgrad_direct_kernel under launch_wgrad_direct's plan: a thread's fma chain over
    tiles_per_cta 4x32 tiles, ctas_x atomic adds and the old value.  Never more than N Ho Wo + 1."""
    Ho, Wo = conv_out_hw(c)
    total = c.N * -(-Ho // 4) * -(-Wo // 32)
    want = max(1, (132 * 8) // (-(-c.K // 16) * -(-c.C // 16)))
    tpc = max(8, -(-total // want))
    return min(tpc * 128 + -(-total // tpc) + 1, c.N * Ho * Wo + 1)


def bias_grad_terms(N, HW):
    """the longest rounding path of bias_grad_kernel: a thread's loop over N images of its share of a chunk, two
    5-level warp trees, `chunks` atomic adds and the old value"""
    chunks = min(64, -(-HW // 65536))
    return N * -(-(-(-HW // chunks)) // 256) + 10 + chunks + 1


# ---- running the direct ops through the C ABI -----------------------------------------------------------------
def _desc(c, N=None):
    algo = _lib.SPC_ALGO_AUTO if c.dtype == F32 else _lib.SPC_ALGO_DIRECT
    return cov.desc(c, N=N, dtype=_lib.dtype_code(c.dtype), algo=algo)


def conv_fwd(d, x, strips, w, b, dtype, split=False):
    L = _lib.lib()
    Ho, Wo = C.c_int(), C.c_int()
    L.spc_conv_out_shape(C.byref(d), C.byref(Ho), C.byref(Wo))
    y = torch.full((d.N, d.K, Ho.value, Wo.value), float("nan"), dtype=dtype, device=DEV)
    halo = _lib.make_halo(strips)
    p = cov._ptr
    if split:
        _lib.check(L.spc_conv2d_fwd_interior(C.byref(d), p(x), p(w), p(b), p(y), None, 0, cov._st()), "fwd_interior")
        _lib.check(L.spc_conv2d_fwd_boundary(C.byref(d), p(x), C.byref(halo), p(w), p(b), p(y), cov._st()),
                   "fwd_boundary")
    else:
        _lib.check(L.spc_conv2d_fwd(C.byref(d), p(x), C.byref(halo), p(w), p(b), p(y), None, 0, cov._st()), "fwd")
    return y


def conv_dgrad(d, dy, w, dtype):
    dx = torch.full((d.N, d.C, d.H, d.W), float("nan"), dtype=dtype, device=DEV)
    _lib.check(_lib.lib().spc_conv2d_dgrad(C.byref(d), cov._ptr(dy), cov._ptr(w), cov._ptr(dx), None, 0, cov._st()),
               "dgrad")
    return dx


def _bits(t):
    return t.view(torch.int16 if t.dtype == BF16 else torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


DFAMILIES = ("conv_direct_kernel", "wgrad_direct_kernel", "bias_grad_kernel")
PFAMILIES = ("pool_fwd_kernel", "pool_fwd_vec_kernel", "pool3_fwd_kernel", "pool3_s1_tma_kernel", "pool3_s1_ring_kernel",
             "pool_bwd_kernel", "pool_bwd_s2_vec_kernel")
WORST = collections.defaultdict(float)


def _record(tag, op, kernels, ratio):
    fams = sorted({n for n, _ in kernels if n in DFAMILIES + PFAMILIES})
    for f in fams:
        WORST[(f, op)] = max(WORST[(f, op)], ratio)
    print("[direct-pool] %-52s %-6s err/bound %.3f  %s" % (tag, op, ratio, "+".join(fams)))


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if WORST:
        print("\n[direct-pool] largest err/bound per kernel family and op:")
        for (f, op), r in sorted(WORST.items()):
            print("[direct-pool]   %-24s %-6s %.3f" % (f, op, r))


@pytest.mark.parametrize("c", DCASES, ids=dcase_id)
def test_direct_case_against_fp64(c):
    L = _lib.lib()
    tag = dcase_id(c)
    x, w, b, dy, strips = make_conv_inputs(c)
    x, w, b, dy, *strips = [t.to(DEV) if t is not None else None for t in (x, w, b, dy, *strips)]
    ref, A = reference(x, w, b, dy, strips, c.stride)
    bnd = conv_bounds(c)
    d = _desc(c)
    for op in range(3):
        assert not L.spc_conv_uses_tcgen05(C.byref(d), op), (tag, op)

    y, kf = traced(lambda: conv_fwd(d, x, strips, w, b, c.dtype))
    _record(tag, "y", kf, check(y, ref["y"], A["y"], *bnd["y"], tag + " y"))
    y2, ks = traced(lambda: conv_fwd(d, x, strips, w, b, c.dtype, split=True))
    assert _same_bits(y2, y), tag + ": fwd_interior + fwd_boundary differs from the one-pass forward"
    dx, kd = traced(lambda: conv_dgrad(d, dy, w, c.dtype))
    _record(tag, "dx", kd, check(dx, ref["dx"], A["dx"], *bnd["dx"], tag + " dx"))
    for _ in range(2):   # no atomics: bit-reproducible
        assert _same_bits(conv_fwd(d, x, strips, w, b, c.dtype), y), tag + " y not reproducible"
        assert _same_bits(conv_fwd(d, x, strips, w, b, c.dtype, split=True), y), tag + " split y not reproducible"
        assert _same_bits(conv_dgrad(d, dy, w, c.dtype), dx), tag + " dx not reproducible"

    dw = torch.full(w.shape, float("nan"), dtype=torch.float32, device=DEV)
    db = torch.full((c.K,), float("nan"), dtype=torch.float32, device=DEV) if c.bias else None
    _, kw = traced(lambda: cov.run_wgrad(d, x, strips, dy, dw, db, 0))
    _record(tag, "dw", kw, check(dw, ref["dw"], A["dw"], *bnd["dw"], tag + " dw"))
    if c.bias:
        _record(tag, "db", kw, check(db, ref["db"], A["db"], *bnd["db"], tag + " db"))
    # accumulate=1 adds onto what dw / db hold
    g = torch.Generator(device=DEV).manual_seed(7)
    dw0 = torch.randn(w.shape, generator=g, device=DEV) * float(ref["dw"].abs().mean())
    dw = dw0.clone()
    db0 = torch.randn((c.K,), generator=g, device=DEV) * float(ref["db"].abs().mean()) if c.bias else None
    db = db0.clone() if c.bias else None
    cov.run_wgrad(d, x, strips, dy, dw, db, 1)
    check(dw, dw0.double() + ref["dw"], dw0.double().abs() + A["dw"], *bnd["dw"], tag + " dw accumulate")
    if c.bias:
        check(db, db0.double() + ref["db"], db0.double().abs() + A["db"], *bnd["db"], tag + " db accumulate")

    def retrace():
        return traced(lambda: (conv_fwd(d, x, strips, w, b, c.dtype), conv_fwd(d, x, strips, w, b, c.dtype, True),
                               conv_dgrad(d, dy, w, c.dtype),
                               cov.run_wgrad(d, x, strips, dy, torch.empty_like(dw),
                                             torch.empty_like(db) if c.bias else None, 0)))[1]
    k = kf | ks | kd | kw
    assert launched(k, lambda k: c.launches <= k, retrace), \
        "%s did not launch %s (launched: %s)" % (tag, sorted(c.launches - k), sorted(k))


# ---- full-size fp32 on the direct path -----------------------------------------------------------------------------
# BASELINE layers at the N = 4 tile of the AmoebaNet-D 8192^2 stage (halo strips on every side the filter reads):
# the stem (8192^2 layer, 4096^2 tile) and a 1x7 of the third cell (2048^2 layer, 1024^2 tile), in fp32 against cuDNN
# fp32 with TF32 off.  db is requested although the layers have no bias: Ho Wo = 2048^2 makes it the 64-chunk bias grad.
FULLSIZE = [(3, 104, 3, 3, 2, 4096), (52, 52, 1, 7, 1, 1024)]


@pytest.mark.parametrize("case", FULLSIZE, ids=["stem-3to104-3x3-s2-4096", "52to52-1x7-1024"])
def test_direct_fullsize_fp32_vs_cudnn(case):
    from tests import test_gpu_fullsize_parity as fs
    Cc, Kk, R, S, st, H = case
    L = _lib.lib()
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        hh, hw = (R - 1) // 2, (S - 1) // 2
        gen = torch.Generator(device=DEV).manual_seed(4242 + Cc + H)
        x = torch.randn((1, Cc, H, H), device=DEV, generator=gen)
        w = torch.randn((Kk, Cc, R, S), device=DEV, generator=gen) / (Cc * R * S) ** 0.5
        strips = [s.float() if s is not None else None for s in fs._halo_strips(1, Cc, H, H, hh, hw, gen)]
        c = DCase(Cc, Kk, R, S, st, 1, H, H, False, F32, "all", frozenset(), "")
        d = _desc(c)
        assert not L.spc_conv_uses_tcgen05(C.byref(d), 0)
        xp = fs._padded(x, strips, hh, hw)
        y = conv_fwd(d, x, strips, w, None, F32)
        fs._check(y, F.conv2d(xp, w, None, stride=st), "y", rel=2.0 ** -16, floor=2.0 ** -16)
        del y
        gy = torch.randn((1, Kk) + conv_out_hw(c), device=DEV, generator=gen)
        dx = conv_dgrad(d, gy, w, F32)
        ref = torch.nn.grad.conv2d_input(xp.shape, w, gy, stride=st)[:, :, hh:hh + H, hw:hw + H]
        fs._check(dx, ref, "dx", rel=2.0 ** -16, floor=2.0 ** -16)
        del dx, ref
        dw = torch.empty(w.shape, device=DEV)
        db = torch.empty((Kk,), device=DEV)
        cov.run_wgrad(d, x, strips, gy, dw, db, 0)
        dw_ref = torch.nn.grad.conv2d_weight(xp, w.shape, gy, stride=st)
        assert float((dw - dw_ref).abs().max()) <= 1e-4 * float(dw_ref.abs().max())
        Ho, Wo = conv_out_hw(c)
        check(db, gy.double().sum((0, 2, 3)), gy.double().abs().sum((0, 2, 3)), 0.0,
              gamma(bias_grad_terms(1, Ho * Wo)), "db")
    finally:
        torch.backends.cudnn.allow_tf32 = old
        torch.cuda.empty_cache()


# ---- pool case table ---------------------------------------------------------------------------------------------
# run_fwd: TMA for 3x3 s1 (+ pool3_s1_ring_kernel when the view has strips), pool3_fwd_kernel for 3x3 s2,
# pool_fwd_vec_kernel for 2x2 s2 -- all three when x and y are 16-byte aligned, Wo % VEC == 0, W % (VEC stride) == 0
# and W == Wo stride (VEC = 4 fp32 / 8 bf16) -- else pool_fwd_kernel.  run_bwd: avg 3x3 s1 = the TMA kernel on dy
# (aligned, W % VEC == 0); pool_bwd_s2_vec_kernel for avg 3x3 s2 and max 2x2 s2 when W % 16 == 0, H = 2 Ho, W = 2 Wo;
# pool_bwd_kernel otherwise.  fwd / bwd name the kernel family; "a|b" is a for fp32, b for bf16.
PCase = collections.namedtuple("PCase", "mode k stride H W fwd bwd note")
TMA, RING, P3, VECK, GEN = "pool3_s1_tma_kernel", "pool3_s1_ring_kernel", "pool3_fwd_kernel", "pool_fwd_vec_kernel", \
    "pool_fwd_kernel"
BGEN, S2A, S2M = "pool_bwd_kernel", "pool_bwd_s2_vec_kernel:avg", "pool_bwd_s2_vec_kernel:max"
PCASES = [
    PCase("avg", 3, 1, 16, 64, TMA, TMA, "one row tile"),
    PCase("avg", 3, 2, 32, 64, P3, S2A, ""),
    PCase("max", 2, 2, 16, 32, VECK, S2M, ""),
    PCase("max", 3, 1, 9, 11, GEN, BGEN, "W not a multiple of VEC"),
    PCase("avg", 3, 1, 7, 13, GEN, BGEN, ""),
    PCase("avg", 3, 2, 10, 18, GEN, BGEN, "W % (VEC stride) != 0"),
    PCase("max", 3, 2, 8, 8, P3 + "|" + GEN, BGEN, "Wo = 4: one fp32 vector; not a bf16 vector"),
    PCase("avg", 5, 1, 12, 12, GEN, BGEN, "5x5: two-row strips"),
    PCase("avg", 3, 1, 20, 256, TMA, TMA, "rows of whole warps of 16-byte vectors"),
    PCase("max", 3, 1, 33, 512, TMA, BGEN, ""),
    PCase("avg", 3, 2, 34, 256, P3, S2A, "Ho = 17 odd"),
    PCase("avg", 3, 1, 70, 136, TMA, TMA, "several row / column tiles, partial edge tiles"),
    PCase("max", 3, 1, 130, 264, TMA, BGEN, "3 x 5 (fp32) / 3 x 3 (bf16) tiles, partial both ways"),
    PCase("avg", 3, 1, 64, 128, TMA, TMA, "exactly one / two tiles"),
    PCase("avg", 3, 1, 2, 16, TMA, TMA, "H = 2"),
    PCase("max", 3, 1, 1, 8, TMA, BGEN, "H = 1"),
    PCase("avg", 3, 2, 10, 16, P3, S2A, "wv = 4 / 2 vectors per row: one warp spans 8 / 16 rows and several planes"),
    PCase("max", 3, 2, 11, 32, P3, BGEN, "odd H at stride 2: last window over the bottom pad / strip"),
    PCase("max", 2, 2, 9, 32, VECK, BGEN, "odd H: the last row is in no window"),
    PCase("avg", 2, 2, 8, 16, VECK, BGEN, "avg 2x2 backward: generic"),
]
PN, PC = 2, 5


def pcase_id(c):
    return "%s%d-s%d-%dx%d" % (c.mode, c.k, c.stride, c.H, c.W)


def _pool_inst(name, dtype):
    t, vec = ("float", 4) if dtype == F32 else ("__nv_bfloat16", 8)
    if name == VECK:
        return "%s<%s, %d, 2, 2>" % (name, t, vec)
    if name == P3:
        return "%s<%s, %d, 2>" % (name, t, vec)
    if name.startswith("pool_bwd_s2_vec_kernel:"):
        mode = _lib.SPC_POOL_AVG if name.endswith("avg") else _lib.SPC_POOL_MAX
        return "pool_bwd_s2_vec_kernel<%s, %d>" % (t, mode)
    return "%s<%s>" % (name, t)


def pool_launches(c, dtype, strips=False):
    """(fwd, bwd) instance sets a case must launch; strips: the view has halo strips (TMA adds the ring kernel)"""
    def pick(s):
        return s.split("|")[0 if dtype == F32 else -1]
    fwd = [pick(c.fwd)] + ([RING] if pick(c.fwd) == TMA and strips else [])
    return K(*[_pool_inst(n, dtype) for n in fwd]), K(_pool_inst(pick(c.bwd), dtype))


def pool_table_instances():
    out = set()
    for c in PCASES:
        for dt in (F32, BF16):
            for s in (False, True):
                f, b = pool_launches(c, dt, s)
                out |= f | b
    return out


def direct_table_instances():
    out = set()
    for c in DCASES:
        out |= c.launches
    return out


def pool_masks(c):
    """the interior tile first, then every other neighbour mask of a 3x3 grid and of 3-way slicing, and none"""
    if c.k == 1 or (c.k - 1) // 2 == 0:
        return [[0] * 9]
    out = [[1, 1, 1, 1, 0, 1, 1, 1, 1]]
    for method, P in cov.GRIDS:
        for r in range(P):
            m = so.neighbour_mask(method, P, r, c.k, c.k)
            if m not in out:
                out.append(m)
    return out + [[0] * 9]


REGIMES = ("normal", "ties", "relu", "inf", "nan")


def make_pool_inputs(c, dtype, mask, regime):
    """x, the strips of mask and dy (CPU, dtype) in one data regime"""
    g = torch.Generator().manual_seed(zlib.crc32(repr((tuple(c[:5]), str(dtype), tuple(mask), regime)).encode()))
    pad = (c.k - 1) // 2

    def data(shape):
        if regime == "ties":
            return torch.randint(-2, 3, shape, generator=g).float()
        v = torch.randn(shape, generator=g)
        if regime == "relu":
            return v.clamp_min(0)
        if regime in ("inf", "nan"):
            u = torch.rand(shape, generator=g)
            if regime == "inf":
                v = torch.where(u < 0.03, math.inf, torch.where(u > 0.97, -math.inf, v))
            else:
                v = torch.where(u < 0.04, math.nan, v)
        return v

    x = data((PN, PC, c.H, c.W))
    if regime == "ties":
        x[:, 0] = -torch.randint(1, 3, x[:, 0].shape, generator=g).float()   # all negative: border maxima = the pad
    if regime == "nan":
        x[:, :, 0, :2] = math.nan                                             # two NaNs in the first windows
    strips = [None] * 9
    for i, (dr, dc) in enumerate(so.DIRS):
        rows, cols = (pad if dr else c.H), (pad if dc else c.W)
        if i != 4 and mask[i] and rows and cols:
            strips[i] = data((PN, PC, rows, cols)).to(dtype)
    Ho, Wo = (c.H + 2 * pad - c.k) // c.stride + 1, (c.W + 2 * pad - c.k) // c.stride + 1
    dy = torch.randn((PN, PC, Ho, Wo), generator=g).to(dtype)
    return x.to(dtype), strips, dy


def pool_reference(c, x, strips, dy):
    """ATen on the padded tile, float64 CPU: y, dx and the bound's A for y (avg) and dx"""
    pad = (c.k - 1) // 2
    xp = padded(x.cpu(), [s.cpu() if s is not None else None for s in strips], pad, pad).requires_grad_(True)
    fn = F.max_pool2d if c.mode == "max" else F.avg_pool2d
    y = fn(xp, c.k, c.stride, 0)
    g64 = dy.cpu().double()
    dxp, = torch.autograd.grad(y, xp, g64, retain_graph=True)
    dxa, = torch.autograd.grad(y, xp, g64.abs())
    crop = (slice(None), slice(None), slice(pad, pad + c.H), slice(pad, pad + c.W))
    ya = F.avg_pool2d(xp.detach().abs(), c.k, c.stride, 0) if c.mode == "avg" else None
    return y.detach(), ya, dxp[crop], dxa[crop]


def pool_bounds(c, dtype):
    """{op: (rel, abs coefficient) or None = bit-exact}"""
    rel = BF16_REL if dtype == BF16 else 0.0
    carry = 1.0 + BF16_REL if dtype == BF16 else 1.0
    if c.mode == "max":
        return {"y": None, "dx": None if c.k == c.stride else (rel, carry * gamma(9))}
    return {"y": (rel, carry * 12 * U), "dx": (rel, carry * 12 * U)}


def check_pool(got, ref, A, bound, name):
    """bound None: bit-exact (NaN where ref is NaN); else non-finite ref values exactly, the finite ones in bound"""
    got, ref = got.double().cpu(), ref.double()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), "%s: NaN at %d places, ATen at %d" % (
        name, int(torch.isnan(got).sum()), int(nan.sum()))
    if bound is None:
        bad = (got != ref) & ~nan
        assert not bad.any(), "%s: %d elements differ from ATen, first at %s (got %r, ref %r)" % (
            name, int(bad.sum()), tuple(bad.nonzero()[0].tolist()), float(got[bad][0]), float(ref[bad][0]))
        return 0.0
    inf = torch.isinf(ref)
    assert torch.equal(got[inf], ref[inf]), name + ": infinities differ"
    fin = torch.isfinite(ref)
    return check(got[fin], ref[fin], A.double()[fin], bound[0], bound[1], name)


def pool_run(c, dtype, x, strips, dy, xoff=0):
    """spc_pool2d_fwd + spc_pool2d_bwd through the C ABI; xoff > 0 views x at that element offset (unaligned)"""
    L = _lib.lib()
    pad = (c.k - 1) // 2
    d = _lib.PoolDesc(PN, PC, c.H, c.W, c.k, c.stride, pad, _lib.SPC_POOL_MAX if c.mode == "max" else _lib.SPC_POOL_AVG,
                      _lib.dtype_code(dtype))
    if xoff:
        buf = torch.empty(x.numel() + xoff, dtype=dtype, device=DEV)
        xd = buf[xoff:].view(x.shape)
        xd.copy_(x)
    else:
        xd = x.to(DEV)
    sd = [s.to(DEV) if s is not None else None for s in strips]
    dyd = dy.to(DEV)
    y = torch.full(dy.shape, float("nan"), dtype=dtype, device=DEV)
    dx = torch.full(x.shape, float("nan"), dtype=dtype, device=DEV)

    # the Halo struct holds raw pointers: it is made from sd in each call, so the closures keep the strips alive
    def fwd():
        halo = _lib.make_halo(sd)
        _lib.check(L.spc_pool2d_fwd(C.byref(d), cov._ptr(xd), C.byref(halo), cov._ptr(y), cov._st()), "pool fwd")
        return y.clone()

    def bwd():
        halo = _lib.make_halo(sd)
        _lib.check(L.spc_pool2d_bwd(C.byref(d), cov._ptr(xd), C.byref(halo), cov._ptr(dyd), cov._ptr(dx), cov._st()),
                   "pool bwd")
        return dx.clone()
    return fwd, bwd, xd


def _pool_check_one(c, dtype, mask, regime, trace=False, xoff=0):
    tag = "%s %s %s %s%s" % (pcase_id(c), "fp32" if dtype == F32 else "bf16", regime, "".join(map(str, mask)),
                             " off%d" % xoff if xoff else "")
    x, strips, dy = make_pool_inputs(c, dtype, mask, regime)
    fwd, bwd, xd = pool_run(c, dtype, x, strips, dy, xoff)
    if trace:
        y, kf = traced(fwd)
        dx, kb = traced(bwd)
    else:
        y, dx, kf, kb = fwd(), bwd(), set(), set()
    ref_y, ya, ref_dx, dxa = pool_reference(c, x, strips, dy)
    bnd = pool_bounds(c, dtype)
    _record(tag, "y", kf, check_pool(y, ref_y, ya, bnd["y"], tag + " y"))
    _record(tag, "dx", kb, check_pool(dx, ref_dx, dxa, bnd["dx"], tag + " dx"))
    if trace:   # no atomics: bit-reproducible
        for _ in range(2):
            assert _same_bits(fwd(), y) and _same_bits(bwd(), dx), tag + " not reproducible"
    return kf, kb, lambda: traced(fwd)[1] | traced(bwd)[1], xd


@pytest.mark.parametrize("dtype", [F32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("c", PCASES, ids=pcase_id)
def test_pool_case_against_aten(c, dtype):
    masks = pool_masks(c)
    for mi, mask in enumerate(masks):
        # every regime on the interior tile, one corner and no neighbours; random and NaN data under every mask
        regimes = REGIMES if mi in (0, 1, len(masks) - 1) else ("normal", "nan")
        for regime in regimes:
            first = regime == "normal" and mi in (0, len(masks) - 1)
            kf, kb, retrace, _ = _pool_check_one(c, dtype, mask, regime, trace=first)
            if first:
                want_f, want_b = pool_launches(c, dtype, any(mask))
                assert launched(kf | kb, lambda k: want_f | want_b <= k, retrace), \
                    "%s did not launch %s (launched %s)" % (pcase_id(c), sorted((want_f | want_b) - (kf | kb)),
                                                            sorted(kf | kb))


@pytest.mark.parametrize("dtype", [F32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("c", [c for c in PCASES if c.fwd != GEN or c.bwd != BGEN][:6], ids=pcase_id)
def test_pool_unaligned_view_falls_back(c, dtype):
    """x viewed one element past a 16-byte boundary: the generic kernels, and the same results"""
    mask = pool_masks(c)[0]
    kf, kb, retrace, xd = _pool_check_one(c, dtype, mask, "nan", trace=True, xoff=1)
    assert xd.data_ptr() % 16 != 0
    want = K(_pool_inst(GEN, dtype), _pool_inst(BGEN, dtype))
    assert launched(kf | kb, lambda k: want <= k, retrace), sorted(kf | kb)
    fast = {n for n, _ in kf | kb} & {TMA, RING, P3, VECK, "pool_bwd_s2_vec_kernel"}
    assert not fast, sorted(fast)
