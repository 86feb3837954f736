"""-m gpu: every wgmma kernel instance, and every halo fix-up configuration, against an fp64 reference per element.

The tensor-core path is a large set of separately compiled template instances -- conv_tap_kernel<NB, S, KS>,
wgrad_tap_kernel<S, QC>, pw_gemm_kernel<MB>, pw_wgrad_kernel<NBLK, NA> -- each with its own register allocation and
its own handling of the spare accumulators of a short last pass.  CASES is one table of small bf16 convolutions chosen
so that together they launch every instance (and every helper kernel of the stride-2 and shifted-copy paths).  Each
case runs fprop, dgrad and wgrad through the C ABI under torch.profiler and asserts that the instances it lists were
launched, so a case keeps testing the path it was written for whatever the test order.  Branches of the shared-memory
plans that do not show in kernel names (resident / streamed weights, operand-ring `group`, wgrad strip width `nbw`,
row splits, tap passes) are named in the comment of the case that reaches them.

Reference: F.conv2d / torch.nn.grad.* in float64 on the padded tile (zeros where the tile has no neighbour, the halo
strips where it has one), together with the same operation on |x|, |w|, |dy| ("A", the absolute sum).  Bounds, per
element (the inputs are bf16-representable, so only the fp32 summation and the final rounding differ):
    y, dx (bf16)       |got - ref| <= 2^-8 |ref| + 2^-12 A
    dw, db (fp32)      |got - ref| <= 2^-12 A           (straight from spc_conv2d_wgrad, not rounded by autograd)
tests/test_tc_coverage_bounds.py checks on the CPU that these bounds reject a dropped channel, a dropped pixel row
and a dropped tap at the table's shapes, and tests/test_tc_coverage_bounds.py::test_instance_table_matches_library
that the table names exactly the instances libspconv.so contains.  Run with -s to see the worst
err / bound of every case and, at the end, per kernel family.
"""
import collections
import ctypes as C
import math
import re
import zlib

import pytest
import torch
import torch.nn.functional as F

from mpi4dl_b200 import _lib
from oracle import spatial_oracle as so

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
REL_Y, ABS_Y, ABS_W = 2.0 ** -8, 2.0 ** -12, 2.0 ** -12


# ---- kernel names ------------------------------------------------------------------------------------------------
def parse_kernel(sig):
    """'void spc::(anonymous namespace)::conv_tap_kernel<2, 7, 3>(CUtensorMap, ...)' -> ('conv_tap_kernel', ('2', '7', '3'))"""
    s = sig.replace("(anonymous namespace)", "anon").split("(", 1)[0].strip()
    if s.startswith("void "):
        s = s[5:]
    m = re.match(r"^(.*?)(?:<(.*)>)?$", s)
    args = tuple(a.strip() for a in m.group(2).split(",")) if m.group(2) else ()
    return m.group(1).split("::")[-1], args


def K(*sigs):
    return frozenset(parse_kernel(s) for s in sigs)


# ---- the case table ----------------------------------------------------------------------------------------------
# KS of conv_tap = cbox / 16, cbox = 64 if the reduction has >= 64 channels else round_up(channels, 16): fprop reduces
# over C, dgrad over K.  QC of wgrad_tap = round_up(min(K, C), 16); mode A if K >= C.  The plan branches named below
# were checked against plan_tap / plan_passes / run_wgrad_tap's host planning.
Case = collections.namedtuple("Case", "C K R S stride N H W bias launches note")
CASES = [
    # ---- S = 1 (R x 1 filters): conv_tap<2, 1, KS>; wgrad on pw_wgrad_kernel (row-shifted boxes, no copies)
    Case(13, 29, 7, 1, 1, 2, 9, 64, True,
         K("conv_tap_kernel<2, 1, 1>", "conv_tap_kernel<2, 1, 2>", "pw_wgrad_kernel<16, 8>", "repack_weights_kernel"),
         "odd H (last 2-row tile half outside); resident weights; wgrad 7 taps on 8 accumulators (one spare)"),
    Case(136, 136, 3, 1, 1, 1, 4, 64, False, K("pw_gemm_kernel<2>", "pw_wgrad_kernel<128, 2>"),
         "M = 136 > 128 both ways: fprop and dgrad on pw_gemm_kernel in tap mode (row-shifted boxes, no copies)"),
    Case(45, 61, 5, 1, 1, 2, 12, 128, False,
         K("conv_tap_kernel<2, 1, 3>", "conv_tap_kernel<2, 1, 4>", "pw_wgrad_kernel<64, 4>"),
         "wgrad TG=4: passes of 4 + 1 taps (3 spare)"),
    Case(128, 104, 7, 1, 1, 1, 10, 64, False,
         K("conv_tap_kernel<2, 1, 4>", "pw_wgrad_kernel<128, 2>"),
         "streamed weights (fprop ast=5, dgrad ast=4), 2 k-chunks, dgrad's second chunk partial (40 of 64); "
         "wgrad NBLK=128: passes of 2 taps, last 1"),
    # ---- S = 3
    Case(13, 29, 3, 3, 1, 2, 11, 64, True,
         K("conv_tap_kernel<2, 3, 1>", "conv_tap_kernel<2, 3, 2>", "wgrad_tap_kernel<3, 16>"),
         "group=1 operand ring; wgrad mode A, QC=16: passes of 2 rows + 1 row on 8 accumulators"),
    Case(45, 29, 3, 3, 1, 1, 9, 256, False,
         K("conv_tap_kernel<2, 3, 3>", "conv_tap_kernel<2, 3, 2>", "wgrad_tap_kernel<3, 32>"),
         "wgrad mode B, nbw=2, 3 one-row passes of 3 taps (1 spare each)"),
    Case(45, 61, 1, 3, 1, 2, 5, 192, False,
         K("conv_tap_kernel<2, 3, 3>", "conv_tap_kernel<2, 3, 4>", "wgrad_tap_kernel<3, 48>"),
         "W = 3 x 64; wgrad column passes 2 + 1 (1 spare)"),
    Case(128, 61, 1, 3, 1, 2, 4, 64, True,
         K("conv_tap_kernel<2, 3, 4>", "wgrad_tap_kernel<3, 64>"),
         "fprop 2 k-chunks; wgrad mode B, column passes 2 + 1"),
    Case(77, 93, 1, 3, 1, 2, 3, 64, False, K("wgrad_tap_kernel<3, 80>"), "fprop group=0, dgrad group=1"),
    Case(128, 93, 1, 3, 1, 2, 3, 64, False, K("wgrad_tap_kernel<3, 96>"), "wgrad mode B, one tap per pass"),
    Case(109, 128, 1, 3, 1, 2, 3, 64, False, K("wgrad_tap_kernel<3, 112>"), "M = 128 fprop"),
    Case(128, 128, 1, 3, 1, 2, 3, 64, True, K("conv_tap_kernel<2, 3, 4>", "wgrad_tap_kernel<3, 128>"), ""),
    Case(8, 3, 3, 3, 1, 2, 10, 128, True,
         K("conv_tap_kernel<2, 3, 1>", "wgrad_tap_kernel<3, 16>"),
         "M = 3 fprop, M = 8 dgrad; wgrad mode B, nbw=2"),
    Case(13, 200, 3, 3, 1, 2, 7, 64, False,
         K("shift_copies_vec_kernel<3, 1>", "pw_gemm_kernel<2>", "conv_tap_kernel<2, 3, 4>", "pw_wgrad_kernel<16, 16>"),
         "M = 200 > 128: fprop on shifted copies; dgrad 4 k-chunks, the last 8 of 64 channels; "
         "wgrad K > 128: copies + NA=16 with 9 taps (7 spare)"),
    Case(136, 136, 3, 3, 1, 1, 4, 64, False,
         K("shift_copies_vec_kernel<3, 1>", "pw_gemm_kernel<2>", "pw_wgrad_kernel<128, 2>"),
         "136 channels both ways: every op on shifted copies; wgrad passes of 2 taps (last 1)"),
    # ---- S = 5
    Case(29, 13, 5, 5, 1, 2, 7, 64, True,
         K("conv_tap_kernel<2, 5, 2>", "conv_tap_kernel<2, 5, 1>", "wgrad_tap_kernel<5, 16>"),
         "wgrad mode B, QC=16: 5 one-row passes of 5 taps (3 spare each)"),
    Case(29, 45, 1, 5, 1, 2, 5, 128, False,
         K("conv_tap_kernel<2, 5, 2>", "conv_tap_kernel<2, 5, 3>", "wgrad_tap_kernel<5, 32>"),
         "wgrad nbw=2, column passes 3 + 2"),
    Case(61, 45, 1, 5, 1, 2, 4, 64, False,
         K("conv_tap_kernel<2, 5, 4>", "conv_tap_kernel<2, 5, 3>", "wgrad_tap_kernel<5, 48>"),
         "fprop group=0; wgrad mode B, column passes 2 + 2 + 1"),
    Case(61, 77, 1, 5, 1, 2, 3, 64, False, K("wgrad_tap_kernel<5, 64>"), "dgrad 2 k-chunks (77)"),
    Case(128, 77, 1, 5, 1, 2, 3, 64, False, K("wgrad_tap_kernel<5, 80>"), "dgrad streamed weights (ast=7)"),
    Case(93, 109, 1, 5, 1, 2, 3, 64, False, K("wgrad_tap_kernel<5, 96>"), "fprop streamed weights (ast=8)"),
    Case(109, 128, 1, 5, 1, 2, 3, 64, False, K("wgrad_tap_kernel<5, 112>"), "streamed weights both ways"),
    Case(128, 128, 1, 5, 1, 2, 3, 64, False, K("wgrad_tap_kernel<5, 128>"), ""),
    Case(13, 16, 1, 5, 1, 1, 6, 512, True,
         K("conv_tap_kernel<2, 5, 1>", "wgrad_tap_kernel<5, 16>"), "wgrad nbw=4 (W = 512)"),
    Case(29, 45, 5, 5, 1, 2, 7, 64, False,
         K("conv_tap_kernel<2, 5, 2>", "conv_tap_kernel<2, 5, 3>", "shift_copies_vec_kernel<5, 2>",
           "pw_wgrad_kernel<32, 8>"),
         "fprop streamed weights with group=1; 5x5 at QC=32 has no wgrad_tap plan: copies + 25 taps in passes of 8 "
         "(last 1)"),
    Case(136, 136, 1, 5, 1, 1, 3, 64, False,
         K("shift_copies_vec_kernel<5, 2>", "pw_gemm_kernel<2>", "pw_wgrad_kernel<128, 2>"),
         "136 channels both ways: every op on shifted copies"),
    # ---- S = 7
    Case(29, 13, 3, 7, 1, 2, 7, 64, False,
         K("conv_tap_kernel<2, 7, 2>", "conv_tap_kernel<2, 7, 1>", "wgrad_tap_kernel<7, 16>"),
         "wgrad mode B, 3 one-row passes of 7 taps (1 spare each)"),
    Case(45, 29, 1, 7, 1, 1, 37, 64, False,
         K("conv_tap_kernel<2, 7, 3>", "conv_tap_kernel<2, 7, 2>", "wgrad_tap_kernel<7, 32>"),
         "wgrad 4 row splits of 10 rows, the last 7; column passes 4 + 3"),
    Case(45, 61, 1, 7, 1, 2, 5, 64, True,
         K("conv_tap_kernel<2, 7, 3>", "conv_tap_kernel<2, 7, 4>", "wgrad_tap_kernel<7, 48>"),
         "wgrad column passes 2 + 2 + 2 + 1"),
    Case(128, 61, 1, 7, 1, 2, 3, 64, False,
         K("conv_tap_kernel<2, 7, 4>", "wgrad_tap_kernel<7, 64>"), "wgrad mode B, passes 2 + 2 + 2 + 1"),
    Case(77, 93, 1, 7, 1, 2, 3, 64, False, K("wgrad_tap_kernel<7, 80>"), "streamed weights both ways"),
    Case(128, 93, 1, 7, 1, 2, 3, 64, False, K("wgrad_tap_kernel<7, 96>"), ""),
    Case(109, 128, 1, 7, 1, 2, 3, 64, False, K("wgrad_tap_kernel<7, 112>"), ""),
    Case(128, 128, 1, 7, 1, 2, 3, 64, False, K("wgrad_tap_kernel<7, 128>"), ""),
    Case(128, 128, 3, 7, 1, 1, 5, 64, False,
         K("conv_tap_kernel<2, 7, 4>", "shift_copies_vec_kernel<7, 3>", "pw_wgrad_kernel<128, 2>"),
         "21 taps x 2 k-chunks: streamed weights; no wgrad_tap plan: copies + passes of 2 taps (last 1)"),
    Case(136, 136, 1, 7, 1, 1, 3, 64, False,
         K("shift_copies_vec_kernel<7, 3>", "pw_gemm_kernel<2>", "pw_wgrad_kernel<128, 2>"),
         "136 channels both ways: every op on shifted copies"),
    # ---- 1x1: pw_gemm_kernel<MB>, pw_wgrad_kernel<NBLK, MG>
    Case(13, 13, 1, 1, 1, 2, 8, 24, True, K("pw_gemm_kernel<1>", "pw_wgrad_kernel<16, 1>"),
         "P = 192: last 128-pixel tile partial"),
    Case(13, 200, 1, 1, 1, 2, 8, 24, False, K("pw_gemm_kernel<2>", "pw_gemm_kernel<1>", "pw_wgrad_kernel<16, 2>"),
         "M = 200: MB=2, rows 200..255 of the second block empty"),
    Case(13, 416, 1, 1, 1, 1, 8, 16, False, K("pw_gemm_kernel<2>", "pw_wgrad_kernel<16, 4>"),
         "M = 416: num_mg = 2; dgrad 7 k-chunks, the last half"),
    Case(29, 100, 1, 1, 1, 2, 6, 20, True, K("pw_wgrad_kernel<32, 1>"), ""),
    Case(29, 200, 1, 1, 1, 2, 6, 20, False, K("pw_wgrad_kernel<32, 2>"), ""),
    Case(29, 416, 1, 1, 1, 2, 6, 20, False, K("pw_wgrad_kernel<32, 4>"), "wgrad 4 blocks of 104 rows"),
    Case(45, 100, 1, 1, 1, 2, 6, 20, False, K("pw_wgrad_kernel<64, 1>"), ""),
    Case(45, 200, 1, 1, 1, 2, 6, 20, False, K("pw_wgrad_kernel<64, 2>"), ""),
    Case(61, 416, 1, 1, 1, 1, 6, 20, False, K("pw_wgrad_kernel<64, 4>"), ""),
    Case(104, 100, 1, 1, 1, 2, 6, 20, False, K("pw_wgrad_kernel<128, 1>"), ""),
    # ---- stride 2
    Case(104, 200, 1, 1, 2, 2, 16, 64, True,
         K("subsample2_kernel", "upsample2_zero_kernel", "pw_gemm_kernel<2>", "pw_gemm_kernel<1>",
           "pw_wgrad_kernel<128, 2>"), "1x1 stride 2"),
    Case(29, 45, 3, 3, 2, 2, 10, 128, False,
         K("shift_copies_s2k3_kernel", "repack_dgrad_s2_kernel", "shift_copies_vec_kernel<2, 0>",
           "interleave_s2_kernel", "pw_gemm_kernel<1>", "pw_wgrad_kernel<32, 8>"),
         "Ho = 5 odd; dgrad = 2x2-tap conv over 4 parity classes; wgrad passes of 8 taps + 1"),
    Case(13, 29, 5, 5, 2, 1, 12, 128, True, K("shift_copies_kernel", "pw_gemm_kernel<1>", "pw_wgrad_kernel<16, 16>"),
         "generic subsampled copies; dgrad on the direct kernel"),
    Case(45, 61, 1, 7, 2, 1, 6, 256, False, K("shift_copies_kernel", "pw_gemm_kernel<1>", "pw_wgrad_kernel<64, 4>"),
         "generic subsampled copies; dgrad on the direct kernel"),
]

# what the bf16 halo fix-up launches (test_halo_masks): im2col of the boundary outputs + one pointwise GEMM
FIXUP_FWD = K("halo_im2col_kernel", "boundary_scatter_kernel")
FIXUP_WGRAD = K("halo_im2col_kernel", "boundary_gather_kernel")


def table_instances():
    out = set()
    for c in CASES:
        out |= c.launches
    return out | FIXUP_FWD | FIXUP_WGRAD


def shifted_copy_only(c):
    """stride-1 multi-tap rows with more than 128 channels on both sides: conv_tap_kernel and wgrad_tap_kernel take at
    most 128, so fprop, dgrad and wgrad all run on pw_gemm_kernel / pw_wgrad_kernel (over shifted copies when S > 1)"""
    return c.stride == 1 and c.R * c.S > 1 and min(c.C, c.K) > 128


def case_id(c):
    return "%dto%d-%dx%d-s%d-n%d-%dx%d%s" % (c.C, c.K, c.R, c.S, c.stride, c.N, c.H, c.W, "-b" if c.bias else "")


def _find(C_, K_, R, S, stride=1):
    return next(c for c in CASES if (c.C, c.K, c.R, c.S, c.stride) == (C_, K_, R, S, stride))


# a 3x3, a 1x7, a 7x1, a 5x5 and a 3x3 stride-2 layer: run under every neighbour mask of a 3x3 grid and of 3-way
# horizontal / vertical slicing
MASK_CASES = [_find(13, 29, 3, 3), _find(45, 61, 1, 7), _find(13, 29, 7, 1), _find(29, 13, 5, 5), _find(29, 45, 3, 3, 2)]
GRIDS = [("square", 9), ("horizontal", 3), ("vertical", 3)]


# ---- inputs, reference, bound ------------------------------------------------------------------------------------
def out_hw(c):
    ph, pw = (c.R - 1) // 2, (c.S - 1) // 2
    return (c.H + 2 * ph - c.R) // c.stride + 1, (c.W + 2 * pw - c.S) // c.stride + 1


def make_inputs(c, mask, salt=0):
    """bf16 tensors (CPU) for one tile: x, w, b, dy and the halo strips the mask asks for."""
    g = torch.Generator().manual_seed(zlib.crc32(repr((tuple(c[:9]), tuple(mask), salt)).encode()))
    ph, pw = (c.R - 1) // 2, (c.S - 1) // 2
    x = torch.randn((c.N, c.C, c.H, c.W), generator=g).bfloat16()
    w = (torch.randn((c.K, c.C, c.R, c.S), generator=g) / math.sqrt(c.C * c.R * c.S)).bfloat16()
    b = torch.randn((c.K,), generator=g).bfloat16() if c.bias else None
    strips = [None] * 9
    for i, (dr, dc) in enumerate(so.DIRS):
        rows, cols = (ph if dr else c.H), (pw if dc else c.W)
        if i != 4 and mask[i] and rows and cols:
            strips[i] = torch.randn((c.N, c.C, rows, cols), generator=g).bfloat16()
    Ho, Wo = out_hw(c)
    dy = torch.randn((c.N, c.K, Ho, Wo), generator=g).bfloat16()
    return x, w, b, dy, strips


def padded(x, strips, ph, pw):
    """the tile with its halo ring: the strips where the tile has a neighbour, zeros elsewhere (float64)"""
    N, Cc, H, W = x.shape
    xp = torch.zeros((N, Cc, H + 2 * ph, W + 2 * pw), dtype=torch.float64, device=x.device)
    xp[:, :, ph:ph + H, pw:pw + W] = x.double()
    rows = [(0, ph), (ph, ph + H), (ph + H, H + 2 * ph)]
    cols = [(0, pw), (pw, pw + W), (pw + W, W + 2 * pw)]
    for i, s in enumerate(strips):
        if s is not None:
            (r0, r1), (c0, c1) = rows[i // 3], cols[i % 3]
            xp[:, :, r0:r1, c0:c1] = s.double()
    return xp


def reference(x, w, b, dy, strips, stride):
    """fp64 conv / dgrad / wgrad / bias grad of one tile, and the same on absolute values (the bound's A)."""
    R, S = w.shape[2:]
    ph, pw = (R - 1) // 2, (S - 1) // 2
    H, W = x.shape[2:]
    xp = padded(x, strips, ph, pw)
    wd, gd = w.double(), dy.double()
    bd = b.double() if b is not None else None
    st = (stride, stride)

    def ops(xp_, w_, b_, g_):
        return {
            "y": F.conv2d(xp_, w_, b_, st),
            "dx": torch.nn.grad.conv2d_input(xp_.shape, w_, g_, st)[:, :, ph:ph + H, pw:pw + W],
            "dw": torch.nn.grad.conv2d_weight(xp_, w_.shape, g_, st),
            "db": g_.sum((0, 2, 3)),
        }

    ref = ops(xp, wd, bd, gd)
    A = ops(xp.abs(), wd.abs(), bd.abs() if bd is not None else None, gd.abs())
    return ref, A


def check(got, ref, A, rel, absk, name):
    """per element |got - ref| <= rel |ref| + absk A; returns the worst err / bound"""
    got, ref, A = got.double(), ref.double().to(got.device), A.double().to(got.device)
    assert got.shape == ref.shape, (name, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    bound = rel * ref.abs() + absk * A
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if worst > 1.0:
        bad = int((ratio > 1).sum())
        i = int(ratio.argmax())
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
        raise AssertionError("%s: %d of %d elements out of bound, worst err/bound %.3g at %s (got %.6g, ref %.6g, A %.6g)"
                             % (name, bad, ratio.numel(), worst, idx, float(got[idx]), float(ref[idx]), float(A[idx])))
    return worst


def check_act(got, ref, A, name):
    return check(got, ref, A, REL_Y, ABS_Y, name)


def check_grad(got, ref, A, name):
    return check(got, ref, A, 0.0, ABS_W, name)


# ---- running the ops through the C ABI ---------------------------------------------------------------------------
def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def desc(c, N=None, dtype=_lib.SPC_BF16, algo=_lib.SPC_ALGO_AUTO):
    return _lib.ConvDesc(c.N if N is None else N, c.C, c.H, c.W, c.K, c.R, c.S, c.stride, c.stride, (c.R - 1) // 2,
                         (c.S - 1) // 2, dtype, algo)


def _ws(d, op):
    n = _lib.lib().spc_conv_workspace_bytes(C.byref(d), op)
    return torch.empty(max(n, 16), dtype=torch.uint8, device=DEV), n


def run_fwd(d, x, strips, w, b, split=False):
    L = _lib.lib()
    Ho, Wo = C.c_int(), C.c_int()
    L.spc_conv_out_shape(C.byref(d), C.byref(Ho), C.byref(Wo))
    y = torch.empty((d.N, d.K, Ho.value, Wo.value), dtype=torch.bfloat16, device=DEV)
    ws, n = _ws(d, 0)
    halo = _lib.make_halo(strips)
    if split:   # the trainer's overlap schedule: interior pass while the exchange runs, then the boundary fix-up
        _lib.check(L.spc_conv2d_fwd_interior(C.byref(d), _ptr(x), _ptr(w), _ptr(b), _ptr(y), _ptr(ws), n, _st()), "fwd_interior")
        _lib.check(L.spc_conv2d_fwd_boundary(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), _st()),
                   "fwd_boundary")
    else:
        _lib.check(L.spc_conv2d_fwd(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), _ptr(ws), n, _st()), "fwd")
    return y


def run_dgrad(d, dy, w):
    dx = torch.empty((d.N, d.C, d.H, d.W), dtype=torch.bfloat16, device=DEV)
    ws, n = _ws(d, 1)
    _lib.check(_lib.lib().spc_conv2d_dgrad(C.byref(d), _ptr(dy), _ptr(w), _ptr(dx), _ptr(ws), n, _st()), "dgrad")
    return dx


def run_wgrad(d, x, strips, dy, dw, db, accumulate):
    ws, n = _ws(d, 2)
    halo = _lib.make_halo(strips)
    _lib.check(_lib.lib().spc_conv2d_wgrad(C.byref(d), _ptr(x), C.byref(halo), _ptr(dy), C.c_void_p(dw.data_ptr()),
                                           _ptr(db), accumulate, _ptr(ws), n, _st()), "wgrad")
    return dw, db


def traced(fn):
    """run fn under the CUDA profiler; returns (result, {(kernel name, template args)}).  In a long-lived process the
    profiler has lost the records of the first launches of a session, so a throw-away kernel goes first; every op
    launches kernels, so an empty trace is retried."""
    for _ in range(3):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device=DEV).add_(1)
            torch.cuda.synchronize()
            out = fn()
            torch.cuda.synchronize()
        names = set()
        for e in prof.profiler.kineto_results.events():
            if e.device_type() == torch.autograd.DeviceType.CUDA and "spc::" in e.name():
                names.add(parse_kernel(e.name()))
        if names:
            break
    return out, names


FAMILIES = ("conv_tap_kernel", "wgrad_tap_kernel", "pw_gemm_kernel", "pw_wgrad_kernel", "conv_direct_kernel",
            "wgrad_direct_kernel")
WORST = collections.defaultdict(float)


def _record(tag, op, kernels, ratio):
    fams = sorted({n for n, _ in kernels if n in FAMILIES})
    for f in fams:
        WORST[(f, op)] = max(WORST[(f, op)], ratio)
    print("[tc-coverage] %-44s %-6s err/bound %.3f  %s" % (tag, op, ratio, "+".join(fams)))


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if WORST:
        print("\n[tc-coverage] largest err/bound per kernel family and op:")
        for (f, op), r in sorted(WORST.items()):
            print("[tc-coverage]   %-20s %-6s %.3f" % (f, op, r))


def _to_dev(*ts):
    return [t.to(DEV) if t is not None else None for t in ts]


def run_and_check(c, mask, tag, split_check=False):
    """all four results of one tile against the fp64 reference; returns the kernels each op launched"""
    L = _lib.lib()
    x, w, b, dy, strips = make_inputs(c, mask)
    x, w, b, dy = _to_dev(x, w, b, dy)
    strips = _to_dev(*strips)
    ref, A = reference(x, w, b, dy, strips, c.stride)
    d = desc(c)
    assert L.spc_conv_uses_tcgen05(C.byref(d), 0) and L.spc_conv_uses_tcgen05(C.byref(d), 2), "left the wgmma path"
    dgrad_direct = c.stride == 2 and c.R * c.S > 1 and (c.R, c.S) != (3, 3)
    assert L.spc_conv_uses_tcgen05(C.byref(d), 1) == (not dgrad_direct)
    y, kf = traced(lambda: run_fwd(d, x, strips, w, b))
    _record(tag, "y", kf, check_act(y, ref["y"], A["y"], tag + " y"))
    if split_check:
        y2 = run_fwd(d, x, strips, w, b, split=True)
        assert torch.equal(y2, y), tag + ": fwd_interior + fwd_boundary differs from fwd"
    dx, kd = traced(lambda: run_dgrad(d, dy, w))
    _record(tag, "dx", kd, check_act(dx, ref["dx"], A["dx"], tag + " dx"))
    dw = torch.full(w.shape, float("nan"), dtype=torch.float32, device=DEV)
    db = torch.full((c.K,), float("nan"), dtype=torch.float32, device=DEV) if c.bias else None
    _, kw = traced(lambda: run_wgrad(d, x, strips, dy, dw, db, 0))
    _record(tag, "dw", kw, check_grad(dw, ref["dw"], A["dw"], tag + " dw"))
    if c.bias:
        check_grad(db, ref["db"], A["db"], tag + " db")

    def retrace():
        return traced(lambda: (run_fwd(d, x, strips, w, b), run_dgrad(d, dy, w),
                               run_wgrad(d, x, strips, dy, torch.empty_like(dw), torch.empty_like(db) if c.bias else None, 0)))[1]
    return kf, kd, kw, (d, x, strips, dy, w, ref, A, retrace)


def launched(kernels, pred, retrace):
    """pred(launched kernels).  A trace is a lower bound of what ran (records can be lost, see traced): if pred does not
    hold, the ops are traced again and their kernels added"""
    k = set(kernels)
    for _ in range(2):
        if pred(k):
            return True
        k |= retrace()
    return pred(k)


def _names(kernels):
    return {n for n, _ in kernels}


# ---- tests -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_case_against_fp64(c):
    kf, kd, kw, (d, x, strips, dy, w, ref, A, retrace) = run_and_check(c, [0] * 9, case_id(c))
    assert launched(kf | kd | kw, lambda k: c.launches <= k, retrace), \
        "%s did not launch %s (launched: %s)" % (case_id(c), sorted(c.launches - (kf | kd | kw)), sorted(kf | kd | kw))
    if shifted_copy_only(c):
        assert not {"conv_tap_kernel", "wgrad_tap_kernel"} & _names(kf | kd | kw), sorted(kf | kd | kw)
    # accumulate=1 adds onto what dw / db hold
    g = torch.Generator(device=DEV).manual_seed(7)
    dw0 = torch.randn(w.shape, generator=g, device=DEV) * float(ref["dw"].abs().mean())
    dw = dw0.clone()
    db0 = torch.randn((c.K,), generator=g, device=DEV) * float(ref["db"].abs().mean()) if c.bias else None
    db = db0.clone() if c.bias else None
    run_wgrad(d, x, strips, dy, dw, db, 1)
    check_grad(dw, dw0.double() + ref["dw"], A["dw"], case_id(c) + " dw accumulate")
    if c.bias:
        check_grad(db, db0.double() + ref["db"], A["db"], case_id(c) + " db accumulate")


def _fixup_expected(c, mask):
    """whether the boundary pass has outputs to redo: a side with a strip whose halo some output window reads (with
    stride 2 on an even tile, no window reaches the bottom / right halo)"""
    ph, pw = (c.R - 1) // 2, (c.S - 1) // 2
    Ho, Wo = out_hw(c)
    reads = {"top": ph > 0, "bottom": (Ho - 1) * c.stride - ph + c.R > c.H,
             "left": pw > 0, "right": (Wo - 1) * c.stride - pw + c.S > c.W}
    sides = {"top": (0, 1, 2), "bottom": (6, 7, 8), "left": (0, 3, 6), "right": (2, 5, 8)}
    return any(reads[s] and any(mask[i] for i in idx) for s, idx in sides.items())


def _masks(c, method, P):
    out = []
    for r in range(P):
        m = so.neighbour_mask(method, P, r, c.R, c.S)
        if m not in out:
            out.append(m)
    return out


# the fix-up paths of test_halo_masks: "fixup" is bf16 on the boundary GEMM (fprop and wgrad); the direct ones are
# spc_conv2d_fwd_interior + spc_conv2d_fwd_boundary with the direct kernel on the boundary rectangles, which fp32 and
# SPC_ALGO_DIRECT use (the overlapped forward of conv_spatial in fp32)
DIRECT_PATHS = {"direct_fp32": (torch.float32, _lib.SPC_F32, _lib.SPC_ALGO_AUTO),
                "direct_bf16": (torch.bfloat16, _lib.SPC_BF16, _lib.SPC_ALGO_DIRECT)}


def run_boundary_direct(c, mask, tag, dtype, spc_dtype, algo):
    """interior pass, then the boundary pass; y against the fp64 reference.  Returns the kernels the boundary pass
    launched and a function that traces it again"""
    L = _lib.lib()
    x, w, b, dy, strips = make_inputs(c, mask)
    ref, A = reference(x, w, b, dy, strips, c.stride)
    x, w, b, *strips = [t.to(DEV, dtype) if t is not None else None for t in (x, w, b, *strips)]
    d = desc(c, dtype=spc_dtype, algo=algo)
    assert not L.spc_conv_uses_tcgen05(C.byref(d), 0), tag
    y = torch.empty((c.N, c.K) + out_hw(c), dtype=dtype, device=DEV)
    _lib.check(L.spc_conv2d_fwd_interior(C.byref(d), _ptr(x), _ptr(w), _ptr(b), _ptr(y), None, 0, _st()), "fwd_interior")
    halo = _lib.make_halo(strips)

    def boundary():
        _lib.check(L.spc_conv2d_fwd_boundary(C.byref(d), _ptr(x), C.byref(halo), _ptr(w), _ptr(b), _ptr(y), _st()),
                   "fwd_boundary")

    _, k = traced(boundary)
    _record(tag, "y", k, check_act(y, ref["y"], A["y"], tag + " y"))
    return k, lambda: traced(boundary)[1]


def run_wgrad_direct(c, mask, tag):
    """fp32 wgrad on the direct kernel, which reads the strips in place; dw, db against the fp64 reference with the
    always-valid bound of an fp32 sum of N Ho Wo exact products: gamma(N Ho Wo + 1) A, u = 2^-24"""
    x, w, b, dy, strips = make_inputs(c, mask)
    ref, A = reference(x, w, b, dy, strips, c.stride)
    x, w, dy, *strips = [t.to(DEV, torch.float32) if t is not None else None for t in (x, w, dy, *strips)]
    d = desc(c, dtype=_lib.SPC_F32)
    assert not _lib.lib().spc_conv_uses_tcgen05(C.byref(d), 2), tag
    Ho, Wo = out_hw(c)
    n = c.N * Ho * Wo + 1
    gam = n * 2.0 ** -24 / (1 - n * 2.0 ** -24)
    dw = torch.full(w.shape, float("nan"), device=DEV)
    db = torch.full((c.K,), float("nan"), device=DEV) if c.bias else None
    _, k = traced(lambda: run_wgrad(d, x, strips, dy, dw, db, 0))
    _record(tag, "dw", k, check(dw, ref["dw"], A["dw"], 0.0, gam, tag + " dw"))
    if c.bias:
        check(db, ref["db"], A["db"], 0.0, gam, tag + " db")
    return k, lambda: traced(lambda: run_wgrad(d, x, strips, dy, dw, db, 0))[1]


@pytest.mark.parametrize("path", ["fixup"] + list(DIRECT_PATHS) + ["wgrad_direct_fp32"])
@pytest.mark.parametrize("grid", GRIDS, ids=[g[0] for g in GRIDS])
@pytest.mark.parametrize("c", MASK_CASES, ids=case_id)
def test_halo_masks(c, grid, path):
    """corner, edge and interior tiles of a 3x3 grid and the end / middle tiles of 3-way slicing: the bf16 halo
    fix-up on the boundary GEMM, the forward fix-up on the direct kernel (fp32, bf16 with SPC_ALGO_DIRECT), and the fp32
    wgrad on the direct kernel"""
    method, P = grid
    for mask in _masks(c, method, P):
        tag = "%s %s%s %s" % (case_id(c), method, "".join(map(str, mask)), path)
        fix = _fixup_expected(c, mask)
        if path == "wgrad_direct_fp32":
            k, retrace = run_wgrad_direct(c, mask, tag)
            assert launched(k, lambda k: "wgrad_direct_kernel" in _names(k), retrace), (tag, sorted(k))
        elif path == "fixup":
            kf, kd, kw, rest = run_and_check(c, mask, tag, split_check=True)
            k = kf | kd | kw
            assert launched(k, lambda k: FIXUP_FWD | FIXUP_WGRAD <= k, rest[-1]) == fix, (tag, fix, sorted(k))
        else:
            k, retrace = run_boundary_direct(c, mask, tag, *DIRECT_PATHS[path])
            assert launched(k, lambda k: "conv_direct_kernel" in _names(k), retrace) == fix, (tag, fix, sorted(k))
            assert "halo_im2col_kernel" not in _names(k), (tag, sorted(k))


def test_wgrad_empty_batch_accumulate():
    """N == 0: accumulate=1 leaves dw / db as they are, accumulate=0 zeroes them"""
    for c in (_find(13, 29, 3, 3), _find(13, 13, 1, 1), _find(29, 45, 3, 3, 2)):
        d = desc(c, N=0)
        dw0 = torch.randn((c.K, c.C, c.R, c.S), device=DEV)
        db0 = torch.randn((c.K,), device=DEV)
        dw, db = dw0.clone(), db0.clone()
        run_wgrad(d, None, [None] * 9, None, dw, db, 1)
        torch.cuda.synchronize()
        assert torch.equal(dw, dw0) and torch.equal(db, db0), case_id(c)
        run_wgrad(d, None, [None] * 9, None, dw, db, 0)
        torch.cuda.synchronize()
        assert not dw.any() and not db.any(), case_id(c)
