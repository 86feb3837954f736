"""Fused training-mode BatchNorm2d + ReLU (csrc/bnrelu.cu, torchgems/fused.py) against fp64, per channel and per element.

The reference is computed in fp64 on the device from the STORED y (bf16 upcast where the dtype is bf16), one channel
at a time: mean and biased variance by two passes, rstd = 1 / sqrt(var + eps), xhat = (y - mean) rstd,
z = relu?(xhat gamma + beta), g = dz [mask], dsum = sum g, dsumx = sum g xhat, dx = gamma rstd (g - dsum/M - xhat dsumx/M).
u = 2^-24 is the fp32 unit roundoff, 2^-8 the bf16 one, M = N*H*W.

Statistics (spc_bn_stats).  A (plane, 16384-element chunk) item sums its values in a tree (6 levels per thread, 5 in
the warp, 3 across the CTA: a sum of n terms has error <= 14u sum|terms|), takes m = fl(sum / n), then sums d = y - m
(one rounding, relative to d) and d^2 in the same trees; mean_i = m + sum d / n and M2_i = sum d^2 - (sum d)^2 / n are
formed in fp64.  With |d| <= |y - mean| + |mean_i - mean| and |mean_i - mean| <= mean_i|y - mean|, the items' sum d
carry <= 15u * 2 sum|y - mean| of error in total, and the fp64 merge plus the final rounding to fp32 add u |mean|:
    |mean - mean64| <= 2^-23 |mean64| + 2^-19 mean|y - mean64|                 (30u <= 2^-19)
M2_i has <= 17u M2_i (d^2: 3u, tree: 14u); an item mean error e_i <= 30u mean_i|y - mean| enters
sum n_i (mean_i - mean)^2 as <= 60u n_i mean_i((y - mean)^2) (Cauchy-Schwarz); the rounding to fp32 adds u:
    |var - var64| <= 2^-16 var64 + 2^-30 mean(y^2)                            (78u <= 2^-16 = 256u)
The second term is there only for a constant channel (var64 = 0), where the item's residual cancellation is
<= u (15u mean|y|)^2 / 2^-30 relative.  Both are tighter than 2^-17 mean|y| and 2^-14 var64 + 2^-30 mean(y^2).

Backward sums (spc_bn_bwd_reduce).  g = dz or 0 is exact, xhat = fl(fl(y - mean) rstd) has <= 2u relative error,
g xhat one more u, the tree 14u, the fp64 merge and the rounding to fp32 u:
    |dsum - dsum64| <= 2^-19 sum|g|,   |dsumx - dsumx64| <= 2^-19 sum|g xhat|  (18u <= 2^-19 = 32u)

Per element, for the apply kernels with the library's own fp32 mean, rstd (and dsum, dsumx):
  z:  xhat 2u, xhat gamma u, + beta u (<= 4u, fewer with an FMA):  |z - z64| <= 4u A_z,  A_z = |xhat gamma| + |beta|.
      Bound 2^-21 A_z (8u); bf16 storage adds 2^-8 |z|:  (2^-8 + 2^-20) A_z.  relu is 1-Lipschitz.
  dx: 1/M 2u, a0 = dsum/M 3u, a1 = dsumx/M 3u, xhat a1 6u, two subtractions u each of their operands' magnitudes,
      gamma rstd u, the product u: <= 9u A_dx,  A_dx = |gamma| rstd (|g| + |dsum|/M + |xhat| |dsumx|/M).
      Bound 2^-20 A_dx (16u); bf16: (2^-8 + 2^-19) A_dx.

End to end (bn_relu), against the EXACT statistics: dm and dv are the statistics bounds above; rstd is
fl(rsqrt(fl(var + eps))) (rsqrtf: 2 ulp), so with t = dv / (var64 + eps), rstd / rstd64 - 1 is at most
rho = (1 - t)^-1/2 (1 + 2^-21) - 1.  xhat then moves by dxh = dm rstd64 (1 + rho) + |xhat64| rho, z by |gamma| dxh on top
of the kernel bound on the moved A_z; dsum by E_s = 2^-19 sum|g| and dsumx by E_x = sum|g| dxh + 2^-19 sum|g| (|xhat64|
+ dxh), and dx by |gamma| rstd64 [rho I + (1 + rho)(E_s/M + (dxh (|dsumx64| + E_x) + |xhat64| E_x)/M)] plus the kernel
bound on the moved A_dx (I = the exact |g| + |dsum64|/M + |xhat64| |dsumx64|/M).  dgamma = dsumx and dbeta = dsum
take the parameters' dtype (bf16: 2^-8 more).  The running buffers take the momentum update of those statistics in
their own dtype (a few roundings: 6 units of that dtype on the magnitudes).

The backward reference takes its ReLU mask from the kernel's forward decision (z_got > 0); separately, that mask may
differ from the fp64 one only where |xhat64 gamma + beta| is within the forward bound.  At the shapes with more than one
chunk per plane or more items than CTAs, every entry point and bn_relu forward + backward run three times and must be
bit-identical.  Run with -s to see the worst err / bound of every case.
"""
import collections
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest
import torch

from mpi4dl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
EPS = 1e-5
BN_CHUNK = 16384       # elements per (plane, chunk) work item (bnrelu.cu)
BN_GRID = 132 * 8      # CTAs of the streaming kernels
SUM_BOUND = 2.0 ** -19
Z_BOUND = {torch.float32: 2.0 ** -21, torch.bfloat16: 2.0 ** -8 + 2.0 ** -20}
DX_BOUND = {torch.float32: 2.0 ** -20, torch.bfloat16: 2.0 ** -8 + 2.0 ** -19}
UNIT = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8}


def mean_bound(mean64, mad):
    """mad = mean|y - mean64|"""
    return 2.0 ** -23 * abs(mean64) + 2.0 ** -19 * mad


def var_bound(var64, ms):
    """ms = mean(y^2)"""
    return 2.0 ** -16 * var64 + 2.0 ** -30 * ms


# ---- the case table ----------------------------------------------------------------------------------------------
Shape = collections.namedtuple("Shape", "N C H W note")
SHAPES = [
    Shape(3, 4, 2, 4, "H*W = 8, the minimum"),
    Shape(2, 3, 40, 72, "H*W = 2880: one partial chunk per plane"),
    Shape(1, 3, 256, 128, "H*W = 2 chunks exactly"),
    Shape(1, 2, 1000, 1000, "61 chunks and a partial one of 576"),
    Shape(2, 5, 2048, 2048, "2560 items on 1056 CTAs: the grid-stride loop wraps, planes map to channels over N = 2"),
    Shape(1, 1, 4096, 4096, "one plane of 1024 chunks"),
]


def _stage_shapes():
    """the BatchNorms of the stage at the N = 4 tile (half the image's extent): the stem's 104 channels at 2048^2 and
    every size of the 208- and 52-channel layers of the AmoebaNet-D layer list"""
    layers = json.load(open(os.path.join(ROOT, "tests", "golden", "layers_amoebanetd_sp4.json")))["layers"]
    out = {(104, 2048)}
    out |= {(l["K"], l["H"] // 2) for l in layers if l["op"] == "conv" and l["K"] in (52, 208)}
    return [Shape(1, c, h, h, "stage") for c, h in sorted(out)]


STAGE = _stage_shapes()
RATIOS = (0.2, 10.0, 100.0)     # |mean| / std of the data


def shape_id(s):
    return "%dx%dx%dx%d" % (s.N, s.C, s.H, s.W)


def multi_item(s):
    chunks = -(-s.H * s.W // BN_CHUNK)
    return chunks > 1 or s.N * s.C * chunks > BN_GRID


DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}
CASES = [pytest.param(s, dt, relu, r, id="%s-%s-%s-m%g" % (shape_id(s), dt, "relu" if relu else "bn", r))
         for s in SHAPES for dt in DTYPES for relu in (False, True) for r in RATIOS]
CASES += [pytest.param(s, "bf16", True, r, id="stage-%s-bf16-relu-m%g" % (shape_id(s), r)) for s in STAGE for r in (0.2, 100.0)]


def make_inputs(s, dtype, ratio, seed):
    """y: per channel std in [0.5, 2], mean = +-ratio * std; channel 0 is the constant 1.5 when C > 1 (a large
    constant would leave the end-to-end bound on rstd vacuous: 2^-30 mean(y^2) would reach eps).
    dz: standard normal.  Both stored in `dtype`."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    sig = torch.rand(s.C, device=DEV, generator=g) * 1.5 + 0.5
    sign = torch.where(torch.arange(s.C, device=DEV) % 2 == 0, 1.0, -1.0)
    mu = sign * ratio * sig
    if s.C > 1:
        sig[0], mu[0] = 0.0, 1.5
    y = torch.randn((s.N, s.C, s.H, s.W), device=DEV, generator=g)
    y = (y.mul_(sig.view(1, -1, 1, 1)).add_(mu.view(1, -1, 1, 1))).to(dtype)
    dz = torch.randn((s.N, s.C, s.H, s.W), device=DEV, generator=g).to(dtype)
    gamma = (torch.rand(s.C, device=DEV, generator=g) + 0.5) * torch.where(torch.rand(s.C, device=DEV, generator=g) < 0.2,
                                                                             -1.0, 1.0)
    beta = torch.rand(s.C, device=DEV, generator=g) - 0.5
    return y, dz, gamma, beta


def seed_of(*key):
    return zlib.crc32(repr(key).encode())


def ref_stats(yc):
    """fp64 two-pass statistics of one channel (any shape): mean, biased var, mean|y - mean|, mean(y^2)"""
    yd = yc.double()
    m = yd.mean()
    d = yd - m
    return float(m), float((d * d).mean()), float(d.abs().mean()), float((yd * yd).mean())


class Worst(dict):
    """worst err / bound per quantity; every check asserts err <= bound per element (NaN fails)"""

    def check(self, name, got, ref, bound):
        dev = next((t.device for t in (got, ref, bound) if torch.is_tensor(t) and t.dim() > 0), "cpu")
        got, ref, bound = (torch.as_tensor(t, dtype=torch.float64, device=dev) for t in (got, ref, bound))
        err = (got - ref).abs()
        ok = err <= bound
        r = float(torch.where(bound > 0, err / bound, torch.where(err > 0, float("inf"), 0.0)).max())
        self[name] = max(self.get(name, 0.0), r)
        if not bool(ok.all()):
            raise AssertionError("%s: %d of %d elements out of bound, worst err/bound %.3g"
                                 % (name, int((~ok).sum()), ok.numel(), r))

    def report(self, tag):
        print("[bn] %-44s %s" % (tag, "  ".join("%s %.3f" % kv for kv in self.items())))


# ---- the C ABI -----------------------------------------------------------------------------------------------------
def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dims(y):
    N, Cc, H, W = y.shape
    return N, Cc, H * W, _lib.dtype_code(y.dtype)


def _ws(N, Cc, HW):
    n = _lib.lib().spc_bn_workspace_bytes(N, Cc, HW)
    assert n > 0
    return torch.empty(n, dtype=torch.uint8, device=DEV), n


def run_stats(y):
    N, Cc, HW, code = _dims(y)
    mean, var = torch.empty(Cc, device=DEV), torch.empty(Cc, device=DEV)
    ws, n = _ws(N, Cc, HW)
    _lib.check(_lib.lib().spc_bn_stats(N, Cc, HW, code, _p(y), _p(mean), _p(var), _p(ws), n, _st()), "spc_bn_stats")
    return mean, var


def run_apply(y, mean, rstd, gamma, beta, relu):
    N, Cc, HW, code = _dims(y)
    z = torch.empty_like(y)
    _lib.check(_lib.lib().spc_bn_apply(N, Cc, HW, code, _p(y), _p(mean), _p(rstd), _p(gamma), _p(beta), int(relu), _p(z),
                                       _st()), "spc_bn_apply")
    return z


def run_bwd_reduce(dz, y, mean, rstd, gamma, beta, relu):
    N, Cc, HW, code = _dims(y)
    dsum, dsumx = torch.empty(Cc, device=DEV), torch.empty(Cc, device=DEV)
    ws, n = _ws(N, Cc, HW)
    _lib.check(_lib.lib().spc_bn_bwd_reduce(N, Cc, HW, code, _p(dz), _p(y), _p(mean), _p(rstd), _p(gamma), _p(beta),
                                            int(relu), _p(dsum), _p(dsumx), _p(ws), n, _st()), "spc_bn_bwd_reduce")
    return dsum, dsumx


def run_bwd_apply(dz, y, mean, rstd, gamma, beta, relu, dsum, dsumx):
    N, Cc, HW, code = _dims(y)
    dx = torch.empty_like(y)
    _lib.check(_lib.lib().spc_bn_bwd_apply(N, Cc, HW, code, _p(dz), _p(y), _p(mean), _p(rstd), _p(gamma), _p(beta),
                                           int(relu), _p(dsum), _p(dsumx), _p(dx), _st()), "spc_bn_bwd_apply")
    return dx


def _host(*ts):
    return [t.detach().double().cpu().tolist() for t in ts]


def _mask_check(w, name, z_got, pre, zb, relu):
    """the kernel's ReLU decision (z_got > 0) differs from the fp64 one (pre > 0) only where |pre| <= the z bound"""
    if relu:
        differ = (z_got > 0) != (pre > 0)
        w.check(name, torch.where(differ, pre.abs(), 0.0), 0.0, torch.where(differ, zb, 0.0))


# ---- CPU -----------------------------------------------------------------------------------------------------------
def test_bounds_detect_planted_errors():
    """at |mean| / std = 100 the statistics bounds reject a variance scaled by 1 + 2^-12 and a mean moved by 2^-14 std
    (the fp64 reference of fp32 data, numpy)"""
    rng = np.random.default_rng(5)
    for sig in (0.5, 1.0, 2.0):
        y = (100.0 * sig + sig * rng.standard_normal(1 << 16)).astype(np.float32).astype(np.float64)
        m = y.mean()
        d = y - m
        v, mad, ms = (d * d).mean(), np.abs(d).mean(), (y * y).mean()
        assert abs(v * (1 + 2.0 ** -12) - v) > var_bound(v, ms)
        assert 2.0 ** -14 * np.sqrt(v) > mean_bound(m, mad)
        assert 0.0 <= var_bound(v, ms) and 0.0 < mean_bound(m, mad)
    # and the bound still admits the final rounding of an exact result to fp32
    assert abs(float(np.float32(m)) - m) <= mean_bound(m, mad)
    assert abs(float(np.float32(v)) - v) <= var_bound(v, ms)


def test_workspace_bytes():
    L = _lib.lib()
    assert L.spc_bn_workspace_bytes(3, 4, 8) == 12 * 16
    assert L.spc_bn_workspace_bytes(1, 2, 1000 * 1000) == 2 * 62 * 16
    assert L.spc_bn_workspace_bytes(2, 5, 2048 * 2048) == 10 * 256 * 16
    for bad in ((0, 4, 8), (1, 0, 8), (1, 4, 0), (1, 4, 12)):
        assert L.spc_bn_workspace_bytes(*bad) == 0


def test_argument_validation_needs_no_gpu():
    """misaligned tensor pointers and a short workspace are SPC_EINVAL before anything is enqueued (fake pointers)"""
    L = _lib.lib()
    N, Cc, HW, f32 = 1, 2, 64, _lib.SPC_F32
    need = L.spc_bn_workspace_bytes(N, Cc, HW)
    A, V = 1 << 20, (1 << 20) + 64           # 16-byte aligned stand-ins for a tensor and a per-channel vector

    def P(x):
        return C.c_void_p(x)

    calls = {
        "stats": (lambda p: L.spc_bn_stats(N, Cc, HW, f32, P(p[0]), P(p[1]), P(p[2]), P(p[3]), need, None), 4,
                  (0, 3), (1, 2)),
        "apply": (lambda p: L.spc_bn_apply(N, Cc, HW, f32, P(p[0]), P(p[1]), P(p[2]), P(p[3]), P(p[4]), 1, P(p[5]),
                                           None), 6, (0, 5), (1, 2, 3, 4)),
        "bwd_reduce": (lambda p: L.spc_bn_bwd_reduce(N, Cc, HW, f32, P(p[0]), P(p[1]), P(p[2]), P(p[3]), P(p[4]), P(p[5]),
                                                     1, P(p[6]), P(p[7]), P(p[8]), need, None), 9, (0, 1, 8),
                       (2, 3, 4, 5, 6, 7)),
        "bwd_apply": (lambda p: L.spc_bn_bwd_apply(N, Cc, HW, f32, P(p[0]), P(p[1]), P(p[2]), P(p[3]), P(p[4]), P(p[5]),
                                                   1, P(p[6]), P(p[7]), P(p[8]), None), 9, (0, 1, 8), (2, 3, 4, 5, 6, 7)),
    }
    for name, (call, nargs, big, small) in calls.items():
        base = [A if i in big else V for i in range(nargs)]
        for i in big:
            for off in (4, 8):
                p = list(base)
                p[i] += off
                assert call(p) == -1, (name, i, off)
                assert b"aligned" in L.spc_last_error(), (name, i, off, L.spc_last_error())
        for i in small:
            p = list(base)
            p[i] += 2
            assert call(p) == -1, (name, i)
            assert b"aligned" in L.spc_last_error(), (name, i, L.spc_last_error())
    # a workspace one byte short
    assert L.spc_bn_stats(N, Cc, HW, f32, P(A), P(V), P(V + 64), P(A + 4096), need - 1, None) == -1
    assert b"workspace" in L.spc_last_error()
    assert L.spc_bn_bwd_reduce(N, Cc, HW, f32, P(A), P(A), P(V), P(V), P(V), P(V), 1, P(V), P(V), P(A + 4096), need - 1,
                               None) == -1
    assert b"workspace" in L.spc_last_error()
    assert L.spc_bn_stats(N, Cc, 12, f32, P(A), P(V), P(V), P(A), need, None) == -1   # H*W % 8


# ---- GPU: the entry points -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("s,dt,relu,ratio", CASES)
def test_kernels_against_fp64(s, dt, relu, ratio):
    dtype = DTYPES[dt]
    tag = "kernels %s %s %s m%g" % (shape_id(s), dt, "relu" if relu else "bn", ratio)
    y, dz, gamma, beta = make_inputs(s, dtype, ratio, seed_of(s[:4], dt, ratio))
    M = s.N * s.H * s.W
    w = Worst()
    mean, var = run_stats(y)
    rstd = torch.rsqrt(var + EPS)
    z = run_apply(y, mean, rstd, gamma, beta, relu)
    dsum, dsumx = run_bwd_reduce(dz, y, mean, rstd, gamma, beta, relu)
    dx = run_bwd_apply(dz, y, mean, rstd, gamma, beta, relu, dsum, dsumx)
    hm, hv, hr, hg, hb, hs, hx = _host(mean, var, rstd, gamma, beta, dsum, dsumx)
    zb, db = Z_BOUND[dtype], DX_BOUND[dtype]
    for c in range(s.C):
        yc = y[:, c]
        m64, v64, mad, ms = ref_stats(yc)
        w.check("mean", hm[c], m64, mean_bound(m64, mad))
        w.check("var", hv[c], v64, var_bound(v64, ms))
        xh = (yc.double() - hm[c]) * hr[c]
        pre = xh * hg[c] + hb[c]
        Az = (xh * hg[c]).abs_() + abs(hb[c])
        w.check("z", z[:, c], pre.clamp(min=0.0) if relu else pre, zb * Az)
        _mask_check(w, "mask", z[:, c], pre, zb * Az, relu)
        g = dz[:, c].double()
        if relu:
            g = torch.where(z[:, c] > 0, g, 0.0)
        gx = g * xh
        w.check("dsum", hs[c], float(g.sum()), SUM_BOUND * float(g.abs().sum()))
        w.check("dsumx", hx[c], float(gx.sum()), SUM_BOUND * float(gx.abs().sum()))
        dx64 = (g - hs[c] / M - xh * (hx[c] / M)) * (hg[c] * hr[c])
        Adx = (g.abs() + abs(hs[c]) / M + xh.abs() * (abs(hx[c]) / M)) * abs(hg[c] * hr[c])
        w.check("dx", dx[:, c], dx64, db * Adx)
    w.report(tag)
    if multi_item(s):
        for _ in range(2):
            m2, v2 = run_stats(y)
            assert torch.equal(m2, mean) and torch.equal(v2, var), tag + ": spc_bn_stats not reproducible"
            assert torch.equal(run_apply(y, mean, rstd, gamma, beta, relu), z), tag + ": spc_bn_apply not reproducible"
            s2, x2 = run_bwd_reduce(dz, y, mean, rstd, gamma, beta, relu)
            assert torch.equal(s2, dsum) and torch.equal(x2, dsumx), tag + ": spc_bn_bwd_reduce not reproducible"
            assert torch.equal(run_bwd_apply(dz, y, mean, rstd, gamma, beta, relu, dsum, dsumx), dx), \
                tag + ": spc_bn_bwd_apply not reproducible"


# ---- GPU: bn_relu end to end ---------------------------------------------------------------------------------------
def _module(s, dtype, gamma, beta, momentum=0.1, affine=True, track=True):
    bn = torch.nn.BatchNorm2d(s.C, eps=EPS, momentum=momentum, affine=affine, track_running_stats=track).to(DEV)
    with torch.no_grad():
        if affine:
            bn.weight.copy_(gamma)
            bn.bias.copy_(beta)
        if track:
            g = torch.Generator(device=DEV).manual_seed(s.C)
            bn.running_mean.copy_(torch.randn(s.C, device=DEV, generator=g))
            bn.running_var.copy_(torch.rand(s.C, device=DEV, generator=g) + 0.5)
            bn.num_batches_tracked.fill_(3)
    return bn.to(dtype)


def _run_bn_relu(bn, y, dz, relu):
    from mpi4dl_b200.torchgems.fused import bn_relu, fusable

    assert fusable(y, bn)
    x = y.clone().requires_grad_(True)
    z = bn_relu(x, bn, relu=relu)
    z.backward(dz)
    return z.detach(), x.grad


def check_bn_relu(s, dtype, relu, ratio, momentum=0.1, affine=True, track=True, repeat=False):
    tag = "bn_relu %s %s %s m%g mom=%s%s%s" % (shape_id(s), str(dtype)[6:], "relu" if relu else "bn", ratio, momentum,
                                              "" if affine else " no-affine", "" if track else " no-running")
    y, dz, gamma, beta = make_inputs(s, dtype, ratio, seed_of(s[:4], str(dtype), ratio, "e2e"))
    if not affine:
        gamma, beta = torch.ones_like(gamma), torch.zeros_like(beta)
    bn = _module(s, dtype, gamma, beta, momentum, affine, track)
    gamma, beta = bn.weight.detach().float() if affine else gamma, bn.bias.detach().float() if affine else beta
    rm0, rv0 = (_host(bn.running_mean, bn.running_var) if track else (None, None))
    first = _run_bn_relu(bn, y, dz, relu) + ((bn.weight.grad, bn.bias.grad) if affine else ()) + \
        ((bn.running_mean.clone(), bn.running_var.clone()) if track else ())
    z, dx = first[:2]
    M = s.N * s.H * s.W
    hg, hb = _host(gamma, beta)
    zb, dxb = Z_BOUND[dtype], DX_BOUND[dtype]
    P = UNIT[dtype] if dtype == torch.bfloat16 else 0.0          # the parameters' (and their gradients') dtype
    w = Worst()
    mom = momentum if momentum is not None else 1.0 / 4.0          # num_batches_tracked 3 -> 4
    for c in range(s.C):
        yc = y[:, c]
        m64, v64, mad, ms = ref_stats(yc)
        dm, dv = mean_bound(m64, mad), var_bound(v64, ms)
        r64 = 1.0 / np.sqrt(v64 + EPS)
        t = dv / (v64 + EPS)
        assert t < 1, (tag, c, t)
        rho = (1.0 - t) ** -0.5 * (1 + 2.0 ** -21) - 1.0
        ga, be = abs(hg[c]), abs(hb[c])
        xh = (yc.double() - m64) * r64
        dxh = xh.abs() * rho + dm * r64 * (1 + rho)
        pre = xh * hg[c] + hb[c]
        bz = ga * dxh + zb * ((xh.abs() + dxh) * ga + be)
        w.check("z", z[:, c], pre.clamp(min=0.0) if relu else pre, bz)
        _mask_check(w, "mask", z[:, c], pre, bz, relu)
        g = dz[:, c].double()
        if relu:
            g = torch.where(z[:, c] > 0, g, 0.0)
        sg = float(g.abs().sum())
        D, S = float(g.sum()), float((g * xh).sum())
        Es = SUM_BOUND * sg
        Ex = float((g.abs() * dxh).sum()) + SUM_BOUND * float((g.abs() * (xh.abs() + dxh)).sum())
        dx64 = (g - D / M - xh * (S / M)) * (hg[c] * r64)
        I = g.abs() + abs(D) / M + xh.abs() * (abs(S) / M)
        moved = (dxh * (abs(S) + Ex) + xh.abs() * Ex + Es) / M
        Adx = (g.abs() + (abs(D) + Es) / M + (xh.abs() + dxh) * ((abs(S) + Ex) / M)) * (ga * r64 * (1 + rho))
        bdx = (I * rho + moved * (1 + rho)) * (ga * r64) + dxb * Adx
        w.check("dx", dx[:, c], dx64, bdx * (1 + 2.0 ** -10))
        if affine:
            w.check("dgamma", first[2][c], S, Ex + P * (abs(S) + Ex))
            w.check("dbeta", first[3][c], D, Es + P * (abs(D) + Es))
        if track:
            R = 6 * UNIT[dtype]
            rm, rv = first[-2][c], first[-1][c]
            k = M / max(M - 1.0, 1.0)
            w.check("running_mean", rm, (1 - mom) * rm0[c] + mom * m64,
                    mom * dm + R * (abs((1 - mom) * rm0[c]) + mom * (abs(m64) + dm)))
            w.check("running_var", rv, (1 - mom) * rv0[c] + mom * k * v64,
                    mom * k * dv + R * (abs((1 - mom) * rv0[c]) + mom * k * (v64 + dv)))
    if track:
        assert int(bn.num_batches_tracked) == 4
    else:
        assert bn.running_mean is None and bn.running_var is None
    if not affine:
        assert bn.weight is None
    w.report(tag)
    if repeat:
        for _ in range(2):
            bn2 = _module(s, dtype, gamma, beta, momentum, affine, track)
            again = _run_bn_relu(bn2, y, dz, relu) + ((bn2.weight.grad, bn2.bias.grad) if affine else ()) + \
                ((bn2.running_mean, bn2.running_var) if track else ())
            names = ["z", "dx"] + (["dgamma", "dbeta"] if affine else []) + (["running_mean", "running_var"] if track else [])
            for n, a, b in zip(names, first, again):
                assert torch.equal(a, b), "%s: %s not reproducible" % (tag, n)


@pytest.mark.gpu
@pytest.mark.parametrize("s,dt,relu,ratio", CASES)
def test_bn_relu_against_fp64(s, dt, relu, ratio):
    check_bn_relu(s, DTYPES[dt], relu, ratio, repeat=multi_item(s))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("variant", ["momentum-none", "no-affine", "no-running-stats"])
def test_bn_relu_module_options(variant, dt):
    s = SHAPES[3]
    kw = {"momentum-none": dict(momentum=None), "no-affine": dict(affine=False), "no-running-stats": dict(track=False)}
    check_bn_relu(s, DTYPES[dt], True, 10.0, **kw[variant])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_misaligned_view_takes_the_module_path(dt):
    """a contiguous view whose data pointer is not 16-byte aligned is not fusable (checked BEFORE bn_relu runs, so a
    missing check fails here and never launches a misaligned kernel); bn_relu then computes what the module computes"""
    from mpi4dl_b200.torchgems.fused import bn_relu, fusable

    dtype = DTYPES[dt]
    shape = (2, 3, 8, 16)
    n = int(np.prod(shape))
    t = torch.randn(n + 1, device=DEV).to(dtype)[1:].view(shape)
    assert t.is_contiguous() and t.data_ptr() % 16
    bn = torch.nn.BatchNorm2d(3).to(DEV).to(dtype)
    ref = torch.nn.BatchNorm2d(3).to(DEV).to(dtype)
    assert not fusable(t, bn)
    assert fusable(t.clone(), bn)
    z = bn_relu(t, bn, relu=True)
    zr = torch.relu(ref(t))
    assert torch.equal(z, zr)
    assert torch.equal(bn.running_mean, ref.running_mean) and torch.equal(bn.running_var, ref.running_var)
