"""-m gpu: pw_px_gemm_kernel<NT> (gemm_px.cu), the pixel-major bf16 1x1 GEMM that large fprop / dgrad problems run on,
against an fp64 reference per element with the bound of test_gpu_tc_coverage:
    |got - ref| <= 2^-8 |ref| + 2^-12 A        (A = the same product on |x|, |w|)

The cases reach every instance (NT = 56, 104, 208), resident and streamed weights, one and several channel groups
(M = 416: 2, M = 1664: 8), reductions that are not a multiple of 64 channels (52, 104), pixel counts that are not a
multiple of 128, both activation / output box modes (3-d boxes, and the 5-d boxes of layers with >= 4 MB channel
planes), bias, and a stride-2 layer (through the subsample / zero-upsample passes).  Each asserts by kernel name that
the op ran on pw_px_gemm_kernel with the expected NT; the small shapes of test_gpu_tc_coverage still run on
pw_gemm_kernel.
"""
import collections

import pytest
import torch

from mpi4dl_b200 import _lib
from tests import test_gpu_tc_coverage as cov

pytestmark = pytest.mark.gpu

DEV = cov.DEV
Case = collections.namedtuple("Case", "C K stride N H W bias nt_fwd nt_dgrad note")
# "large" = at least 2 x SM count 128-pixel tiles (264 on a 132-SM H100); every case has more than that.  The C ABI's
# bf16 1x1 path needs P % 8 == 0.
CASES = [
    Case(52, 52, 1, 1, 184, 197, True, 56, 56,
         "P = 36248 (284 tiles, the last 24 pixels); Cin = 52 both ways; resident weights; 3-d boxes"),
    Case(104, 208, 1, 2, 130, 132, True, 208, 104,
         "2 images of 135 tiles; fprop Cin = 104 (second k-chunk 40 of 64), dgrad NT = 104 over 4 chunks, resident"),
    Case(104, 416, 1, 1, 190, 196, False, 208, 104,
         "fprop M = 416: 2 groups, streamed weights; dgrad 7 k-chunks resident"),
    Case(416, 1664, 1, 1, 180, 190, True, 208, 208,
         "fprop M = 1664: 8 groups streamed; dgrad M = 416 over 26 k-chunks, streamed"),
    Case(208, 52, 1, 1, 1024, 2048, True, 56, 208,
         "4 MB planes: fprop 5-d activation box, 3-d output box (52 % 8 != 0); dgrad 3-d activation, 5-d output box"),
    Case(104, 416, 1, 1, 1024, 2048, False, 208, 104,
         "4 MB planes: 5-d boxes both ways, fprop 2 groups streamed"),
    Case(104, 208, 2, 1, 384, 384, False, 208, 104,
         "stride 2: 192 x 192 subsampled pixels (288 tiles); dgrad through the zero-upsample pass"),
]


def case_id(c):
    return "%dto%d-s%d-n%d-%dx%d%s" % (c.C, c.K, c.stride, c.N, c.H, c.W, "-b" if c.bias else "")


def desc(c):
    return _lib.ConvDesc(c.N, c.C, c.H, c.W, c.K, 1, 1, c.stride, c.stride, 0, 0, _lib.SPC_BF16, _lib.SPC_ALGO_AUTO)


def check_sliced(got, a, w, b, name, step=104):
    """got[N][M][P] against a[N][Cin][P] contracted with w[M][Cin] (+b) in fp64, `step` output channels at a time (the
    fp64 temporaries of the 4 MB-plane cases would not fit otherwise)"""
    worst = 0.0
    for m0 in range(0, w.shape[0], step):
        ws = w[m0:m0 + step].double()
        ref = torch.einsum("mc,ncp->nmp", ws, a.double())
        A = torch.einsum("mc,ncp->nmp", ws.abs(), a.double().abs())
        if b is not None:
            ref += b[m0:m0 + step].double()[None, :, None]
            A += b[m0:m0 + step].double().abs()[None, :, None]
        worst = max(worst, cov.check_act(got[:, m0:m0 + step], ref, A, "%s channels %d.." % (name, m0)))
        del ref, A
    torch.cuda.empty_cache()   # the fp64 temporaries of the large cases are not needed by the next one
    return worst


def px_kernels(kernels):
    return {args for n, args in kernels if n == "pw_px_gemm_kernel"}


def cuda_events(fn):
    """every CUDA activity name one profiled run of fn records (for the failure message: an empty list means the
    profiler recorded nothing, not that nothing ran)"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({e.name()[:60] for e in prof.profiler.kineto_results.events()
                   if e.device_type() == torch.autograd.DeviceType.CUDA})


def assert_ran_px(kernels, nt, fn):
    """fn launched pw_px_gemm_kernel<nt> and no other instance of it.  A trace is a lower bound of what ran (records
    can be lost in a long-lived process, see test_gpu_tc_coverage.traced): a trace without the kernel is repeated"""
    ok = cov.launched(kernels, lambda k: px_kernels(k) == {(str(nt),)}, lambda: cov.traced(fn)[1])
    assert ok, "expected pw_px_gemm_kernel<%d>; traced: %s; all CUDA events of one more run: %s" % (
        nt, sorted(kernels), cuda_events(fn))


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_px_against_fp64(c):
    g = torch.Generator().manual_seed(c.C * 7919 + c.K * 31 + c.H)
    x = torch.randn((c.N, c.C, c.H, c.W), generator=g).bfloat16().to(DEV)
    w = (torch.randn((c.K, c.C, 1, 1), generator=g) / c.C ** 0.5).bfloat16().to(DEV)
    b = torch.randn((c.K,), generator=g).bfloat16().to(DEV) if c.bias else None
    Ho, Wo = c.H // c.stride, c.W // c.stride
    dy = torch.randn((c.N, c.K, Ho, Wo), generator=g).bfloat16().to(DEV)
    d = desc(c)
    strips = [None] * 9

    y, kf = cov.traced(lambda: cov.run_fwd(d, x, strips, w, b))
    assert_ran_px(kf, c.nt_fwd, lambda: cov.run_fwd(d, x, strips, w, b))
    xs = x[:, :, ::c.stride, ::c.stride] if c.stride > 1 else x
    wf = w[:, :, 0, 0]
    rf = check_sliced(y.reshape(c.N, c.K, -1), xs.reshape(c.N, c.C, -1), wf, b, case_id(c) + " y")
    del y

    dx, kd = cov.traced(lambda: cov.run_dgrad(d, dy, w))
    assert_ran_px(kd, c.nt_dgrad, lambda: cov.run_dgrad(d, dy, w))
    if c.stride > 1:   # the zero-upsample pass: only the even pixels carry the GEMM's result
        assert not dx[:, :, 1::2].any() and not dx[:, :, :, 1::2].any()
        dx = dx[:, :, ::2, ::2]
    rd = check_sliced(dx.reshape(c.N, c.C, -1), dy.reshape(c.N, c.K, -1), wf.t(), None, case_id(c) + " dx")
    print("[pw-px] %-28s y err/bound %.3f  dx err/bound %.3f" % (case_id(c), rf, rd))


SMALL = [cov._find(13, 13, 1, 1), cov._find(13, 200, 1, 1), cov._find(13, 416, 1, 1), cov._find(104, 200, 1, 1, 2)]


@pytest.mark.parametrize("c", SMALL, ids=cov.case_id)
def test_small_shapes_stay_on_pw_gemm(c):
    x, w, b, dy, strips = cov.make_inputs(c, [0] * 9)
    x, w, b, dy = cov._to_dev(x, w, b, dy)
    d = cov.desc(c)
    for fn in (lambda: cov.run_fwd(d, x, [None] * 9, w, b), lambda: cov.run_dgrad(d, dy, w)):
        _, k = cov.traced(fn)
        assert cov.launched(k, lambda k: "pw_gemm_kernel" in cov._names(k), lambda: cov.traced(fn)[1]), sorted(k)
        assert "pw_px_gemm_kernel" not in cov._names(k), sorted(k)
