"""-m gpu: spc_conv2d_wgrad_deterministic and PyTorch's deterministic mode on the spatial stages.

1. Every row of the wgrad coverage tables -- test_gpu_tc_coverage.CASES (bf16 wgmma), the CASES of test_tf32_pointwise,
   test_tf32_tap and test_tf32_strided (TF32), and the direct / bias rows of test_gpu_direct_pool_coverage -- runs
   through the deterministic entry point, with all eight halo strips on the rows of the MASK_CASES lists.  Each row:
   dw / db within the row's fp64 bound; bit-identical across a call alone, a call while a large matmul runs on a
   second stream (the CTAs land on other SMs, in another order), and a CUDA-graph replay; the same with
   accumulate = 1; the kernels launched are those of spc_conv2d_wgrad plus the in-order reduce.
2. A TF32 tap case whose split count exceeds what a small workspace holds runs in several passes and gives the bits of
   the single-pass run.
3. torch.use_deterministic_algorithms(True) (uninitialised memory filled with NaN): the first six AmoebaNet-D cells and a
   ResNet-v2 spatial stage on four tiles over the peer transport (the harness of test_gpu_recompute), fp32 AUTO, fp32
   SPCONV_ALLOW_TF32=strided and bf16 autocast, exact backward off and on.  Every .grad is bit-identical between two
   runs, and the checkpointed stage's parameter gradients equal the plain stage's bit for bit.

Parts 1 and 2 run in one spawned process (part 3 in four), and the test process only collects their results.  They
capture a few hundred CUDA graphs and open a few hundred profiler sessions.  Run in the test process, they left
torch.profiler losing the records of the first kernels of later sessions, so the kernel-name checks of the modules
that run after this one (test_tf32_pointwise, test_tf32_strided) saw only a session's last launches.
"""
import ctypes as C
import os
import time
import traceback
import zlib

import pytest
import torch
import torch.multiprocessing as mp

from mpi4dl_b200 import _lib
from oracle import spatial_oracle as so
from tests import test_gpu_direct_pool_coverage as dp
from tests import test_gpu_recompute as rc
from tests import test_gpu_tc_coverage as cov
from tests import test_tf32_pointwise as pw
from tests import test_tf32_strided as s2
from tests import test_tf32_tap as tap

pytestmark = pytest.mark.gpu
DEV = cov.DEV
TF32_ABS = 2.0 ** -9 + 2.0 ** -12          # spconv.h: TF32 wgrad on arbitrary fp32 inputs
ALL = [1, 1, 1, 1, 0, 1, 1, 1, 1]
NONE = [0] * 9
REDUCE = "wgrad_reduce_kernel"


class Row:
    """one wgrad problem: cov-style geometry, storage dtype, algo, halo mask, and the bound (rel, A coefficient) of dw
    and db"""

    def __init__(self, rid, C_, K_, R, S, stride, N, H, W, bias, dtype, algo, mask, bw, bb):
        self.id, self.C, self.K, self.R, self.S, self.stride = rid, C_, K_, R, S, stride
        self.N, self.H, self.W, self.bias, self.dtype, self.algo, self.mask = N, H, W, bias, dtype, algo, mask
        self.bw, self.bb = bw, bb


def _rows():
    rows = []
    for c in cov.CASES:
        rows.append(Row("bf16-" + cov.case_id(c), c.C, c.K, c.R, c.S, c.stride, c.N, c.H, c.W, c.bias, torch.bfloat16,
                        _lib.SPC_ALGO_AUTO, ALL if c in cov.MASK_CASES else NONE, (0.0, cov.ABS_W), (0.0, cov.ABS_W)))
    for c in pw.CASES:
        rows.append(Row("tf32pw-" + pw.case_id(c), c.C, c.K, 1, 1, c.stride, c.N, c.H, c.W, c.bias, torch.float32,
                        _lib.SPC_ALGO_TF32, NONE, (0.0, TF32_ABS), (0.0, TF32_ABS)))
    for c in tap.CASES:
        rows.append(Row("tf32tap-" + tap.case_id(c), c.C, c.K, c.R, c.S, 1, c.N, c.H, c.W, c.bias, torch.float32,
                        _lib.SPC_ALGO_TF32_ALL, ALL if c in tap.MASK_CASES else NONE, (0.0, TF32_ABS), (0.0, TF32_ABS)))
    for c in s2.CASES:
        rows.append(Row("tf32s2-" + s2.case_id(c), c.C, c.K, c.R, c.S, 2, c.N, c.H, c.W, c.bias, torch.float32,
                        _lib.SPC_ALGO_TF32_STRIDED, ALL if c in s2.MASK_CASES else NONE, (0.0, TF32_ABS),
                        (0.0, TF32_ABS)))
    for c in dp.DCASES:
        names = {n for n, _ in c.launches}
        if not names & {"wgrad_direct_kernel", "bias_grad_kernel"}:
            continue
        b = dp.conv_bounds(c)
        rows.append(Row("direct-" + dp.dcase_id(c), c.C, c.K, c.R, c.S, c.stride, c.N, c.H, c.W, c.bias, c.dtype,
                        _lib.SPC_ALGO_AUTO if c.dtype == torch.float32 else _lib.SPC_ALGO_DIRECT, dp.MASKS[c.mask],
                        b["dw"], b["db"]))
    return rows


ROWS = _rows()


def _desc(r, N=None):
    return _lib.ConvDesc(r.N if N is None else N, r.C, r.H, r.W, r.K, r.R, r.S, r.stride, r.stride, (r.R - 1) // 2,
                         (r.S - 1) // 2, _lib.dtype_code(r.dtype), r.algo)


def _inputs(r):
    g = torch.Generator().manual_seed(zlib.crc32(r.id.encode()))
    ph, pw_ = (r.R - 1) // 2, (r.S - 1) // 2
    x = torch.randn((r.N, r.C, r.H, r.W), generator=g).to(r.dtype)
    strips = [None] * 9
    for i, (dr, dc) in enumerate(so.DIRS):
        rows, cols = (ph if dr else r.H), (pw_ if dc else r.W)
        if i != 4 and r.mask[i] and rows and cols:
            strips[i] = torch.randn((r.N, r.C, rows, cols), generator=g).to(r.dtype)
    Ho, Wo = (r.H + 2 * ph - r.R) // r.stride + 1, (r.W + 2 * pw_ - r.S) // r.stride + 1
    dy = torch.randn((r.N, r.K, Ho, Wo), generator=g).to(r.dtype)
    return [t.to(DEV) if t is not None else None for t in (x, dy, *strips)]


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def wgrad(d, x, strips, dy, dw, db, accumulate, deterministic=True, ws_bytes=None):
    L = _lib.lib()
    op = 3 if deterministic else 2
    n = L.spc_conv_workspace_bytes(C.byref(d), op) if ws_bytes is None else ws_bytes
    ws = torch.empty(max(n, 16), dtype=torch.uint8, device=DEV)
    fn = L.spc_conv2d_wgrad_deterministic if deterministic else L.spc_conv2d_wgrad
    halo = _lib.make_halo(strips)
    _lib.check(fn(C.byref(d), _ptr(x), C.byref(halo), _ptr(dy), C.c_void_p(dw.data_ptr()), _ptr(db), accumulate,
                  _ptr(ws), n, C.c_void_p(torch.cuda.current_stream().cuda_stream)), "wgrad")
    return dw, db


def _three_ways(d, x, strips, dy, dw0, db0, accumulate):
    """(dw, db) of a call alone, a call under a concurrent matmul on a second stream, and a CUDA-graph replay"""
    outs = []

    def fresh():
        return dw0.clone(), db0.clone() if db0 is not None else None

    dw, db = fresh()
    outs.append(wgrad(d, x, strips, dy, dw, db, accumulate))
    big = torch.randn(4096, 4096, device=DEV)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for _ in range(3):
            big = big @ big
            big /= big.abs().max()
    dw, db = fresh()
    outs.append(wgrad(d, x, strips, dy, dw, db, accumulate))
    torch.cuda.synchronize()
    dw, db = fresh()
    n = _lib.lib().spc_conv_workspace_bytes(C.byref(d), 3)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        wgrad(d, x, strips, dy, dw, db, accumulate, ws_bytes=n)
    dw.copy_(dw0)
    if db is not None:
        db.copy_(db0)
    g.replay()
    torch.cuda.synchronize()
    outs.append((dw, db))
    return outs


def _same(a, b):
    return a is None and b is None or torch.equal(a.view(torch.int32), b.view(torch.int32))


def _check_row(r):
    x, dy, *strips = _inputs(r)
    ref, A = cov.reference(x, torch.zeros((r.K, r.C, r.R, r.S), device=DEV), torch.zeros(r.K, device=DEV), dy, strips,
                           r.stride)
    d = _desc(r)
    nan = float("nan")
    for accumulate in (0, 1):
        g = torch.Generator(device=DEV).manual_seed(5)
        if accumulate:
            dw0 = torch.randn((r.K, r.C, r.R, r.S), generator=g, device=DEV) * float(ref["dw"].abs().mean())
            db0 = torch.randn((r.K,), generator=g, device=DEV) * float(ref["db"].abs().mean()) if r.bias else None
        else:
            dw0 = torch.full((r.K, r.C, r.R, r.S), nan, device=DEV)
            db0 = torch.full((r.K,), nan, device=DEV) if r.bias else None
        outs = _three_ways(d, x, strips, dy, dw0, db0, accumulate)
        base_w = dw0.double() if accumulate else 0.0
        cov.check(outs[0][0], base_w + ref["dw"], A["dw"], r.bw[0], r.bw[1], r.id + " dw")
        if r.bias:
            base_b = db0.double() if accumulate else 0.0
            cov.check(outs[0][1], base_b + ref["db"], A["db"], r.bb[0], r.bb[1], r.id + " db")
        for i, (dw, db) in enumerate(outs[1:], 1):
            assert _same(dw, outs[0][0]), "%s accumulate=%d: call %d dw differs in %d elements" % (
                r.id, accumulate, i, int((dw != outs[0][0]).sum()))
            assert _same(db, outs[0][1]), "%s accumulate=%d: call %d db differs" % (r.id, accumulate, i)
    # the kernels: spc_conv2d_wgrad's, plus the reduce
    dw = torch.empty((r.K, r.C, r.R, r.S), device=DEV)
    db = torch.empty((r.K,), device=DEV) if r.bias else None

    def default():
        return cov.traced(lambda: wgrad(d, x, strips, dy, dw, db, 0, deterministic=False))[1]

    def det():
        return cov.traced(lambda: wgrad(d, x, strips, dy, dw, db, 0))[1]

    kd, kt = default(), det()
    assert cov.launched(kt, lambda k: kd <= k, det), (r.id, sorted(kd - kt))
    assert cov.launched(kd, lambda k: {n for n, _ in kt - k} <= {REDUCE}, default), (r.id, sorted(kt - kd))


def test_empty_batch():
    """N == 0: accumulate=1 leaves dw / db as they are, accumulate=0 zeroes them"""
    for r in (ROWS[0], next(r for r in ROWS if r.algo == _lib.SPC_ALGO_TF32_STRIDED)):
        d = _desc(r, N=0)
        dw0 = torch.randn((r.K, r.C, r.R, r.S), device=DEV)
        db0 = torch.randn((r.K,), device=DEV)
        dw, db = dw0.clone(), db0.clone()
        wgrad(d, None, [None] * 9, None, dw, db, 1)
        torch.cuda.synchronize()
        assert torch.equal(dw, dw0) and torch.equal(db, db0), r.id
        wgrad(d, None, [None] * 9, None, dw, db, 0)
        torch.cuda.synchronize()
        assert not dw.any() and not db.any(), r.id


def _check_passes():
    """a TF32 tap wgrad whose item chains cap forces many splits (chunks_total / 512): with a workspace that holds two
    slices it runs in passes, with one that holds them all in one; and with op 2's workspace one slice per launch.  All
    three give the same bits, and the passes reduce in order"""
    r = Row("tf32tap-passes", 16, 16, 3, 3, 1, 2, 256, 1024, True, torch.float32, _lib.SPC_ALGO_TF32_ALL, ALL,
            (0.0, TF32_ABS), (0.0, TF32_ABS))
    x, dy, *strips = _inputs(r)
    d = _desc(r)
    L = _lib.lib()
    full = L.spc_conv_workspace_bytes(C.byref(d), 3)
    own = L.spc_conv_workspace_bytes(C.byref(d), 2)
    wn = r.K * r.C * r.R * r.S
    chunks = r.N * r.H * (r.W // 32)
    assert chunks // 512 > 2 and full - own >= (chunks // 512) * wn * 4, (full, own, chunks)
    outs = []
    for nbytes in (full, own + 256 + 2 * wn * 4, own):
        dw = torch.full((r.K, r.C, r.R, r.S), float("nan"), device=DEV)
        db = torch.full((r.K,), float("nan"), device=DEV)
        _, k = cov.traced(lambda: wgrad(d, x, strips, dy, dw, db, 0, ws_bytes=nbytes))
        outs.append((dw, db, {n for n, _ in k}))
    assert REDUCE in outs[0][2] and REDUCE in outs[1][2], [sorted(o[2]) for o in outs]
    for dw, db, _ in outs[1:]:
        assert _same(dw, outs[0][0]) and _same(db, outs[0][1])
    ref, A = cov.reference(x, torch.zeros((r.K, r.C, r.R, r.S), device=DEV), torch.zeros(r.K, device=DEV), dy, strips, 1)
    cov.check(outs[0][0], ref["dw"], A["dw"], 0.0, TF32_ABS, "passes dw")


PASSES = "tf32tap-passes"
ROW_BY_ID = {r.id: r for r in ROWS}


def _child(q, names):
    """run the checks named (row ids, PASSES) in this process; puts {name: None or the failure text}"""
    out = {}
    for name in names:
        try:
            _check_passes() if name == PASSES else _check_row(ROW_BY_ID[name])
            out[name] = None
        except Exception:  # one failing row does not hide the others
            out[name] = traceback.format_exc()[-3000:]
    torch.cuda.synchronize()
    q.put(out)


@pytest.fixture(scope="module")
def child_results(request):
    """the results of every selected part-1 / part-2 check, computed in one spawned process"""
    names = []
    for item in request.session.items:
        if item.module is None or item.module.__name__ != __name__:
            continue
        if item.originalname == "test_row_within_bound_and_reproducible":
            names.append(item.callspec.params["r"])
        elif item.originalname == "test_passes_give_the_single_pass_bits":
            names.append(PASSES)
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    p = ctx.Process(target=_child, args=(q, names))
    p.start()
    while q.empty() and p.is_alive():
        time.sleep(0.5)
    res = None if q.empty() else q.get()
    p.join(60)
    if p.is_alive():
        p.kill()
    assert res is not None, "the checking process ended without results (exit code %s)" % p.exitcode
    return res


@pytest.mark.parametrize("r", [r.id for r in ROWS])
def test_row_within_bound_and_reproducible(r, child_results):
    err = child_results[r]
    assert err is None, err


def test_passes_give_the_single_pass_bits(child_results):
    err = child_results[PASSES]
    assert err is None, err


# ---- 3. the spatial stages under torch.use_deterministic_algorithms(True) -----------------------------------------
def _det_worker(rank, port, ngpu, q):
    import sys
    sys.path.insert(0, rc.ROOT)
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), SPCONV_HALO_TRANSPORT="peer", SPCONV_ARENA_MB="64",
                      SPCONV_HALO_OVERLAP="1")
    multi = ngpu >= rc.P
    dev = torch.device("cuda", rank if multi else 0)
    torch.cuda.set_device(dev)
    if multi:
        dist.init_process_group("nccl", rank=rank, world_size=rc.P, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=rc.P)
    from mpi4dl_b200.torchgems import recompute
    torch.use_deterministic_algorithms(True)
    errs = []
    try:
        g = torch.Generator().manual_seed(11 + rank)
        x = torch.randn(1, 3, rc.IMG // 2, rc.IMG // 2, generator=g).cuda()
        for allow in ("0", "strided"):
            os.environ["SPCONV_ALLOW_TF32"] = allow
            for kind in ("amoebanet", "resnet"):
                plain, ckpt = rc._stage(kind, rank), recompute.checkpoint_spatial_cells(rc._stage(kind, rank))
                with torch.no_grad():
                    shape = rc._out(plain(x)).shape
                    ckpt(x)
                gy = torch.randn(shape, generator=g).cuda()
                arms = [("fp32", False)] if allow == "strided" else [("fp32", False), ("bf16_amp", True)]
                for arm, amp in arms:
                    for exact in (False, True):
                        tag = (kind, allow, arm, exact)
                        a = rc._run(plain, x, gy, amp, exact)
                        b = rc._run(plain, x, gy, amp, exact)
                        c = rc._run(ckpt, x, gy, amp, exact)
                        if not torch.equal(a["dx"], b["dx"]):
                            errs.append((tag, "dx differs between two runs"))
                        for i, (ga, gb, gc) in enumerate(zip(a["grads"], b["grads"], c["grads"])):
                            if ga is None:
                                continue
                            if not _same(ga, gb):
                                errs.append((tag, "grad %d differs between two runs" % i, int((ga != gb).sum())))
                            if not _same(ga, gc):
                                errs.append((tag, "grad %d: recompute differs from plain" % i, int((ga != gc).sum())))
        torch.cuda.synchronize()
    except Exception as ex:  # report instead of hanging the peers
        import traceback
        errs.append(("exception", repr(ex), traceback.format_exc()[-1500:]))
    q.put((rank, errs))
    try:
        dist.barrier()
        dist.destroy_process_group()
    except Exception:
        pass


def test_stages_bit_reproducible_under_deterministic_mode():
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    procs = [ctx.Process(target=_det_worker, args=(r, 29881, torch.cuda.device_count(), q)) for r in range(rc.P)]
    for p in procs:
        p.start()
    res = [q.get() for _ in range(rc.P)]
    for p in procs:
        p.join(120)
        if p.is_alive():
            p.kill()
    bad = [(r, e) for r, e in res if e]
    assert not bad, bad
