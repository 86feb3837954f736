"""-m gpu: FULL-SIZE parity of every distinct BASELINE layer shape against an INDEPENDENT reference.

For each unique (shape, op) of the AmoebaNet-D 8192^2 spatial stage (tests/golden/layers_amoebanetd_sp4.json)
and the ResNet-v2-101 4096^2 spatial stage (layers_resnet101_sp2.json), at the N=1 tile (whole
image, true zero borders on all four sides) and at the N=4 square tile (half the extent, halo
strips PRESENT on every side the kernel shape exchanges on, i.e. an interior tile), the CUDA path
(bf16 storage, through the C ABI) is compared -- the whole tensor, every border and every tile seam
of the persistent wgmma schedule -- with what the reference computes at spatial.py:1019-1029:

    y      = F.conv2d(padded_tile, w, b, stride, padding=0)          cuDNN, fp32, TF32 OFF
    dx     = crop(conv2d_input(padded.shape, w, gy))                 (N2: halos are constants)
    dw, db = conv2d_weight(padded, w.shape, gy), gy.sum((0,2,3))     over the padded tile incl. halos
    pools  = F.{avg,max}_pool2d(padded_tile, k, stride, padding=0)

Inputs are bf16-representable, so the only differences are the fp32 summation order and the final
bf16 rounding of y / dx (half an ulp = 2^-9 relative).  Tolerances (written here, checked per element):
    y, dx :  |got - ref| <= 2^-7 * |ref| + 2^-8 * rms(ref)      (one bf16 ulp = 2^-8 relative, plus a floor)
    dw    :  fp32 straight from spc_conv2d_wgrad:  |got - ref| <= 1e-3 * max|ref|
These shapes exercise num_tiles > 132 (persistent multi-tile loop, stage-ring wrap), num_mg > 1
(416->1248-class M groups come from dgrad of 1664->416), wres on/off, stride 2, all wgrad MG variants
and the multi-wave split-P schedule -- none of which the small oracle cases reach.  The largest tensors
(13 GB in fp32) are checked in channel slices so that every case fits an 80 GB GPU.
"""
import ctypes as C
import json
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def _unique_layers():
    out, seen = [], set()
    for fn, tag in (("layers_amoebanetd_sp4.json", "amoeba"), ("layers_resnet101_sp2.json", "resnet")):
        d = json.load(open(os.path.join(ROOT, "tests", "golden", fn)))
        first = True
        for l in d["layers"]:
            key = json.dumps({k: v for k, v in l.items() if k != "kind"}, sort_keys=True)
            if key not in seen:
                seen.add(key)
                out.append((tag, dict(l), first))
            first = False
    return out


LAYERS = _unique_layers()
CONVS = [(t, l, f) for t, l, f in LAYERS if l["op"] == "conv"]
POOLS = [(t, l, f) for t, l, f in LAYERS if l["op"] == "pool"]


def _cid(p):
    t, l, _ = p
    if l["op"] == "conv":
        return "%s-%dto%d-%dx%d-s%d-%d" % (t, l["C"], l["K"], l["R"], l["S"], l["stride_h"], l["H"])
    return "%s-%s%d-s%d-C%d-%d" % (t, l["mode"], l["k"], l["stride"], l["C"], l["H"])


@pytest.fixture(autouse=True)
def _no_tf32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    torch.cuda.empty_cache()


def _check(got, ref, name, rel=2.0 ** -7, floor=2.0 ** -8):
    """per-element |got-ref| <= rel*|ref| + floor*rms(ref), whole tensor, on the device (in slices of dim 1, so the
    fp32 temporaries stay small next to the operands)."""
    assert got.shape == ref.shape, (name, tuple(got.shape), tuple(ref.shape))
    step = max(1, (1 << 26) // max(1, ref[:, :1].numel()))
    sq = 0.0
    for i in range(0, ref.shape[1], step):
        sq += float(ref[:, i:i + step].float().square().sum(dtype=torch.float64))
    rms = (sq / ref.numel()) ** 0.5
    assert rms > 0, name
    worst, bad = float("-inf"), 0
    for i in range(0, ref.shape[1], step):
        r = ref[:, i:i + step].float()
        viol = (got[:, i:i + step].float() - r).abs_() - (r.abs() * rel + floor * rms)
        worst = max(worst, float(viol.max()))
        bad += int((viol > 0).sum())
        del r, viol
    assert worst <= 0, "%s: %d elements out of tolerance, worst excess %.3g (rms %.3g)" % (name, bad, worst, rms)


def _halo_strips(N, Cc, H, W, hh, hw, gen):
    """Strips for an interior tile: every direction the kernel shape exchanges on (spatial.py:921-939)."""
    strips = [None] * 9
    dirs = [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 0), (0, 1), (1, -1), (1, 0), (1, 1)]
    for i, (dr, dc) in enumerate(dirs):
        if i == 4 or (dr != 0 and hh == 0) or (dc != 0 and hw == 0):
            continue
        shp = (N, Cc, H if dr == 0 else hh, W if dc == 0 else hw)
        strips[i] = torch.randn(shp, device=DEV, generator=gen).to(torch.bfloat16)
    return strips


def _padded(x, strips, hh, hw):
    """The tensor the reference hands to nn.Conv2d: ZeroPad2d + copy_halo_exchange_values (spatial.py:1020,405-413)."""
    N, Cc, H, W = x.shape
    xp = torch.zeros((N, Cc, H + 2 * hh, W + 2 * hw), dtype=torch.float32, device=DEV)
    xp[:, :, hh:hh + H, hw:hw + W] = x.float()
    rows = [(0, hh), (hh, hh + H), (hh + H, H + 2 * hh)]
    cols = [(0, hw), (hw, hw + W), (hw + W, W + 2 * hw)]
    for i, s in enumerate(strips):
        if s is not None:
            (r0, r1), (c0, c1) = rows[i // 3], cols[i % 3]
            xp[:, :, r0:r1, c0:c1] = s.float()
    return xp


@pytest.mark.parametrize("tile", ["n1", "n4"])
@pytest.mark.parametrize("case", CONVS, ids=_cid)
def test_conv_fullsize_vs_cudnn_fp32(case, tile):
    from mpi4dl_b200 import _lib
    from mpi4dl_b200.torchgems.spatial import _ConvSpatialFn

    tag, l, first = case
    L = _lib.lib()
    div = 1 if tile == "n1" else 2
    Cc, K, R, S = l["C"], l["K"], l["R"], l["S"]
    H, W = l["H"] // div, l["W"] // div
    sh, sw, hh, hw = l["stride_h"], l["stride_w"], l["pad_h"], l["pad_w"]
    gen = torch.Generator(device=DEV).manual_seed(1000 + Cc * 7 + K * 3 + R * 11 + S + H)
    x = torch.randn((1, Cc, H, W), device=DEV, generator=gen).to(torch.bfloat16)
    w = (torch.randn((K, Cc, R, S), device=DEV, generator=gen) / (Cc * R * S) ** 0.5).to(torch.bfloat16)
    b = torch.randn(K, device=DEV, generator=gen).to(torch.bfloat16) if l.get("bias") else None
    strips = _halo_strips(1, Cc, H, W, hh, hw, gen) if tile == "n4" else [None] * 9
    desc = (1, Cc, H, W, K, R, S, sh, sw, hh, hw, _lib.SPC_BF16, _lib.SPC_ALGO_AUTO)
    d = _lib.ConvDesc(*desc)
    assert L.spc_conv_uses_tcgen05(C.byref(d), 0), "BASELINE shape fell off the tensor-core path: %r" % (l,)

    xg = x.clone().requires_grad_(not first)
    wg = w.clone().requires_grad_(True)
    bg = b.clone().requires_grad_(True) if b is not None else None
    y = _ConvSpatialFn.apply(xg, wg, bg, desc, *strips)
    gy = (torch.randn(y.shape, device=DEV, generator=gen) * 0.25).to(torch.bfloat16)
    y.backward(gy)

    xp = _padded(x, strips, hh, hw)
    wf = w.float()
    ref = F.conv2d(xp, wf, b.float() if b is not None else None, stride=(sh, sw), padding=0)
    _check(y.detach(), ref, "y")
    del ref
    gyf = gy.float()
    if not first:
        dxp = torch.nn.grad.conv2d_input(xp.shape, wf, gyf, stride=(sh, sw), padding=0)
        _check(xg.grad, dxp[:, :, hh:hh + H, hw:hw + W], "dx")
        del dxp
    dw_ref = torch.nn.grad.conv2d_weight(xp, wf.shape, gyf, stride=(sh, sw), padding=0)
    # fp32 dw straight from the C ABI (the autograd Function rounds it to the weight dtype)
    dw = torch.empty(w.shape, dtype=torch.float32, device=DEV)
    db = torch.empty(K, dtype=torch.float32, device=DEV) if b is not None else None
    nb = L.spc_conv_workspace_bytes(C.byref(d), 2)
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
    halo = _lib.make_halo(strips)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(L.spc_conv2d_wgrad(C.byref(d), C.c_void_p(x.data_ptr()), C.byref(halo), C.c_void_p(gy.data_ptr()),
                                  C.c_void_p(dw.data_ptr()), C.c_void_p(db.data_ptr()) if db is not None else None, 0,
                                  C.c_void_p(ws.data_ptr()), nb, st), "wgrad")
    tol = 1e-3 * float(dw_ref.abs().max())
    err = float((dw - dw_ref).abs().max())
    assert err <= tol, "dw: max err %.3g > %.3g" % (err, tol)
    _check(wg.grad, dw_ref, "dw(bf16)")
    if b is not None:
        db_ref = gyf.sum((0, 2, 3))
        assert float((db - db_ref).abs().max()) <= 1e-3 * float(db_ref.abs().max()) + 1e-3


@pytest.mark.parametrize("tile", ["n1", "n4"])
@pytest.mark.parametrize("case", POOLS, ids=_cid)
def test_pool_fullsize_vs_aten_fp32(case, tile):
    from mpi4dl_b200 import _lib
    from mpi4dl_b200.torchgems.spatial import _PoolFn

    tag, l, _ = case
    div = 1 if tile == "n1" else 2
    Cc, k, s, pad = l["C"], l["k"], l["stride"], l["pad"]
    H, W = l["H"] // div, l["W"] // div
    gen = torch.Generator(device=DEV).manual_seed(77 + Cc + k * 5 + s + H)
    x = torch.randn((1, Cc, H, W), device=DEV, generator=gen).to(torch.bfloat16)
    strips = _halo_strips(1, Cc, H, W, pad, pad, gen) if (tile == "n4" and pad) else [None] * 9
    mode = _lib.SPC_POOL_MAX if l["mode"] == "max" else _lib.SPC_POOL_AVG
    xg = x.clone().requires_grad_(True)
    y = _PoolFn.apply(xg, (1, Cc, H, W, k, s, pad, mode, _lib.SPC_BF16), *strips)
    gy = torch.randn(y.shape, device=DEV, generator=gen).to(torch.bfloat16)
    y.backward(gy)
    xp = _padded(x, strips, pad, pad).requires_grad_(True)
    ref = F.max_pool2d(xp, k, s, 0) if l["mode"] == "max" else F.avg_pool2d(xp, k, s, 0)
    _check(y.detach(), ref.detach(), "y", rel=2.0 ** -8, floor=2.0 ** -9)
    ref.backward(gy.float())
    _check(xg.grad, xp.grad[:, :, pad:pad + H, pad:pad + W], "dx", rel=2.0 ** -7, floor=2.0 ** -8)
