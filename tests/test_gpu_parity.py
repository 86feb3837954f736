"""-m gpu: parity of the CUDA path (through the C ABI) against
  (1) the committed golden vectors produced by the unmodified reference, and
  (2) the oracle on seeded inputs, incl. edge cases and size-independent properties.
Tolerances: fp32 path  atol = 1e-4 * sqrt(C*R*S) relative to max|ref| (SURVEY 8c);
            bf16 path  y, dx per element against fp64 on bf16-rounded inputs (test_gpu_tc_coverage.check_act);
                       dw (rounded to bf16 by autograd) and db against the fp32 oracle, rtol 2e-2."""
import numpy as np
import pytest
import torch

from oracle import spatial_oracle as so
from tests import gpu_util as gu
from tests import test_gpu_tc_coverage as cov

pytestmark = pytest.mark.gpu


def _tol(ref, C, R, S, scale=1e-4):
    return scale * np.sqrt(C * R * S) * max(1.0, float(np.abs(ref).max()))


def _close(a, b, atol, name):
    err = float(np.abs(a - b).max()) if a.size else 0.0
    assert a.shape == b.shape, (name, a.shape, b.shape)
    assert err <= atol, "%s: max err %g > %g" % (name, err, atol)


@pytest.mark.parametrize("gi", range(5))
def test_conv_against_reference_golden(golden, gi):
    z, meta = golden
    g = meta["grids"][gi]
    P, method, gname = g["P"], g["method"], g["name"]
    for case in meta["cases"]:
        if case["kind"] != "conv":
            continue
        cname = case["name"]
        x, w = z[f"{cname}/x"], z[f"{cname}/w"]
        b = z[f"{cname}/b"] if case["bias"] else None
        R, S = w.shape[2:]
        hh, hw = (R - 1) // 2, (S - 1) // 2
        tiles = so.split(x, method, P)
        padded = so.exchange_halos(tiles, method, hh, hw, kh=R, kw=S)
        for r in range(P):
            mask = so.neighbour_mask(method, P, r, R, S)
            strips = gu.strips_from_padded(padded[r], mask, hh, hw, torch.float32)
            out = gu.conv_tile(tiles[r], w, b, z[f"{gname}/{cname}/gy/{r}"], strips, tuple(case["stride"]))
            C = x.shape[1]
            key = f"{gname}/{cname}"
            ref_y = z[f"{key}/y/{r}"]
            if case["data"] == "kat" and np.abs(ref_y).max() < 2 ** 24:
                # the reference's own known-answer test: exact equality (SURVEY section 4)
                assert np.array_equal(out["y"], ref_y), f"{key}/y/{r} KAT not exact"
            else:
                _close(out["y"], ref_y, _tol(ref_y, C, R, S), f"{key}/y/{r}")
            _close(out["dx"], z[f"{key}/dx/{r}"], _tol(z[f"{key}/dx/{r}"], w.shape[0], R, S), f"{key}/dx/{r}")
            ref_dw = z[f"{key}/dw/{r}"]
            _close(out["dw"], ref_dw, 1e-5 * np.sqrt(tiles[r][0, 0].size * 2) * max(1.0, np.abs(ref_dw).max()), f"{key}/dw/{r}")
            if case["bias"]:
                ref_db = z[f"{key}/db/{r}"]
                _close(out["db"], ref_db, 1e-4 * max(1.0, np.abs(ref_db).max()), f"{key}/db/{r}")


@pytest.mark.parametrize("gi", range(5))
def test_pool_against_reference_golden(golden, gi):
    z, meta = golden
    g = meta["grids"][gi]
    P, method, gname = g["P"], g["method"], g["name"]
    for case in meta["cases"]:
        if case["kind"] != "pool":
            continue
        cname = case["name"]
        x = z[f"{cname}/x"]
        k, halo = case["k"], (case["k"] - 1) // 2
        tiles = so.split(x, method, P)
        padded = so.exchange_halos(tiles, method, halo, halo)
        mode = "max" if case["mode"] == "MaxPool2d" else "avg"
        for r in range(P):
            mask = so.neighbour_mask(method, P, r) if halo else [0] * 9
            strips = gu.strips_from_padded(padded[r], mask, halo, halo, torch.float32)
            out = gu.pool_tile(tiles[r], z[f"{gname}/{cname}/gy/{r}"], strips, mode, k, case["stride"])
            _close(out["y"], z[f"{gname}/{cname}/y/{r}"], 1e-5, f"{gname}/{cname}/y/{r}")
            _close(out["dx"], z[f"{gname}/{cname}/dx/{r}"], 1e-5, f"{gname}/{cname}/dx/{r}")


@pytest.mark.parametrize("gi", range(5))
def test_halo_pad_against_reference_golden(golden, gi):
    from mpi4dl_b200.torchgems.spatial import _HaloPadFn

    z, meta = golden
    g = meta["grids"][gi]
    P, method, gname = g["P"], g["method"], g["name"]
    for case in meta["cases"]:
        if case["kind"] != "halo":
            continue
        cname, h = case["name"], case["halo"]
        tiles = so.split(z[f"{cname}/x"], method, P)
        padded = so.exchange_halos(tiles, method, h, h)
        for r in range(P):
            mask = so.neighbour_mask(method, P, r)
            strips = gu.strips_from_padded(padded[r], mask, h, h, torch.float32)
            x = gu.t(tiles[r], grad=True)
            y = _HaloPadFn.apply(x, h, *strips)
            assert np.array_equal(y.detach().cpu().numpy(), z[f"{gname}/{cname}/y/{r}"])
            y.backward(gu.t(z[f"{gname}/{cname}/gy/{r}"]))
            assert np.array_equal(x.grad.cpu().numpy(), z[f"{gname}/{cname}/dx/{r}"])


def test_halo_pack_matches_oracle_send_regions():
    """spc_halo_pack cuts exactly the strips the reference sends (spatial.py:239-309)."""
    import ctypes as C
    from mpi4dl_b200 import _lib

    rng = np.random.default_rng(3)
    for (N, Cc, H, W, hh, hw) in [(2, 3, 8, 12, 1, 1), (1, 2, 9, 7, 2, 3), (1, 1, 4, 4, 0, 2), (1, 4, 5, 6, 3, 0)]:
        x_np = rng.standard_normal((N, Cc, H, W)).astype(np.float32)
        for dtype in (torch.float32, torch.bfloat16):
            x = gu.t(x_np, dtype)
            xp = np.pad(x.float().cpu().numpy(), ((0, 0), (0, 0), (hh, hh), (hw, hw)))
            bufs, ptrs = [None] * 9, [0] * 9
            for i in range(9):
                (r0, r1), (c0, c1) = so._send_region(i, hh, hw, H + 2 * hh, W + 2 * hw)
                if i != 4 and r1 > r0 and c1 > c0:
                    bufs[i] = torch.empty((N, Cc, r1 - r0, c1 - c0), dtype=dtype, device="cuda:0")
                    ptrs[i] = bufs[i].data_ptr()
            arr = (C.c_void_p * 9)(*[C.c_void_p(p) if p else C.c_void_p(None) for p in ptrs])
            _lib.check(_lib.lib().spc_halo_pack(N, Cc, H, W, hh, hw, _lib.dtype_code(dtype), C.c_void_p(x.data_ptr()),
                                                C.byref(arr), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "pack")
            for i in range(9):
                if bufs[i] is not None:
                    (r0, r1), (c0, c1) = so._send_region(i, hh, hw, H + 2 * hh, W + 2 * hw)
                    assert np.array_equal(bufs[i].float().cpu().numpy(), xp[:, :, r0:r1, c0:c1]), (i, hh, hw)


CONV_CASES = [
    # C, K, (R,S), stride, H, W, bias
    (3, 16, (3, 3), (1, 1), 20, 36, True),
    (16, 16, (3, 3), (1, 1), 33, 130, False),     # ragged: crosses direct-kernel tile edges
    (52, 52, (3, 3), (2, 2), 32, 64, False),
    (3, 104, (3, 3), (2, 2), 64, 64, False),
    (52, 52, (1, 7), (1, 1), 16, 160, False),
    (52, 52, (7, 1), (1, 1), 40, 48, False),
    (104, 208, (1, 1), (1, 1), 24, 40, False),
    (208, 52, (1, 1), (1, 1), 16, 16, True),
    (64, 128, (1, 1), (2, 2), 16, 32, False),
    (5, 7, (5, 5), (1, 1), 12, 12, True),
    (17, 19, (3, 3), (1, 1), 7, 5, True),         # odd everything, tile smaller than a CTA tile
    # shapes that take the tensor-core (wgmma) path in bf16 (W % 64 == 0 for multi-tap, H*W % 8 == 0 for 1x1)
    (52, 52, (1, 7), (1, 1), 8, 128, False),
    (104, 104, (7, 1), (1, 1), 16, 64, False),
    (64, 16, (3, 3), (1, 1), 12, 192, True),
    (104, 104, (3, 3), (1, 1), 9, 64, False),
    (1664, 416, (1, 1), (1, 1), 8, 48, False),    # 4 M-blocks, streamed weights
    (416, 1248, (1, 1), (1, 1), 8, 32, False),    # > 512 output channels: M groups
    (104, 208, (1, 1), (2, 2), 16, 64, False),    # stride-2 pointwise (FactorizedReduce)
    (52, 52, (3, 3), (2, 2), 32, 256, False),     # stride-2 3x3 on wgmma (column-subsampled copies)
    (104, 104, (3, 3), (2, 2), 8, 128, False),
    (3, 104, (3, 3), (2, 2), 16, 128, False),     # the AmoebaNet stem
    # stride-1 multi-tap convolutions: small / partial channel boxes, odd row counts
    # (tile rows past the image), 5-wide filters, several 64-channel chunks, resident and streamed weights
    (3, 16, (3, 3), (1, 1), 20, 64, True),
    (16, 16, (3, 3), (1, 1), 7, 128, False),
    (24, 40, (5, 5), (1, 1), 10, 64, True),
    (128, 64, (3, 3), (1, 1), 6, 64, True),
    (200, 104, (1, 7), (1, 1), 5, 128, False),
    (104, 104, (1, 7), (1, 1), 3, 192, False),
    (104, 104, (7, 1), (1, 1), 23, 64, False),
    (52, 128, (7, 1), (1, 1), 4, 64, True),
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_conv_against_oracle_seeded(case, dtype):
    C, K, (R, S), stride, H, W, bias = case
    rng = np.random.default_rng(hash((C, K, R, S, H, W)) % (2 ** 31))
    hh, hw = (R - 1) // 2, (S - 1) // 2
    x = rng.standard_normal((2, C, H, W)).astype(np.float32)
    w = (rng.standard_normal((K, C, R, S)) / np.sqrt(C * R * S)).astype(np.float32)
    b = rng.standard_normal(K).astype(np.float32) if bias else None
    # a tile in the middle of a 3x3 grid: all 8 neighbours present
    xp = np.pad(x, ((0, 0), (0, 0), (hh, hh), (hw, hw)))
    halo_vals = rng.standard_normal(xp.shape).astype(np.float32)
    inner = np.zeros(xp.shape, dtype=bool)
    inner[:, :, hh:hh + H, hw:hw + W] = True
    xp = np.where(inner, xp, halo_vals)
    if dtype == torch.bfloat16:
        xp, w = gu.bf16_round(xp), gu.bf16_round(w)
        b = gu.bf16_round(b) if b is not None else None
        x = xp[:, :, hh:hh + H, hw:hw + W]
    mask = [1, 1, 1, 1, 0, 1, 1, 1, 1]
    if R == 1:
        mask = [0, 0, 0, 1, 0, 1, 0, 0, 0]
    if S == 1:
        mask = [0, 1, 0, 0, 0, 0, 0, 1, 0] if R > 1 else [0] * 9
    strips = gu.strips_from_padded(xp, mask, hh, hw, dtype)
    y_ref = so.conv2d_fwd(xp, w, b, stride)
    gy = rng.standard_normal(y_ref.shape).astype(np.float32)
    if dtype == torch.bfloat16:
        gy = gu.bf16_round(gy)
    dxp, dw_ref, db_ref = so.conv2d_bwd(xp, w, gy, stride, need_db=bias)
    dx_ref = so.crop(dxp, hh, hw)
    out = gu.conv_tile(x, w, b, gy, strips, stride, dtype)
    if dtype == torch.float32:
        _close(out["y"], y_ref, _tol(y_ref, C, R, S), "y")
        _close(out["dx"], dx_ref, _tol(dx_ref, K, R, S), "dx")
        _close(out["dw"], dw_ref, 1e-5 * np.sqrt(2 * H * W) * max(1.0, np.abs(dw_ref).max()), "dw")
    else:
        # y, dx per element against fp64 (|got - ref| <= 2^-8 |ref| + 2^-12 A, see test_gpu_tc_coverage.py); dw has
        # been rounded to bf16 by autograd, hence the looser check
        ref, A = cov.reference(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b) if b is not None else None,
                               torch.from_numpy(gy), gu.strips_from_padded(xp, mask, hh, hw, torch.float32, "cpu"),
                               stride[0])
        cov.check_act(torch.from_numpy(out["y"]), ref["y"], A["y"], "y")
        cov.check_act(torch.from_numpy(out["dx"]), ref["dx"], A["dx"], "dx")
        np.testing.assert_allclose(out["dw"], dw_ref, rtol=2e-2, atol=2e-2 * np.abs(dw_ref).max())
    if bias:
        np.testing.assert_allclose(out["db"], db_ref, rtol=2e-2 if dtype == torch.bfloat16 else 1e-4,
                                   atol=(2e-2 if dtype == torch.bfloat16 else 1e-4) * np.abs(db_ref).max())


# the pools are checked per element against ATen in tests/test_gpu_direct_pool_coverage.py


def test_empty_batch_and_border_tile():
    """N == 0 is a no-op; a tile with no neighbours equals zero-padded conv."""
    rng = np.random.default_rng(1)
    x = rng.standard_normal((0, 3, 8, 8)).astype(np.float32)
    w = rng.standard_normal((4, 3, 3, 3)).astype(np.float32)
    out = gu.conv_tile(x, w, None, None, [None] * 9, (1, 1))
    assert out["y"].shape == (0, 4, 8, 8)
    x = rng.standard_normal((1, 3, 8, 8)).astype(np.float32)
    out = gu.conv_tile(x, w, None, None, [None] * 9, (1, 1))
    ref = so.conv2d_fwd(np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1))), w, None, (1, 1))
    _close(out["y"], ref, _tol(ref, 3, 3, 3), "border")


def test_full_size_properties_linearity_and_tile_equals_slice():
    """Size-independent properties at a BASELINE-scale tile (ResNet 16->16 3x3 on a 2048^2 tile,
    bf16): (a) linearity conv(a*x) == a*conv(x) for a power-of-two a (exact in floating point),
    (b) a tile with oracle-cut halos equals the same slice of the 'full image' conv computed by
    the same kernel, (c) checksum of avg-pool: sum(y)*k*k == sum over windows."""
    from mpi4dl_b200 import _lib
    from mpi4dl_b200.torchgems.spatial import _ConvSpatialFn, _PoolFn

    torch.manual_seed(0)
    dev = "cuda:0"
    C = K = 16
    H = W = 2048
    full = torch.randn(1, C, H, 2 * W, device=dev, dtype=torch.bfloat16)
    w = (torch.randn(K, C, 3, 3, device=dev) / 12).to(torch.bfloat16)
    code = _lib.dtype_code(torch.bfloat16)

    def conv(x, strips=(None,) * 9):
        N, Cc, h, ww = x.shape
        return _ConvSpatialFn.apply(x.contiguous(), w, None, (N, Cc, h, ww, K, 3, 3, 1, 1, 1, 1, code, 0), *strips)

    y_full = conv(full)
    y2 = conv(full * 2)
    assert torch.equal(y2, y_full * 2)
    # left tile of a vertical-2 split: right neighbour's first column is its halo strip 5
    left = full[:, :, :, :W].contiguous()
    strips = [None] * 9
    strips[5] = full[:, :, :, W:W + 1].contiguous()
    y_left = conv(left, strips)
    # interior columns come from the same (wgmma) kernel in both runs: bit-exact.  The last
    # column is recomputed by the boundary kernel from the halo strip (different fp32 summation
    # order), so it may differ by one bf16 rounding step.
    assert torch.equal(y_left[..., :W - 1], y_full[..., :W - 1])
    edge, ref_edge = y_left[..., W - 1].float(), y_full[..., W - 1].float()
    assert torch.allclose(edge, ref_edge, rtol=1e-2, atol=1e-2)
    # avg-pool checksum on the same tensor
    N, Cc, h, ww = left.shape
    yp = _PoolFn.apply(left, (N, Cc, h, ww, 3, 1, 1, _lib.SPC_POOL_AVG, code), *([None] * 9))
    ref = torch.nn.functional.avg_pool2d(left.float(), 3, 1, 1, count_include_pad=True)
    assert torch.allclose(yp.float(), ref, atol=2e-2, rtol=2e-2)


@pytest.mark.parametrize("rank", range(4))
@pytest.mark.parametrize("k,stride", [((3, 3), 1), ((1, 7), 1), ((3, 3), 2)])
def test_fused_halo_conv_variant(rank, k, stride):
    """conv_spatial(halo_len=0) (D2): zero padding only on image-border sides, none (valid conv)
    on neighbour-facing sides, no exchange.  Oracle: asymmetric np.pad + padding=0 conv."""
    from mpi4dl_b200.torchgems import spatial

    rng = np.random.default_rng(11 + rank)
    C, K, H, W = 8, 6, 20, 24
    R, S = k
    ph, pw = (R - 1) // 2, (S - 1) // 2
    x = rng.standard_normal((1, C, H, W)).astype(np.float32)
    m = spatial.conv_spatial(rank, 1, 4, C, K, k, stride=stride, padding=(ph, pw), halo_len=0, bias=True).cuda()
    w = m.weight.detach().cpu().numpy()
    b = m.bias.detach().cpu().numpy()
    top, bottom, left, right = m._inner_sides
    xp = np.pad(x, ((0, 0), (0, 0), (0 if top else ph, 0 if bottom else ph), (0 if left else pw, 0 if right else pw)))
    ref = so.conv2d_fwd(xp, w, b, (stride, stride))
    xt = gu.t(x, grad=True)
    y = m(xt)      # (strided on a tile whose top / left faces a neighbour: phase re-aligned by _fused_pre)
    assert tuple(y.shape) == ref.shape, (y.shape, ref.shape)
    _close(y.detach().cpu().numpy(), ref, _tol(ref, C, R, S), "fused y")
    gy = rng.standard_normal(ref.shape).astype(np.float32)
    y.backward(gu.t(gy))
    dxp, dw, db = so.conv2d_bwd(xp, w, gy, (stride, stride))
    Hp, Wp = xp.shape[2:]
    dx_ref = dxp[:, :, (0 if top else ph):Hp - (0 if bottom else ph), (0 if left else pw):Wp - (0 if right else pw)]
    _close(xt.grad.cpu().numpy(), dx_ref, _tol(dx_ref, K, R, S), "fused dx")
    _close(m.weight.grad.cpu().numpy(), dw, 1e-4 * max(1.0, np.abs(dw).max()), "fused dw")
