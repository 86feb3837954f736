"""CPU: the exact backward's algebra.  With the reverse halo exchange (tests/exact_oracle.py) every tile's input
gradient equals the matching slice of the same op's gradient on the unsplit image -- zero padding at true borders,
avg pool / k^2, max pool routing to the first maximum with 0 at true borders -- up to one final fp32 rounding:
|err| <= 2^-22 * A, A = the same op on absolute values in float64.  The same bound rejects the reference's
tile-local gradient (SURVEY 8a N2) and a reverse exchange that adds strip d at edge d instead of 8-d."""
import numpy as np
import pytest

from oracle import spatial_oracle as so
from tests import exact_oracle as xo

GRIDS = [("square", 4), ("vertical", 2), ("vertical", 4), ("horizontal", 2), ("horizontal", 4)]
CONVS = [(3, 3, 1), (3, 3, 2), (1, 7, 1), (7, 1, 1), (5, 5, 1), (1, 1, 1)]
POOLS = [("avg", 1), ("avg", 2), ("max", 1), ("max", 2)]
HALOS = [1, 2, 3]
BOUND = 2.0 ** -22


def _cases():
    for method, P in GRIDS:
        for R, S, st in CONVS:
            yield pytest.param(method, P, ("conv", R, S, st), id="%s%d-conv%dx%ds%d" % (method, P, R, S, st))
        for mode, st in POOLS:
            yield pytest.param(method, P, ("pool", mode, st), id="%s%d-%spool3s%d" % (method, P, mode, st))
        for h in HALOS:
            yield pytest.param(method, P, ("halo", h), id="%s%d-halo%d" % (method, P, h))


def _violates(got, ref, A):
    return bool((np.abs(got.astype(np.float64) - ref) > BOUND * A).any())


def run_case(method, P, op, seed=0):
    """(per-rank oracle results, per-rank fp64 full-image reference, per-rank A, whether any strip travels)"""
    rng = np.random.default_rng(seed)
    full = rng.standard_normal((2, 3, 24, 24)).astype(np.float32)
    tiles = so.split(full, method, P)
    if op[0] == "conv":
        _, R, S, st = op
        w = rng.standard_normal((4, 3, R, S)).astype(np.float32)
        ys = so.conv_spatial(tiles, w, None, method, (st, st))
        gys = [rng.standard_normal(y["y"].shape).astype(np.float32) for y in ys]
        res = xo.conv_spatial(tiles, w, method, (st, st), gys)
        ref, A = xo.full_reference("conv", full, gys, method, P, w=w, stride=(st, st))
        moves = (R > 1 or S > 1) and any(any(so.neighbour_mask(method, P, r, R, S)) for r in range(P))
    elif op[0] == "pool":
        _, mode, st = op
        ys = so.pool_spatial(tiles, method, mode, 3, st, 1)
        gys = [rng.standard_normal(y["y"].shape).astype(np.float32) for y in ys]
        res = xo.pool_spatial(tiles, method, mode, 3, st, gys)
        ref, A = xo.full_reference("pool", full, gys, method, P, mode=mode, k=3, stride=st)
        moves = True
    else:
        h = op[1]
        gys = [rng.standard_normal((t.shape[0], t.shape[1], t.shape[2] + 2 * h, t.shape[3] + 2 * h)).astype(np.float32)
               for t in tiles]
        res = xo.halo_exchange_layer(tiles, method, h, gys)
        ref, A = xo.full_reference("halo", full, gys, method, P, halo_len=h)
        moves = True
    return res, ref, A, moves


@pytest.mark.parametrize("method,P,op", list(_cases()))
def test_exact_dx_equals_full_image_gradient(method, P, op):
    res, ref, A, moves = run_case(method, P, op)
    for r in range(P):
        err = np.abs(res[r]["exact"].astype(np.float64) - ref[r])
        assert (err <= BOUND * A[r]).all(), "rank %d: max err/bound %.3g" % (
            r, float((err / np.maximum(BOUND * A[r], 1e-300)).max()))
    if moves:
        # the test has teeth: the reference's tile-local dx and a reverse exchange into the wrong band both fail
        assert any(_violates(res[r]["n2"], ref[r], A[r]) for r in range(P)), "N2 dx passes the bound"
        assert any(_violates(res[r]["flipped"], ref[r], A[r]) for r in range(P)), "flipped pairing passes the bound"
    else:
        for r in range(P):
            np.testing.assert_array_equal(res[r]["exact64"], res[r]["n2"])
