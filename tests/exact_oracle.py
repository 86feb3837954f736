"""Exact-backward restatement for the tests (numpy, all ranks in one process, float64 throughout).

Built on oracle/spatial_oracle.py: the same tiling, neighbour masks and _send_region / _recv_region helpers.  The
forward exchange copies neighbour i's send band 8-i into this tile's pad strip i; the exact backward reverses every
such copy: the gradient in pad strip i of this tile's padded input gradient is added into neighbour i's band 8-i.
The reference drops it (SURVEY 8a N2: received strips are detached constants).

Each op returns per rank dict(exact=..., n2=..., flipped=...): the exact dx, the reference's tile-local dx, and a
deliberately wrong variant that adds strip i into band i instead of 8-i (so a test can show it has teeth).
`full_reference` gives the fp64 gradient of the same op on the unsplit image, sliced per tile, and the same op on
absolute values (the error scale A)."""
import numpy as np

from oracle import spatial_oracle as so


def conv_dgrad64(shape, w, gy, stride):
    """d(conv2d_fwd)/d(padded input) in float64."""
    sh, sw = stride
    K, C, R, S = w.shape
    Ho, Wo = gy.shape[2:]
    dxp = np.zeros(shape, dtype=np.float64)
    w64, g64 = w.astype(np.float64), gy.astype(np.float64)
    for r in range(R):
        for s in range(S):
            dxp[:, :, r:r + (Ho - 1) * sh + 1:sh, s:s + (Wo - 1) * sw + 1:sw] += np.einsum("kc,nkhw->nchw", w64[:, :, r, s], g64)
    return dxp


def pool_bwd64(xp, gy, mode, k, stride):
    """so.pool_bwd without the final fp32 rounding (max: first maximum in row-major window order)."""
    Ho, Wo = gy.shape[2:]
    dxp = np.zeros(xp.shape, dtype=np.float64)
    g64 = gy.astype(np.float64)
    sl = [(slice(None), slice(None), slice(r, r + (Ho - 1) * stride + 1, stride), slice(s, s + (Wo - 1) * stride + 1, stride))
          for r in range(k) for s in range(k)]
    if mode == "avg":
        for idx in sl:
            dxp[idx] += g64 / (k * k)
        return dxp
    arg = np.stack([xp[idx] for idx in sl], axis=0).argmax(axis=0)
    for j, idx in enumerate(sl):
        dxp[idx] += np.where(arg == j, g64, 0.0)
    return dxp


def reverse_exchange(dxps, method, hh, hw, kh=3, kw=3, flip=False):
    """dxps: per-rank padded input gradients.  Returns per-rank cropped dx with the strip gradients added into the
    neighbours' send bands (flip=True: into band i instead of 8-i -- wrong on purpose)."""
    P = len(dxps)
    acc = [d.astype(np.float64).copy() for d in dxps]
    for rank in range(P):
        mask = so.neighbour_mask(method, P, rank, kh, kw)
        nbr = so.neighbour_ranks(method, P, rank, mask)
        Hp, Wp = dxps[rank].shape[2:]
        for i in range(9):
            if not mask[i]:
                continue
            (rr0, rr1), (rc0, rc1) = so._recv_region(i, hh, hw, Hp, Wp)
            peer = acc[nbr[i]]
            e = i if flip else 8 - i
            (sr0, sr1), (sc0, sc1) = so._send_region(e, hh, hw, peer.shape[2], peer.shape[3])
            peer[:, :, sr0:sr1, sc0:sc1] += dxps[rank][:, :, rr0:rr1, rc0:rc1]
    return [so.crop(a, hh, hw) for a in acc]


def _result(dxps, method, hh, hw, kh=3, kw=3):
    exact = reverse_exchange(dxps, method, hh, hw, kh, kw)
    flipped = reverse_exchange(dxps, method, hh, hw, kh, kw, flip=True)
    return [dict(exact=exact[r].astype(np.float32), exact64=exact[r], n2=so.crop(dxps[r], hh, hw), flipped=flipped[r])
            for r in range(len(dxps))]


def conv_spatial(tiles, w, method, stride, gys):
    R, S = w.shape[2:]
    hh, hw = (R - 1) // 2, (S - 1) // 2
    padded = so.exchange_halos(tiles, method, hh, hw, kh=R, kw=S)
    dxps = [conv_dgrad64(xp.shape, w, gy, stride) for xp, gy in zip(padded, gys)]
    return _result(dxps, method, hh, hw, R, S)


def pool_spatial(tiles, method, mode, k, stride, gys):
    h = (k - 1) // 2
    padded = so.exchange_halos(tiles, method, h, h)
    return _result([pool_bwd64(xp, gy, mode, k, stride) for xp, gy in zip(padded, gys)], method, h, h)


def halo_exchange_layer(tiles, method, halo_len, gys):
    return _result([g.astype(np.float64) for g in gys], method, halo_len, halo_len)


# ---- the same ops on the unsplit image ---------------------------------------------------------------------------

def assemble(parts, method, P):
    """Per-rank output tiles -> the full-image tensor (tile outputs are disjoint slices of it)."""
    rows, cols = so.grid_shape(method, P)
    return np.concatenate([np.concatenate(parts[r * cols:(r + 1) * cols], axis=3) for r in range(rows)], axis=2)


def full_reference(op, full, gys, method, P, **kw):
    """(ref, A): per-rank slices of the float64 full-image input gradient, and of the same op on |w| and |gy|.
    op: "conv" (kw: w, stride), "pool" (kw: mode, k, stride) or "halo" (kw: halo_len)."""
    N, Cc, H, W = full.shape

    def run(absolute):
        if op == "halo":
            h = kw["halo_len"]
            acc = np.zeros((N, Cc, H + 2 * h, W + 2 * h))
            for r, g in enumerate(gys):   # the padded tiles overlap in the padded image: sum their gradients
                hs, ws = so.tile_slices(method, P, r, H, W)
                acc[:, :, hs.start:hs.stop + 2 * h, ws.start:ws.stop + 2 * h] += np.abs(g) if absolute else g
            return so.crop(acc, h, h)
        gy = assemble(gys, method, P).astype(np.float64)
        if op == "conv":
            w = kw["w"]
            R, S = w.shape[2:]
            hh, hw = (R - 1) // 2, (S - 1) // 2
            shape = (N, Cc, H + 2 * hh, W + 2 * hw)
            d = conv_dgrad64(shape, np.abs(w) if absolute else w, np.abs(gy) if absolute else gy, kw["stride"])
            return so.crop(d, hh, hw)
        k = kw["k"]
        h = (k - 1) // 2
        xp = np.pad(full.astype(np.float64), ((0, 0), (0, 0), (h, h), (h, h)))
        return so.crop(pool_bwd64(xp, np.abs(gy) if absolute else gy, kw["mode"], k, kw["stride"]), h, h)

    ref, A = run(False), run(True)
    return so.split(ref, method, P), so.split(A, method, P)
