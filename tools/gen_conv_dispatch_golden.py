"""Record libspconv's host-side convolution decisions for a grid of descriptors:

    python tools/gen_conv_dispatch_golden.py path/to/libspconv.so [out.json]

For every descriptor it stores spc_conv_uses_tcgen05(d, 0..2), spc_conv_workspace_bytes(d, 0..3) and, under
SPC_ALGO_TCGEN05, the return code of spc_conv2d_fwd / spc_conv2d_dgrad on the ops that have no tensor-core path (those
reject the call before any launch, so dummy pointers do).  All of it is host arithmetic; without a device the library
plans for the H100 SXM's 132 SMs.  tests/test_conv_dispatch_cpu.py checks the built library against the result
(default: tests/golden/conv_dispatch.npz), so a change to the path decision or to a workspace formula shows up there.

Grid: every conv of the two bench layer lists at 1 and 2 tiles per side and N in {1, 4}, and synthetic shapes on both
sides of each predicate of the path choice (filter, stride, W % 4 / 8 / 32 / 64, odd H, H*W / stride^2 % 8, few
channels, output-channel counts, the 24 GiB workspace cut of the bf16 tap path), each under bf16 AUTO / DIRECT /
TCGEN05 and fp32 AUTO / DIRECT / TF32 / TF32_ALL / TF32_STRIDED / TCGEN05.

Output arrays, one row per descriptor: desc (the spc_conv_desc fields), uses (ops 0..2), ws (ops 0..3) and rc (fprop,
dgrad; 1 where the call was not made because it would launch -- the library's return codes are <= 0).
"""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "conv_dispatch.npz")
NOT_CALLED = 1
FIELDS = ("N", "C", "H", "W", "K", "R", "S", "stride_h", "stride_w", "pad_h", "pad_w", "dtype", "algo")
SPC_F32, SPC_BF16 = 0, 1
AUTO, DIRECT, TCGEN05, TF32, TF32_ALL, TF32_STRIDED = range(6)
ALGOS = [(SPC_BF16, a) for a in (AUTO, DIRECT, TCGEN05)] + \
        [(SPC_F32, a) for a in (AUTO, DIRECT, TF32, TF32_ALL, TF32_STRIDED, TCGEN05)]


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in FIELDS]


def shapes():
    """(N, C, H, W, K, R, S, stride) of the grid, without the dtype / algo"""
    out = []
    for fn in ("layers_amoebanetd_sp4.json", "layers_resnet101_sp2.json"):
        for l in json.load(open(os.path.join(ROOT, "tests", "golden", fn)))["layers"]:
            if l["op"] != "conv":
                continue
            for tiles in (1, 2):
                for n in (1, 4):
                    out.append((n, l["C"], l["H"] // tiles, l["W"] // tiles, l["K"], l["R"], l["S"], l["stride_h"]))
    filters = [(1, 1), (3, 3), (5, 5), (7, 7), (1, 7), (7, 1)]
    for r, s in filters:
        for stride in (1, 2):
            for h in (32, 33):
                for w in (32, 36, 40, 60, 62, 64, 96, 128):
                    out.append((1, 64, h, w, 104, r, s, stride))
            for c in (3, 8, 64, 256):
                for k in (16, 52, 104, 128, 208, 300):
                    out.append((4 if k in (16, 208) else 1, c, 64, 64, k, r, s, stride))
    # 1x1: H*W / stride^2 on and off a multiple of 8, W on and off a multiple of 32
    for h, w in ((2, 32), (6, 32), (10, 96), (3, 8), (3, 6), (5, 5), (34, 48), (2, 16)):
        for stride in (1, 2):
            out.append((1, 16, h, w, 32, 1, 1, stride))
    # the bf16 tap path's 24 GiB workspace cut (shifted copies of a 3x3 layer of 256 channels)
    for hw in (1024, 2048, 2560):
        for n in (1, 4):
            out.append((n, 256, hw, hw, 256, 3, 3, 1))
    return sorted(set(out))


def record(lib_path):
    L = C.CDLL(os.path.abspath(lib_path))
    L.spc_conv_uses_tcgen05.restype = C.c_int
    L.spc_conv_uses_tcgen05.argtypes = [C.POINTER(ConvDesc), C.c_int]
    L.spc_conv_workspace_bytes.restype = C.c_size_t
    L.spc_conv_workspace_bytes.argtypes = [C.POINTER(ConvDesc), C.c_int]
    desc, uses, ws, rc = [], [], [], []
    for n, c, h, w, k, r, s, stride in shapes():
        for dtype, algo in ALGOS:
            d = ConvDesc(n, c, h, w, k, r, s, stride, stride, (r - 1) // 2, (s - 1) // 2, dtype, algo)
            u, b, e = row(L, d)
            desc.append([getattr(d, f) for f in FIELDS]); uses.append(u); ws.append(b); rc.append(e)
    return dict(desc=np.array(desc, np.int32), uses=np.array(uses, np.int8), ws=np.array(ws, np.int64),
                rc=np.array(rc, np.int8))


def row(L, d):
    """(uses of ops 0..2, workspace of ops 0..3, fprop and dgrad rc) of descriptor d"""
    uses = [L.spc_conv_uses_tcgen05(C.byref(d), op) for op in range(3)]
    ws = [L.spc_conv_workspace_bytes(C.byref(d), op) for op in range(4)]
    rcs = [NOT_CALLED, NOT_CALLED]
    if d.algo == TCGEN05:
        p = C.c_void_p(8)
        if not uses[0]:
            rcs[0] = L.spc_conv2d_fwd(C.byref(d), p, None, p, None, p, None, C.c_size_t(0), None)
        if not uses[1]:
            rcs[1] = L.spc_conv2d_dgrad(C.byref(d), p, p, p, None, C.c_size_t(0), None)
    return uses, ws, rcs


def main():
    if len(sys.argv) < 2:
        sys.exit(__doc__)
    out = sys.argv[2] if len(sys.argv) > 2 else OUT
    golden = record(sys.argv[1])
    np.savez_compressed(out, **golden)
    print("%d descriptors -> %s" % (len(golden["desc"]), out))


if __name__ == "__main__":
    main()
