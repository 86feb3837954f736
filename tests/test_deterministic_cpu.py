"""CPU-only: the deterministic wgrad's argument checks and workspace bound, and the scripts' --deterministic /
--enable-deterministic flags.  No GPU work: the checks fail before any launch, and spc_conv_workspace_bytes is host
arithmetic (without a device it plans for the H100 SXM's 132 SMs)."""
import ctypes as C
import importlib.util
import json
import os

import pytest

from mpi4dl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIB = 1 << 20


def _call(d, dw):
    L = _lib.lib()
    return L.spc_conv2d_wgrad_deterministic(C.byref(d), C.c_void_p(8), None, C.c_void_p(8), dw, None, 0, None, 0, None)


def test_rejects_null_dw_and_bad_dtype():
    L = _lib.lib()
    d = _lib.ConvDesc(1, 3, 8, 8, 4, 3, 3, 1, 1, 1, 1, _lib.SPC_F32, 0)
    assert _call(d, None) == -1
    assert b"null tensor pointer" in L.spc_last_error()
    d = _lib.ConvDesc(1, 3, 8, 8, 4, 3, 3, 1, 1, 1, 1, 7, 0)
    assert _call(d, C.c_void_p(8)) == -1
    assert b"dtype" in L.spc_last_error()


def _layers(fn):
    return json.load(open(os.path.join(ROOT, "tests", "golden", fn)))["layers"]


@pytest.mark.parametrize("fn", ["layers_amoebanetd_sp4.json", "layers_resnet101_sp2.json"])
def test_workspace_bound(fn):
    """op 3 - op 2 <= SPC_WGRAD_SLICE_BYTES_MAX (256 MiB) for every conv of both bench layer lists, on the whole image
    (N = 1 tile) and on a quarter of it (4 tiles), in bf16 and fp32 SPC_ALGO_TF32_STRIDED; and op 3 > 0 everywhere"""
    L = _lib.lib()
    seen = 0
    for l in _layers(fn):
        if l["op"] != "conv":
            continue
        for tiles in (1, 2):
            for dtype, algo in ((_lib.SPC_BF16, _lib.SPC_ALGO_AUTO), (_lib.SPC_F32, _lib.SPC_ALGO_TF32_STRIDED)):
                d = _lib.ConvDesc(1, l["C"], l["H"] // tiles, l["W"] // tiles, l["K"], l["R"], l["S"], l["stride_h"],
                                  l["stride_w"], l["pad_h"], l["pad_w"], dtype, algo)
                w2, w3 = L.spc_conv_workspace_bytes(C.byref(d), 2), L.spc_conv_workspace_bytes(C.byref(d), 3)
                assert 0 < w3 and w3 - w2 <= 256 * MIB + 256, (l, tiles, dtype, w2, w3)
                seen += 1
    assert seen > 0


def _load(rel):
    spec = importlib.util.spec_from_file_location(os.path.basename(rel)[:-3], os.path.join(ROOT, "benchmarks", rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("rel", ["spatial_parallelism/benchmark_sp.py",
                                 "gems_master_with_spatial_parallelism/benchmark_gems_master_with_sp.py"])
def test_training_scripts_parse_deterministic(rel):
    p = _load(rel).get_parser()
    assert p.parse_args(["--deterministic", "--recompute"]).deterministic
    assert not p.parse_args([]).deterministic


def test_halo_conv_benchmark_parses_enable_deterministic():
    p = _load("communication/halo/benchmark_sp_halo_exchange_conv.py").get_parser()
    assert p.parse_args(["--enable-deterministic"]).enable_deterministic
    assert not p.parse_args([]).enable_deterministic
