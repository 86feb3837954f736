"""CPU-only: libspconv.so loads and exports exactly the spc_* symbols include/spconv.h declares; argument
validation works without a GPU (no compute calls here)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from mpi4dl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "spconv.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(spc_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    names = _declared()
    assert len(names) >= 20
    bound = {s[0] for s in _lib.SYMBOLS}
    for n in names:
        assert hasattr(L, n), "libspconv.so does not export %s" % n
        assert n in bound, "%s is declared in spconv.h but not bound in _lib.py" % n
    assert bound == set(names)


def test_library_exports_only_declared_symbols():
    """an entry point removed from spconv.h does not stay behind as an undeclared export"""
    if shutil.which("nm") is None:
        pytest.skip("nm (binutils) is not installed")
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {ln.split()[-1] for ln in out.splitlines() if ln.split() and ln.split()[-1].startswith("spc_")}
    assert exported == set(_declared()), "exported but not declared: %s; declared but not exported: %s" % (
        sorted(exported - set(_declared())), sorted(set(_declared()) - exported))


def test_version_102_and_structs():
    """SPC_VERSION 102: the immediate-mode halo protocol (spc_halo_post / spc_halo_collect, spc_mailbox_signal /
    spc_mailbox_wait) and spc_reload_env are gone"""
    L = _lib.lib()
    assert L.spc_version() == 102
    assert C.sizeof(_lib.ConvDesc) == 13 * 4
    assert C.sizeof(_lib.PoolDesc) == 9 * 4
    assert C.sizeof(_lib.Halo) == 9 * C.sizeof(C.c_void_p)


def test_argument_validation_needs_no_gpu():
    L = _lib.lib()
    # "same" padding rule of the reference (spatial.py:119-121)
    d = _lib.ConvDesc(1, 3, 8, 8, 4, 3, 3, 1, 1, 0, 0, _lib.SPC_F32, 0)
    rc = L.spc_conv2d_fwd(C.byref(d), C.c_void_p(8), None, C.c_void_p(8), None, C.c_void_p(8), None, 0, None)
    assert rc == -1
    assert b"Spatial not supported yet" in L.spc_last_error()
    d = _lib.ConvDesc(1, 3, 8, 8, 4, 3, 3, 1, 1, 1, 1, 7, 0)
    assert L.spc_conv2d_fwd(C.byref(d), C.c_void_p(8), None, C.c_void_p(8), None, C.c_void_p(8), None, 0, None) == -1
    assert b"dtype" in L.spc_last_error()
    p = _lib.PoolDesc(1, 3, 8, 8, 3, 1, 0, _lib.SPC_POOL_AVG, _lib.SPC_F32)
    assert L.spc_pool2d_fwd(C.byref(p), C.c_void_p(8), None, C.c_void_p(8), None) == -1
    ho, wo = C.c_int(), C.c_int()
    d = _lib.ConvDesc(1, 3, 16, 32, 4, 3, 3, 2, 2, 1, 1, _lib.SPC_F32, 0)
    L.spc_conv_out_shape(C.byref(d), C.byref(ho), C.byref(wo))
    assert (ho.value, wo.value) == (8, 16)
