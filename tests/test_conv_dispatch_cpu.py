"""CPU-only: the convolution path libspconv picks for each op and the workspace it asks for match
tests/golden/conv_dispatch.npz (tools/gen_conv_dispatch_golden.py) row for row, and SPC_ALGO_TCGEN05 rejects the
same fprop / dgrad shapes before any launch.  Host arithmetic only: without a device the library plans for the H100
SXM's 132 SMs, as the golden was recorded."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

from mpi4dl_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tool():
    path = os.path.join(ROOT, "tools", "gen_conv_dispatch_golden.py")
    spec = importlib.util.spec_from_file_location("gen_conv_dispatch_golden", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _device_sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else None


def test_conv_dispatch_matches_golden():
    sms = _device_sms()
    if sms is not None and sms != 132:
        pytest.skip("the golden plans for 132 SMs; this device has %d" % sms)
    tool = _tool()
    L = _lib.lib()
    g = np.load(os.path.join(ROOT, "tests", "golden", "conv_dispatch.npz"))
    assert len(g["desc"]) > 5000
    bad = []
    for desc, uses, ws, rc in zip(g["desc"], g["uses"], g["ws"], g["rc"]):
        # fprop / dgrad are called only where this library has no tensor-core path: SPC_ALGO_TCGEN05 rejects those
        # before any launch
        got = tool.row(L, _lib.ConvDesc(*map(int, desc)))
        want = (list(map(int, uses)), list(map(int, ws)), list(map(int, rc)))
        if tuple(got) != want:
            bad.append((list(map(int, desc)), want, got))
    assert not bad, "%d of %d descriptors differ, first: %s: want %s got %s" % (len(bad), len(g["desc"]), *bad[0])
