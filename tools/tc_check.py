"""GPU check of the wgmma path against a torch fp32 matmul of the same bf16 inputs (dev tool)."""
import sys, os, time
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import torch
from mpi4dl_b200 import _lib
from mpi4dl_b200.torchgems.spatial import _ConvSpatialFn

torch.manual_seed(0)
dev = "cuda:0"
cases = [(64, 128, 16, 16), (104, 208, 32, 64), (208, 52, 64, 64), (52, 208, 24, 40), (416, 416, 32, 32),
         (1664, 416, 32, 32), (416, 104, 40, 24), (104, 416, 64, 128), (16, 64, 128, 128), (8, 8, 8, 8)]
if len(sys.argv) > 1 and sys.argv[1] == "big":
    cases = [(104, 208, 4096, 4096), (208, 52, 4096, 4096), (416, 416, 1024, 1024), (1664, 416, 1024, 1024),
             (104, 416, 1024, 1024), (416, 104, 1024, 1024), (624, 416, 2048, 2048)]
ok = True
for (C, K, H, W) in cases:
    x = torch.randn(1, C, H, W, device=dev).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(K, C, 1, 1, device=dev) / C ** 0.5).to(torch.bfloat16).requires_grad_(True)
    b = torch.randn(K, device=dev).to(torch.bfloat16)
    desc = (1, C, H, W, K, 1, 1, 1, 1, 0, 0, _lib.SPC_BF16, _lib.SPC_ALGO_TCGEN05)
    y = _ConvSpatialFn.apply(x, w, b, desc, *([None] * 9))
    torch.cuda.synchronize()
    if H * W <= 1 << 20:
        ref = torch.einsum("kc,nchw->nkhw", w.float().view(K, C), x.float()) + b.float().view(1, K, 1, 1)
        err = (y.float() - ref).abs().max().item()
        scale = ref.abs().max().item()
        good = err <= 2e-2 * scale
        ok &= good
        print("fwd C=%d K=%d %dx%d  max_err %.4g (scale %.3g) %s" % (C, K, H, W, err, scale, "OK" if good else "FAIL"), flush=True)
        gy = torch.randn_like(y)
        # dgrad only (wgrad via direct kernel is slow but fine at these sizes)
        L = _lib.lib()
        import ctypes as Cc
        d = _lib.ConvDesc(*desc)
        dx = torch.empty_like(x)
        nb = L.spc_conv_workspace_bytes(Cc.byref(d), 1)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        _lib.check(L.spc_conv2d_dgrad(Cc.byref(d), Cc.c_void_p(gy.data_ptr()), Cc.c_void_p(w.data_ptr()), Cc.c_void_p(dx.data_ptr()),
                                      Cc.c_void_p(ws.data_ptr()), nb, Cc.c_void_p(torch.cuda.current_stream().cuda_stream)), "dgrad")
        torch.cuda.synchronize()
        refdx = torch.einsum("kc,nkhw->nchw", w.float().view(K, C), gy.float())
        err = (dx.float() - refdx).abs().max().item()
        scale = refdx.abs().max().item()
        good = err <= 2e-2 * scale
        ok &= good
        print("dgrad                       max_err %.4g (scale %.3g) %s" % (err, scale, "OK" if good else "FAIL"), flush=True)
        dw = torch.empty(K, C, dtype=torch.float32, device=dev)
        nb = L.spc_conv_workspace_bytes(Cc.byref(d), 2)
        ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=dev)
        _lib.check(L.spc_conv2d_wgrad(Cc.byref(d), Cc.c_void_p(x.data_ptr()), None, Cc.c_void_p(gy.data_ptr()), Cc.c_void_p(dw.data_ptr()), None, 0,
                                      Cc.c_void_p(ws.data_ptr()), nb, Cc.c_void_p(torch.cuda.current_stream().cuda_stream)), "wgrad")
        torch.cuda.synchronize()
        refdw = torch.einsum("nkhw,nchw->kc", gy.float(), x.float())
        err = (dw - refdw).abs().max().item()
        scale = refdw.abs().max().item()
        good = err <= 2e-3 * scale
        ok &= good
        print("wgrad                       max_err %.4g (scale %.3g) %s" % (err, scale, "OK" if good else "FAIL"), flush=True)
    else:
        # timing
        with torch.no_grad():
            for _ in range(3):
                y = _ConvSpatialFn.apply(x.detach(), w.detach(), None, desc, *([None] * 9))
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                y = _ConvSpatialFn.apply(x.detach(), w.detach(), None, desc, *([None] * 9))
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
        byts = (C + K) * H * W * 2
        fl = 2.0 * C * K * H * W
        # spot check a slab
        ref = torch.einsum("kc,nchw->nkhw", w.float().view(K, C), x[:, :, :8].float())
        err = (y[:, :, :8].float() - ref).abs().max().item()
        print("fwd C=%d K=%d %dx%d  %.3f ms  %.0f GB/s  %.0f TF/s  spot_err %.3g" % (C, K, H, W, ms, byts / ms / 1e6, fl / ms / 1e9, err), flush=True)
        import ctypes as Cc
        L = _lib.lib()
        d = _lib.ConvDesc(*desc)
        gy = torch.randn_like(y)
        dx = torch.empty_like(x)
        dw = torch.zeros(K, C, dtype=torch.float32, device=dev)
        nb1 = L.spc_conv_workspace_bytes(Cc.byref(d), 1)
        ws = torch.empty(max(nb1, 16), dtype=torch.uint8, device=dev)
        sp = Cc.c_void_p(torch.cuda.current_stream().cuda_stream)
        def dg():
            _lib.check(L.spc_conv2d_dgrad(Cc.byref(d), Cc.c_void_p(gy.data_ptr()), Cc.c_void_p(w.data_ptr()), Cc.c_void_p(dx.data_ptr()), Cc.c_void_p(ws.data_ptr()), nb1, sp), "dgrad")
        def wg():
            _lib.check(L.spc_conv2d_wgrad(Cc.byref(d), Cc.c_void_p(x.data_ptr()), None, Cc.c_void_p(gy.data_ptr()), Cc.c_void_p(dw.data_ptr()), None, 0, None, 0, sp), "wgrad")
        for nm, fn in (("dgrad", dg), ("wgrad", wg)):
            fn(); fn(); torch.cuda.synchronize()
            e0.record()
            for _ in range(5): fn()
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            print("   %s %.3f ms  %.0f GB/s  %.0f TF/s" % (nm, ms, byts / ms / 1e6, fl / ms / 1e9), flush=True)
        refdw = torch.einsum("nkhw,nchw->kc", gy[:, :, :64].float(), x[:, :, :64].float())
        # full check of wgrad on a cropped problem is not possible; check dw magnitude sanity only
        print("   dw abs max %.3g" % dw.abs().max().item(), flush=True)
# multi-tap convs vs cuDNN fp32 (dev check only)
import torch.nn.functional as F
taps = [(52, 52, 1, 7, 32, 128), (104, 104, 7, 1, 32, 64), (104, 104, 3, 3, 16, 128), (64, 16, 3, 3, 8, 192)]
if len(sys.argv) > 1 and sys.argv[1] == "big":
    taps = [(104, 104, 1, 7, 1024, 1024), (104, 104, 7, 1, 1024, 1024), (52, 52, 1, 7, 2048, 2048), (64, 16, 3, 3, 4096, 4096)]
torch.backends.cudnn.allow_tf32 = False
for (C, K, R, S, H, W) in taps:
    x = torch.randn(1, C, H, W, device=dev).to(torch.bfloat16)
    w = (torch.randn(K, C, R, S, device=dev) / (C * R * S) ** 0.5).to(torch.bfloat16)
    desc = (1, C, H, W, K, R, S, 1, 1, (R - 1) // 2, (S - 1) // 2, _lib.SPC_BF16, _lib.SPC_ALGO_TCGEN05)
    with torch.no_grad():
        y = _ConvSpatialFn.apply(x, w, None, desc, *([None] * 9))
        torch.cuda.synchronize()
        hs = min(H, 64)
        ref = F.conv2d(x[:, :, :hs + R].float(), w.float(), None, 1, ((R - 1) // 2, (S - 1) // 2))[:, :, :hs]
        err = (y[:, :, :hs].float() - ref).abs().max().item()
        scale = ref.abs().max().item()
        good = err <= 2e-2 * scale
        ok &= good
        import ctypes as Cc
        L = _lib.lib(); d = _lib.ConvDesc(*desc)
        gy = torch.randn_like(y); dx = torch.empty_like(x)
        nb1 = L.spc_conv_workspace_bytes(Cc.byref(d), 1)
        ws = torch.empty(max(nb1, 16), dtype=torch.uint8, device=dev)
        sp = Cc.c_void_p(torch.cuda.current_stream().cuda_stream)
        def dg():
            _lib.check(L.spc_conv2d_dgrad(Cc.byref(d), Cc.c_void_p(gy.data_ptr()), Cc.c_void_p(w.data_ptr()), Cc.c_void_p(dx.data_ptr()), Cc.c_void_p(ws.data_ptr()), nb1, sp), "dgrad")
        dg(); torch.cuda.synchronize()
        refdx = F.conv_transpose2d(gy[:, :, :hs + R].float(), w.float(), None, 1, ((R - 1) // 2, (S - 1) // 2))[:, :, :hs]
        e2 = (dx[:, :, :hs].float() - refdx).abs().max().item(); s2 = refdx.abs().max().item()
        good2 = e2 <= 2e-2 * s2
        ok &= good2
        def fw():
            return _ConvSpatialFn.apply(x, w, None, desc, *([None] * 9))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        res = []
        for fn in (fw, dg):
            fn(); torch.cuda.synchronize(); e0.record()
            for _ in range(3): fn()
            e1.record(); torch.cuda.synchronize(); res.append(e0.elapsed_time(e1) / 3)
        fl = 2.0 * C * K * R * S * H * W
        print("tap C=%d K=%d %dx%d @%dx%d fwd err %.3g/%.3g %s  dgrad err %.3g/%.3g %s | fwd %.3f ms %.0f TF/s dgrad %.3f ms %.0f TF/s" % (
            C, K, R, S, H, W, err, scale, "OK" if good else "FAIL", e2, s2, "OK" if good2 else "FAIL", res[0], fl / res[0] / 1e9, res[1], fl / res[1] / 1e9), flush=True)
print("ALL OK" if ok else "SOME FAILED")
