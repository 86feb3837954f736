"""Fused BatchNorm2d (+ ReLU) for the cells of a spatial stage (SURVEY 8f-2), on libspconv (csrc/bnrelu.cu).

The reference's spatial cells are eager chains  ReLU -> conv -> nn.BatchNorm2d  (src/models/amoebanet.py:365-398)
with plain, per-tile batch statistics (SURVEY 8a N4: not synchronised over the tiles).  `bn_relu` computes the
same training-mode BatchNorm2d -- batch statistics of the local tensor, biased variance for normalisation,
unbiased for running_var, momentum update of the running buffers -- and, when asked, the ReLU that FOLLOWS it
in the chain, in one pass over HBM each way instead of three (stats, apply, relu) / five (backward).
`relu_conv_bn_chain` is the drop-in forward for the  [ReLU, conv, BN] * k  Sequential of a spatial cell: same
submodules, same state-dict keys, same numerics up to rounding (the BN output feeding a ReLU is rounded once, not
twice).  Eval mode, non-CUDA tensors, H*W not a multiple of 8 and misaligned views take the module's own
PyTorch path.
"""
import ctypes as C

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _workspace(L, N, Cc, HW, device):
    """per-(plane, chunk) partials of spc_bn_stats / spc_bn_bwd_reduce"""
    n = L.spc_bn_workspace_bytes(N, Cc, HW)
    ws = torch.empty(n, dtype=torch.uint8, device=device)
    return ws, C.c_void_p(ws.data_ptr()), n


class _BnReluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, gamma, beta, eps, relu, stats_out):
        L = _lib.lib()
        y = y.contiguous()
        N, Cc, H, W = y.shape
        HW = H * W
        code = _lib.dtype_code(y.dtype)
        st = torch.empty(2, Cc, dtype=torch.float32, device=y.device)
        mean, var = st[0], st[1]                                   # var: biased (normalisation)
        ws, wsp, nws = _workspace(L, N, Cc, HW, y.device)
        _lib.check(L.spc_bn_stats(N, Cc, HW, code, _p(y), _p(mean), _p(var), wsp, nws, _st()), "spc_bn_stats")
        m = float(N * HW)
        rstd = torch.rsqrt(var + eps)
        g32 = gamma.detach().float().contiguous() if gamma is not None else torch.ones(Cc, device=y.device)
        b32 = beta.detach().float().contiguous() if beta is not None else torch.zeros(Cc, device=y.device)
        z = torch.empty_like(y)
        _lib.check(L.spc_bn_apply(N, Cc, HW, code, _p(y), _p(mean), _p(rstd), _p(g32), _p(b32), int(relu), _p(z), _st()),
                   "spc_bn_apply")
        stats_out.append((mean, var, m))
        ctx.save_for_backward(y, mean, rstd, g32, b32)
        ctx.relu = bool(relu)
        ctx.has_affine = gamma is not None
        ctx.param_dtype = gamma.dtype if gamma is not None else None
        return z

    @staticmethod
    def backward(ctx, dz):
        L = _lib.lib()
        y, mean, rstd, g32, b32 = ctx.saved_tensors
        dz = dz.contiguous()
        if dz.data_ptr() % 16:                                     # the kernels read 16-byte vectors
            dz = dz.clone()
        N, Cc, H, W = y.shape
        HW = H * W
        code = _lib.dtype_code(y.dtype)
        d = torch.empty(2, Cc, dtype=torch.float32, device=y.device)
        ws, wsp, nws = _workspace(L, N, Cc, HW, y.device)
        _lib.check(L.spc_bn_bwd_reduce(N, Cc, HW, code, _p(dz), _p(y), _p(mean), _p(rstd), _p(g32), _p(b32), int(ctx.relu),
                                       _p(d[0]), _p(d[1]), wsp, nws, _st()), "spc_bn_bwd_reduce")
        dy = None
        if ctx.needs_input_grad[0]:
            dy = torch.empty_like(y)
            _lib.check(L.spc_bn_bwd_apply(N, Cc, HW, code, _p(dz), _p(y), _p(mean), _p(rstd), _p(g32), _p(b32), int(ctx.relu),
                                          _p(d[0]), _p(d[1]), _p(dy), _st()), "spc_bn_bwd_apply")
        dgamma = d[1].to(ctx.param_dtype) if ctx.has_affine and ctx.needs_input_grad[1] else None
        dbeta = d[0].to(ctx.param_dtype) if ctx.has_affine and ctx.needs_input_grad[2] else None
        return dy, dgamma, dbeta, None, None, None


def fusable(x, bn):
    """The kernels read and write 16-byte vectors: a contiguous view whose storage offset breaks that alignment (the
    kernels would read it in place) takes the module's path."""
    return (isinstance(bn, nn.BatchNorm2d) and bn.training and x.is_cuda and x.dim() == 4 and
            (x.shape[2] * x.shape[3]) % 8 == 0 and x.dtype in (torch.float32, torch.bfloat16) and x.numel() > 0 and
            (x.data_ptr() % 16 == 0 or not x.is_contiguous()))


def bn_relu(x, bn, relu=False):
    """relu?(bn(x)) for a training-mode nn.BatchNorm2d `bn` (its parameters and running buffers are used and
    updated exactly as the module would); falls back to the module (+ F.relu) when not fusable."""
    if not fusable(x, bn):
        z = bn(x)
        return F.relu(z) if relu else z
    stats = []
    z = _BnReluFn.apply(x, bn.weight, bn.bias, bn.eps, relu, stats)
    if bn.track_running_stats and bn.running_mean is not None:
        mean, var, m = stats[0]
        with torch.no_grad():
            bn.num_batches_tracked += 1
            # momentum=None (cumulative average): the factor 1 / num_batches_tracked stays on the device -- reading
            # the counter on the host would synchronise, which a CUDA-graph capture forbids
            mom = bn.momentum if bn.momentum is not None else 1.0 / bn.num_batches_tracked.double()
            unbiased = var * (m / max(m - 1.0, 1.0))
            if bn.momentum is not None:
                bn.running_mean.mul_(1 - mom).add_(mean.to(bn.running_mean.dtype), alpha=mom)
                bn.running_var.mul_(1 - mom).add_(unbiased.to(bn.running_var.dtype), alpha=mom)
            else:
                keep, mom = (1 - mom).to(bn.running_mean.dtype), mom.to(bn.running_mean.dtype)
                bn.running_mean.mul_(keep).addcmul_(mean.to(bn.running_mean.dtype), mom)
                bn.running_var.mul_(keep).addcmul_(unbiased.to(bn.running_var.dtype), mom)
    return z


class relu_conv_bn_chain(nn.Sequential):
    """[ReLU, conv, BatchNorm2d] * k as ONE module with the Sequential's children and keys ("0", "1", "2", ...).
    forward: the first ReLU runs as it is; every BatchNorm2d is fused with the ReLU of the NEXT triple."""

    def forward(self, x):
        mods = list(self)
        assert len(mods) % 3 == 0
        x = mods[0](x)
        for i in range(0, len(mods), 3):
            conv, bn = mods[i + 1], mods[i + 2]
            last = i + 3 >= len(mods)
            x = bn_relu(conv(x), bn, relu=not last)
        return x
