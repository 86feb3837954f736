"""torchgems.graphs -- run a spatial stage's forward and backward from captured CUDA graphs.

    graph_stage(module, sample_inputs, *, amp_dtype=None)   warm up, capture and return a GraphedStage
    GraphedStage(x, part_number)                            the stage's forward for micro-batch `part_number`,
                                                            replayed; its backward replays the captured backward

On small tiles the eager step of a spatial stage is bound by host time: every ctypes call, autograd node and
allocation is launched from the host.  A GraphedStage captures, per micro-batch slot, one forward graph and one
backward graph of the whole stage (cells, fused BatchNorm, halo exchanges, recompute, autocast, exact backward,
deterministic wgrad) and replays them; the step then launches two graphs per micro-batch instead of thousands of
kernels.  What the capture needs, and why:

* Warm-up.  Capture records launches without running them, so everything a first call does on the host has to
  happen before it: the peer transport's IPC handle and slot-offset swaps with each neighbour (`PeerTransport._peer`
  / `_peer_slot`, forward and reverse slots), the transport's launch plans, the lazy module loads.  graph_stage runs
  WARMUP eager forwards + backwards first.  They update the BatchNorm running buffers, which are saved before and
  restored after (recompute.save_batchnorm_buffers), so step 1 of a graphed run equals step 1 of an eager one.  They
  also advance the device-side sequence numbers of the halo slots; that is harmless only because every tile of the
  stage warms up the same number of times, in the same order, so the tiles' slots stay paired.
* No host work inside the captured region: fused.bn_relu keeps the momentum=None factor on the device, and the
  recompute's checkpoint does not save the RNG state (neither is allowed during capture).
* Transport.  Only the peer transport exchanges from the device with fixed launch arguments; a stage that would
  exchange through DistTransport (host-driven torch.distributed P2P) is refused when it is built.
* Autocast is entered with cache_enabled=False (a cached cast would outlive the capture).  The bf16 weight casts of
  conv_spatial happen inside _ConvSpatialFn, so they are captured and read the fp32 masters the optimizer updates
  in place.
* Static buffers.  The input is copied into the slot's static input, the output is the slot's static output
  (valid until the slot's next forward), and the incoming gradient is copied into the static output gradient.
  The replayed backward returns the parameter and input gradients, and autograd accumulates them into `.grad`
  exactly as it accumulates an eager backward's (also into the flat-buffer views of train_spatial_model_master).
* Memory pools.  GPipe runs all forwards, then backwards 0..parts-1 -- not in the reverse order a shared pool would
  need.  So each micro-batch slot has a private pool, shared only by its own forward and backward graph, which
  are captured in the order they replay.
* Frozen configuration.  A capture freezes what the eager path reads at call time: each layer's `algo` and
  `exact_backward`, SPCONV_HALO_OVERLAP, torch.are_deterministic_algorithms_enabled(), and the input's shape, dtype
  and requires_grad.  A call that differs in any of them, or that runs without grad mode, raises; nothing is
  captured again behind the caller's back.
"""
import os

import torch
import torch.nn as nn

from . import halo_transport, spatial
from .recompute import restore_batchnorm_buffers, save_batchnorm_buffers

WARMUP = 2


class GraphCaptureError(RuntimeError):
    pass


def _tensors(x):
    return list(x) if isinstance(x, (tuple, list)) else [x]


def _rebuild(flat, is_tuple):
    return tuple(flat) if is_tuple else flat[0]


def has_spatial_layer(module):
    return any(isinstance(m, spatial._SpatialTopology) for m in module.modules())


def _exchanges(module):
    """True when a layer of `module` exchanges halos with a neighbour tile."""
    return any(isinstance(m, spatial._SpatialTopology) and m.neighbours is not None and any(m.neighbours)
               for m in module.modules())


def check_graphable(module):
    """Raise, before any work, when `module` cannot run from CUDA graphs: no CUDA device, a DistributedDataParallel
    wrapper (its hooks run on the host between the graphs' kernels), or halo exchanges through DistTransport."""
    if not torch.cuda.is_available():
        raise GraphCaptureError("cuda_graph=True needs a CUDA device")
    if isinstance(module, nn.parallel.DistributedDataParallel):
        raise GraphCaptureError("cuda_graph=True: a DistributedDataParallel-wrapped stage cannot be captured")
    if _exchanges(module) and (os.environ.get("SPCONV_HALO_TRANSPORT") == "dist" or
                               isinstance(halo_transport._transport, halo_transport.DistTransport)):
        raise GraphCaptureError("cuda_graph=True: this stage exchanges halos through DistTransport (torch.distributed "
                                "P2P, driven from the host), which cannot be captured; use the peer transport")


def _frozen_config(module):
    """What the eager path reads at call time and a capture freezes."""
    layers = tuple((getattr(m, "algo", None), getattr(m, "exact_backward", None)) for m in module.modules()
                   if hasattr(m, "algo") or hasattr(m, "exact_backward"))
    return layers, halo_transport.overlap_enabled(), torch.are_deterministic_algorithms_enabled()


def _autocast(amp_dtype):
    return torch.autocast("cuda", dtype=amp_dtype or torch.bfloat16, enabled=amp_dtype is not None, cache_enabled=False)


class _Slot:
    """Static buffers and the forward / backward graphs of one micro-batch."""

    def __init__(self, sample):
        self.in_tuple = isinstance(sample, (tuple, list))
        self.static_in = [t.detach().clone().requires_grad_(t.requires_grad) for t in _tensors(sample)]
        self.meta = [(tuple(t.shape), t.dtype, t.requires_grad) for t in self.static_in]

    def capture(self, module, params, amp_dtype):
        self.fwd, self.bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with _autocast(amp_dtype):
            with torch.cuda.graph(self.fwd):
                res = module(_rebuild(self.static_in, self.in_tuple))
        self.out_tuple = isinstance(res, (tuple, list))
        outs = _tensors(res)
        del res
        self.static_out = [o.detach() for o in outs]
        diff = [i for i, o in enumerate(outs) if o.requires_grad]
        self.grad_out = [torch.empty_like(o) if o.requires_grad else None for o in outs]
        wrt = [t for t in self.static_in if t.requires_grad] + params
        with torch.cuda.graph(self.bwd, pool=self.fwd.pool()):
            grads = torch.autograd.grad([outs[i] for i in diff], wrt, [self.grad_out[i] for i in diff],
                                        allow_unused=True)
        it = iter(grads)
        # held here for the slot's lifetime: autograd then copies them into an empty .grad instead of adopting the
        # static buffer that the next replay overwrites
        self.static_grads = [next(it) if t.requires_grad else None for t in self.static_in] + list(it)


class _ReplayFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, slot, n_in, *args):
        for dst, src in zip(slot.static_in, args[:n_in]):
            if dst.data_ptr() != src.data_ptr():
                dst.detach().copy_(src)
        slot.fwd.replay()
        ctx.slot = slot
        return tuple(o.detach() for o in slot.static_out)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, *grads):
        slot = ctx.slot
        for dst, g in zip(slot.grad_out, grads):
            if dst is not None:
                if g is None:
                    dst.zero_()
                else:
                    dst.copy_(g)
        slot.bwd.replay()
        return (None, None) + tuple(slot.static_grads)


class GraphedStage:
    """Callable returned by graph_stage: stage(x, part_number) replays micro-batch `part_number`'s forward."""

    def __init__(self, module, slots, params, config):
        self.module, self.slots, self.params, self.config = module, slots, params, config

    def __call__(self, x, part_number=0):
        slot = self.slots[part_number]
        flat = _tensors(x)
        if not torch.is_grad_enabled():
            raise GraphCaptureError("graphed stage: called without grad mode, but the stage was captured for training "
                                    "(forward and backward); run the module itself under torch.no_grad()")
        meta = [(tuple(t.shape), t.dtype, t.requires_grad) for t in flat]
        if meta != slot.meta:
            raise GraphCaptureError("graphed stage, micro-batch %d: input (shape, dtype, requires_grad) %s differs from "
                                    "the capture's %s" % (part_number, meta, slot.meta))
        if _frozen_config(self.module) != self.config:
            raise GraphCaptureError("graphed stage: a layer's algo / exact_backward, SPCONV_HALO_OVERLAP or "
                                    "torch.are_deterministic_algorithms_enabled() changed since the capture")
        outs = _ReplayFn.apply(slot, len(flat), *flat, *self.params)
        return _rebuild(list(outs), slot.out_tuple)


def graph_stage(module, sample_inputs, *, amp_dtype=None, warmup=WARMUP):
    """Capture `module` (a spatial stage in training mode) once per entry of `sample_inputs` (one per micro-batch:
    a tensor or a tuple of tensors of the shape, dtype and requires_grad the calls will pass) and return a
    GraphedStage.  amp_dtype=torch.bfloat16 captures the forward under torch.autocast.  COLLECTIVE over the tiles of
    the stage: each of them must call it at the same point, with the same number of samples."""
    check_graphable(module)
    sample_inputs = list(sample_inputs)
    if not sample_inputs:
        raise ValueError("graph_stage: no sample inputs")
    dev = _tensors(sample_inputs[0])[0].device
    if _exchanges(module) and isinstance(halo_transport.get_transport(dev), halo_transport.DistTransport):
        raise GraphCaptureError("graph_stage: this stage exchanges halos through DistTransport (torch.distributed "
                                "P2P, driven from the host), which cannot be captured; use the peer transport")
    params = [p for p in module.parameters() if p.requires_grad]
    slots = [_Slot(s) for s in sample_inputs]
    saved = save_batchnorm_buffers(module)
    try:
        s0 = slots[0]
        for _ in range(warmup):
            with _autocast(amp_dtype):
                outs = [o for o in _tensors(module(_rebuild(s0.static_in, s0.in_tuple))) if o.requires_grad]
            wrt = [t for t in s0.static_in if t.requires_grad] + params
            torch.autograd.grad(outs, wrt, [torch.ones_like(o) for o in outs], allow_unused=True)
            del outs
        torch.cuda.synchronize()
        for s in slots:
            s.capture(module, params, amp_dtype)
        torch.cuda.synchronize()
    finally:
        restore_batchnorm_buffers(saved)
    return GraphedStage(module, slots, params, _frozen_config(module))
