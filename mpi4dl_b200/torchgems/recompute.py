"""torchgems.recompute -- activation checkpointing for the cells of a spatial stage.

    checkpoint_spatial_cells(model)   keep only each spatial cell's input (and its received halo strips) for
                                      backward, and run the cell's forward a second time in backward

A spatial layer keeps its whole input tile for backward, and so do the BatchNorm / ReLU around it; at a 4096^2 tile
that, not compute, decides how many GPUs a stage needs.  Each checkpointed cell runs under non-reentrant
torch.utils.checkpoint with a per-call `_HaloRecorder`:

* forward (grad enabled): every halo exchange inside the cell runs as usual, and the 9 strips it received are
  appended to the recorder (spatial._SpatialTopology._exchange, the one place every spatial layer exchanges).
* recompute (in backward): the exchanges take the recorded strips back in the same order and call no transport.
  The recompute therefore moves no halo bytes, and cannot pair a peer-transport slot with a neighbour that
  recomputes its cells in another order.  The exact backward's reverse exchanges run in the backward of the
  recomputed graph, in autograd order, as they do without recompute.
* BatchNorm: the running buffers of the cell's BatchNorm modules (fused bn_relu or plain nn.BatchNorm2d) are
  saved when the recompute starts and put back when it ends, so they get one update per real forward.  The batch
  statistics the recompute uses are the forward's: same kernels, same input.

The recorder lives in the checkpoint call's context_fn closure, so its strips are freed with the graph, also when
no backward runs.  Under torch.no_grad() a cell runs its plain forward and records nothing.
"""
import types

import torch
import torch.nn as nn
from torch.nn.modules.batchnorm import _BatchNorm
from torch.utils.checkpoint import checkpoint

from . import spatial


class _HaloRecorder:
    """Received halo strips of one checkpointed cell call, in exchange order."""

    def __init__(self, module):
        self.module = module
        self.strips = []
        self.replaying = False
        self._pos = 0

    def record(self, strips):
        self.strips.append(strips)

    def replay(self, x, hh, hw):
        if self._pos >= len(self.strips):
            raise RuntimeError("recompute: the cell's recompute exchanges more halos than its forward did (%d)"
                               % len(self.strips))
        strips = self.strips[self._pos]
        self._pos += 1
        N, Cc, H, W = x.shape
        for i, s in enumerate(strips):
            if s is not None and (tuple(s.shape) != spatial._strip_shape(i, N, Cc, H, W, hh, hw) or s.dtype != x.dtype):
                raise RuntimeError("recompute: recorded halo strip %d is %s %s, the recompute needs %s %s" % (
                    i, tuple(s.shape), s.dtype, spatial._strip_shape(i, N, Cc, H, W, hh, hw), x.dtype))
        return strips

    def nbytes(self):
        return sum(s.numel() * s.element_size() for strips in self.strips for s in strips if s is not None)

    def contexts(self):
        return _Record(self), _Replay(self)


class _Record:
    def __init__(self, rec):
        self.rec = rec

    def __enter__(self):
        self.prev = spatial._set_halo_recorder(self.rec)

    def __exit__(self, *exc):
        spatial._set_halo_recorder(self.prev)


class _Replay:
    """Entered once per recompute (a second backward through a retained graph recomputes again)."""

    def __init__(self, rec):
        self.rec = rec

    def __enter__(self):
        self.saved = save_batchnorm_buffers(self.rec.module)
        self.rec.replaying, self.rec._pos = True, 0
        self.prev = spatial._set_halo_recorder(self.rec)

    def __exit__(self, *exc):
        # also on the early stop of torch.utils.checkpoint, which ends the recompute with an exception
        spatial._set_halo_recorder(self.prev)
        self.rec.replaying = False
        restore_batchnorm_buffers(self.saved)
        self.saved = None


def save_batchnorm_buffers(module):
    """Copies of the running buffers of every BatchNorm in `module` (fused bn_relu or plain nn.BatchNorm2d), for
    restore_batchnorm_buffers: a forward that must not count as a training step (a recompute, a CUDA-graph warm-up)
    runs between the two."""
    return [(m, m.running_mean.clone(), m.running_var.clone(), m.num_batches_tracked.clone()) for m in module.modules()
            if isinstance(m, _BatchNorm) and m.track_running_stats and m.running_mean is not None]


def restore_batchnorm_buffers(saved):
    with torch.no_grad():
        for m, mean, var, n in saved:
            m.running_mean.copy_(mean)
            m.running_var.copy_(var)
            m.num_batches_tracked.copy_(n)


def _flatten(args):
    """Tensors nested one level in tuples / lists (the AmoebaNet cells take (x, x_prev)) become positional
    arguments of the checkpointed function, so torch.utils.checkpoint saves them as the region's inputs."""
    flat, spec = [], []
    for a in args:
        if isinstance(a, (tuple, list)):
            spec.append((type(a), len(a)))
            flat.extend(a)
        else:
            spec.append(None)
            flat.append(a)
    return flat, spec


def _unflatten(flat, spec):
    out, i = [], 0
    for s in spec:
        if s is None:
            out.append(flat[i])
            i += 1
        else:
            out.append(s[0](flat[i:i + s[1]]))
            i += s[1]
    return out


def _checkpointed_forward(self, *args):
    cls_forward = type(self).forward
    if not torch.is_grad_enabled():
        return cls_forward(self, *args)
    flat, spec = _flatten(args)
    rec = _HaloRecorder(self)
    # preserve_rng_state=False: the spatial cells draw no random numbers, so there is no RNG state to give the
    # recompute back; saving and restoring it is what a CUDA-graph capture of the region (torchgems.graphs) forbids
    return checkpoint(lambda *t: cls_forward(self, *_unflatten(t, spec)), *flat, use_reentrant=False,
                      context_fn=rec.contexts, preserve_rng_state=False)


def _has_spatial_layer(module):
    return any(isinstance(m, spatial._SpatialTopology) for m in module.modules())


def checkpoint_spatial_cells(model):
    """Recompute, in backward, every top-level child of the stage `model` (an nn.Sequential, or a
    DistributedDataParallel around one) that contains a spatial layer: the stem and the cells of a spatial stage.
    Each such child keeps only its input and its received halo strips for backward.  The module tree and every
    state_dict key stay as they are: the children's instances get a forward of their own, their class is
    untouched.  Children without a spatial layer are left alone.  Returns `model`."""
    seq = model.module if isinstance(model, nn.parallel.DistributedDataParallel) else model
    for child in seq.children():
        if _has_spatial_layer(child) and "forward" not in child.__dict__:
            child.forward = types.MethodType(_checkpointed_forward, child)
    return model
