"""torchgems.mp_pipeline -- model splitter and the layer-parallel (pipeline) trainer the spatial
trainer builds on.  Mirrors the reference's public surface (src/torchgems/mp_pipeline.py):

    model_generator(model, split_size, input_size, balance=None, shape_list=None)   :28-168
        .get_start_end_layer_index / .get_model / .ready_model / .DDP_model / .get_output_shapes
        .models  .shape_list
    train_model(model_gen, local_rank, batch_size, epochs, criterion=None, optimizer=None,
                parts=1, ASYNC=True, GEMS_INVERSE=False, *, amp_dtype=None,
                recompute=False, cuda_graph=False)                                :171-538
        .run_step(x, y) -> (loss, corrects)  .forward_pass  .backward_pass  .update

Host-side orchestration only (no kernels): activations travel forward and their gradients
backward with torch.distributed point-to-point ops.  What changed from the reference: the device
is whatever this process is bound to (CUDA when present, else CPU -- which is what lets the
pipeline logic be tested on gloo against the reference itself), transfers are stream-ordered
NCCL/gloo sends (no torch.cuda.synchronize() fences, no MPI tags: tensors of one message are
sent in a fixed order), and receive buffers are plain `torch.empty`.
"""
from collections import OrderedDict

import contextlib
import os

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.optim as optim
from torch.nn.parallel import DistributedDataParallel as DDP

from . import graphs
from .recompute import checkpoint_spatial_cells


def _device():
    if torch.cuda.is_available():
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


class model_generator:
    def __init__(self, model, split_size, input_size, balance=None, shape_list=None):
        self.model = model
        self.input_size = input_size
        self.split_size = split_size
        self.balance = balance
        self.shape_list = shape_list
        if balance is not None:
            assert len(balance) == split_size, "Length of balance should be equal to split size "

    def get_start_end_layer_index(self, split_rank):
        """Layers [start, end) of `self.model` owned by pipeline stage `split_rank` (:41-69)."""
        n = len(self.model)
        if self.balance is None:
            per = int(n / self.split_size)
            start = split_rank * per
            end = (split_rank + 1) * per if split_rank != self.split_size - 1 else n
            return start, end
        assert sum(self.balance) == n, "balance and number of layers differs"
        start = sum(self.balance[:split_rank])
        return start, start + self.balance[split_rank]

    def get_model(self, split_rank):
        start, end = self.get_start_end_layer_index(split_rank)
        layers = OrderedDict()
        for i, (name, layer) in enumerate(self.model.named_children()):
            if start <= i < end:
                layers[name] = layer
        return nn.Sequential(layers)

    def ready_model(self, split_rank, GET_SHAPES_ON_CUDA=False):
        if self.shape_list is None:
            self.get_output_shapes(GET_SHAPES_ON_CUDA)
        self.models = self.get_model(split_rank=split_rank).to(_device())

    def DDP_model(self, mpi_comm, num_spatial_parts, spatial_size, bucket_size=25, local_rank=None):
        """Gradient averaging over the tiles of a spatial stage (or over DP replicas) through
        DistributedDataParallel, as the reference does (:92-124)."""
        if local_rank is None:
            local_rank = mpi_comm.local_rank
        dev = _device()
        kw = dict(device_ids=[dev.index]) if dev.type == "cuda" else {}
        if local_rank < mpi_comm.total_spatial_processes:
            grp, bb = mpi_comm.spatial_allreduce_grp, False
        elif mpi_comm.LOCAL_DP_LP > 1:
            grp, bb = mpi_comm.LOCAL_DP_MP_Comm, True
        else:
            grp, bb = mpi_comm.allreduce_grp, False
        if not any(p.requires_grad for p in self.models.parameters()):
            return
        self.models = DDP(self.models, bucket_cap_mb=bucket_size, process_group=grp, broadcast_buffers=bb, **kw)

    def get_output_shapes(self, GET_SHAPES_ON_CUDA):
        """Run a batch-1 tensor of zeros through every stage and record output shapes with the real
        batch size put back (:126-168).  Stages with several outputs record a list of shapes."""
        dev = _device() if GET_SHAPES_ON_CUDA else torch.device("cpu")
        self.shape_list = []
        probe = list(self.input_size)
        probe[0] = 1
        cur = torch.zeros(probe, device=dev)
        with torch.no_grad():
            for i in range(self.split_size):
                stage = self.get_model(split_rank=i)
                if GET_SHAPES_ON_CUDA:
                    stage = stage.to(dev)
                out = stage(cur)
                if isinstance(out, tuple):
                    self.shape_list.append([(self.input_size[0],) + tuple(o.shape[1:]) for o in out])
                    cur = tuple(torch.zeros(o.shape, device=dev) for o in out)
                else:
                    self.shape_list.append((self.input_size[0],) + tuple(out.shape[1:]))
                    cur = torch.zeros(out.shape, device=dev)
                if GET_SHAPES_ON_CUDA:
                    stage.to("cpu")
        # the model was moved around; leave it where it started
        if GET_SHAPES_ON_CUDA and torch.cuda.is_available():
            torch.cuda.empty_cache()


class train_model:
    def __init__(self, model_gen, local_rank, batch_size, epochs, criterion=None, optimizer=None, parts=1, ASYNC=True,
                 GEMS_INVERSE=False, *, amp_dtype=None, recompute=False, cuda_graph=False):
        """amp_dtype=torch.bfloat16: the forward of this stage runs under torch.autocast with fp32 parameters (fp32
        master weights, gradients and optimizer); activations and their gradients travel in bf16.
        recompute=True: the cells of this stage that contain a spatial layer keep only their inputs and received halo
        strips for backward and run their forward again there (torchgems.recompute.checkpoint_spatial_cells).
        cuda_graph=True: a stage that contains a spatial layer runs its forward and backward from CUDA graphs
        (torchgems.graphs), captured at the first step; sends, receives, the loss and the optimizer stay eager."""
        self.models = model_gen.models
        if recompute:
            checkpoint_spatial_cells(self.models)
        if cuda_graph:
            graphs.check_graphable(self.models)
        self.cuda_graph = cuda_graph and graphs.has_spatial_layer(self.models)
        self.graphed = None
        self.shape_list = model_gen.shape_list
        self.input_size = model_gen.input_size
        self.parts = parts
        self.epochs = epochs
        self.local_rank = local_rank
        self.ENABLE_ASYNC = ASYNC
        self.GEMS_INVERSE = GEMS_INVERSE
        self.batch_size = batch_size
        self.device = _device()
        # activations travel in the model's dtype (fp32 as in the reference; bf16 when the model was cast), or in the
        # autocast dtype
        self.amp_dtype = amp_dtype
        self.dtype = amp_dtype or next((p.dtype for p in self.models.parameters() if p.is_floating_point()), torch.float32)
        # subclasses (train_model_spatial) set these before calling us
        if not hasattr(self, "num_spatial_parts"):
            self.num_spatial_parts = 1
        if not hasattr(self, "split_rank"):
            self.split_rank = local_rank
        if not hasattr(self, "mp_size"):
            self.mp_size = model_gen.split_size
        if not hasattr(self, "split_size"):
            self.split_size = self.mp_size
        self.MULTIPLE_INPUT = self.split_rank > 0 and isinstance(self.shape_list[self.split_rank - 1], list)
        self.MULTIPLE_OUTPUT = isinstance(self.shape_list[self.split_rank], list)
        self.criterion = nn.CrossEntropyLoss() if criterion is None else criterion
        self.optimizer = optim.SGD(self.models.parameters(), lr=0.001, momentum=0.9) if optimizer is None else optimizer
        self.initialize_recv_buffers()
        self.initialize_send_recv_ranks()

    # ---- topology -----------------------------------------------------------------------------
    def _replica_base(self, my_process_offset):
        """First process rank of the pipeline replica this process belongs to.  The reference addresses
        peers by their position on the rank line (:238-248), which is only right for the first replica;
        with data-parallel replicas (world = k * mp_size) the peers of rank 5 are 4 and 6, not 0 and 2."""
        return dist.get_rank() - my_process_offset if dist.is_initialized() else 0

    def initialize_send_recv_ranks(self):
        r = self.local_rank if not self.GEMS_INVERSE else self.mp_size - 1 - self.local_rank
        step = 1 if not self.GEMS_INVERSE else -1          # the inverse replica runs down the rank line
        base = self._replica_base(r)
        self.to_send_forward = base + r + step
        self.to_recv_forward = base + r - step
        self.to_send_backward = base + r - step
        self.to_recv_backward = base + r + step

    def _parts_shape(self, shape):
        """shape_list already carries the micro-batch size: the scripts build model_generator with
        input_size = (batch_size / parts, ...) (benchmark_amoebanet_sp.py:150-168)."""
        return tuple(shape)

    def _empty_like_shapes(self, shapes, requires_grad):
        if isinstance(shapes, list):
            return tuple(torch.zeros(self._parts_shape(s), device=self.device, dtype=self.dtype, requires_grad=requires_grad)
                         for s in shapes)
        return torch.zeros(self._parts_shape(shapes), device=self.device, dtype=self.dtype, requires_grad=requires_grad)

    def initialize_recv_buffers(self):
        """One activation buffer per micro-batch (their .grad is what travels back) and one buffer
        for the incoming gradient of this stage's output (:251-290)."""
        self.input_x_list = []
        for _ in range(self.parts):
            self.input_x_list.append(self._empty_like_shapes(self.shape_list[self.split_rank - 1], True)
                                     if self.split_rank != 0 else [])
        if self.split_rank != self.split_size - 1:
            g = self._empty_like_shapes(self.shape_list[self.split_rank], False)
            self.grad_overhead = list(g) if isinstance(g, tuple) else g

    # ---- point-to-point -----------------------------------------------------------------------
    @staticmethod
    def _as_list(x):
        return list(x) if isinstance(x, (tuple, list)) else [x]

    @staticmethod
    def _host_staged(t):
        """gloo cannot move CUDA tensors point-to-point: stage through the host (debug / single-GPU
        test configuration only; NCCL sends device buffers directly)."""
        return t.is_cuda and dist.get_backend() != "nccl"

    def _send(self, tensors, dst):
        for t in self._as_list(tensors):
            t = t.detach().contiguous()
            dist.send(t.cpu() if self._host_staged(t) else t, dst=dst)

    def _recv(self, tensors, src):
        for t in self._as_list(tensors):
            if self._host_staged(t):
                h = torch.empty(t.shape, dtype=t.dtype)
                dist.recv(h, src=src)
                t.copy_(h)
            else:
                dist.recv(t, src=src)

    # names kept from the reference; sync and async variants behave the same on stream-ordered backends
    def receive_input_sync(self, part_number):
        with torch.no_grad():
            self._recv(self.input_x_list[part_number], self.to_recv_forward)

    receive_input_async = receive_input_sync

    def send_input_sync(self, y):
        if self.amp_dtype is not None:      # an op autocast runs in fp32 may end the stage: match the receive buffers
            y = [t.to(self.dtype) for t in self._as_list(y)]
        self._send(y, self.to_send_forward)

    send_input_async = send_input_sync

    def receive_grad_sync(self):
        self._recv(self.grad_overhead, self.to_recv_backward)

    receive_grad_async = receive_grad_sync

    def send_grad_sync(self, input_x):
        self._send([t.grad for t in self._as_list(input_x)], self.to_send_backward)

    send_grad_async = send_grad_sync

    # ---- one micro-batch ----------------------------------------------------------------------
    def _autocast(self):
        if self.amp_dtype is None:
            return contextlib.nullcontext()
        return torch.autocast(self.device.type, dtype=self.amp_dtype)

    def _run_stage(self, input_x, part_number):
        """The stage's forward: eager, or replayed from the micro-batch's CUDA graph.  The graphs are captured at the
        first call, on every tile of the stage at the same step (graph_stage is collective over them)."""
        if not self.cuda_graph:
            with self._autocast():
                return self.models(input_x)
        if self.graphed is None:
            self.graphed = graphs.graph_stage(self.models, [input_x] * self.parts, amp_dtype=self.amp_dtype)
        return self.graphed(input_x, part_number)

    def forward_pass(self, data_x, data_y, part_number=0):
        if self.split_rank == 0:
            input_x = data_x
        else:
            self.receive_input_async(part_number)
            input_x = self.input_x_list[part_number]
        y = self._run_stage(input_x, part_number)
        if self.split_rank != self.split_size - 1:
            self.send_input_async(y)
            return y, None
        loss = self.criterion(y.float(), data_y)          # no-op for fp32 models
        corrects = (data_y.eq(torch.argmax(y, dim=-1).long())).sum().float()
        return loss, corrects / self.batch_size

    def backward_pass(self, y, part_number=0):
        if self.split_rank != self.split_size - 1:
            self.receive_grad_async()
            torch.autograd.backward(y, self.grad_overhead)
        else:
            y.backward()
        if self.split_rank != 0:
            self.send_grad_async(self.input_x_list[part_number])
            # fresh leaves for the next step (the old .grad has been shipped)
            buf = self.input_x_list[part_number]
            if isinstance(buf, tuple):
                self.input_x_list[part_number] = tuple(t.detach().requires_grad_() for t in buf)
            else:
                self.input_x_list[part_number] = buf.detach().requires_grad_()

    def run_step(self, data_x, data_y):
        """GPipe-style fill/drain: all micro-batch forwards, then all backwards (:509-534)."""
        data_x = data_x.to(self.device, non_blocking=True)
        data_y = data_y.to(self.device, non_blocking=True)
        if data_x.is_floating_point() and data_x.dtype != self.dtype and self.amp_dtype is None:
            data_x = data_x.to(self.dtype)
        per = int(self.batch_size / self.parts)
        outs, loss, corrects = [], 0, 0
        for i in range(self.parts):
            y, c = self.forward_pass(data_x[i * per:(i + 1) * per], data_y[i * per:(i + 1) * per], part_number=i)
            outs.append(y)
            if self.split_rank == self.split_size - 1:
                loss += y.item()
                corrects += c.item()
        for i in range(self.parts):
            self.backward_pass(outs[i], part_number=i)
        return loss, corrects

    def update(self):
        """optimizer.step() + zero the gradients IN PLACE.  The reference calls zero_grad() (mp_pipeline.py:536-538),
        which since torch 2.0 drops `p.grad` (set_to_none=True): that severs the views
        train_spatial_model_master points into its flat gradient buffers (train_spatial_master.py:126-131), so
        --enable-master-comm-opt would ship stale buffers from the second step on.  Zeroing in place keeps
        the aliases and is numerically identical for every other trainer.  SPCONV_REFERENCE_ZERO_GRAD=1
        restores the reference's call (used by the loss-sequence parity test)."""
        self.optimizer.step()
        self.optimizer.zero_grad(set_to_none=os.environ.get("SPCONV_REFERENCE_ZERO_GRAD") == "1")
