"""torchgems.train_spatial -- the SP+LP trainer: spatial stages (tiles of one image on P ranks,
convolutions exchanging halos) followed by ordinary pipeline stages.  Mirrors the reference's
surface (src/torchgems/train_spatial.py):

    verify_spatial_config(slice_method, image_size, num_spatial_parts_list)              :33-58
    get_shapes_spatial(shape_list, slice_method, spatial_size, num_spatial_parts_list,
                       image_size_times)                                               :61-238
    split_input(inputs, image_size, slice_method, local_rank, num_spatial_parts_list)    :241-290
    train_model_spatial(model_gen, local_rank, batch_size, epochs, spatial_size=1,
                        num_spatial_parts=4, ..., slice_method="square", LOCAL_DP_LP=1,
                        mpi_comm=None, *, amp_dtype=None, recompute=False,
                        cuda_graph=False)                                              :293-1440

Rank line of one model replica (P tiles per spatial stage, S spatial stages):

    [stage 0: P tiles][stage 1: P tiles]...[stage S-1: P tiles][join = stage S][stage S+1]...

Tile t of stage s feeds tile t of stage s+1; every tile of stage S-1 feeds the join rank, which
stitches the P tiles back into one feature map (cat along W for "vertical", H for "horizontal",
a sqrt(P) x sqrt(P) grid for "square") and, in backward, returns each tile's slice of the gradient.

Scope: equal tile counts per spatial stage -- the only configuration verify_spatial_config
accepts (:54-57), so the reference's "skewed" intermediate merges (:453-504, 1190-1254) are
unreachable through its own scripts and are not built.  LOCAL_DP_LP > 1 (LBANN-style data
parallelism in the LP tail, :809-1028) is not built yet and raises.
"""
import math

import torch
import torch.distributed as dist

from .mp_pipeline import train_model
from .utils import isPowerTwo


def verify_spatial_config(slice_method, image_size, num_spatial_parts_list):
    """Power-of-two image and tile sizes only: odd sizes would truncate under strided layers and
    neighbouring tiles would disagree on their shapes (:26-31)."""
    p0 = num_spatial_parts_list[0]
    assert slice_method in ["square", "vertical", "horizontal"], \
        "Possible slice methods are ['square', 'vertical', 'horizontal']"
    assert isPowerTwo(int(image_size)), "Image size should be power of Two"
    per_side = math.sqrt(p0) if slice_method == "square" else p0
    assert isPowerTwo(int(image_size / per_side)), "Image size of each partition should be power of Two"
    for p in num_spatial_parts_list:
        assert p == p0, "Size of each SP partition should be same"


def _tile_divisors(slice_method, parts):
    """(rows, cols) a feature map is cut into."""
    if slice_method == "square":
        return math.sqrt(parts), math.sqrt(parts)
    if slice_method == "vertical":
        return 1, parts
    return parts, 1


def get_shapes_spatial(shape_list, slice_method, spatial_size, num_spatial_parts_list, image_size_times):
    """Per-stage output shapes at the real image size, derived from shapes traced at a small
    image (`image_size_seq`): H and W scale by `image_size_times`, and stages that are spatial
    (index < spatial_size) additionally shrink to one tile.  2-D shapes (the classifier) pass
    through.  "square" divides by sqrt(parts of stage 0), the strips by the stage's own count."""
    out = []
    for idx, entry in enumerate(shape_list):
        spatial = idx < spatial_size
        if slice_method == "square":
            parts = num_spatial_parts_list[0]
        else:
            parts = num_spatial_parts_list[idx] if spatial else 1
        dh, dw = _tile_divisors(slice_method, parts) if spatial else (1, 1)

        def scale(s):
            if len(s) == 2:
                return (int(s[0]), s[1])
            return (int(s[0]), s[1], int(s[2] * image_size_times / dh), int(s[3] * image_size_times / dw))

        if isinstance(entry, list):
            out.append([scale(s) for s in entry])
        else:
            out.append(scale(entry))
    return out


def split_input(inputs, image_size, slice_method, local_rank, num_spatial_parts_list):
    """This rank's tile of a batch of full images.  Strips give the remainder to the last rank."""
    parts = num_spatial_parts_list[0]
    if slice_method == "square":
        side = int(math.sqrt(parts))
        t = int(image_size / math.sqrt(parts))
        row, col = int(local_rank / side), int(local_rank % side)
        return inputs[:, :, row * t:(row + 1) * t, col * t:(col + 1) * t]
    t = int(image_size / parts)
    lo = local_rank * t
    hi = None if local_rank == parts - 1 else lo + t
    if slice_method == "vertical":
        return inputs[:, :, :, lo:hi]
    if slice_method == "horizontal":
        return inputs[:, :, lo:hi, :]


class train_model_spatial(train_model):
    def __init__(self, model_gen, local_rank, batch_size, epochs, spatial_size=1, num_spatial_parts=4, criterion=None,
                 optimizer=None, parts=1, ASYNC=True, GEMS_INVERSE=False, slice_method="square", LOCAL_DP_LP=1,
                 mpi_comm=None, *, amp_dtype=None, recompute=False, cuda_graph=False):
        if LOCAL_DP_LP != 1:
            raise NotImplementedError("LOCAL_DP_LP > 1 (data parallelism inside the LP tail) is not built yet")
        self.slice_method = slice_method
        self.LOCAL_DP_LP = LOCAL_DP_LP
        self.ENABLE_LOCAL_DP_LP = False
        self.spatial_size = spatial_size
        self.local_rank = local_rank
        if isinstance(num_spatial_parts, list):
            assert spatial_size == len(num_spatial_parts), "Spatial size is not equal to lenght of num_spatial_parts"
            assert all(p == num_spatial_parts[0] for p in num_spatial_parts), "Size of each SP partition should be same"
            self.num_spatial_parts_list = num_spatial_parts
            self.num_spatial_parts = num_spatial_parts[0]
        else:
            assert spatial_size == 1, "Spatial size is not 1"
            self.num_spatial_parts_list = [num_spatial_parts]
            self.num_spatial_parts = num_spatial_parts
        P = self.num_spatial_parts
        self.total_spatial_processes = P * spatial_size
        self.split_size = model_gen.split_size
        if local_rank < self.total_spatial_processes:
            self.split_rank = local_rank // P
            self.spatial_local_rank = local_rank % P
        else:
            self.split_rank = local_rank - self.total_spatial_processes + spatial_size
            self.spatial_local_rank = local_rank
        self.mp_size = mpi_comm.mp_size if mpi_comm is not None else self.total_spatial_processes + self.split_size - spatial_size
        self.is_join = self.split_rank == spatial_size
        super().__init__(model_gen, local_rank, batch_size, epochs, criterion=criterion, optimizer=optimizer,
                         parts=parts, ASYNC=ASYNC, GEMS_INVERSE=GEMS_INVERSE, amp_dtype=amp_dtype,
                         recompute=recompute, cuda_graph=cuda_graph)
        if self.is_join:
            self.initialize_recv_buffers_joint()

    # ---- topology -----------------------------------------------------------------------------
    def _line(self, r):
        """Position on the rank line -> process rank (the inverse replica is mirrored, :624-640;
        offset by the first rank of this model replica when the world holds several)."""
        off = self.mp_size - 1 - r if self.GEMS_INVERSE else r
        if not hasattr(self, "_base"):
            mine = self.mp_size - 1 - self.local_rank if self.GEMS_INVERSE else self.local_rank
            self._base = self._replica_base(mine)
        return self._base + off

    def initialize_send_recv_ranks(self):
        P, r = self.num_spatial_parts, self.local_rank
        fwd = back = 1
        if r < self.total_spatial_processes:
            # tile -> same tile of the next spatial stage, or -> the join rank from the last one
            fwd = P if self.split_rank < self.spatial_size - 1 else self.total_spatial_processes - r
            back = P
        self.to_send_forward = self.to_recv_backward = self._line(r + fwd)
        self.to_recv_forward = self.to_send_backward = self._line(r - back)

    def _tile_ranks(self):
        """Process ranks of the P tiles feeding the join rank, in tile order (:691-697)."""
        return [self._line(self.local_rank - self.num_spatial_parts + t) for t in range(self.num_spatial_parts)]

    # ---- join rank ----------------------------------------------------------------------------
    def initialize_recv_buffers_joint(self):
        """P receive buffers per micro-batch, one per tile (:506-555)."""
        shapes = self.shape_list[self.split_rank - 1]
        self.input_x_list = [[self._empty_like_shapes(shapes, True) for _ in range(self.num_spatial_parts)]
                             for _ in range(self.parts)]

    def receive_input_async_joint(self, part_number, ranks=None):
        """All P tiles (every tensor of each) in one batched receive."""
        bufs = [t for buf in self.input_x_list[part_number] for t in self._as_list(buf)]
        srcs = [src for buf, src in zip(self.input_x_list[part_number], self._tile_ranks()) for _ in self._as_list(buf)]
        with torch.no_grad():
            staged = [torch.empty(t.shape, dtype=t.dtype) if self._host_staged(t) else t for t in bufs]
            for w in dist.batch_isend_irecv([dist.P2POp(dist.irecv, h, s) for h, s in zip(staged, srcs)]):
                w.wait()
            for t, h in zip(bufs, staged):
                if h is not t:
                    t.copy_(h)

    recv_inputs_joint = receive_input_async_joint

    def send_grad_async_joint(self, input_x_list):
        ops = []
        for buf, dst in zip(input_x_list, self._tile_ranks()):
            for t in self._as_list(buf):
                g = t.grad.contiguous()
                ops.append(dist.P2POp(dist.isend, g.cpu() if self._host_staged(g) else g, dst))
        for w in dist.batch_isend_irecv(ops):
            w.wait()

    def _stitch(self, tiles):
        P = self.num_spatial_parts
        if self.slice_method == "vertical":
            return torch.cat(tiles, dim=-1)
        if self.slice_method == "horizontal":
            return torch.cat(tiles, dim=-2)
        side = int(math.sqrt(P))
        rows = [torch.cat(tiles[i * side:(i + 1) * side], dim=-1) for i in range(side)]
        return torch.cat(rows, dim=-2)

    def merge_inputs_joint_cat(self, part_number):
        """Stitch the P tiles (of every input, when the stage takes several) into full maps
        (:1083-1188).  The cat is differentiable, so backward leaves each tile's slice of the
        gradient in its receive buffer's .grad."""
        bufs = self.input_x_list[part_number]
        if self.MULTIPLE_INPUT:
            n = len(self.shape_list[self.split_rank - 1])
            return tuple(self._stitch([b[i] for b in bufs]) for i in range(n))
        return self._stitch(list(bufs))

    # ---- one micro-batch ----------------------------------------------------------------------
    def _no_sync_ctx(self, part_number):
        """Gradient all-reduce of a DDP-wrapped stage only on the last micro-batch (:1298-1307)."""
        if isinstance(self.models, torch.nn.parallel.DistributedDataParallel) and part_number != self.parts - 1:
            return self.models.no_sync()
        import contextlib
        return contextlib.nullcontext()

    def forward_pass(self, data_x, data_y, part_number=0):
        if self.split_rank == 0:
            input_x = data_x
        elif self.is_join:
            self.recv_inputs_joint(part_number)
            input_x = self.merge_inputs_joint_cat(part_number)
        else:
            self.receive_input_async(part_number)
            input_x = self.input_x_list[part_number]
        with self._no_sync_ctx(part_number):
            y = self._run_stage(input_x, part_number)
            if self.split_rank != self.split_size - 1:
                self.send_input_async(y)
                return y, None
            loss = self.criterion(y.float(), data_y)          # no-op for fp32 models
        corrects = (data_y.eq(torch.argmax(y, dim=-1).long())).sum().float()
        return loss, corrects / self.batch_size

    def backward_pass(self, y, part_number=0):
        last = self.split_rank == self.split_size - 1
        if not last:
            self.receive_grad_async()
        with self._no_sync_ctx(part_number):
            if last:
                y.backward()
            else:
                torch.autograd.backward(y, self.grad_overhead)
        if self.split_rank == 0:
            return
        bufs = self.input_x_list[part_number]
        if self.is_join:
            self.send_grad_async_joint(bufs)
            self.input_x_list[part_number] = [
                tuple(t.detach().requires_grad_() for t in b) if isinstance(b, tuple) else b.detach().requires_grad_()
                for b in bufs]
        else:
            self.send_grad_async(bufs)
            self.input_x_list[part_number] = (tuple(t.detach().requires_grad_() for t in bufs)
                                              if isinstance(bufs, tuple) else bufs.detach().requires_grad_())
