"""torchgems.comm -- rank arithmetic, process groups and the flat-gradient allreduce of the
reference (src/torchgems/comm.py), re-targeted from `torch.distributed` over CUDA-aware MPI to
one process per GPU with NCCL (gloo on CPU for the plumbing tests).

Mirrors: initialize_cuda (comm.py:34-41), MPIComm (comm.py:44-310), sync_comms_for_master
(comm.py:312-332), SyncAllreduce (comm.py:335-522).  Same constructor signatures, attribute names
and group semantics.  Differences that are deliberate:
  * backend is "nccl" (or "gloo" without CUDA) instead of the patched "mpi" build;
  * every rank creates EVERY group in the same order (NCCL/gloo `new_group` is collective over
    the world; the reference relies on MPI letting each rank create only its own group);
  * initialize_cuda() selects `cuda:LOCAL_RANK` (8 GPUs per node) instead of masking
    CUDA_VISIBLE_DEVICES to `local_rank % 4`;
  * SyncAllreduce flattens with one torch.cat and writes back in place (no per-parameter
    clone/detach chain), same numerics: sum over the group, divided by `divide_bs`.
"""
import math
import os

import numpy as np
import torch
import torch.distributed as dist


def env2int(env_list, default=-1):
    for e in env_list:
        val = int(os.environ.get(e, -1))
        if val >= 0:
            return val
    return default


_LOCAL_RANK_ENV = ["LOCAL_RANK", "MPI_LOCALRANKID", "OMPI_COMM_WORLD_LOCAL_RANK", "MV2_COMM_WORLD_LOCAL_RANK"]


def initialize_cuda():
    """One process per GPU: bind this process to cuda:<local rank> (comm.py:34-41)."""
    if not torch.cuda.is_available():
        return
    my_local_rank = env2int(_LOCAL_RANK_ENV, 0)
    torch.cuda.set_device(my_local_rank % torch.cuda.device_count())
    torch.cuda.init()


def _default_backend():
    b = os.environ.get("SPCONV_DIST_BACKEND")
    if b:
        return b
    return "nccl" if torch.cuda.is_available() else "gloo"


class MPIComm:
    def __init__(self, split_size, ENABLE_MASTER=False, ENABLE_SPATIAL=False, num_spatial_parts=None,
                 spatial_size=None, LOCAL_DP_LP=1, DISABLE_INIT=False):
        self.ENABLE_MASTER = ENABLE_MASTER
        self.ENABLE_SPATIAL = ENABLE_SPATIAL
        self.split_size = split_size
        if not ENABLE_SPATIAL:
            self.mp_size = split_size
        else:  # comm.py:59-67
            self.mp_size = int(split_size + np.sum(num_spatial_parts) - spatial_size
                               + (split_size - spatial_size) * (LOCAL_DP_LP - 1))
        if DISABLE_INIT:
            self.rank = dist.get_rank()
            self.size = dist.get_world_size()
        else:
            self.size, self.rank = self.init_comm(backend=_default_backend())
        self.local_rank = self.rank % self.mp_size
        if self.ENABLE_MASTER:  # the second (inverse) replica lives on mirrored ranks, comm.py:77-80
            self.local_rank = self.mp_size - 1 - self.local_rank
            self.first_local_rank = self.mp_size - 1 - self.local_rank
            self.second_local_rank = self.local_rank
        self.num_spatial_parts = num_spatial_parts
        self.spatial_size = spatial_size
        self.LOCAL_DP_LP = LOCAL_DP_LP
        if ENABLE_SPATIAL and (num_spatial_parts is None or spatial_size is None):
            assert False, "Spatial enabled but num_spatial_parts or spatial_size is None"
        if ENABLE_SPATIAL:
            if isinstance(num_spatial_parts, list):
                assert spatial_size == len(num_spatial_parts), \
                    "spatial size should be equal to elements in num_spatial_parts"
                self.total_spatial_processes = sum(num_spatial_parts)
                self.num_spatial_parts_list = num_spatial_parts
            else:
                self.total_spatial_processes = num_spatial_parts
            self.spatial_allreduce_grp = self.create_allreduce_comm_spatial()
        else:
            self.spatial_allreduce_grp = None

        if ENABLE_SPATIAL:  # comm.py:107-125
            if self.local_rank < self.total_spatial_processes:
                self.split_rank = self.get_split_rank(num_spatial_parts, self.local_rank)
            else:
                self.split_rank = (math.floor((self.local_rank - self.total_spatial_processes) / self.LOCAL_DP_LP)
                                   + spatial_size)
        else:
            self.split_rank = self.local_rank

        if LOCAL_DP_LP > 1:
            self.LP_SP_Groups, self.SP_LP_group = self.create_scatter_gather_spatial_MP_comm()
            self.LOCAL_DP_MP_Comm = self.create_local_DP_in_MP_comm()
            self.test_allreduce_comm(self.LOCAL_DP_MP_Comm)
        else:
            self.LP_SP_Groups, self.SP_LP_group = None, None
            self.LOCAL_DP_MP_Comm = None
        self.allreduce_grp = self.create_allreduce_comm()
        self.test_allreduce_comm(self.allreduce_grp)
        if ENABLE_SPATIAL and torch.cuda.is_available():
            # every rank is here: agree once on the halo transport (peer mailboxes vs torch.distributed P2P)
            from . import halo_transport
            halo_transport.negotiate(torch.device("cuda", torch.cuda.current_device()))

    # ---------------------------------------------------------------------------------------
    def get_split_rank(self, num_spatial_parts_list, local_rank):
        if isinstance(num_spatial_parts_list, list):
            acc = 0
            for stage, parts in enumerate(num_spatial_parts_list):
                if local_rank < acc + parts:
                    return stage
                acc += parts
            return None
        return math.floor(local_rank / num_spatial_parts_list)

    def init_comm(self, backend=None):
        """torchrun / mpirun environment -> process group (comm.py:154-159)."""
        if not dist.is_initialized():
            if "RANK" not in os.environ:  # launched by mpirun: translate the MPI variables
                r = env2int(["OMPI_COMM_WORLD_RANK", "PMI_RANK", "MV2_COMM_WORLD_RANK"], -1)
                s = env2int(["OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "MV2_COMM_WORLD_SIZE"], -1)
                if r >= 0 and s > 0:
                    os.environ["RANK"], os.environ["WORLD_SIZE"] = str(r), str(s)
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29500")
            kw = {}
            if backend == "nccl":
                kw["device_id"] = torch.device("cuda", torch.cuda.current_device())
            dist.init_process_group(backend or _default_backend(), **kw)
        return dist.get_world_size(), dist.get_rank()

    def _new_group(self, ranks):
        return dist.new_group(ranks=sorted(int(r) for r in ranks))

    def create_allreduce_comm_basic(self):
        """Data-parallel replicas of the same model-parallel rank (comm.py:161-168); all groups are
        created on all ranks, this rank keeps its own."""
        mine = None
        for r in range(self.mp_size):
            ranks = [self.mp_size * i + r for i in range(int(self.size / self.mp_size))]
            g = self._new_group(ranks)
            if r == self.local_rank:
                mine = g
        return mine

    def create_allreduce_comm_master(self):
        """GEMS-MASTER: rank r pairs with its mirror (comm.py:170-195)."""
        if self.ENABLE_SPATIAL:
            for first in range(self.total_spatial_processes, self.mp_size):
                second = self.mp_size - 1 - first
                g = self._new_group([first, second])
                if self.first_local_rank in (first, second):
                    self.first_LP_master_group = g
                if self.second_local_rank in (first, second):
                    self.second_LP_master_group = g
            return None
        mine = None
        for r in range(self.mp_size):
            mirror = self.mp_size - 1 - r
            if mirror < r:
                continue
            ranks = [t for t in range(self.size) if t % self.mp_size in (r, mirror)]
            g = self._new_group(ranks)
            if self.local_rank in (r, mirror):
                mine = g
        return mine

    def _stage_ranks(self, j):
        if self.spatial_size == 1:
            parts = self.num_spatial_parts if not isinstance(self.num_spatial_parts, list) else self.num_spatial_parts[0]
            return [parts * j + i for i in range(parts)]
        lst = self.num_spatial_parts_list
        return [sum(lst[:j]) + i for i in range(lst[j])]

    def create_allreduce_comm_spatial(self):
        """The tiles of one spatial stage (+ their mirrors under MASTER) (comm.py:197-248)."""
        if self.ENABLE_MASTER:
            first_local_rank = self.mp_size - 1 - self.local_rank
            second_local_rank = self.local_rank
        mine = None
        for j in range(self.spatial_size):
            base = self._stage_ranks(j)
            ranks = list(base)
            if self.ENABLE_MASTER:
                ranks += [self.mp_size - 1 - r for r in base]
            g = self._new_group(ranks)
            if self.ENABLE_MASTER:
                if first_local_rank in base:
                    self.first_spatial_allreduce_grp = g
                elif second_local_rank in base:
                    self.second_spatial_allreduce_grp = g
            if self.spatial_size == 1 or self.local_rank in base:
                mine = g
        return mine

    def create_scatter_gather_spatial_MP_comm(self):
        """LBANN-style local DP: each tile of the last spatial stage + the LOCAL_DP_LP first LP
        ranks (comm.py:250-276)."""
        prev = self.num_spatial_parts if self.spatial_size == 1 and not isinstance(self.num_spatial_parts, list) \
            else self.num_spatial_parts_list[-1]
        start = self.total_spatial_processes - prev
        lp = [i + self.total_spatial_processes for i in range(self.LOCAL_DP_LP)]
        groups, mine = [], None
        for j in range(prev):
            ranks = [start + j] + lp
            if self.ENABLE_MASTER:
                ranks = [self.mp_size - 1 - r for r in ranks]
            g = self._new_group(ranks)
            groups.append(g)
            if self.local_rank == start + j:
                mine = g
        return groups, mine

    def create_local_DP_in_MP_comm(self):
        n_lp = self.mp_size - self.total_spatial_processes
        mine = None
        for j in range(int(n_lp / self.LOCAL_DP_LP)):
            s = self.total_spatial_processes + j * self.LOCAL_DP_LP
            ranks = [s + i for i in range(self.LOCAL_DP_LP)]
            if self.ENABLE_MASTER:
                ranks = [self.mp_size - 1 - r for r in ranks]
            g = self._new_group(ranks)
            if self.local_rank in ranks:
                mine = g
        return mine

    def create_allreduce_comm(self):
        if self.LOCAL_DP_LP > 1:
            return dist.new_group()
        if not self.ENABLE_MASTER:
            return self.create_allreduce_comm_basic()
        return self.create_allreduce_comm_master()

    def test_allreduce_comm(self, allreduce_grp):
        t = torch.zeros(32, 32, 3, 3, device="cuda" if (torch.cuda.is_available() and dist.get_backend() == "nccl") else "cpu")
        if allreduce_grp is not None:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=allreduce_grp)


def sync_comms_for_master(comm1, comm2):
    """Wire the MASTER groups (created on comm2) into both communicators (comm.py:312-332)."""
    first_local_rank = comm1.local_rank
    second_local_rank = comm2.local_rank
    if first_local_rank < comm1.total_spatial_processes:
        comm1.spatial_allreduce_grp = comm2.first_spatial_allreduce_grp
        comm1.allreduce_grp_master = comm2.first_spatial_allreduce_grp
    if second_local_rank < comm1.total_spatial_processes:
        comm2.spatial_allreduce_grp = comm2.second_spatial_allreduce_grp
        comm2.allreduce_grp_master = comm2.second_spatial_allreduce_grp
    if comm1.LOCAL_DP_LP == 1:
        if first_local_rank >= comm1.total_spatial_processes:
            comm1.allreduce_grp = comm2.first_LP_master_group
            comm1.allreduce_grp_master = comm2.first_LP_master_group
        if second_local_rank >= comm1.total_spatial_processes:
            comm2.allreduce_grp = comm2.second_LP_master_group
            comm2.allreduce_grp_master = comm2.second_LP_master_group


class SyncAllreduce:
    """Flat-gradient allreduce over a group, then grad / divide_bs (comm.py:335-522)."""

    def __init__(self, mpi_comm):
        self.ENABLE_MASTER = mpi_comm.ENABLE_MASTER
        self.mp_size = mpi_comm.mp_size
        self.size = mpi_comm.size
        self.local_rank = mpi_comm.local_rank
        self.allreduce_grp = mpi_comm.allreduce_grp
        self.rank = mpi_comm.rank
        self.num_spatial_parts = mpi_comm.num_spatial_parts
        self.spatial_size = mpi_comm.spatial_size
        self.spatial_allreduce_grp = mpi_comm.spatial_allreduce_grp
        if self.ENABLE_MASTER:  # comm.py:349-358
            self.divide_bs = 2 * (self.size / self.mp_size)
        elif self.spatial_size is not None:
            self.divide_bs = self.num_spatial_parts[0] if isinstance(self.num_spatial_parts, list) else self.num_spatial_parts
        else:
            self.divide_bs = self.size / self.mp_size

    # ---- parameter broadcast --------------------------------------------------------------
    def sync_broadcast(self, model, src, grp_comm):
        for param in model.parameters():
            dist.broadcast(param.data, src=src, group=grp_comm, async_op=False)

    def sync_model_spatial(self, model_gen):
        if self.local_rank < self.spatial_size * self.num_spatial_parts:
            self.sync_broadcast(model_gen.models, src=math.floor(self.local_rank / self.num_spatial_parts),
                                grp_comm=self.spatial_allreduce_grp)

    def sync_model(self, model_gen1, model_gen2):
        if self.local_rank >= self.mp_size / 2:
            self.sync_broadcast(model_gen1.models, src=self.local_rank, grp_comm=self.allreduce_grp)
            self.sync_broadcast(model_gen2.models, src=self.local_rank, grp_comm=self.allreduce_grp)
        else:
            self.sync_broadcast(model_gen2.models, src=self.mp_size - self.local_rank - 1, grp_comm=self.allreduce_grp)
            self.sync_broadcast(model_gen1.models, src=self.mp_size - self.local_rank - 1, grp_comm=self.allreduce_grp)

    # ---- flat gradients -------------------------------------------------------------------
    @staticmethod
    def _grads(model):
        return [p.grad for p in model.parameters() if p.grad is not None]

    def get_grad_flatten(self, model, back=False):
        grads = self._grads(model)
        if not grads:
            return None
        return torch.cat([g.detach().reshape(-1) for g in grads])

    def modify_grads(self, model, flat_grad, *_unused):
        """Scatter the reduced flat buffer back, divided by divide_bs (comm.py:440-458)."""
        off = 0
        inv = 1.0 / self.divide_bs
        for g in self._grads(model):
            n = g.numel()
            g.copy_(flat_grad[off:off + n].view_as(g) * inv)
            off += n

    def apply_allreduce(self, model_gen, allreduce_grp):
        models = model_gen.models
        flat = self.get_grad_flatten(models)
        if flat is None:
            return
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=allreduce_grp)
        self.modify_grads(models, flat)

    def apply_allreduce_master(self, model_gen1, model_gen2):
        m1, m2 = model_gen1.models, model_gen2.models
        f1, f2 = self.get_grad_flatten(m1), self.get_grad_flatten(m2, back=True)
        order = [(f1, None), (f2, None)] if self.local_rank >= self.mp_size / 2 else [(f2, None), (f1, None)]
        for f, _ in order:
            dist.all_reduce(f, op=dist.ReduceOp.SUM, group=self.allreduce_grp)
        self.modify_grads(m1, f1)
        self.modify_grads(m2, f2)

    def apply_allreduce_master_master(self, model_gen1, model_gen2, comm1, comm2):
        """Both replicas, ordered by split rank so mirrored pairs never deadlock (comm.py:479-504)."""
        m1, m2 = model_gen1.models, model_gen2.models
        f1, f2 = self.get_grad_flatten(m1), self.get_grad_flatten(m2, back=True)
        seq = [(f1, comm1.allreduce_grp_master), (f2, comm2.allreduce_grp_master)]
        if comm1.split_rank > comm2.split_rank:
            seq.reverse()
        for f, grp in seq:
            dist.all_reduce(f, op=dist.ReduceOp.SUM, group=grp)
        self.modify_grads(m1, f1)
        self.modify_grads(m2, f2)

    def apply_allreduce_master_and_update(self, tm_master, model_gen1, model_gen2):
        self.apply_allreduce_master(model_gen1, model_gen2)
        tm_master.train_model1.update()
        tm_master.train_model2.update()
