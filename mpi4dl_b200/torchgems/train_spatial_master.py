"""torchgems.train_spatial_master -- GEMS master on top of SP+LP: two replicas of the spatial
pipeline on mirrored rank lines (replica 2: position r runs on rank mp_size-1-r), so the GPUs that
hold replica 1's tiles hold replica 2's tail stages and vice versa.  Mirrors reference
src/torchgems/train_spatial_master.py:

    verify_spatial_master_config(slice_method, image_size, num_spatial_parts_list, spatial_size, mp_size)  :33-84
    train_spatial_model_master(model_gen1, model_gen2, batch_size, spatial_size, num_spatial_parts,
                               slice_method, mpi_comm_first, mpi_comm_second, LOCAL_DP_LP, ...,
                               *, amp_dtype=None, recompute=False, cuda_graph=False)                        :87-501
        .run_step(inputs, labels)                 two (x replications) passes, one per replica
        .run_step_allreduce(inputs, labels, odd)  the --enable-master-comm-opt protocol: instead of an
                                                  allreduce between the replicas, rank r and its mirror
                                                  swap flat parameter / gradient buffers around each pass

Parameters and gradients of each replica are views into one flat buffer per replica (as in the
reference, :104-131), so shipping a replica is a single send of one contiguous tensor.
"""
import torch
import torch.distributed as dist

from .mp_pipeline import _device
from .train_spatial import train_model_spatial, verify_spatial_config


def verify_spatial_master_config(slice_method, image_size, num_spatial_parts_list, spatial_size, mp_size):
    """The tiles of replica 1 (ranks 0..P-1) and of the mirrored replica 2 (ranks mp_size-1..mp_size-P)
    must not share GPUs."""
    verify_spatial_config(slice_method, image_size, num_spatial_parts_list)
    assert mp_size >= 2 * num_spatial_parts_list[0], (
        "Spatial parts from each models i.e. model1 and model2 should use different ranks (cuda devices); "
        "To avoid this, increase the split size by keeping other configuration same.")


class train_spatial_model_master:
    def __init__(self, model_gen1, model_gen2, batch_size, spatial_size, num_spatial_parts, slice_method, mpi_comm_first,
                 mpi_comm_second, LOCAL_DP_LP, criterion=None, optimizer=None, parts=1, ASYNC=True, replications=1, *,
                 amp_dtype=None, recompute=False, cuda_graph=False):
        self.mp_size = mpi_comm_first.mp_size
        self.split_size = model_gen1.split_size
        self.local_rank = mpi_comm_first.local_rank
        self.mpi_comm_first, self.mpi_comm_second = mpi_comm_first, mpi_comm_second
        self.model_gen1, self.model_gen2 = model_gen1, model_gen2
        self.device = _device()
        self.model1_size = self.get_model_parameter_size(model_gen1)
        self.model2_size = self.get_model_parameter_size(model_gen2)
        self.flat_params_model1, self.flat_grads_model1 = self._flatten(model_gen1.models, self.model1_size)
        self.flat_params_model2, self.flat_grads_model2 = self._flatten(model_gen2.models, self.model2_size)
        common = dict(epochs=1, spatial_size=spatial_size, num_spatial_parts=num_spatial_parts, criterion=criterion,
                      optimizer=optimizer, parts=parts, ASYNC=ASYNC, slice_method=slice_method, LOCAL_DP_LP=LOCAL_DP_LP,
                      amp_dtype=amp_dtype, recompute=recompute, cuda_graph=cuda_graph)
        self.train_model1 = train_model_spatial(model_gen1, mpi_comm_first.local_rank, batch_size, GEMS_INVERSE=False,
                                                mpi_comm=mpi_comm_first, **common)
        self.train_model2 = train_model_spatial(model_gen2, mpi_comm_second.local_rank, batch_size, GEMS_INVERSE=True,
                                                mpi_comm=mpi_comm_second, **common)
        self.parts = parts
        self.ENABLE_ASYNC = ASYNC
        self.batch_size = batch_size
        self.replications = replications

    # ---- flat storage -------------------------------------------------------------------------
    def _flatten(self, model, size):
        """Move every parameter (and its gradient) of `model` into one flat buffer, in the parameters' dtype (fp32 under
        amp_dtype: the flat buffers hold the master weights and their gradients).

        Deliberate deviation: the reference re-points `param.data` at a freshly ZEROED buffer without
        copying the values in (:104-131, :187-192), i.e. it silently zero-initialises both replicas
        (every loss starts at ln(num_classes) and only the last bias ever trains).  Here the initial
        values are kept.  SPCONV_GEMS_REFERENCE_ZERO_INIT=1 reproduces the reference's behaviour
        bit for bit (used by the parity test)."""
        import os
        dtype = next((p.dtype for p in model.parameters()), torch.float32)
        flat_p = torch.zeros([size], device=self.device, dtype=dtype)
        flat_g = torch.zeros([size], device=self.device, dtype=dtype)
        off = 0
        if os.environ.get("SPCONV_GEMS_REFERENCE_ZERO_INIT") != "1":
            with torch.no_grad():
                for p in model.parameters():
                    n = p.numel()
                    flat_p[off:off + n].copy_(p.detach().reshape(-1))
                    off += n
        self.update_model_params_loc(model, flat_p)
        self.update_model_grads_loc(model, flat_g)
        return flat_p, flat_g

    def update_model_params_loc(self, model, flat_params):
        off = 0
        for p in model.parameters():
            n = p.numel()
            p.data = flat_params[off:off + n].view(p.shape)
            off += n

    def update_model_grads_loc(self, model, flat_grads):
        off = 0
        for p in model.parameters():
            n = p.numel()
            p.grad = flat_grads[off:off + n].view(p.shape)
            off += n

    def get_model_parameter_size(self, model_gen):
        return sum(p.numel() for p in model_gen.models.parameters())

    def model_parameters(self, model_gen):
        ps = [p.detach().reshape(-1) for p in model_gen.models.parameters()]
        return torch.cat(ps) if ps else None

    def update_model_paramters(self, model_gen, flat_params):
        off = 0
        with torch.no_grad():
            for p in model_gen.models.parameters():
                n = p.numel()
                p.copy_(flat_params[off:off + n].view(p.shape))
                off += n

    # ---- replica shipping between a rank and its mirror ----------------------------------------
    def _mirror(self):
        return self.mp_size - 1 - self.local_rank

    def _exchange(self, send_t, recv_t, peer):
        ops = [dist.P2POp(dist.isend, send_t, peer), dist.P2POp(dist.irecv, recv_t, peer)]
        for w in dist.batch_isend_irecv(ops):
            w.wait()

    def send_recv_params(self, odd_iteration=False):
        """Send the replica this pass trained, receive the other one (:248-273)."""
        send_t = self.flat_params_model2 if odd_iteration else self.flat_params_model1
        recv_t = self.flat_params_model1 if odd_iteration else self.flat_params_model2
        with torch.no_grad():
            self._exchange(send_t, recv_t, self._mirror())

    def send_recv_grads(self, odd_iteration=False):
        """Swap gradient buffers with the mirror rank and accumulate what arrives into the replica
        the second half of the step trains (:296-325)."""
        send_t = self.flat_grads_model2 if odd_iteration else self.flat_grads_model1
        acc = self.flat_grads_model1 if odd_iteration else self.flat_grads_model2
        got = torch.zeros_like(acc)
        self._exchange(send_t, got, self._mirror())
        acc += got

    # ---- steps ---------------------------------------------------------------------------------
    def run_step(self, inputs, labels):
        loss = correct = 0
        bs = self.batch_size
        for j in range(2 * self.replications):
            tm = self.train_model1 if j % 2 == 0 else self.train_model2
            l, c = tm.run_step(inputs[j * bs:(j + 1) * bs], labels[j * bs:(j + 1) * bs])
            loss += l
            correct += c
        return loss, correct

    def _half_step(self, tm, data_x, data_y, between):
        per = int(self.batch_size / self.parts)
        outs, loss, corrects = [], 0, 0
        for i in range(self.parts):
            y, c = tm.forward_pass(data_x[i * per:(i + 1) * per], data_y[i * per:(i + 1) * per], part_number=i)
            outs.append(y)
            if tm.split_rank == tm.split_size - 1:
                loss += y.item()
                corrects += c.item()
        between()
        for i in range(self.parts):
            tm.backward_pass(outs[i], part_number=i)
        return loss, corrects

    def run_step_allreduce(self, inputs, labels, odd_iteration):
        """Two half steps (:327-455).  First half trains replica A (1 on even iterations, 2 on odd):
        ranks other than the last position swap parameters with their mirror between forward and
        backward; the last position receives them before and sends after.  Second half trains
        replica B with the same pattern on gradient buffers, accumulating the mirror's gradients."""
        inputs = inputs.to(self.device)
        labels = labels.to(self.device)
        tm1, tm2 = (self.train_model2, self.train_model1) if odd_iteration else (self.train_model1, self.train_model2)
        peer = self._mirror()
        last = self.mp_size - 1
        recv_p = self.flat_params_model1 if odd_iteration else self.flat_params_model2
        send_p = self.flat_params_model2 if odd_iteration else self.flat_params_model1
        send_g = self.flat_grads_model2 if odd_iteration else self.flat_grads_model1
        acc_g = self.flat_grads_model1 if odd_iteration else self.flat_grads_model2

        if tm1.local_rank == last:
            with torch.no_grad():
                dist.recv(recv_p, src=peer)
        l1, c1 = self._half_step(tm1, inputs[:self.batch_size], labels[:self.batch_size],
                                 (lambda: self.send_recv_params(odd_iteration)) if tm1.local_rank != last else (lambda: None))
        if tm1.local_rank == last:
            dist.send(send_p, dst=peer)

        if tm2.local_rank == last:
            got = torch.zeros_like(acc_g)
            dist.recv(got, src=peer)
            acc_g += got
        l2, c2 = self._half_step(tm2, inputs[self.batch_size:], labels[self.batch_size:],
                                 (lambda: self.send_recv_grads(odd_iteration)) if tm2.local_rank != last else (lambda: None))
        if tm2.local_rank == last:
            dist.send(send_g, dst=peer)
        return l1 + l2, c1 + c2
