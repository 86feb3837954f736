"""torchgems.gems_master -- GEMS "master" training of a layer-parallel model: two replicas of the
pipeline share the same GPUs, the second one laid out in the opposite direction (its stage i runs
on rank mp_size-1-i), so that a rank is busy with replica 2 while it would idle in replica 1's
pipeline bubble.  Mirrors reference src/torchgems/gems_master.py:23-103 (train_model_master)."""
from .mp_pipeline import train_model


class train_model_master:
    def __init__(self, model_gen1, model_gen2, local_rank, batch_size, epochs, criterion=None, optimizer=None, parts=1,
                 ASYNC=True, replications=1, *, amp_dtype=None, recompute=False, cuda_graph=False):
        self.mp_size = self.split_size = model_gen1.split_size
        self.second_rank = self.split_size - local_rank - 1
        # as in the reference (:41-62) both replicas get the default criterion / optimizer
        self.train_model1 = train_model(model_gen1, local_rank, batch_size, epochs, parts=parts, ASYNC=True,
                                        GEMS_INVERSE=False, amp_dtype=amp_dtype, recompute=recompute,
                                        cuda_graph=cuda_graph)
        self.train_model2 = train_model(model_gen2, self.second_rank, batch_size, epochs, parts=parts, ASYNC=True,
                                        GEMS_INVERSE=True, amp_dtype=amp_dtype, recompute=recompute,
                                        cuda_graph=cuda_graph)
        self.parts, self.epochs, self.local_rank = parts, epochs, local_rank
        self.ENABLE_ASYNC = ASYNC
        self.batch_size = batch_size
        self.replications = replications

    def run_step(self, inputs, labels):
        """`inputs` holds 2 * replications batches; even ones go through replica 1, odd ones through
        the mirrored replica 2."""
        loss = correct = 0
        bs = self.batch_size
        for j in range(2 * self.replications):
            tm = self.train_model1 if j % 2 == 0 else self.train_model2
            l, c = tm.run_step(inputs[j * bs:(j + 1) * bs], labels[j * bs:(j + 1) * bs])
            loss += l
            correct += c
        return loss, correct
