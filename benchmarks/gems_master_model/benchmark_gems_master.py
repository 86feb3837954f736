"""GEMS-master training benchmark on a layer-parallel model: two replicas of the pipeline on the same
ranks, the second one mirrored (its stage i on rank split_size-1-i), each step trains 2 x --times/2
batches; afterwards the two replicas' gradients are combined rank <-> mirror rank
(SyncAllreduce.apply_allreduce_master_and_update).  Flags of the reference's
benchmarks/gems_master_model scripts; torchrun launch; runs on CPU/gloo too.

    torchrun --nproc-per-node 2 benchmarks/gems_master_model/benchmark_resnet_gems_master.py \\
        --split-size 2 --image-size 64 --batch-size 2 --times 2
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", ".."), os.path.join(HERE, "..")]

import common  # noqa: E402
from mpi4dl_b200.torchgems import comm as gems_comm  # noqa: E402
from mpi4dl_b200.torchgems import parser  # noqa: E402
from mpi4dl_b200.torchgems.gems_master import train_model_master  # noqa: E402
from mpi4dl_b200.torchgems.mp_pipeline import model_generator  # noqa: E402


def main(kind):
    p = parser.get_parser()
    p.add_argument("--dtype", choices=["fp32", "bf16", "bf16-amp"], default="fp32",
                   help="bf16-amp: fp32 parameters, the forward under torch.autocast(dtype=torch.bfloat16)")
    p.add_argument("--steps", type=int, default=10)
    args = p.parse_args()
    gems_comm.initialize_cuda()
    np.random.seed(seed=1405)
    batch_size, parts, image_size, mp_size = args.batch_size, args.parts, int(args.image_size), args.split_size
    times = max(2, args.times)                          # one batch per replica at least
    balance = [int(v) for v in args.balance.split(",")] if args.balance else None
    mb = int(batch_size / parts)
    dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float32
    amp_dtype = torch.bfloat16 if args.dtype == "bf16-amp" else None

    mpi_comm = gems_comm.MPIComm(split_size=mp_size, ENABLE_MASTER=True)
    local_rank = mpi_comm.rank % mp_size
    seq, seq_size, make_model = common.build_sequential(kind, args, mb, image_size)
    gen_seq = model_generator(model=seq, split_size=mp_size, input_size=(mb, 3, seq_size, seq_size), balance=balance)
    gen_seq.get_output_shapes(GET_SHAPES_ON_CUDA=torch.cuda.is_available())
    shapes = common.scale_shapes(gen_seq.shape_list, int(image_size / seq_size))
    del seq, gen_seq

    gens = []
    for stage in (local_rank, mp_size - local_rank - 1):            # replica 1, mirrored replica 2
        g = model_generator(model=make_model().to(dtype), split_size=mp_size, input_size=(mb, 3, image_size, image_size),
                            balance=balance, shape_list=shapes)
        g.ready_model(split_rank=stage)
        gens.append(g)
    tm_master = train_model_master(gens[0], gens[1], local_rank, batch_size, args.num_epochs, parts=parts, ASYNC=True,
                                   replications=int(times / 2), amp_dtype=amp_dtype)
    sync_allreduce = gems_comm.SyncAllreduce(mpi_comm)
    sync_allreduce.sync_model(gens[0], gens[1])

    perf = []
    for epoch in range(args.num_epochs):
        loss_sum = correct_sum = 0.0
        n = 0
        for inputs, labels in common.batches(args, image_size, batch_size * 2 * int(times / 2), args.steps):
            with common.StepTimer() as t:
                loss, correct = tm_master.run_step(inputs, labels)
                sync_allreduce.apply_allreduce_master_and_update(tm_master, gens[0], gens[1])
            loss_sum += loss
            correct_sum += correct
            n += 1
            if mpi_comm.rank == 0:
                print("Epoch: %d images per sec:%s" % (epoch, batch_size * 2 * int(times / 2) / t.seconds), flush=True)
                perf.append(batch_size * 2 * int(times / 2) / t.seconds)
            if mpi_comm.rank == mp_size - 1:
                print("Step :%d, LOSS: %s, Global loss: %s Acc: %s" % (n - 1, loss, loss_sum / n, correct), flush=True)
        if mpi_comm.rank == mp_size - 1 and n:
            print("Epoch %d Global loss: %s Acc %s" % (epoch, loss_sum / n, correct_sum / n), flush=True)
    if mpi_comm.rank == 0:
        common.report(perf)
    import torch.distributed as dist
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main(common.pop_model_flag(sys.argv, "resnet"))
