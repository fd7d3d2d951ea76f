"""Launcher with the reference's flags (main.py:10-64): generate the graph (or read its published files with
``--data-source files``; nothing is downloaded), partition it into the on-disk store (``data/store.py``:
``graph_partition`` unless ``--skip-partition``), start one process per partition / GPU; each loads its part
(``load_partition``; with ``--eval --parallel-eval --inductive`` also its parts of the two evaluation graphs,
``load_eval_partition``) and runs ``train.run``.  ogbn-papers100M is never built whole: its store is written by
streaming (``store.papers100m_partition``), and the configurations that would need its whole graph are refused at
launch (``store.check_papers100m``).

    python -m bns_gcn_b200.main --dataset ogbn-papers100m --data-source files --data-path ./dataset/ \
        --n-partitions 8 --partition-method random --use-pp --parallel-eval

    python -m bns_gcn_b200.main --dataset reddit --n-partitions 4 --model graphsage --n-layers 3 --n-hidden 256 \
        --sampling-rate 0.1 --use-pp --partition-method random --n-epochs 50 --no-eval

Under torchrun (RANK / WORLD_SIZE set) it joins the existing job instead of spawning.
"""
import os
import random
import warnings

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from .data.store import (EVAL_GRAPHS, check_papers100m, default_graph_name, graph_partition, load_eval_partition,
                         load_partition, wants_eval_partitions)
from .helper.parser import create_parser


def init_processes(rank, size, args):
    """train.py:459-470: rendezvous, load this rank's partition, run."""
    from . import train
    os.environ.setdefault('MASTER_ADDR', args.master_addr)
    os.environ.setdefault('MASTER_PORT', '%d' % args.port)
    local = rank % max(torch.cuda.device_count(), 1)
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    dist.init_process_group('nccl', rank=rank, world_size=size, device_id=dev)
    # Without --fix-seed every process drew its own args.seed (main(): random.randint).  The weights are created from
    # it on every rank and never broadcast (only gradients are all-reduced), so the replicas must agree on it:
    # rank 0's seed wins.  (The mp.spawn path pickles one args object to all ranks; under torchrun each rank ran main().)
    seed = [int(args.seed)]
    dist.broadcast_object_list(seed, src=0)
    args.seed = int(seed[0])
    if getattr(args, '_partition_in_job', False):          # torchrun: nobody partitioned before the ranks started
        if rank == 0:
            graph_partition(args, device=dev)
        dist.barrier()
    g, node_dict, gpb = load_partition(args, rank)          # train.py:469 (fills args.n_feat / n_class / n_train)
    eval_parts = None
    if wants_eval_partitions(args):                         # --eval --parallel-eval --inductive
        eval_parts = {w: load_eval_partition(args, w, rank) for w in EVAL_GRAPHS}
    train.run(g, node_dict, gpb, args, dev, eval_parts=eval_parts)
    dist.destroy_process_group()


def main(argv=None):
    args = create_parser(argv)
    check_papers100m(args)                                  # before anything is read or written
    if args.fix_seed is False:
        if args.parts_per_node < args.n_partitions:
            warnings.warn('Please enable `--fix-seed` for multi-node training.')
        args.seed = random.randint(0, 1 << 31)
    if args.backend in ('gloo', 'mpi'):
        warnings.warn(f'--backend {args.backend}: host-staged transports are what this build replaces; using nccl')
        args.backend = 'nccl'
    if args.graph_name == '':                               # main.py:17-23
        args.graph_name = default_graph_name(args)
    under_torchrun = 'RANK' in os.environ and 'WORLD_SIZE' in os.environ
    if not args.skip_partition:                             # main.py:25-30
        if under_torchrun:
            args._partition_in_job = True
        elif args.node_rank == 0:
            graph_partition(args)
    print(args)
    if under_torchrun:
        init_processes(int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), args)
        return
    mp.set_start_method('spawn', force=True)
    start = args.node_rank * args.parts_per_node
    procs = []
    for i in range(start, min(start + args.parts_per_node, args.n_partitions)):
        p = mp.Process(target=init_processes, args=(i, args.n_partitions, args))
        p.start()
        procs.append(p)
    for p in procs:
        p.join()


if __name__ == '__main__':
    main()
