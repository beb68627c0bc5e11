"""End-to-end tier (SURVEY 4.2): a few hundred ResNet-50 iterations through the flagship trainer on
N GPUs -- the loss must go down and the replicas must stay in consensus.

    torchrun --nproc-per-node 8 benchmarks/e2e_convergence.py --algo sgp --iters 300 --out gpurun_out/e2e_sgp.json

Data: a fixed synthetic pool per rank (64 batches, labels are a deterministic function of the image
so that the task is learnable by every rank and the ranks' optima agree).  Reported per run:
mean loss / prec@1 over the first and last 20 iterations (averaged over ranks), the relative consensus
distance  max_i ||z_i - zbar|| / ||zbar||  (zbar: the push-sum weighted average) after the run and at a few checkpoints, push-sum
weights, images/s.  Nothing here is timed for the headline; it is a correctness run.
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stochastic_gradient_push_b200 as sgp                                        # noqa: E402
from stochastic_gradient_push_b200 import models                                   # noqa: E402
from stochastic_gradient_push_b200.optim import FusedGossipSGD                     # noqa: E402
from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel  # noqa: E402
from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer           # noqa: E402


def consensus(tr):
    """max_i ||z_i - zbar|| / ||zbar|| over the push-sum average zbar = sum_i w_i z_i / sum_i w_i
    (GossipDataParallel.average_model; finish() first: under Overlap-SGP the trainer holds the last
    residual)"""
    tr.finish()
    tr.model.average_model()
    st = tr.model.last_consensus
    return max(d ** 0.5 for d in st.rank_distance_sq) / max(st.average_norm_sq ** 0.5, 1e-12)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--algo', default='sgp', choices=['sgp', 'osgp', 'dpsgd'])
    ap.add_argument('--model', default='resnet50')
    ap.add_argument('--iters', type=int, default=300)
    ap.add_argument('--batch-size', type=int, default=32)
    ap.add_argument('--classes', type=int, default=16)
    ap.add_argument('--image', type=int, default=224)
    ap.add_argument('--lr', type=float, default=0.05)
    ap.add_argument('--dtype', default='fp32')
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', 0)))
    dev = torch.device('cuda', torch.cuda.current_device())
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)                    # same initial weights on every rank
    net = models.MODEL_ZOO[args.model](num_classes=args.classes)
    if hasattr(models, 'init_imagenet_in_1hr') and args.model.startswith('resnet'):
        models.init_imagenet_in_1hr(net)
    net = net.to(dev).to(memory_format=torch.channels_last)
    if args.algo == 'dpsgd':
        graph = sgp.RingGraph(rank, world)
    else:
        graph = sgp.NPeerDynamicDirectedExponentialGraph(rank, world)
    amp = torch.bfloat16 if args.dtype == 'bf16' else None
    model = GossipDataParallel(net, graph=graph, push_sum=(args.algo != 'dpsgd'), overlap=(args.algo == 'osgp'),
                               rank=rank, world_size=world, heartbeat_timeout=120, compute_dtype=amp)
    opt = FusedGossipSGD(model, lr=args.lr, momentum=0.9, weight_decay=1e-4, nesterov=True)
    tr = GossipTrainer(model, opt, amp_dtype=amp, use_cuda_graph=True)

    # learnable synthetic task: class = which of `classes` fixed random templates was added to noise
    g = torch.Generator().manual_seed(4242)
    templates = torch.randn(args.classes, 3, args.image, args.image, generator=g)
    gr = torch.Generator().manual_seed(1000 + rank)
    pool = []
    for _ in range(64):
        y = torch.randint(0, args.classes, (args.batch_size,), generator=gr)
        x = 0.7 * templates[y] + torch.randn(args.batch_size, 3, args.image, args.image, generator=gr)
        pool.append((x.pin_memory(), y.pin_memory()))

    slots, cons = [], []
    t0 = time.time()
    for i in range(args.iters):
        x, y = pool[i % len(pool)]
        slots.append(tr.step(x, y))
        if (i + 1) % 100 == 0 or i == 19:
            tr.stream.synchronize()
            tr.check()
            rows = [tr.metrics_ring[s].tolist() for s in slots]
            slots = []
            cons.append({'iter': i + 1, 'consensus': consensus(tr),
                         'loss': sum(r[0] for r in rows[-20:]) / len(rows[-20:]),
                         'prec1': sum(r[1] for r in rows[-20:]) / len(rows[-20:])})
    tr.finish()
    wall = time.time() - t0
    final = consensus(tr)
    stats = torch.tensor([cons[0]['loss'], cons[-1]['loss'], cons[0]['prec1'], cons[-1]['prec1'],
                          float(model.ps_weight)], device=dev, dtype=torch.float64)
    lo, hi = stats.clone(), stats.clone()
    if world > 1:
        dist.all_reduce(stats)
        stats /= world
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    if rank == 0:
        out = {'algo': args.algo, 'model': args.model, 'world': world, 'iters': args.iters, 'dtype': args.dtype,
               'per_gpu_batch': args.batch_size, 'loss_first20': round(stats[0].item(), 4),
               'loss_last20': round(stats[1].item(), 4), 'prec1_first20': round(stats[2].item(), 2),
               'prec1_last20': round(stats[3].item(), 2), 'consensus_rel_final': final,
               'ps_weight_min_max': [round(lo[4].item(), 6), round(hi[4].item(), 6)],
               'checkpoints_rank0': cons, 'images_per_s_wall': round(args.batch_size * world * args.iters / wall, 1),
               'pass': bool(stats[1] < 0.7 * stats[0] and final < 0.05)}
        print(json.dumps(out))
        if args.out:
            with open(args.out, 'w') as f:
                json.dump(out, f, indent=1)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
