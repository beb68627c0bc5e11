"""
Shared machinery of the two training entry points (``gossip_sgd.py`` and
``gossip_sgd_adpsgd.py``): flag parsing, environment bootstrap, schedules,
data loaders, CSV logging, accuracy, checkpoint state.

Flag surface = the reference's (``gossip_sgd.py:72-159``,
``gossip_sgd_adpsgd.py:69-144``): same names, same defaults, booleans accepted
as the strings ``'True'/'False'`` so the shipped SLURM job scripts keep working.
Additions are opt-in: ``--synthetic`` (no dataset on the box), ``--fused``
(FusedGossipSGD instead of torch.optim.SGD), ``--amp`` (bf16 autocast),
``--channels_last``, ``--transport``; rank / world / master are also read from
torchrun's ``RANK / WORLD_SIZE / MASTER_ADDR`` when SLURM/OMPI variables are
absent.

The per-rank CSV is byte-compatible with the reference's (4 header lines, the
``Epoch,itr,BT(s),...,val`` column row; ``gossip_sgd.py:262-274``) so
``visualization/plotting.py`` reads either.
"""

from __future__ import annotations

import argparse
import copy
import os
import time

import torch
import torch.distributed as dist

from .. import (GRAPH_TOPOLOGIES, MIXING_STRATEGIES)
from ..experiment import ClusterManager, Meter, get_tcp_interface_name, make_logger


# --------------------------------------------------------------------------- #
# flags
# --------------------------------------------------------------------------- #
def str2bool(v):
    if isinstance(v, bool):
        return v
    if str(v).lower() in ('true', '1', 'yes', 'y'):
        return True
    if str(v).lower() in ('false', '0', 'no', 'n'):
        return False
    raise argparse.ArgumentTypeError('expected True/False, got %r' % (v,))


def build_parser(adpsgd: bool = False) -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description='Gossip SGD (H100-native)')
    B = dict(type=str2bool, nargs='?', const=True)
    p.add_argument('--all_reduce', default=False, **B, help='all-reduce instead of gossip')
    p.add_argument('--batch_size', default=32, type=int, help='per-agent batch size')
    p.add_argument('--lr', default=0.1, type=float,
                   help='reference learning rate (for a 256-sample batch)')
    p.add_argument('--num_dataloader_workers', default=10, type=int)
    p.add_argument('--num_epochs', default=90, type=int)
    p.add_argument('--momentum', default=0.9, type=float)
    p.add_argument('--weight_decay', default=1e-4, type=float)
    p.add_argument('--nesterov', default=False, **B)
    p.add_argument('--no_bias_decay', default=False, **B,
                   help='no weight decay on parameters with ndim <= 1 (BatchNorm weight and bias, all '
                        'biases): two parameter groups (optim.no_bias_decay_groups), for --fused True '
                        'and False alike.  SGP / OSGP / D-PSGD')
    p.add_argument('--lars', default=False, **B,
                   help='LARS (layer-wise adaptive rate scaling) inside the fused gossip step '
                        '(FusedGossipSGD(lars=True)); with --no_bias_decay True the groups are '
                        'optim.lars_groups (no decay and no LARS for ndim <= 1 parameters).  --fused True '
                        'with SGP / OSGP / D-PSGD only')
    p.add_argument('--lars_trust', default=0.001, type=float, help='LARS trust coefficient eta')
    p.add_argument('--clip_grad_norm', default=0.0, type=float,
                   help='clip each rank\'s gradient to this global 2-norm inside the fused gossip step '
                        '(FusedGossipSGD(max_grad_norm=...), torch.nn.utils.clip_grad_norm_ semantics); '
                        '0 = off.  --fused True with SGP / OSGP / D-PSGD only')
    p.add_argument('--skip_nonfinite', default=False, **B,
                   help='skip the SGD of a step whose gradient norm is inf or NaN on that rank (the rank '
                        'keeps gossiping; FusedGossipSGD(skip_nonfinite=True)).  --fused True with SGP / '
                        'OSGP / D-PSGD only')
    p.add_argument('--push_sum', default=True, **B, help='push-sum (SGP) or push-pull (D-PSGD)')
    p.add_argument('--graph_type', default=5, type=int, choices=list(GRAPH_TOPOLOGIES))
    p.add_argument('--mixing_strategy', default=0, type=int, choices=list(MIXING_STRATEGIES))
    p.add_argument('--schedule', nargs='+', default=None, type=float,
                   help='epoch factor epoch factor ... (default 30 0.1 60 0.1 80 0.1)')
    p.add_argument('--peers_per_itr_schedule', nargs='+', type=int,
                   help='epoch num_peers epoch num_peers ...; must contain epoch 0')
    p.add_argument('--overlap', default=False, **B)
    p.add_argument('--synch_freq', default=0, type=int)
    p.add_argument('--warmup', default=False, **B, help='linear LR warm-up over --warmup_epochs epochs')
    p.add_argument('--warmup_epochs', default=5, type=int,
                   help='length of the --warmup ramp from --lr to the scaled target learning rate')
    p.add_argument('--lr_policy', default='step', choices=['step', 'poly'],
                   help='after the warm-up: step = multiply by the --schedule factors (Goyal et al.); '
                        'poly = end_lr + (target - end_lr) * (1 - progress) ** poly_power, set every '
                        'iteration (the MLPerf ResNet-50 recipe, with --lars)')
    p.add_argument('--poly_power', default=2.0, type=float, help='exponent of --lr_policy poly')
    p.add_argument('--end_lr', default=0.0001, type=float,
                   help='learning rate that --lr_policy poly reaches at the end (absolute, not scaled)')
    p.add_argument('--label_smoothing', default=0.0, type=float,
                   help='label smoothing eps in [0, 1] of the training loss (as in '
                        'torch.nn.CrossEntropyLoss(label_smoothing=eps); on the fused loss kernel with '
                        '--cuda_graph True); validation keeps the plain cross-entropy')
    p.add_argument('--mixup_alpha', default=0.0, type=float,
                   help='mixup (Zhang et al. 2018) on the training batch: lam ~ Beta(a, a), each image mixed '
                        'with its partner in the flipped batch, two-target loss; 0 = off.  Fused into the '
                        'input copy and the fused loss kernel with --cuda_graph True; validation is never mixed')
    p.add_argument('--cutmix_alpha', default=0.0, type=float,
                   help='CutMix (Yun et al. 2019): a box of area 1 - lam, lam ~ Beta(a, a), pasted from the '
                        'partner image; 0 = off.  With --mixup_alpha too, one of the two per step')
    p.add_argument('--mix_prob', default=1.0, type=float,
                   help='probability that a training step is mixed (mixup or CutMix)')
    p.add_argument('--mix_switch_prob', default=0.5, type=float,
                   help='with both alphas > 0: probability that a mixed step uses CutMix rather than mixup')
    p.add_argument('--model_ema_decay', default=0.0, type=float,
                   help='keep an exponential moving average of the weights and BatchNorm statistics '
                        '(ops.model_ema.ModelEma) with this decay in [0, 1), updated after every step (inside '
                        'the captured step with --cuda_graph True), validated at each epoch end and logged to '
                        '<checkpoint_dir><tag>ema_r<rank>_n<world>.csv; 0 = off.  Not with AD-PSGD')
    p.add_argument('--model_ema_warmup', default=False, **B,
                   help='EMA decay warm-up: min(decay, (1 + t) / (10 + t)) after t updates')
    p.add_argument('--drop_path_rate', default=0.0, type=float,
                   help='stochastic depth (Huang et al. 2016; timm drop_path_rate) in [0, 1) on the ResNet residual '
                        'blocks, linear in the block index (block 0 never drops, the last drops with this rate); '
                        'applied inside the fused BatchNorm kernels, drawn from (--seed, rank); 0 = off.  Not with '
                        '--model tiny')
    p.add_argument('--distill_alpha', default=0.0, type=float,
                   help='knowledge distillation (Hinton et al. 2015) weight alpha in [0, 1]: the training loss is '
                        '(1 - alpha) CE + alpha T^2 KL(softmax(teacher / T) || softmax(student / T)), the teacher '
                        'being --teacher_model loaded from --teacher_checkpoint, frozen in eval mode; 0 = off.  '
                        'On the fused loss kernel inside the captured step with --cuda_graph True; validation '
                        'never distils.  Not with AD-PSGD')
    p.add_argument('--distill_temperature', default=1.0, type=float,
                   help='softmax temperature T > 0 of --distill_alpha')
    p.add_argument('--teacher_model', default=None, type=str,
                   help='architecture of the --distill_alpha teacher, a models.MODEL_ZOO key (with --num_classes)')
    p.add_argument('--teacher_checkpoint', default=None, type=str,
                   help='weights of the --distill_alpha teacher: a model state_dict, or a checkpoint this '
                        'trainer wrote.  Loaded again on --resume (the teacher is not checkpointed)')
    p.add_argument('--seed', default=47, type=int)
    p.add_argument('--resume', default=False, **B)
    p.add_argument('--backend', default='nccl', choices=['nccl', 'gloo', 'mpi'])
    p.add_argument('--tag', default='', type=str)
    p.add_argument('--print_freq', default=10, type=int)
    p.add_argument('--verbose', default=True, **B)
    p.add_argument('--train_fast', default=False, **B)
    p.add_argument('--checkpoint_all', default=True, **B)
    p.add_argument('--master_port', default='40100', type=str)
    p.add_argument('--checkpoint_dir', type=str, default='./checkpoints/')
    p.add_argument('--network_interface_type', default='infiniband',
                   choices=['infiniband', 'ethernet'])
    p.add_argument('--dataset_dir', type=str, default=None)
    if adpsgd:
        p.add_argument('--bilat', default=True, **B)
        p.add_argument('--shared_fpath', default='', type=str,
                       help='file on a shared FS used as the global iteration counter')
        p.add_argument('--bs_fpath', default='', type=str, help='(accepted, unused; parity)')
    else:
        p.add_argument('--num_iterations_per_training_epoch', default=None, type=int,
                       help='testing only: leave the training loop early')
        p.add_argument('--overwrite_checkpoints', default=True, **B)
        p.add_argument('--num_itr_ignore', type=int, default=10)
        p.add_argument('--no_cuda_streams', action='store_true')
    # ---- H100-native additions (all optional) ----
    p.add_argument('--synthetic', default=None, **B,
                   help='synthetic 3x224x224 data (default: True when --dataset_dir is unset)')
    p.add_argument('--synthetic_len', default=1281167, type=int, help='images per synthetic epoch')
    p.add_argument('--data_format', default='folder', choices=['folder', 'shards'],
                   help="folder: torchvision ImageFolder + DataLoader workers (the reference's pipeline); "
                        "shards: pre-decoded uint8 shards under DATASET_DIR/{train,val} (python -m "
                        "stochastic_gradient_push_b200.data.make_shards) gathered by a background thread, "
                        "crop / flip / normalisation on the GPU (data/shards.py)")
    p.add_argument('--auto_augment', default='none', choices=['none', 'ta_wide', 'ra', 'imagenet'],
                   help='augmentation policy on the training images: ta_wide TrivialAugmentWide (torchvision\'s '
                        'ResNet-50 recipe), ra RandAugment (--ra_num_ops, --ra_magnitude), imagenet AutoAugment '
                        'with the ImageNet policy; with --data_format shards inside the GPU augment kernel '
                        '(data.GpuAugment), with --data_format folder the torchvision transform after the '
                        'flip.  Not with synthetic data')
    p.add_argument('--ra_num_ops', default=2, type=int,
                   help='--auto_augment ra: ops applied in sequence to each image, in [0, 4]')
    p.add_argument('--ra_magnitude', default=9, type=int,
                   help='--auto_augment ra: magnitude bin of every op, in [0, 30]')
    p.add_argument('--random_erase', default=0.0, type=float,
                   help='probability p in [0, 1] of RandomErasing(p, value=0) after the normalisation of each '
                        'training image (GPU augment kernel with --data_format shards, '
                        'transforms.RandomErasing(p) with --data_format folder); 0 = off.  Not with synthetic data')
    p.add_argument('--fused', default=True, **B, help='FusedGossipSGD (SGD inside the gossip kernel)')
    p.add_argument('--amp', default=True, **B, help='bf16 autocast for forward/backward')
    p.add_argument('--channels_last', default=True, **B)
    p.add_argument('--transport', default='auto', choices=['auto', 'nvlink', 'c10d'])
    p.add_argument('--gossip_dtype', default='fp32', choices=['fp32', 'bf16'],
                   help='precision of the gossip messages (GossipDataParallel(gossip_dtype=...)): bf16 '
                        'halves the bytes sent per in-neighbour and conserves push-sum mass exactly; '
                        'parameters stay fp32.  Synchronous SGP and D-PSGD only')
    p.add_argument('--consensus_freq', default=0, type=int,
                   help='every N iterations and at each epoch end, log the consensus distance of the '
                        'ranks\' models (GossipDataParallel.consensus_distance) to stdout and to '
                        '<checkpoint_dir><tag>consensus_r<rank>_n<world>.csv; 0 = off.  SGP / OSGP / D-PSGD')
    p.add_argument('--validate_average', default=False, **B,
                   help='at each epoch end, also validate the push-sum average model (BatchNorm running '
                        'statistics averaged over the ranks for the purpose) and log its prec@1 in the '
                        'consensus CSV.  SGP / OSGP / D-PSGD')
    p.add_argument('--slowmo_frequency', default=0, type=int,
                   help='SlowMo (GossipDataParallel(slowmo_frequency=N)): every N iterations, average the '
                        'ranks\' models exactly and take a slow-momentum step; 0 = off.  SGP / OSGP / '
                        'D-PSGD with --nprocs_per_node 1')
    p.add_argument('--slowmo_lr', default=1.0, type=float, help='SlowMo slow learning rate alpha')
    p.add_argument('--slowmo_momentum', default=0.5, type=float, help='SlowMo slow momentum beta')
    p.add_argument('--nprocs_per_node', default=1, type=int,
                   help='hierarchical mode (GossipDataParallel(nprocs_per_node=K), reference '
                        'gossip/distributed.py:62-80; it has no flag for it): K consecutive ranks form a '
                        'node -- only its first rank gossips, on a graph over the NODES; parameters are '
                        'broadcast and gradients averaged inside the node every iteration (NVLS kernels on '
                        'one NVLink domain).  E.g. N hosts x 8 GPUs: --nprocs_per_node 8')
    p.add_argument('--model', default='resnet50')
    p.add_argument('--num_classes', default=1000, type=int)
    p.add_argument('--image_size', default=224, type=int)
    p.add_argument('--device', default=None, help="'cuda' / 'cpu' (default: cuda if available)")
    p.add_argument('--trace_file', default='', type=str,
                   help='write a Chrome trace (PREFIX_r<rank>.json; NVTX ranges on CUDA) of the '
                        'first --trace_iters training iterations')
    p.add_argument('--trace_iters', default=50, type=int)
    return p


def pairs_to_dict(flat, cast=float):
    """[e0, v0, e1, v1, ...] -> {e0: v0, e1: v1, ...}"""
    flat = list(flat)
    assert len(flat) % 2 == 0, 'schedule needs (epoch, value) pairs'
    return {int(flat[i]): cast(flat[i + 1]) for i in range(0, len(flat), 2)}


def resolve_env(args):
    """rank / world / master from SLURM, OpenMPI or torchrun variables."""
    env = os.environ
    if args.backend == 'mpi' and 'OMPI_COMM_WORLD_RANK' in env:
        args.rank = int(env['OMPI_COMM_WORLD_RANK'])
        args.world_size = int(env.get('OMPI_UNIVERSE_SIZE', env.get('OMPI_COMM_WORLD_SIZE', 1)))
    elif 'SLURM_PROCID' in env and 'RANK' not in env:
        args.rank = int(env['SLURM_PROCID'])
        args.world_size = int(env['SLURM_NTASKS'])
    else:
        args.rank = int(env.get('RANK', 0))
        args.world_size = int(env.get('WORLD_SIZE', 1))
    args.local_rank = int(env.get('LOCAL_RANK', env.get('SLURM_LOCALID', 0)))
    args.master_addr = env.get('MASTER_ADDR') or env.get('HOSTNAME') or '127.0.0.1'
    if 'MASTER_PORT' in env and 'SLURM_PROCID' not in env:
        args.master_port = env['MASTER_PORT']
    return args


def resolve_backend(args) -> str:
    """``--backend mpi`` (reference ``gossip_sgd.py:127-129, 600-602``): ranks come from the
    ``mpirun`` environment (``OMPI_COMM_WORLD_*``, see :func:`resolve_env`).  A PyTorch built with
    MPI uses the MPI process group as in the reference; otherwise MPI stays the *launcher* and the
    control plane is a TCP rendezvous (MASTER_ADDR / MASTER_PORT, exported by the job script) over
    nccl (CUDA) or gloo (CPU).  Either way the data plane on one NVLink domain is the kernel
    transport, which never touches the process group."""
    if args.backend != 'mpi':
        return args.backend
    if dist.is_mpi_available():
        return 'mpi'
    return 'nccl' if (args.device == 'cuda' and dist.is_nccl_available()) else 'gloo'


def finalize_args(args, adpsgd=False):
    """Derived settings + process-group / graph / mixing construction."""
    resolve_env(args)
    if args.checkpoint_dir and not args.checkpoint_dir.endswith('/'):
        args.checkpoint_dir += '/'
    os.makedirs(args.checkpoint_dir, exist_ok=True)
    ClusterManager.set_checkpoint_dir(args.checkpoint_dir)
    args.out_fname = '{}{}out_r{}_n{}.csv'.format(args.checkpoint_dir, args.tag, args.rank,
                                                  args.world_size)
    if args.device is None:
        args.device = 'cuda' if torch.cuda.is_available() else 'cpu'
    if args.device == 'cpu' and args.backend == 'nccl':
        args.backend = 'gloo'
    if args.synthetic is None:
        args.synthetic = args.dataset_dir is None
    args.cpu_comm = (args.backend == 'gloo' and not args.push_sum and not args.all_reduce) \
        or args.device == 'cpu'
    args.comm_device = torch.device('cpu') if args.cpu_comm else torch.device('cuda')
    args.lr_schedule = pairs_to_dict(args.schedule if args.schedule is not None
                                     else [30, 0.1, 60, 0.1, 80, 0.1], float)
    args.ppi_schedule = pairs_to_dict(args.peers_per_itr_schedule
                                      if args.peers_per_itr_schedule is not None else [0, 1], int)
    assert 0 in args.ppi_schedule, 'peers_per_itr_schedule must define epoch 0'
    if args.all_reduce:
        assert args.graph_type == -1, '--all_reduce needs --graph_type -1'
    if args.gossip_dtype == 'bf16':
        unsupported = ('AD-PSGD' if adpsgd else '--all_reduce' if args.all_reduce else
                       '--overlap (OSGP)' if getattr(args, 'overlap', False) else
                       '--nprocs_per_node > 1' if getattr(args, 'nprocs_per_node', 1) > 1 else None)
        if unsupported:
            raise ValueError('--gossip_dtype bf16 is not supported with %s; bf16 messages are '
                             'implemented for synchronous SGP and D-PSGD' % unsupported)
    if getattr(args, 'consensus_freq', 0) or getattr(args, 'validate_average', False):
        unsupported = 'AD-PSGD' if adpsgd else '--all_reduce' if args.all_reduce else None
        if unsupported:
            raise ValueError('--consensus_freq / --validate_average are not supported with %s: they '
                             'measure gossip (SGP, OSGP, D-PSGD)' % unsupported)
        if args.consensus_freq < 0:
            raise ValueError('--consensus_freq must be >= 0')
    if getattr(args, 'no_bias_decay', False):
        unsupported = 'AD-PSGD' if adpsgd else '--all_reduce' if args.all_reduce else None
        if unsupported:
            raise ValueError('--no_bias_decay is not supported with %s: parameter groups are '
                             'implemented for SGP, OSGP and D-PSGD' % unsupported)
    if getattr(args, 'lars', False):
        unsupported = ('AD-PSGD' if adpsgd else '--all_reduce' if args.all_reduce else
                       '--fused False' if not getattr(args, 'fused', True) else None)
        if unsupported:
            raise ValueError('--lars is not supported with %s: LARS is implemented in the fused gossip '
                             'step (FusedGossipSGD) for SGP, OSGP and D-PSGD' % unsupported)
        if not args.lars_trust > 0:
            raise ValueError('--lars_trust must be > 0')
    check_grad_clip_flags(args, adpsgd)
    if getattr(args, 'slowmo_frequency', 0):
        unsupported = ('AD-PSGD' if adpsgd else '--all_reduce' if args.all_reduce else
                       '--nprocs_per_node > 1' if getattr(args, 'nprocs_per_node', 1) > 1 else None)
        if unsupported:
            raise ValueError('--slowmo_frequency is not supported with %s: SlowMo is implemented for '
                             'SGP, OSGP and D-PSGD' % unsupported)
        from ..parallel.distributed import check_slowmo_args
        check_slowmo_args(args.slowmo_frequency, args.slowmo_lr, args.slowmo_momentum)
    check_schedule_args(args)
    if not 0.0 <= getattr(args, 'label_smoothing', 0.0) <= 1.0:
        raise ValueError('--label_smoothing must be in [0, 1], got %r' % (args.label_smoothing,))
    check_mix_flags(args)
    check_augment_flags(args)
    check_ema_flags(args, adpsgd)
    check_drop_path_flags(args)
    check_distill_flags(args, adpsgd)
    args.ema_fname = '{}{}ema_r{}_n{}.csv'.format(args.checkpoint_dir, args.tag, args.rank, args.world_size)
    args.consensus_fname = '{}{}consensus_r{}_n{}.csv'.format(args.checkpoint_dir, args.tag, args.rank,
                                                              args.world_size)

    if args.backend == 'gloo' and args.network_interface_type == 'ethernet':
        try:
            os.environ['GLOO_SOCKET_IFNAME'] = get_tcp_interface_name('ethernet')
        except Exception:
            pass
    elif args.network_interface_type == 'ethernet' and args.backend == 'nccl':
        os.environ['NCCL_SOCKET_IFNAME'] = get_tcp_interface_name('ethernet')
        os.environ['NCCL_IB_DISABLE'] = '1'

    if args.device == 'cuda':
        torch.cuda.set_device(args.local_rank % max(torch.cuda.device_count(), 1))
    os.environ['MASTER_ADDR'] = str(args.master_addr)
    # one control-plane world is enough (the reference's AD-PSGD script needs
    # master_port and master_port+1 because its gossip PROCESS owns a second world)
    os.environ['MASTER_PORT'] = str(args.master_port)
    if not dist.is_initialized() and args.world_size > 1:
        dist.init_process_group(backend=resolve_backend(args), world_size=args.world_size, rank=args.rank)
        dist.barrier()        # create the communicator now, not >5 min apart (reference :678-682)

    args.graph, args.mixing = None, None
    graph_class = GRAPH_TOPOLOGIES[args.graph_type]
    args.graph_class = graph_class
    args.mixing_class = MIXING_STRATEGIES[args.mixing_strategy]
    k = max(1, int(getattr(args, 'nprocs_per_node', 1)))
    args.nprocs_per_node = k
    if k > 1:
        assert not adpsgd and not args.all_reduce, '--nprocs_per_node applies to SGP / OSGP / D-PSGD'
        assert args.world_size % k == 0, '--nprocs_per_node must divide the number of ranks'
    if graph_class is not None and not adpsgd:
        # (hierarchical mode: the graph connects NODES; edges address each node's first rank)
        args.graph = graph_class(args.rank // k, args.world_size // k, nprocs_per_node=k,
                                 local_rank=args.rank % k, peers_per_itr=args.ppi_schedule[0])
        if args.mixing_class is not None:
            args.mixing = args.mixing_class(args.graph, args.comm_device)
    return args


# --------------------------------------------------------------------------- #
# schedules
# --------------------------------------------------------------------------- #
def check_mix_flags(args):
    """ValueError for mixup / CutMix flags out of range."""
    for flag in ('mixup_alpha', 'cutmix_alpha'):
        v = getattr(args, flag, 0.0)
        if not 0.0 <= v < float('inf'):
            raise ValueError('--%s must be a finite value >= 0, got %r' % (flag, v))
    for flag in ('mix_prob', 'mix_switch_prob'):
        v = getattr(args, flag, 0.0)
        if not 0.0 <= v <= 1.0:
            raise ValueError('--%s must be in [0, 1], got %r' % (flag, v))


def check_augment_flags(args):
    """ValueError for --random_erase outside [0, 1], --ra_num_ops outside [0, 4], --ra_magnitude
    outside [0, 30], and for --auto_augment / --random_erase with synthetic data (there are no images
    to augment)."""
    p = getattr(args, 'random_erase', 0.0)
    if not 0.0 <= p <= 1.0:
        raise ValueError('--random_erase must be in [0, 1], got %r' % (p,))
    for flag, hi in (('ra_num_ops', 4), ('ra_magnitude', 30)):
        v = getattr(args, flag, 0)
        if not 0 <= v <= hi:
            raise ValueError('--%s must be in [0, %d], got %r' % (flag, hi, v))
    if (getattr(args, 'auto_augment', 'none') != 'none' or p > 0) and args.synthetic:
        raise ValueError('--auto_augment / --random_erase need image data (--dataset_dir); synthetic data '
                         'has no images to augment')


def check_grad_clip_flags(args, adpsgd=False):
    """ValueError for --clip_grad_norm / --skip_nonfinite outside the fused gossip step, or for a
    negative or non-finite --clip_grad_norm."""
    clip = getattr(args, 'clip_grad_norm', 0.0)
    if not (clip >= 0 and clip != float('inf')):
        raise ValueError('--clip_grad_norm must be a finite number >= 0 (0 = off), got %r' % (clip,))
    for flag, on in (('--clip_grad_norm', clip > 0), ('--skip_nonfinite', getattr(args, 'skip_nonfinite', False))):
        if not on:
            continue
        unsupported = ('AD-PSGD' if adpsgd else '--all_reduce' if args.all_reduce else
                       '--fused False' if not getattr(args, 'fused', True) else None)
        if unsupported:
            raise ValueError('%s is not supported with %s: gradient clipping and non-finite step skipping '
                             'are implemented in the fused gossip step (FusedGossipSGD) for SGP, OSGP and '
                             'D-PSGD' % (flag, unsupported))


def check_eval_graph_flags(args):
    """ValueError for --eval_graph True outside the captured fused gossip step (GossipTrainer), whose
    ``evaluate()`` it calls."""
    if not getattr(args, 'eval_graph', False):
        return
    unsupported = ('--all_reduce' if args.all_reduce else
                   '--fused False' if not args.fused else
                   '--cuda_graph False' if not args.cuda_graph else
                   '--transport c10d' if args.transport == 'c10d' else
                   '--device cpu' if args.device == 'cpu' else None)
    if unsupported:
        raise ValueError('--eval_graph is not supported with %s: the captured evaluation is '
                         'GossipTrainer.evaluate, which needs the captured fused gossip step (--cuda_graph True '
                         '--fused True on the CUDA kernel transport) for SGP, OSGP and D-PSGD' % unsupported)


def check_precise_bn_flags(args):
    """ValueError for --precise_bn_batches < 0, and for N > 0 outside the captured fused gossip step
    (GossipTrainer), whose ``update_bn()`` it calls."""
    n = getattr(args, 'precise_bn_batches', 0)
    if n < 0:
        raise ValueError('--precise_bn_batches must be >= 0, got %r' % (n,))
    if n == 0:
        return
    unsupported = ('--all_reduce' if args.all_reduce else
                   '--fused False' if not args.fused else
                   '--cuda_graph False' if not args.cuda_graph else
                   '--transport c10d' if args.transport == 'c10d' else
                   '--device cpu' if args.device == 'cpu' else None)
    if unsupported:
        raise ValueError('--precise_bn_batches is not supported with %s: the statistics are recomputed by '
                         'GossipTrainer.update_bn, which needs the captured fused gossip step (--cuda_graph True '
                         '--fused True on the CUDA kernel transport) for SGP, OSGP and D-PSGD' % unsupported)


def check_accumulation_flags(args):
    """ValueError for --accumulation_steps < 1, for K > 1 outside the captured fused gossip step
    (GossipTrainer), and for a --batch_size that K does not divide."""
    k = args.accumulation_steps
    if k < 1:
        raise ValueError('--accumulation_steps must be >= 1, got %r' % (k,))
    if k == 1:
        return
    unsupported = ('--all_reduce' if args.all_reduce else
                   '--fused False' if not args.fused else
                   '--cuda_graph False' if not args.cuda_graph else
                   '--transport c10d' if args.transport == 'c10d' else
                   '--device cpu' if args.device == 'cpu' else
                   '--nprocs_per_node > 1' if args.nprocs_per_node > 1 else None)
    if unsupported:
        raise ValueError('--accumulation_steps > 1 is not supported with %s: gradient accumulation is '
                         'implemented in the captured fused gossip step (--cuda_graph True --fused True) for '
                         'SGP, OSGP and D-PSGD' % unsupported)
    if args.batch_size % k:
        raise ValueError('--batch_size %d is not divisible by --accumulation_steps %d'
                         % (args.batch_size, k))


def check_drop_path_flags(args):
    """ValueError for --drop_path_rate outside [0, 1), and for a rate > 0 with --model tiny (no residual blocks)."""
    p = getattr(args, 'drop_path_rate', 0.0)
    if not 0.0 <= p < 1.0:
        raise ValueError('--drop_path_rate must be in [0, 1), got %r' % (p,))
    if p > 0 and args.model == 'tiny':
        raise ValueError('--drop_path_rate is not supported with --model tiny: stochastic depth drops residual '
                         'blocks, and TinyConvNet has none')


def model_num_classes(name, args) -> int:
    """the number of classes ``init_model`` gives model ``name`` (``tiny`` keeps TinyConvNet's default)"""
    if name == 'tiny':
        import inspect
        from ..models import TinyConvNet
        return inspect.signature(TinyConvNet).parameters['num_classes'].default
    return args.num_classes


def check_distill_flags(args, adpsgd=False):
    """ValueError for --distill_alpha outside [0, 1], --distill_temperature not finite and > 0, and for
    alpha > 0 with AD-PSGD, without both --teacher_model and --teacher_checkpoint, or with a teacher whose
    class count differs from the student's."""
    import math
    alpha = getattr(args, 'distill_alpha', 0.0)
    temp = getattr(args, 'distill_temperature', 1.0)
    if not 0.0 <= alpha <= 1.0:
        raise ValueError('--distill_alpha must be in [0, 1], got %r' % (alpha,))
    if not (math.isfinite(temp) and temp > 0.0):
        raise ValueError('--distill_temperature must be finite and > 0, got %r' % (temp,))
    if alpha == 0.0:
        return
    if adpsgd:
        raise ValueError('--distill_alpha is not supported with AD-PSGD: only the SGP / OSGP / D-PSGD and '
                         'all-reduce trainers run a teacher')
    if not getattr(args, 'teacher_model', None) or not getattr(args, 'teacher_checkpoint', None):
        raise ValueError('--distill_alpha > 0 needs --teacher_model and --teacher_checkpoint')
    from ..models import MODEL_ZOO
    if args.teacher_model not in MODEL_ZOO:
        raise ValueError('--teacher_model must be one of %s, got %r' % (', '.join(sorted(MODEL_ZOO)), args.teacher_model))
    nt, ns = model_num_classes(args.teacher_model, args), model_num_classes(args.model, args)
    if nt != ns:
        raise ValueError('the teacher --teacher_model %s has %d classes but the student --model %s has %d'
                         % (args.teacher_model, nt, args.model, ns))


def teacher_state_dict(obj):
    """the model ``state_dict`` inside a loaded --teacher_checkpoint: the object itself, or from a checkpoint this
    trainer wrote its ``'state_dict'`` (of the data-parallel wrapper: its own ``'state_dict'`` again for the
    gossip wrappers), with the wrapper's ``module.`` key prefix stripped and the wrapper's own entries dropped"""
    sd = obj
    for _ in range(2):                                 # checkpoint -> wrapper state -> module state
        if isinstance(sd, dict) and isinstance(sd.get('state_dict'), dict):
            sd = sd['state_dict']
    if not isinstance(sd, dict):
        raise ValueError('--teacher_checkpoint holds no state_dict (got %s)' % type(obj).__name__)
    if any(k.startswith('module.') for k in sd):
        sd = {k[len('module.'):]: v for k, v in sd.items() if k.startswith('module.')}
    return sd


def load_teacher(args):
    """The --distill_alpha teacher: --teacher_model with --num_classes, loaded strictly from
    --teacher_checkpoint (the same file on every rank), on ``args.device`` (channels_last with
    --channels_last on CUDA), in eval mode without gradients.  None when --distill_alpha is 0."""
    if not getattr(args, 'distill_alpha', 0.0) > 0:
        return None
    from .. import models
    kw = {} if args.teacher_model == 'tiny' else {'num_classes': args.num_classes}
    net = models.MODEL_ZOO[args.teacher_model](**kw)
    ckpt = torch.load(args.teacher_checkpoint, map_location='cpu', weights_only=False)
    net.load_state_dict(teacher_state_dict(ckpt), strict=True)
    net = net.to(args.device)
    if args.channels_last and args.device == 'cuda':
        net = net.to(memory_format=torch.channels_last)
    return net.eval().requires_grad_(False)


def stochastic_depth_of(model):
    """the ``ops.stochastic_depth.StochasticDepth`` of ``model`` (through a data-parallel wrapper), or None"""
    return getattr(getattr(model, 'module', model), 'stochastic_depth', None)


def save_stochastic_depth(state, model):
    """checkpoint the draw counter under ``stochastic_depth`` (--drop_path_rate > 0 only)"""
    sd = stochastic_depth_of(model)
    if sd is not None:
        state['stochastic_depth'] = sd.state_dict()


def load_stochastic_depth(ckpt, state, model, log):
    """--resume: continue the draw sequence where the checkpoint left it"""
    sd = stochastic_depth_of(model)
    if sd is None:
        return
    if 'stochastic_depth' in ckpt:
        sd.load_state_dict(ckpt['stochastic_depth'])
        state['stochastic_depth'] = ckpt['stochastic_depth']
    else:
        log.warning('checkpoint has no stochastic_depth: the drop masks start again from draw 0')


def check_ema_flags(args, adpsgd=False):
    """ValueError for --model_ema_decay out of [0, 1) or with AD-PSGD."""
    d = getattr(args, 'model_ema_decay', 0.0)
    if not 0.0 <= d < 1.0:
        raise ValueError('--model_ema_decay must be in [0, 1), got %r' % (d,))
    if d > 0 and adpsgd:
        raise ValueError('--model_ema_decay is not supported with AD-PSGD: its gossip daemon rewrites the '
                         'parameters concurrently on another stream')


def make_model_ema(args, model):
    """The ``ops.model_ema.ModelEma`` of ``model`` for --model_ema_decay (None when it is 0)."""
    if not getattr(args, 'model_ema_decay', 0.0) > 0:
        return None
    from ..ops.model_ema import ModelEma
    return ModelEma(model, decay=args.model_ema_decay, warmup=args.model_ema_warmup)


def check_schedule_args(args):
    """ValueError for learning-rate policy flags that contradict each other."""
    policy = getattr(args, 'lr_policy', 'step')
    warmup_epochs = getattr(args, 'warmup_epochs', 5)
    if warmup_epochs < 0:
        raise ValueError('--warmup_epochs must be >= 0, got %r' % (warmup_epochs,))
    if policy != 'poly':
        return
    if getattr(args, 'schedule', None) is not None:
        raise ValueError('--schedule sets the step policy\'s factors; it cannot be combined with '
                         '--lr_policy poly')
    if not args.poly_power > 0:
        raise ValueError('--poly_power must be > 0, got %r' % (args.poly_power,))
    if not args.end_lr >= 0:
        raise ValueError('--end_lr must be >= 0, got %r' % (args.end_lr,))
    if args.warmup and warmup_epochs >= args.num_epochs:
        raise ValueError('--lr_policy poly needs the warm-up (%d epochs) to end before --num_epochs (%d)'
                         % (warmup_epochs, args.num_epochs))


def learning_rate_at(args, epoch, itr=None, itr_per_epoch=None, scale=1):
    """Goyal et al. policy (``gossip_sgd.py:508-536``): target = lr*bs*ws/256,
    optional linear warm-up from ``lr`` over ``warmup_epochs`` (default 5) epochs, then
    multiplicative steps (``lr_policy='step'``) or polynomial decay to ``end_lr``
    (``lr_policy='poly'``, the MLPerf ResNet-50 recipe): with ``count`` iterations done,
    ``T`` in all and ``W`` of warm-up, ``p = clamp((count - W) / (T - W), 0, 1)`` and
    ``lr = end_lr + (target - end_lr) * (1 - p) ** poly_power``.  So the first iteration after the
    warm-up runs at ``target``.  Without ``itr`` the counts are whole epochs."""
    target = args.lr * args.batch_size * scale * args.world_size / 256
    warmup_epochs = getattr(args, 'warmup_epochs', 5)
    if args.warmup and epoch < warmup_epochs:
        if target <= args.lr:
            return target
        assert itr is not None and itr_per_epoch is not None
        count = epoch * itr_per_epoch + itr + 1
        return args.lr + (target - args.lr) * (count / (warmup_epochs * itr_per_epoch))
    if getattr(args, 'lr_policy', 'step') == 'poly':
        per_epoch = 1 if itr is None else itr_per_epoch
        count = epoch * per_epoch + (0 if itr is None else itr)
        total = args.num_epochs * per_epoch
        warm = (warmup_epochs if args.warmup else 0) * per_epoch
        p = min(max((count - warm) / max(total - warm, 1), 0.0), 1.0)
        return args.end_lr + (target - args.end_lr) * (1.0 - p) ** args.poly_power
    lr = target
    for e, factor in args.lr_schedule.items():
        if epoch >= e:
            lr *= factor
    return lr


def update_learning_rate(args, optimizer, epoch, itr=None, itr_per_epoch=None, scale=1):
    lr = learning_rate_at(args, epoch, itr, itr_per_epoch, scale)
    for group in optimizer.param_groups:
        group['lr'] = lr
    return lr


def peers_per_itr_at(schedule, epoch):
    """Latest schedule entry whose epoch is <= ``epoch``."""
    best, ppi = -1, None
    for e, v in schedule.items():
        if best <= e <= epoch:
            best, ppi = e, v
    return ppi


def update_peers_per_itr(args, model, epoch):
    model.update_gossiper('peers_per_itr', peers_per_itr_at(args.ppi_schedule, epoch))


# --------------------------------------------------------------------------- #
# data
# --------------------------------------------------------------------------- #
class SyntheticLoader(object):
    """Epoch-length stream of (pinned-host) random batches; a small pool is
    generated once and cycled, like a page-cache-resident dataset."""

    def __init__(self, n_images, batch_size, world_size, rank, image_size=224,
                 num_classes=1000, seed=0, pool=8, pin=True):
        self.batch_size = batch_size
        self.n_batches = max(1, n_images // (batch_size * world_size))
        g = torch.Generator().manual_seed(seed * 1000003 + rank)
        self.pool = []
        for _ in range(min(pool, self.n_batches)):
            x = torch.randn(batch_size, 3, image_size, image_size, generator=g)
            y = torch.randint(0, num_classes, (batch_size,), generator=g)
            if pin and torch.cuda.is_available():
                x, y = x.pin_memory(), y.pin_memory()
            self.pool.append((x, y))
        self.sampler = self

    def set_epoch(self, epoch):
        self._epoch = epoch

    def __len__(self):
        return self.n_batches

    def __iter__(self):
        for i in range(self.n_batches):
            yield self.pool[i % len(self.pool)]


def make_dataloader(args, train=True):
    """(loader, sampler) for training, loader for validation."""
    if args.synthetic:
        n = args.synthetic_len if train else max(args.batch_size * args.world_size * 4, 1)
        loader = SyntheticLoader(n, args.batch_size, args.world_size if train else 1, args.rank,
                                 args.image_size, args.num_classes, seed=args.seed + (0 if train else 1))
        return (loader, loader) if train else loader
    if getattr(args, 'data_format', 'folder') == 'shards':
        from ..data import ShardLoader
        if train:
            loader = ShardLoader(os.path.join(args.dataset_dir, 'train'), args.batch_size, args.world_size,
                                 args.rank, shuffle=True, drop_last=True, seed=args.seed)
            return loader, loader
        return ShardLoader(os.path.join(args.dataset_dir, 'val'), args.batch_size, 1, 0, shuffle=False,
                           drop_last=False, seed=args.seed)
    import torchvision.datasets as datasets
    if train:
        ds = datasets.ImageFolder(os.path.join(args.dataset_dir, 'train'), folder_transforms(args, train=True))
        sampler = torch.utils.data.distributed.DistributedSampler(
            ds, num_replicas=args.world_size, rank=args.rank)
        loader = torch.utils.data.DataLoader(
            ds, batch_size=args.batch_size, shuffle=False, sampler=sampler,
            num_workers=args.num_dataloader_workers, pin_memory=True, drop_last=True,
            persistent_workers=args.num_dataloader_workers > 0)
        return loader, sampler
    ds = datasets.ImageFolder(os.path.join(args.dataset_dir, 'val'), folder_transforms(args, train=False))
    return torch.utils.data.DataLoader(ds, batch_size=args.batch_size, shuffle=False,
                                       num_workers=args.num_dataloader_workers, pin_memory=True)


def folder_transforms(args, train=True):
    """The ``--data_format folder`` pipeline: RandomResizedCrop, flip, [TrivialAugmentWide |
    RandAugment | AutoAugment], ToTensor, Normalize, [RandomErasing] for training (torchvision's
    recipe order), Resize + CenterCrop for validation, which never augments."""
    import torchvision.transforms as transforms
    norm = transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
    if not train:
        return transforms.Compose([transforms.Resize(int(args.image_size * 256 / 224)),
                                   transforms.CenterCrop(args.image_size), transforms.ToTensor(), norm])
    steps = [transforms.RandomResizedCrop(args.image_size), transforms.RandomHorizontalFlip()]
    policy = getattr(args, 'auto_augment', 'none')
    if policy == 'ta_wide':
        steps.append(transforms.TrivialAugmentWide())
    elif policy == 'ra':
        steps.append(transforms.RandAugment(num_ops=args.ra_num_ops, magnitude=args.ra_magnitude))
    elif policy == 'imagenet':
        steps.append(transforms.AutoAugment(transforms.AutoAugmentPolicy.IMAGENET))
    steps += [transforms.ToTensor(), norm]
    if getattr(args, 'random_erase', 0.0) > 0:
        steps.append(transforms.RandomErasing(p=args.random_erase))
    return transforms.Compose(steps)


def device_batch(args, batch, train=True):
    """uint8 shard batches (``--data_format shards``): copy the bytes to the device and run the
    crop / flip / normalisation, and --auto_augment / --random_erase on training batches, there
    (``data.GpuAugment``); anything else passes through."""
    if batch.dtype != torch.uint8:
        return batch
    aug = getattr(args, '_gpu_augment', None)
    if aug is None:
        from ..data import GpuAugment
        ta = getattr(args, 'auto_augment', 'none')
        aug = args._gpu_augment = GpuAugment(out_size=args.image_size, seed=args.seed * 7919 + args.rank,
                                             auto_augment=None if ta == 'none' else ta,
                                             random_erase=getattr(args, 'random_erase', 0.0),
                                             ra_num_ops=getattr(args, 'ra_num_ops', 2),
                                             ra_magnitude=getattr(args, 'ra_magnitude', 9))
    return aug(batch.to(args.device, non_blocking=True), train=train)


def make_batch_mix(args):
    """The training batches' ``ops.batch_mix.BatchMix`` for --mixup_alpha / --cutmix_alpha (None
    when both are 0): one draw per step, a pure function of (--seed, rank, iteration)."""
    if not (getattr(args, 'mixup_alpha', 0.0) > 0 or getattr(args, 'cutmix_alpha', 0.0) > 0):
        return None
    from ..ops.batch_mix import BatchMix
    return BatchMix(args.mixup_alpha, args.cutmix_alpha, args.mix_prob, args.mix_switch_prob,
                    seed=args.seed, rank=args.rank)


def mix_train_batch(args, batch_mix, batch, itr):
    """Eager training loops: the batch of iteration ``itr`` mixed on ``args.device`` (the sm_90a
    kernel on CUDA) and the mix state its loss needs."""
    if batch.device.type != torch.device(args.device).type:
        batch = batch.to(args.device, non_blocking=True)
    batch_mix.iteration = itr
    return batch_mix.apply(batch), batch_mix.state


def train_loss(criterion, output, target, mix, label_smoothing, teacher_logits=None, args=None):
    """Training loss of the eager loops: ``criterion`` or, for a mixed batch, the two-target
    cross-entropy (fused kernel on CUDA) with the same label smoothing.  With ``teacher_logits`` the
    --distill_alpha / --distill_temperature objective of ``args`` (``reference_distillation_loss``)."""
    if teacher_logits is not None:
        from ..ops.fused_loss import reference_distillation_loss
        return reference_distillation_loss(output.float(), target, teacher_logits.float(), args.distill_alpha,
                                           args.distill_temperature, label_smoothing,
                                           lam=None if mix is None else mix[0])[0]
    if mix is None:
        return criterion(output.float(), target)
    from ..ops.fused_loss import fused_cross_entropy
    return fused_cross_entropy(output.float(), target, label_smoothing, mix=mix)[0]


# --------------------------------------------------------------------------- #
# metrics / logging / state
# --------------------------------------------------------------------------- #
def accuracy(output, target, topk=(1,)):
    """precision@k in percent as 1-element tensors (no host sync)."""
    with torch.no_grad():
        maxk = max(topk)
        _, pred = output.topk(maxk, 1, True, True)
        hit = pred.eq(target.view(-1, 1))
        return [hit[:, :k].any(dim=1).float().sum(0, keepdim=True).mul_(100.0 / target.size(0))
                for k in topk]


CSV_COLUMNS = ('Epoch,itr,BT(s),avg:BT(s),std:BT(s),NT(s),avg:NT(s),std:NT(s),'
               'DT(s),avg:DT(s),std:DT(s),Loss,avg:Loss,Prec@1,avg:Prec@1,Prec@5,avg:Prec@5,val')


class CSVLog(object):

    def __init__(self, fname, world_size, num_workers, batch_size):
        self.fname = fname
        if not os.path.exists(fname):
            with open(fname, 'w') as f:
                print('BEGIN-TRAINING\nWorld-Size,{}\nNum-DLWorkers,{}\nBatch-Size,{}\n{}'.format(
                    world_size, num_workers, batch_size, CSV_COLUMNS), file=f)

    def train_row(self, epoch, itr, bt, nt, dt, loss, top1, top5):
        with open(self.fname, 'a') as f:
            print('{},{},{},{},{},{:.4f},{:.4f},{:.3f},{:.3f},{:.3f},{:.3f},-1'.format(
                epoch, itr, bt, nt, dt, loss.val, loss.avg, top1.val, top1.avg,
                top5.val, top5.avg), file=f)

    def val_row(self, epoch, bt, nt, dt, prec1):
        with open(self.fname, 'a') as f:
            print('{},-1,{},{},{},-1,-1,-1,-1,-1,-1,{}'.format(epoch, bt, nt, dt, prec1), file=f)


class ConsensusLog(object):
    """``--consensus_freq`` / ``--validate_average``: one row per measurement; ``avg_prec1`` is
    the prec@1 of the push-sum average model (epoch-end rows with ``--validate_average``)."""

    COLUMNS = 'epoch,itr,distance_sq,average_norm_sq,relative,avg_prec1'

    def __init__(self, fname):
        self.fname = fname
        if not os.path.exists(fname):
            with open(fname, 'w') as f:
                print(self.COLUMNS, file=f)

    def row(self, epoch, itr, stats, avg_prec1=None):
        with open(self.fname, 'a') as f:
            print('{},{},{!r},{!r},{!r},{}'.format(epoch, itr, stats.distance_sq, stats.average_norm_sq,
                                                    stats.relative, '' if avg_prec1 is None else avg_prec1),
                  file=f)


class EmaLog(object):
    """``--model_ema_decay``: one row per validation of the EMA model."""

    COLUMNS = 'epoch,num_updates,prec1,prec5'

    def __init__(self, fname):
        self.fname = fname
        if not os.path.exists(fname):
            with open(fname, 'w') as f:
                print(self.COLUMNS, file=f)

    def row(self, epoch, num_updates, prec1, prec5):
        with open(self.fname, 'a') as f:
            print('{},{},{!r},{!r}'.format(epoch, num_updates, prec1, prec5), file=f)


def update_state(state, update_dict):
    for key, value in update_dict.items():
        state[key] = copy.deepcopy(value)


def fresh_state(model_sd, optim_sd):
    return {'epoch': 0, 'itr': 0, 'best_prec1': 0, 'is_best': True, 'state_dict': model_sd,
            'optimizer': optim_sd, 'elapsed_time': 0,
            'batch_meter': Meter(ptag='Time').__dict__, 'data_meter': Meter(ptag='Data').__dict__,
            'nn_meter': Meter(ptag='Forward/Backward').__dict__}


def init_model(args):
    """ResNet (default resnet50) initialised as in "ImageNet in 1 hour"."""
    from .. import models
    kw = {} if args.model == 'tiny' else {'num_classes': args.num_classes}
    if getattr(args, 'drop_path_rate', 0.0) > 0:
        kw['drop_path_rate'] = args.drop_path_rate
    net = models.MODEL_ZOO[args.model](**kw)
    if isinstance(net, models.ResNet):
        models.init_imagenet_in_1hr(net)
        if net.stochastic_depth is not None:
            net.stochastic_depth.reseed(args.seed, args.rank)
    net = net.to(args.device)
    if args.channels_last and args.device == 'cuda':
        net = net.to(memory_format=torch.channels_last)
    return net
