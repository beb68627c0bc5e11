"""Gradient accumulation (``GossipTrainer(accumulation_steps=k)``, ``gossip_sgd.py --accumulation_steps``)
without a GPU: the argument's validation, the scaled gradient the optimizer stages, the trainer's
accumulating backward on a bare instance, BatchMix's per-micro-batch mixing under one draw, and the
command line's parsing, rejections and help."""
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import batch_mix as bm
from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer, check_accumulation_steps

import test_distributed_c10d as sim


@pytest.mark.parametrize('k', [1, 2, 7, np.int64(4), torch.tensor(3).item()])
def test_accumulation_steps_accepts_integers_from_one(k):
    assert check_accumulation_steps(k) == int(k)
    assert type(check_accumulation_steps(k)) is int


@pytest.mark.parametrize('k', [0, -1, 2.0, 1.5, True, False, '2', None, np.float64(2)])
def test_accumulation_steps_rejects_everything_else(k):
    with pytest.raises(ValueError, match='accumulation_steps must be an integer >= 1'):
        check_accumulation_steps(k)


def test_trainer_validates_before_touching_the_model():
    """the check runs first, so it needs no CUDA engine: a bad k, or k > 1 in hierarchical mode"""
    with pytest.raises(ValueError, match='accumulation_steps must be an integer'):
        GossipTrainer(object(), None, accumulation_steps=0)
    hier = types.SimpleNamespace(nprocs_per_node=2, _kernel=None)
    with pytest.raises(ValueError, match='nprocs_per_node > 1'):
        GossipTrainer(hier, None, accumulation_steps=2)
    with pytest.raises(AssertionError):                  # k = 1 gets past the check to the engine assert
        GossipTrainer(hier, None, accumulation_steps=1)


class _Engine(object):
    def __init__(self):
        self.grad_scale = None

    def set_hyper(self, lr, mu, wd, nest, do_sgd=True, grad_scale=1.0, groups=None, max_grad_norm=None):
        self.grad_scale = grad_scale


@pytest.mark.parametrize('grad_scale', [1.0, 0.125, 1.0 / 3.0])
@pytest.mark.parametrize('k', [1, 2, 3, 5])
def test_set_engine_hyper_stages_grad_scale_over_k(grad_scale, k):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    model = GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, grad_scale=grad_scale)
    e = _Engine()
    opt.set_engine_hyper(e, micro_batches=k)
    assert e.grad_scale == grad_scale / k                # divided in fp64 ...
    assert opt.grad_scale == grad_scale                  # ... and the optimizer's own value is kept
    # the engine rounds the fp64 quotient to fp32 once, in its hyper-parameter row
    row = torch.zeros(1, dtype=torch.float32)
    row[0] = e.grad_scale
    assert float(row[0]) == float(np.float32(grad_scale / k))


# -- the trainer's accumulating backward on a bare instance (as in test_trainer_backward_cpu) ---------- #
class _C(object):
    """stand-in for the extension: counts grad_accumulate calls and does dst += float(src)"""

    def __init__(self):
        self.calls = []

    def grad_accumulate(self, dst, src):
        self.calls.append(len(dst))
        for d, s in zip(dst, src):
            d.add_(s.float())


def _bare(net):
    t = GossipTrainer.__new__(GossipTrainer)
    t.batched_grad_copy = True
    t._grad_slots = None
    t._accum_dst = None
    t.accum_fallbacks = 0
    t.model = types.SimpleNamespace(_twin=[])
    t.engine = types.SimpleNamespace(C=_C())
    return t


def _net():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Flatten(), nn.Linear(8 * 6 * 6, 5))


def _bind(net, foreign=None):
    """.grad of every parameter = a view of one flat fp32 buffer; ``foreign``: index of a parameter
    whose slot gets transposed strides (its fresh gradient then has a foreign layout)"""
    params = list(net.parameters())
    flat = torch.zeros(sum(p.numel() for p in params))
    off = 0
    for i, p in enumerate(params):
        v = flat[off:off + p.numel()]
        p.grad = v.view(p.shape[::-1]).t() if i == foreign else v.view_as(p)
        off += p.numel()
    return flat


@pytest.mark.parametrize('foreign', [None, 3])
def test_accumulating_backward_sums_the_micro_batches(foreign):
    xs = [torch.randn(4, 3, 6, 6, generator=torch.Generator().manual_seed(s)) for s in range(3)]
    ref = _net()
    for x in xs:                                           # torch: .grad accumulates over backward calls
        ref(x).square().mean().backward()
    want = torch.cat([p.grad.reshape(-1) for p in ref.parameters()])

    net = _net()
    flat = _bind(net, foreign)
    views = [p.grad for p in net.parameters()]
    t = _bare(net)
    for j, x in enumerate(xs):
        t._backward(net(x).square().mean(), net, accumulate=j > 0)
    if foreign is not None:        # the (5, 288) weight's slot is transposed: gather it back to logical order
        w = list(net.parameters())[foreign]
        off = sum(p.numel() for p in list(net.parameters())[:foreign])
        flat = flat.clone()
        flat[off:off + w.numel()] = views[foreign].reshape(-1)
    torch.testing.assert_close(flat, want, rtol=1e-6, atol=1e-7)
    for p, v in zip(net.parameters(), views):
        assert p.grad is v                                 # the views are re-bound after every pass
    n = len(views)
    fallback = 0 if foreign is None else 1
    assert t.engine.C.calls == [n - fallback] * 2          # ONE launch per later micro-batch
    assert t.accum_fallbacks == 2 * fallback


# -- BatchMix: k micro-batches under one draw ------------------------------------------------------------ #
@pytest.mark.parametrize('k', [1, 2, 4])
@pytest.mark.parametrize('alphas', [(0.4, 0.0), (0.0, 1.0)], ids=['mixup', 'cutmix'])
def test_batch_mix_mixes_each_micro_batch_with_itself(k, alphas):
    x = torch.randn(8, 3, 10, 12, generator=torch.Generator().manual_seed(5))
    mix = bm.BatchMix(*alphas, seed=3)
    mix.iteration = 11
    out = mix.apply(x, micro_batches=k)
    assert mix.iteration == 12                             # one draw for the whole step
    p = mix.sample(10, 12, itr=11)
    assert mix.last == p and p.mode != bm.NO_MIX
    m = 8 // k
    for j in range(k):
        assert torch.equal(out[j * m:(j + 1) * m], bm.reference_batch_mix(x[j * m:(j + 1) * m], p))
    if k == 1:
        assert torch.equal(out, bm.reference_batch_mix(x, p))


@pytest.mark.parametrize('k', [0, 3])
def test_batch_mix_rejects_micro_batches_that_do_not_divide(k):
    with pytest.raises(ValueError, match='micro_batches'):
        bm.BatchMix(0.4).apply(torch.randn(8, 3, 4, 4), micro_batches=k)


# -- command line ---------------------------------------------------------------------------------------- #
def _parse(argv, tmp_path):
    from stochastic_gradient_push_b200.cli import gossip_sgd
    return gossip_sgd.parse_args(argv + ['--checkpoint_dir', str(tmp_path) + '/'])


def test_cli_default_and_accepted_combination(tmp_path, monkeypatch):
    from stochastic_gradient_push_b200.cli import gossip_sgd
    assert _parse(['--device', 'cpu'], tmp_path).accumulation_steps == 1
    # the supported combinations (finalize_args, which would set up the GPU, is skipped)
    monkeypatch.setattr(gossip_sgd, 'finalize_args', lambda args, adpsgd=False: args)
    for extra in ([], ['--overlap', 'True'], ['--push_sum', 'False'], ['--cuda_graph']):
        args = _parse(['--device', 'cuda', '--cuda_graph', 'True', '--batch_size', '256',
                       '--accumulation_steps', '4'] + extra, tmp_path)
        assert args.accumulation_steps == 4 and args.batch_size == 256


@pytest.mark.parametrize('extra,what', [
    (['--all_reduce', 'True', '--graph_type', '-1', '--cuda_graph', 'True'], '--all_reduce'),
    (['--fused', 'False', '--cuda_graph', 'True'], '--fused False'),
    ([], '--cuda_graph False'),
    (['--cuda_graph', 'True', '--transport', 'c10d'], '--transport c10d'),
    (['--cuda_graph', 'True', '--device', 'cpu'], '--device cpu'),
    (['--cuda_graph', 'True', '--device', 'cuda', '--nprocs_per_node', '2'], '--nprocs_per_node > 1'),
])
def test_cli_rejects_every_other_path(tmp_path, extra, what):
    with pytest.raises(ValueError, match='--accumulation_steps > 1 is not supported with %s' % what):
        _parse(['--accumulation_steps', '2'] + extra, tmp_path)


@pytest.mark.parametrize('bs,k', [(32, 3), (30, 4), (8, 16)])
def test_cli_rejects_a_batch_size_that_k_does_not_divide(tmp_path, bs, k):
    with pytest.raises(ValueError, match='--batch_size %d is not divisible by --accumulation_steps %d' % (bs, k)):
        _parse(['--accumulation_steps', str(k), '--batch_size', str(bs), '--cuda_graph', 'True',
                '--device', 'cuda'], tmp_path)


@pytest.mark.parametrize('k', ['0', '-2'])
def test_cli_rejects_k_below_one(tmp_path, k):
    with pytest.raises(ValueError, match='--accumulation_steps must be >= 1'):
        _parse(['--accumulation_steps', k, '--device', 'cpu'], tmp_path)


def test_cli_rejects_a_non_integer_k(tmp_path, capsys):
    with pytest.raises(SystemExit):
        _parse(['--accumulation_steps', '2.5', '--device', 'cpu'], tmp_path)
    assert 'invalid int value' in capsys.readouterr().err


def test_help_documents_the_flag_and_adpsgd_has_none(tmp_path, capsys):
    with pytest.raises(SystemExit):
        _parse(['--help'], tmp_path)
    text = ' '.join(capsys.readouterr().out.split())
    assert '--accumulation_steps' in text
    for words in ('gradient accumulation', 'summed in fp32', '--batch_size stays the per-rank step batch',
                  'divisible by K', '--cuda_graph True --fused True'):
        assert words in text, words
    from stochastic_gradient_push_b200.cli.common import build_parser
    assert '--accumulation_steps' not in build_parser(adpsgd=True).format_help()
    with pytest.raises(SystemExit):
        build_parser(adpsgd=True).parse_args(['--accumulation_steps', '2'])


def test_binding_rejects_bad_lists_without_a_gpu():
    """the extension's argument checks run before anything touches a device"""
    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    a = torch.zeros(8)
    C.grad_accumulate([], [])                                   # an empty list: nothing to do
    for dst, src, what in (([], [a], '0 dst tensors but 1 src tensors'),
                           ([a], [a.clone()], 'pair 0: every tensor must be a CUDA tensor')):
        with pytest.raises(RuntimeError, match=what):
            C.grad_accumulate(dst, src)
    assert C.ACCUM_MAX_SEGS >= 465 and C.ACCUM_CHUNK % 8 == 0  # ResNet-152's list fits one launch
