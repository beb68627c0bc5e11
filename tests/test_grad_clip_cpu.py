"""Gradient-norm clipping and non-finite step skipping in FusedGossipSGD (``max_grad_norm=``,
``skip_nonfinite=``) on the c10d plane (gloo, CPU): one rank against ``torch.nn.utils.clip_grad_norm_``
followed by ``torch.optim.SGD`` (one and several groups, Nesterov, clipping and non-clipping
thresholds, a threshold change between steps), LARS after clipping against a per-tensor LARC, torch's
NaN propagation for non-finite norms, the skip on a four-rank SGP world, the checkpoint round trip,
and the rejections of the constructor and the command line."""

import math
import re

import pytest
import torch

import stochastic_gradient_push_b200 as sgp

import test_distributed_c10d as sim
from dist_utils import run_distributed

SELF_W = [0.3, 0.5, 0.6, 0.45]
ETA, EPS = 0.05, 1e-8


def _single():
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    model = GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1)
    assert model.transport == 'c10d'
    return model


def _groups(params, kind, lars=False):
    """parameters of sim._model: [W1 (5x6), b1 (5), W2 (3x5), b2 (3)]"""
    w1, b1, w2, b2 = params
    if kind == 'one':
        return None
    return [dict(params=[w1, w2], weight_decay=2e-2, lars=lars),
            dict(params=[b1, b2], weight_decay=0.0, lr=0.05, lars=False)]


def _ours(kind, nesterov, norms, lars=False, poison=None, **kw):
    """FusedGossipSGD on one rank without gossip; `norms[s]` is the threshold of step s; `poison`:
    (step, value) written into the first gradient element after backward"""
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    model = _single()
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-3, nesterov=nesterov,
                         param_groups=_groups(list(model.module.parameters()), kind, lars), lars=lars,
                         trust_coefficient=ETA, lars_eps=EPS, max_grad_norm=norms[0], **kw)
    model.train()
    seen = []
    for step, mx in enumerate(norms):
        opt.max_grad_norm = mx
        x, y = sim._batch(0, step)
        ((model(x) - y) ** 2).mean().backward()
        if poison is not None and poison[0] == step:
            opt.grad_flat[torch.float32][0] = poison[1]
        opt.step()
        seen.append(float(opt.grad_norm) if opt.grad_norm is not None else None)
        opt.zero_grad()
    model.unbias()
    return sim._flat(model.module), seen, opt


def _reference(kind, nesterov, norms, lars=False, poison=None):
    """torch: clip_grad_norm_ over every parameter, [per-tensor LARC(clip=False)], torch.optim.SGD"""
    net = sim._model(0)
    groups = _groups(list(net.parameters()), kind, lars)
    opt = torch.optim.SGD(groups if groups is not None else net.parameters(), lr=0.1, momentum=0.9,
                          weight_decay=1e-3, nesterov=nesterov)
    lars_of = {id(p): g.get('lars', False) for g in (groups or []) for p in g['params']}
    totals = []
    for step, mx in enumerate(norms):
        opt.zero_grad()
        x, y = sim._batch(0, step)
        ((net(x) - y) ** 2).mean().backward()
        if poison is not None and poison[0] == step:
            next(net.parameters()).grad.view(-1)[0] = poison[1]
        totals.append(float(torch.nn.utils.clip_grad_norm_(net.parameters(), mx if mx is not None else math.inf)))
        if lars:
            with torch.no_grad():
                for g in opt.param_groups:
                    for p in g['params']:
                        if not lars_of[id(p)]:
                            continue
                        nx, ng = p.norm(), p.grad.norm()
                        if nx != 0 and ng != 0:
                            t = ETA * nx / (ng + g['weight_decay'] * nx + EPS)
                            p.grad.add_(p, alpha=g['weight_decay']).mul_(t)
                            p.grad.sub_(p, alpha=g['weight_decay'])    # SGD adds wd * p back
        opt.step()
    return sim._flat(net), totals


@pytest.mark.parametrize('kind', ['one', 'groups'])
@pytest.mark.parametrize('nesterov', [False, True])
@pytest.mark.parametrize('norms', [(0.05, 0.05, 0.05), (100.0, 100.0, 100.0), (0.05, 100.0, 0.02, 0.3)],
                         ids=['clipping', 'not-clipping', 'changing'])
def test_matches_clip_grad_norm_then_sgd(kind, nesterov, norms):
    got, seen, _ = _ours(kind, nesterov, norms)
    want, totals = _reference(kind, nesterov, norms)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6)
    assert seen == pytest.approx(totals, rel=1e-5)
    if norms[0] < 1:
        assert max(totals) > norms[0]                  # the threshold did clip
    # clipping changed the result relative to the plain step
    plain, _ = _reference(kind, nesterov, [math.inf] * len(norms))
    if min(norms) < 1:
        assert (plain - want).abs().max() > 1e-4


@pytest.mark.parametrize('norms', [(0.05, 0.05, 0.05), (100.0, 100.0)], ids=['clipping', 'not-clipping'])
def test_lars_sees_the_clipped_gradient(norms):
    got, _, opt = _ours('groups', True, norms, lars=True)
    assert opt._lars_flags == (True, False)
    want, _ = _reference('groups', True, norms, lars=True)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6)


def test_skip_only_runs_the_plain_step():
    got, seen, opt = _ours('one', False, (None, None), skip_nonfinite=True)
    want, totals = _reference('one', False, (None, None))
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-7)
    assert seen == pytest.approx(totals, rel=1e-5) and opt.nonfinite_steps == 0


@pytest.mark.parametrize('value', [math.inf, math.nan], ids=['inf', 'nan'])
def test_nonfinite_norm_without_skip_propagates_as_torch(value):
    norms = (0.05, 0.05)                                # the poisoned step is the last one
    got, seen, opt = _ours('one', False, norms, poison=(1, value))
    want, totals = _reference('one', False, norms, poison=(1, value))
    assert torch.isnan(want).any()
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6, equal_nan=True)
    assert torch.isnan(got).equal(torch.isnan(want))
    assert (math.isinf(seen[1]) if value == math.inf else math.isnan(seen[1]))
    if value == math.inf:
        assert not torch.isnan(want).all()              # coef 0: only the inf element turns NaN
    assert opt.nonfinite_steps == 0


def _skip_worker(rank, world, steps, bad_rank, bad_step):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    graph = sgp.NPeerDynamicDirectedExponentialGraph(rank, world, peers_per_itr=1)
    mix = sgp.SelfWeightedMixing(graph, 'cpu', self_weight=SELF_W)
    model = GossipDataParallel(sim._model(rank), graph=graph, mixing=mix, push_sum=True, overlap=False,
                               rank=rank, world_size=world, verbose=False)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-3, max_grad_norm=0.5,
                         skip_nonfinite=True)
    arena = model._arenas[torch.float32]
    model.train()
    checks = {}
    for step in range(steps):
        x, y = sim._batch(rank, step)
        ((model(x) - y) ** 2).mean().backward()
        if rank == bad_rank and step == bad_step:
            opt.grad_flat[torch.float32][3] = math.nan
            model.ps_numerator()
            x_before = arena.flat.clone()
            m_before = opt.momentum_flat[torch.float32].clone()
            opt.step()
            checks = dict(x_same=torch.equal(arena.flat, x_before),
                          m_same=torch.equal(opt.momentum_flat[torch.float32], m_before),
                          norm_nan=math.isnan(float(opt.grad_norm)))
        else:
            opt.step()
        opt.zero_grad()
        checks.setdefault('grad_zero_after', True)
        if rank == bad_rank and step == bad_step:
            checks['grad_zero_after'] = bool((opt.grad_flat[torch.float32] == 0).all())
        model.transfer_params()
    model.sync_comms()
    w = float(model.ps_weight)
    model.unbias()
    flat = sim._flat(model.module)
    return dict(checks, finite=bool(torch.isfinite(flat).all()), w=w, skipped=opt.nonfinite_steps)


def test_skip_nonfinite_on_a_four_rank_sgp_world():
    world, steps, bad = 4, 5, 1
    out = run_distributed(_skip_worker, world, steps, bad, 2)
    assert out[bad]['x_same'] and out[bad]['m_same'] and out[bad]['norm_nan']
    assert out[bad]['grad_zero_after']
    assert [o['skipped'] for o in out] == [1 if r == bad else 0 for r in range(world)]
    assert all(o['finite'] for o in out)
    # the skipping rank kept gossiping: the push-sum weights still sum to the world size
    assert sum(o['w'] for o in out) == pytest.approx(world, abs=1e-5)
    assert any(abs(o['w'] - 1) > 1e-3 for o in out)


def test_state_dict_round_trip_and_old_checkpoints():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    _, _, opt = _ours('one', False, (0.05, 0.05), skip_nonfinite=True, poison=(1, math.nan))
    assert opt.nonfinite_steps == 1
    sd = opt.state_dict()
    assert sd['grad_clip'] == {'max_grad_norm': 0.05, 'skip_nonfinite': True, 'nonfinite_steps': 1}
    other = FusedGossipSGD(_single(), lr=0.1)
    assert other.grad_norm is None and other.nonfinite_steps == 0
    other.load_state_dict(sd)
    assert (other.max_grad_norm, other.skip_nonfinite, other.nonfinite_steps) == (0.05, True, 1)
    assert other.grad_norm is not None and other.state_dict()['grad_clip'] == sd['grad_clip']
    # a checkpoint from before these options keeps the constructor's values
    old = {k: v for k, v in sd.items() if k != 'grad_clip'}
    kept = FusedGossipSGD(_single(), lr=0.1, max_grad_norm=2.0)
    kept.load_state_dict(old)
    assert (kept.max_grad_norm, kept.skip_nonfinite, kept.nonfinite_steps) == (2.0, False, 0)


@pytest.mark.parametrize('bad', [0, 0.0, -1.0, math.inf, math.nan, 'x'])
def test_constructor_rejects_bad_thresholds(bad):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    with pytest.raises(ValueError, match='max_grad_norm'):
        FusedGossipSGD(_single(), lr=0.1, max_grad_norm=bad)
    opt = FusedGossipSGD(_single(), lr=0.1, max_grad_norm=1.0)
    with pytest.raises(ValueError, match='max_grad_norm'):
        opt.max_grad_norm = bad


def test_cli_parses_the_flags_and_rejects_unsupported_modes(tmp_path):
    from stochastic_gradient_push_b200.cli.common import build_parser, finalize_args
    base = ['--device', 'cpu', '--checkpoint_dir', str(tmp_path) + '/']
    args = build_parser().parse_args(['--clip_grad_norm', '2.5', '--skip_nonfinite', 'True'] + base)
    assert args.clip_grad_norm == 2.5 and args.skip_nonfinite is True
    finalize_args(args)
    defaults = build_parser().parse_args([])
    assert defaults.clip_grad_norm == 0.0 and defaults.skip_nonfinite is False
    for flag in (['--clip_grad_norm', '1.0'], ['--skip_nonfinite', 'True']):
        for adpsgd, extra, what in ((False, ['--all_reduce', 'True', '--graph_type', '-1'], '--all_reduce'),
                                    (False, ['--fused', 'False'], '--fused False'),
                                    (True, [], 'AD-PSGD')):
            args = build_parser(adpsgd=adpsgd).parse_args(flag + base + extra)
            with pytest.raises(ValueError, match='%s is not supported with %s' % (flag[0], re.escape(what))):
                finalize_args(args, adpsgd=adpsgd)
    for bad in ('-1', 'inf'):
        args = build_parser().parse_args(['--clip_grad_norm', bad] + base)
        with pytest.raises(ValueError, match='--clip_grad_norm'):
            finalize_args(args)


def test_gossip_sgd_cli_with_clipping_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    args = COMMON + ['--push_sum', 'True', '--graph_type', '5', '--num_epochs', '1', '--num_itr_ignore', '0',
                     '--seed', '47', '--clip_grad_norm', '0.5', '--skip_nonfinite', 'True',
                     '--checkpoint_dir', str(tmp_path) + '/']
    out = _torchrun(2, 'gossip_sgd.py', args, master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    assert re.search(r'epoch 0 last gradient norm \S+ non-finite steps skipped 0', out.stdout), out.stdout[-3000:]
    for r in range(2):
        assert len(open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()) > 2
