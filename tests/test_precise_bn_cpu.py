"""Precise BatchNorm statistics without a GPU: the reference path of ops.fused_bn.precise_bn_stats and
BNStatsAccumulator against the momentum-1 oracle, what it leaves alone, and the --precise_bn_batches flag."""
import copy

import pytest
import torch
import torch.nn as nn

from stochastic_gradient_push_b200 import models
from stochastic_gradient_push_b200.ops import fused_bn
from stochastic_gradient_push_b200.ops.fused_bn import BNStatsAccumulator, FusedBatchNormAct2d, precise_bn_stats


def _bns(net):
    return [m for m in net.modules() if isinstance(m, FusedBatchNormAct2d)]


def oracle(net, batches):
    """per BN layer (running_mean, running_var): one eager train-mode forward per batch with the running
    buffers zeroed and momentum 1, so that they hold exactly that batch's statistics; summed in fp64 in
    batch order, divided by K, rounded to fp32"""
    net = copy.deepcopy(net).train()
    bns = _bns(net)
    sums = [(torch.zeros(m.num_features, dtype=torch.float64), torch.zeros(m.num_features, dtype=torch.float64))
            for m in bns]
    for x in batches:
        for m in bns:
            m.running_mean.zero_()
            m.running_var.zero_()
            m.momentum = 1.0
        with torch.no_grad():
            net(x)
        sums = [(sm + m.running_mean.cpu().double(), sv + m.running_var.cpu().double())
                for (sm, sv), m in zip(sums, bns)]
    k = len(batches)
    return [((sm / k).float(), (sv / k).float()) for sm, sv in sums]


def _precise(net, batches):
    acc = BNStatsAccumulator(net)
    net.train()
    with torch.no_grad(), precise_bn_stats(acc):
        for x in batches:
            net(x)
    acc.commit(len(batches))
    return acc


def _small_resnet():
    torch.manual_seed(0)
    net = models.resnet50(num_classes=10)
    for m in _bns(net):              # non-trivial running statistics and affine parameters to start from
        m.running_mean.uniform_(-1, 1)
        m.running_var.uniform_(0.5, 2)
        m.weight.data.uniform_(0.5, 1.5)
        m.bias.data.uniform_(-0.5, 0.5)
        m.num_batches_tracked.fill_(7)
    return net


def _batches():
    g = torch.Generator().manual_seed(1)
    return [torch.randn(n, 3, 32, 32, generator=g) for n in (4, 4, 3)]      # the last one partial


@pytest.fixture
def reference_path(monkeypatch):
    monkeypatch.setattr(fused_bn, 'FORCE_REFERENCE', True)


def test_reference_path_equals_the_oracle(reference_path):
    net, batches = _small_resnet(), _batches()
    want = oracle(net, batches)
    _precise(net, batches)
    bns = _bns(net)
    assert len(bns) == 53
    for m, (rm, rv) in zip(bns, want):
        assert torch.equal(m.running_mean, rm)
        assert torch.equal(m.running_var, rv)


def test_only_the_running_statistics_change(reference_path):
    net, batches = _small_resnet(), _batches()
    params = [p.detach().clone() for p in net.parameters()]
    stats = [(m.running_mean.clone(), m.running_var.clone()) for m in _bns(net)]
    net.eval()
    acc = BNStatsAccumulator(net)
    net.train()
    with torch.no_grad(), precise_bn_stats(acc):
        pass                                            # K = 0: no batch, no commit
    for m, (rm, rv) in zip(_bns(net), stats):
        assert torch.equal(m.running_mean, rm) and torch.equal(m.running_var, rv)
    assert int(acc.flat.abs().sum()) == 0
    with pytest.raises(ValueError, match='k >= 1'):
        acc.commit(0)
    _precise(net, batches)
    assert all(torch.equal(p, q) for p, q in zip(net.parameters(), params))
    assert all(int(m.num_batches_tracked) == 7 for m in _bns(net))
    assert not all(torch.equal(m.running_mean, rm) for m, (rm, _) in zip(_bns(net), stats))


def test_outputs_are_those_of_the_training_forward(reference_path):
    net, batches = _small_resnet(), _batches()
    plain = copy.deepcopy(net).train()
    acc = BNStatsAccumulator(net)
    net.train()
    with torch.no_grad():
        want = plain(batches[0])
        with precise_bn_stats(acc):
            got = net(batches[0])
    assert torch.equal(got, want)
    # the training forward blended the batch statistics in; inside the block they went to the accumulator
    assert int(plain.bn1.num_batches_tracked) == 8 and int(net.bn1.num_batches_tracked) == 7
    c = net.bn1.num_features
    assert torch.equal(acc.views[0][:c], acc.views[0][:c].float().double())     # fp32 values, summed in fp64


def test_accumulator_layout():
    net = models.TinyConvNet(width=8)
    acc = BNStatsAccumulator(net)
    assert acc.flat.dtype == torch.float64 and acc.flat.numel() == 2 * (8 + 16)
    assert [v.numel() for v in acc.views] == [16, 32]
    assert all(v.data_ptr() == acc.flat.data_ptr() + 8 * off for v, off in zip(acc.views, (0, 16)))
    assert acc.layers == _bns(net)


def test_eval_mode_layers_and_plain_forwards_are_untouched(reference_path):
    net = models.TinyConvNet(width=8).eval()
    x = torch.randn(2, 3, 16, 16)
    acc = BNStatsAccumulator(net)
    with torch.no_grad():
        want = net(x)
        with precise_bn_stats(acc):
            got = net(x)
    assert torch.equal(got, want) and int(acc.flat.abs().sum()) == 0


def test_foreign_batchnorm_layers_are_rejected():
    net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8))
    with pytest.raises(ValueError, match='FusedBatchNormAct2d; found BatchNorm2d'):
        BNStatsAccumulator(net)


def test_a_layer_outside_the_accumulator_is_rejected(reference_path):
    net, other = models.TinyConvNet(width=8).train(), models.TinyConvNet(width=8).train()
    with torch.no_grad(), precise_bn_stats(BNStatsAccumulator(other)):
        with pytest.raises(ValueError, match="not one of the accumulator's layers"):
            net(torch.randn(2, 3, 16, 16))


# --------------------------------------------------------------------------- #
# CLI
# --------------------------------------------------------------------------- #
def _parse(argv, tmp_path):
    from stochastic_gradient_push_b200.cli import gossip_sgd
    return gossip_sgd.parse_args(argv + ['--checkpoint_dir', str(tmp_path) + '/'])


def test_cli_default_is_off_and_the_flag_parses(tmp_path, monkeypatch):
    from stochastic_gradient_push_b200.cli import gossip_sgd
    assert _parse(['--device', 'cpu'], tmp_path).precise_bn_batches == 0
    monkeypatch.setattr(gossip_sgd, 'finalize_args', lambda args, adpsgd=False: args)
    for extra in ([], ['--overlap', 'True'], ['--push_sum', 'False'], ['--eval_graph', 'True']):
        args = _parse(['--device', 'cuda', '--cuda_graph', 'True', '--precise_bn_batches', '5'] + extra, tmp_path)
        assert args.precise_bn_batches == 5


def test_cli_rejects_a_negative_count(tmp_path):
    with pytest.raises(ValueError, match='--precise_bn_batches must be >= 0, got -1'):
        _parse(['--device', 'cuda', '--cuda_graph', 'True', '--precise_bn_batches', '-1'], tmp_path)


@pytest.mark.parametrize('extra,what', [
    (['--all_reduce', 'True', '--graph_type', '-1', '--cuda_graph', 'True'], '--all_reduce'),
    (['--fused', 'False', '--cuda_graph', 'True'], '--fused False'),
    ([], '--cuda_graph False'),
    (['--cuda_graph', 'True', '--transport', 'c10d'], '--transport c10d'),
    (['--cuda_graph', 'True', '--device', 'cpu'], '--device cpu'),
])
def test_cli_rejects_the_flag_without_the_captured_trainer(tmp_path, extra, what):
    with pytest.raises(ValueError, match='--precise_bn_batches is not supported with %s' % what):
        _parse(['--precise_bn_batches', '2'] + extra, tmp_path)


def test_help_documents_the_flag(tmp_path, capsys):
    with pytest.raises(SystemExit):
        _parse(['--help'], tmp_path)
    text = ' '.join(capsys.readouterr().out.split())
    assert '--precise_bn_batches' in text and 'GossipTrainer.update_bn' in text


def test_bindings_exist():
    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    assert callable(C.bn_stats_commit) and C.BN_COMMIT_MAX_SEGS == 1000
    assert 'acc' in C.bn_forward.__doc__ and 'acc' in C.conv1x1_bn_forward.__doc__


def test_commit_binding_rejects_bad_tables():
    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    acc, m, v = torch.zeros(16, dtype=torch.float64), torch.zeros(8), torch.zeros(8)
    with pytest.raises(RuntimeError, match='same length'):
        C.bn_stats_commit([acc], [m], [], 1)
    with pytest.raises(RuntimeError, match='k must be >= 1'):
        C.bn_stats_commit([acc], [m], [v], 0)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        C.bn_stats_commit([acc], [m], [v], 1)
    C.bn_stats_commit([], [], [], 1)                    # nothing to do: no launch
