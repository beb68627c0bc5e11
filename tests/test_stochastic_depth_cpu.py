"""Stochastic depth (``drop_path_rate``) on the CPU: the rate rule, the hash oracle of the draw kernel, the
model wiring (parameters, state_dict, eval / precise-statistics forwards), the reference composition's
gradients, the command-line checks and the checkpointed draw counter."""
import argparse
import copy
import logging

import pytest
import torch
import torch.nn.functional as F

from stochastic_gradient_push_b200 import models
from stochastic_gradient_push_b200.cli import common
from stochastic_gradient_push_b200.ops import oracle
from stochastic_gradient_push_b200.ops.fused_bn import (BNStatsAccumulator, fused_bn_act, precise_bn_stats,
                                                        reference_bn_act)
from stochastic_gradient_push_b200.ops.stochastic_depth import (StochasticDepth, block_rates,
                                                                keep_threshold)


def test_linear_rate_rule():
    assert block_rates(16, 0.05) == [0.05 * l / 15 for l in range(16)]
    assert block_rates(16, 0.05)[0] == 0.0 and block_rates(16, 0.05)[-1] == pytest.approx(0.05)
    assert block_rates(1, 0.3) == [0.0]
    sd = StochasticDepth(8, 0.1)
    assert sd.num_blocks == 8 and sd.rates[0] == 0.0 and sd.rates[7] == pytest.approx(0.1)
    assert sd.thresholds[0] == 1 << 24 and sd.keep_scales[0] == 1.0
    assert sd.thresholds[7] == keep_threshold(0.1) == round(0.9 * (1 << 24))
    assert sd.keep_scales[7] == float(torch.tensor(1 / 0.9, dtype=torch.float32))
    for bad in (-0.1, 1.0, 1.5):
        with pytest.raises(ValueError):
            StochasticDepth(8, bad)


def test_oracle_is_deterministic_and_keyed():
    sd = StochasticDepth(16, 0.5)
    a = oracle.drop_path_scales(47, 0, 3, sd.thresholds, sd.keep_scales, 256)
    assert a.shape == (16, 256) and a.dtype == torch.float32
    assert torch.equal(a, oracle.drop_path_scales(47, 0, 3, sd.thresholds, sd.keep_scales, 256))
    for other in ((48, 0, 3), (47, 1, 3), (47, 0, 4)):          # seed, rank and draw index all matter
        assert not torch.equal(a, oracle.drop_path_scales(*other, sd.thresholds, sd.keep_scales, 256))
    # the first n columns do not depend on n
    assert torch.equal(a[:, :100], oracle.drop_path_scales(47, 0, 3, sd.thresholds, sd.keep_scales, 100))
    # values: 0 or the block's keep scale; block 0 never drops
    for l in range(16):
        assert set(a[l].unique().tolist()) <= {0.0, sd.keep_scales[l]}
    assert torch.all(a[0] == 1.0)
    # negative seeds are taken as uint64
    oracle.drop_path_scales(-5, 0, 0, sd.thresholds, sd.keep_scales, 4)


def test_keep_frequencies():
    sd = StochasticDepth(4, 0.6)                                 # rates 0, 0.2, 0.4, 0.6
    n = 200000
    s = oracle.drop_path_scales(1, 2, 0, sd.thresholds, sd.keep_scales, n)
    for l, p in enumerate(sd.rates):
        kept = (s[l] > 0).double().mean().item()
        assert abs(kept - (1 - p)) < 0.005, (l, kept, p)
        # scale_by_keep: the expected scale is 1
        assert abs(s[l].double().mean().item() - 1.0) < 0.01


def test_cpu_draws_advance_the_counter():
    sd = StochasticDepth(16, 0.2, seed=3, rank=1)
    assert sd.draws == 0
    a = sd.draw(8, 'cpu')
    b = sd.draw(8, 'cpu')
    assert sd.draws == 2 and not torch.equal(a, b)
    assert torch.equal(a, oracle.drop_path_scales(3, 1, 0, sd.thresholds, sd.keep_scales, 8))
    assert torch.equal(b, oracle.drop_path_scales(3, 1, 1, sd.thresholds, sd.keep_scales, 8))
    sd.reseed(4, 1)
    assert torch.equal(sd.draw(8, 'cpu'), oracle.drop_path_scales(4, 1, 2, sd.thresholds, sd.keep_scales, 8))
    assert copy.deepcopy(sd) is sd                              # model copies share the draw sequence


def test_parameters_and_state_dict_unchanged():
    ref = models.resnet50()
    net = models.resnet50(drop_path_rate=0.05)
    assert ref.stochastic_depth is None and net.stochastic_depth.num_blocks == 16
    params = list(net.parameters())
    assert len(params) == 161 and sum(p.numel() for p in params) == 25557032
    assert list(net.state_dict().keys()) == list(ref.state_dict().keys())
    assert [n for n, _ in net.named_buffers()] == [n for n, _ in ref.named_buffers()]
    twin = copy.deepcopy(net)
    assert twin.stochastic_depth is net.stochastic_depth
    with pytest.raises(ValueError):
        models.resnet18(drop_path_rate=1.0)
    with pytest.raises(ValueError):
        models.resnet18(drop_path_rate=-0.1)


def _pair(rate, seed=0):
    torch.manual_seed(seed)
    a = models.resnet18(num_classes=10)
    b = models.resnet18(num_classes=10, drop_path_rate=rate)
    b.load_state_dict(a.state_dict())
    return a, b


def test_eval_and_precise_bn_forwards_do_not_drop():
    a, b = _pair(0.5)
    x = torch.randn(4, 3, 32, 32)
    a.eval(), b.eval()
    with torch.no_grad():
        assert torch.equal(a(x), b(x))
    assert b.stochastic_depth.draws == 0
    a.train(), b.train()
    acc_a, acc_b = BNStatsAccumulator(a), BNStatsAccumulator(b)
    with torch.no_grad():
        with precise_bn_stats(acc_a):
            ya = a(x)
        with precise_bn_stats(acc_b):
            yb = b(x)
    assert torch.equal(ya, yb) and torch.equal(acc_a.flat, acc_b.flat)
    assert b.stochastic_depth.draws == 0
    # a training forward draws once and differs
    with torch.no_grad():
        yb = b(x)
    assert b.stochastic_depth.draws == 1 and not torch.equal(ya, yb)


def test_training_forward_is_the_drop_path_composition():
    """the model's CPU training forward == the blocks run by hand with the oracle's scales applied as
    relu(bn(conv(x)) * s + identity)"""
    _, b = _pair(0.4, seed=1)
    b.train()
    x = torch.randn(6, 3, 32, 32)
    sd = b.stochastic_depth
    scales = oracle.drop_path_scales(sd.seed, sd.rank, 0, sd.thresholds, sd.keep_scales, 6)
    state = copy.deepcopy(b.state_dict())
    with torch.no_grad():
        got = b(x)
    b.load_state_dict(state)                                   # the running statistics before the forward
    with torch.no_grad():
        h = b.maxpool(b.bn1(b.conv1(x), relu=True))
        blocks = [blk for layer in (b.layer1, b.layer2, b.layer3, b.layer4) for blk in layer]
        for l, blk in enumerate(blocks):
            identity = h if blk.downsample is None else blk.downsample[1](blk.downsample[0](h))
            out = blk.bn1(blk.conv1(h), relu=True)
            z = blk.bn2(blk.conv2(out))
            h = F.relu(z * scales[l].view(-1, 1, 1, 1) + identity)
        want = b.fc(torch.flatten(b.avgpool(h), 1))
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def test_reference_composition_gradients():
    torch.manual_seed(0)
    N, C = 4, 6
    x = torch.randn(N, C, 3, 3, dtype=torch.float64, requires_grad=True)
    res = torch.randn(N, C, 3, 3, dtype=torch.float64, requires_grad=True)
    w = (torch.rand(C, dtype=torch.float64) + 0.5).requires_grad_(True)
    bias = torch.randn(C, dtype=torch.float64, requires_grad=True)
    s = torch.tensor([0.0, 1.25, 1.25, 0.0], dtype=torch.float64)

    def f(x, res, w, bias):
        return reference_bn_act(x, w, bias, None, None, None, residual=res, relu=True, training=True,
                                branch_scale=s)
    assert torch.autograd.gradcheck(f, (x, res, w, bias))
    y = f(x, res, w, bias)
    # a dropped sample's output is relu(residual), and its input still gets a gradient through the
    # batch statistics
    assert torch.equal(y[0], F.relu(res[0])) and torch.equal(y[3], F.relu(res[3]))
    y.sum().backward()
    assert x.grad[0].abs().sum() > 0
    with pytest.raises(ValueError, match='residual'):
        fused_bn_act(x, w, bias, None, None, branch_scale=s.float())


def _args(**kw):
    base = dict(drop_path_rate=0.0, model='resnet50')
    base.update(kw)
    return argparse.Namespace(**base)


def test_cli_validation():
    common.check_drop_path_flags(_args())
    common.check_drop_path_flags(_args(drop_path_rate=0.05))
    common.check_drop_path_flags(_args(model='tiny'))
    for bad in (-0.01, 1.0, 2.0):
        with pytest.raises(ValueError, match='drop_path_rate'):
            common.check_drop_path_flags(_args(drop_path_rate=bad))
    with pytest.raises(ValueError, match='tiny'):
        common.check_drop_path_flags(_args(model='tiny', drop_path_rate=0.1))
    p = common.build_parser()
    assert p.parse_args([]).drop_path_rate == 0.0
    assert p.parse_args(['--drop_path_rate', '0.05']).drop_path_rate == 0.05


def test_init_model_seeds_with_seed_and_rank():
    ns = argparse.Namespace(model='resnet18', num_classes=10, drop_path_rate=0.1, seed=9, rank=3, device='cpu',
                            channels_last=False)
    net = common.init_model(ns)
    assert (net.stochastic_depth.seed, net.stochastic_depth.rank) == (9, 3)
    assert net.stochastic_depth.rates[-1] == pytest.approx(0.1)
    ns.drop_path_rate = 0.0
    assert common.init_model(ns).stochastic_depth is None


class _Wrapper(object):
    def __init__(self, module):
        self.module = module


def test_checkpoint_round_trip_of_the_counter(tmp_path):
    log = logging.getLogger('test')
    net = models.resnet18(num_classes=10, drop_path_rate=0.1)
    sd = net.stochastic_depth
    for _ in range(5):
        sd.draw(2, 'cpu')
    state = {}
    common.save_stochastic_depth(state, _Wrapper(net))
    assert state == {'stochastic_depth': {'draws': 5}}
    torch.save(state, tmp_path / 'ckpt.pth')
    ckpt = torch.load(tmp_path / 'ckpt.pth', weights_only=False)
    fresh = models.resnet18(num_classes=10, drop_path_rate=0.1)
    new_state = {}
    common.load_stochastic_depth(ckpt, new_state, _Wrapper(fresh), log)
    assert fresh.stochastic_depth.draws == 5 and new_state['stochastic_depth'] == {'draws': 5}
    assert torch.equal(fresh.stochastic_depth.draw(3, 'cpu'), sd.draw(3, 'cpu'))
    # rate 0: nothing is saved or loaded
    state = {}
    common.save_stochastic_depth(state, _Wrapper(models.resnet18()))
    assert state == {}
