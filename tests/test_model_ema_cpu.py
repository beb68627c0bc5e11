"""ModelEma without a GPU: the plain-torch update against an independent fp64 emulation of
fmaf(1 - d_t, s - e, e), the warm-up decay, applied() and state_dict round trips, argument
validation (decay range, AD-PSGD), the command line's --model_ema_decay / --model_ema_warmup, and
two-rank gloo runs of gossip_sgd.py with and without the EMA."""

import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from stochastic_gradient_push_b200.ops.model_ema import ModelEma, decay_at


def _net(dtype=torch.float32):
    torch.manual_seed(0)
    net = nn.Sequential(nn.Linear(7, 13), nn.BatchNorm1d(13), nn.ReLU(), nn.Linear(13, 3))
    return net.to(dtype)


def _emulate(e, s, d_t):
    """fp32 e, s; fp32 w = 1 - d_t and fp32 s - e; w * (s - e) + e in fp64, rounded once to fp32"""
    w = np.float32(1.0) - np.float32(d_t)
    diff = (s.astype(np.float32) - e).astype(np.float32)
    return (np.float64(w) * diff.astype(np.float64) + e.astype(np.float64)).astype(np.float32)


def _float_state(net):
    return {k: v.detach().float().numpy().copy() for k, v in net.state_dict().items() if v.is_floating_point()}


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('warmup', [False, True])
def test_cpu_update_matches_formula(dtype, warmup):
    net = _net(dtype)
    ema = ModelEma(net, decay=0.9, warmup=warmup)
    ref = _float_state(net)
    for t in range(6):
        with torch.no_grad():
            for p in net.parameters():
                p.add_(torch.randn_like(p.float()).to(dtype))
        net.train()
        net(torch.randn(5, 7).to(dtype))           # moves the BatchNorm running statistics
        ema.update()
        d = decay_at(0.9, warmup, t)
        src = _float_state(net)
        ref = {k: _emulate(ref[k], src[k], d) for k in ref}
        got = ema.state_dict()['state_dict']
        assert set(got) == set(ref)
        for k in ref:
            assert np.array_equal(got[k].numpy(), ref[k]), (t, k)
    assert ema.num_updates == 6
    assert 'num_batches_tracked' not in ' '.join(ema.state_dict()['state_dict'])


def test_warmup_decay_rule():
    for t in range(21):
        r = np.float32(np.float32(1 + t) / np.float32(10 + t))
        assert decay_at(0.9999, True, t) == min(np.float32(0.9999), r)
        assert decay_at(0.5, True, t) == min(np.float32(0.5), r)
        assert decay_at(0.9999, False, t) == np.float32(0.9999)


def test_applied_swaps_in_and_restores_bits():
    net = _net()
    ema = ModelEma(net, decay=0.5)
    with torch.no_grad():
        for p in net.parameters():
            p.mul_(3.0)
    net.train()
    net(torch.randn(4, 7))
    ema.update()
    before = {k: v.clone() for k, v in net.state_dict().items()}
    fresh = _net()
    fresh.load_state_dict(ema.state_dict()['state_dict'], strict=False)
    x = torch.randn(6, 7)
    fresh.eval()
    net.eval()
    with ema.applied():
        inside = net(x)
    assert torch.equal(inside, fresh(x))
    for k, v in net.state_dict().items():
        assert torch.equal(v, before[k]), k


def test_state_dict_round_trip_continues_bit_for_bit():
    net = _net()
    a = ModelEma(net, decay=0.8, warmup=True)
    for _ in range(3):
        with torch.no_grad():
            net[0].weight.add_(1.0)
        a.update()
    sd = a.state_dict()
    b = ModelEma(net, decay=0.1)
    b.load_state_dict(sd)
    assert (b.decay, b.warmup, b.num_updates) == (0.8, True, 3)
    for _ in range(3):
        with torch.no_grad():
            net[0].weight.mul_(0.5)
        a.update()
        b.update()
    for k, v in a.state_dict()['state_dict'].items():
        assert torch.equal(v, b.state_dict()['state_dict'][k]), k


def test_set_decay_and_reset():
    net = _net()
    ema = ModelEma(net, decay=0.9)
    ema.set_decay(0.0)                      # d = 0: the EMA becomes the model
    with torch.no_grad():
        net[0].bias.add_(2.0)
    ema.update()
    assert torch.equal(ema.state_dict()['state_dict']['0.bias'], net[0].bias.detach())
    ema.reset()
    assert ema.num_updates == 0


@pytest.mark.parametrize('decay', [-0.1, 1.0, 1.5, float('nan')])
def test_decay_out_of_range_raises(decay):
    with pytest.raises(ValueError, match=r'\[0, 1\)'):
        ModelEma(_net(), decay=decay)
    ema = ModelEma(_net(), decay=0.5)
    with pytest.raises(ValueError):
        ema.set_decay(decay)


def test_unsupported_dtype_raises():
    with pytest.raises(ValueError, match='fp32 and bf16'):
        ModelEma(_net(torch.float16))


def test_adpsgd_trainer_rejects_ema():
    from stochastic_gradient_push_b200.parallel.ad_psgd import make_bilat_trainer
    with pytest.raises(ValueError, match='AD-PSGD'):
        make_bilat_trainer(None, lr=0.1, ema=object())


def test_cli_parsing_and_rejections(tmp_path):
    from stochastic_gradient_push_b200.cli.common import build_parser, finalize_args
    d = str(tmp_path) + '/'
    args = build_parser().parse_args([])
    assert args.model_ema_decay == 0.0 and args.model_ema_warmup is False
    args = finalize_args(build_parser().parse_args(
        ['--model_ema_decay', '0.999', '--model_ema_warmup', 'True', '--device', 'cpu', '--checkpoint_dir', d]))
    assert args.model_ema_decay == 0.999 and args.model_ema_warmup is True
    assert args.ema_fname == d + 'ema_r0_n1.csv'
    for bad in ('1.0', '-0.5'):
        with pytest.raises(ValueError, match='model_ema_decay'):
            finalize_args(build_parser().parse_args(['--model_ema_decay', bad, '--device', 'cpu',
                                                     '--checkpoint_dir', d]))
    args = build_parser(adpsgd=True).parse_args(['--model_ema_decay', '0.99', '--device', 'cpu',
                                                 '--checkpoint_dir', d])
    with pytest.raises(ValueError, match='AD-PSGD'):
        finalize_args(args, adpsgd=True)
    from stochastic_gradient_push_b200.cli import gossip_sgd_adpsgd
    with pytest.raises(ValueError, match='AD-PSGD'):
        gossip_sgd_adpsgd.main(['--model_ema_decay', '0.99', '--device', 'cpu', '--checkpoint_dir', d])


def test_gossip_sgd_cli_ema_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    base = COMMON + ['--push_sum', 'True', '--graph_type', '5', '--num_epochs', '2', '--num_itr_ignore', '0']
    runs = {}
    for tag, extra in (('plain', []), ('ema', ['--model_ema_decay', '0.99', '--model_ema_warmup', 'True'])):
        d = tmp_path / tag
        d.mkdir()
        out = _torchrun(2, 'gossip_sgd.py', base + ['--checkpoint_dir', str(d) + '/'] + extra, master_port)
        assert out.returncode == 0, out.stdout[-3000:]
        runs[tag] = (d, out.stdout)
    d, stdout = runs['ema']
    assert ' * EMA Prec@1' in stdout
    for r in range(2):
        lines = open(str(d / ('ema_r%d_n2.csv' % r))).read().splitlines()
        assert lines[0] == 'epoch,num_updates,prec1,prec5'
        rows = [l.split(',') for l in lines[1:]]
        assert [row[0] for row in rows] == ['0', '1']
        assert int(rows[1][1]) > int(rows[0][1]) > 0
        assert all(0.0 <= float(row[2]) <= float(row[3]) <= 100.0 for row in rows)
        ck = torch.load(str(d / ('checkpoint_r%d_n2.pth.tar' % r)), map_location='cpu', weights_only=False)
        em = ck['model_ema']
        assert em['decay'] == 0.99 and em['warmup'] is True and em['num_updates'] == int(rows[1][1])
        model_keys = {k for k, v in ck['state_dict']['state_dict'].items() if v.is_floating_point()}
        assert {'module.' + k for k in em['state_dict']} == model_keys
        assert all(torch.isfinite(v).all() for v in em['state_dict'].values())
        # without the flag: today's files and keys
        pd = runs['plain'][0]
        assert not os.path.exists(str(pd / ('ema_r%d_n2.csv' % r)))
        pk = torch.load(str(pd / ('checkpoint_r%d_n2.pth.tar' % r)), map_location='cpu', weights_only=False)
        assert 'model_ema' not in pk
        assert set(pk) == set(ck) - {'model_ema'}
        plain = open(str(pd / ('out_r%d_n2.csv' % r))).read().splitlines()
        withema = open(str(d / ('out_r%d_n2.csv' % r))).read().splitlines()
        assert [len(l.split(',')) for l in plain] == [len(l.split(',')) for l in withema]
    assert ' * EMA' not in runs['plain'][1]


def test_gossip_sgd_cli_ema_resume_without_key_warns(tmp_path, master_port):
    """A checkpoint written without the EMA, resumed with it on: the EMA restarts from the loaded model."""
    from test_cli_and_experiment import COMMON, _torchrun
    base = COMMON + ['--push_sum', 'True', '--graph_type', '5', '--num_itr_ignore', '0',
                     '--checkpoint_dir', str(tmp_path) + '/']
    out = _torchrun(2, 'gossip_sgd.py', base + ['--num_epochs', '1'], master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    out = _torchrun(2, 'gossip_sgd.py', base + ['--num_epochs', '2', '--resume', 'True', '--model_ema_decay', '0.9'],
                    master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    assert 'checkpoint has no model_ema' in out.stdout
    for r in range(2):
        ck = torch.load(str(tmp_path / ('checkpoint_r%d_n2.pth.tar' % r)), map_location='cpu', weights_only=False)
        assert ck['model_ema']['num_updates'] > 0 and ck['epoch'] == 2
