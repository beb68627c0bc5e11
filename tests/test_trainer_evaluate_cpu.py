"""GossipTrainer.evaluate without a GPU: EvalResult arithmetic, the --eval_graph flag (default off, parse,
rejection outside the captured trainer) and the bindings' argument checks."""
import math

import pytest
import torch

from stochastic_gradient_push_b200.parallel.trainer import EvalResult


def test_eval_result_from_sums():
    r = EvalResult.from_sums(1234.5, 600, 900, 1000)
    assert r == EvalResult(1.2345, 60.0, 90.0, 1000)
    assert isinstance(r.count, int) and r.loss == 1234.5 / 1000
    r = EvalResult.from_sums(3.0, 1, 2, 3)
    assert r.prec1 == 100.0 / 3 and r.prec5 == 200.0 / 3 and r.loss == 1.0
    assert r.prec1 <= r.prec5 <= 100.0


def test_eval_result_with_no_counted_row_is_nan():
    r = EvalResult.from_sums(0.0, 0, 0, 0)
    assert r.count == 0 and all(math.isnan(v) for v in (r.loss, r.prec1, r.prec5))


def test_eval_result_is_a_tuple_with_named_fields():
    loss, p1, p5, n = EvalResult.from_sums(2.0, 1, 1, 2)
    assert (loss, p1, p5, n) == (1.0, 50.0, 50.0, 2)
    assert EvalResult._fields == ('loss', 'prec1', 'prec5', 'count')


def _parse(argv, tmp_path):
    from stochastic_gradient_push_b200.cli import gossip_sgd
    return gossip_sgd.parse_args(argv + ['--checkpoint_dir', str(tmp_path) + '/'])


def test_cli_default_is_off_and_the_flag_parses(tmp_path, monkeypatch):
    from stochastic_gradient_push_b200.cli import gossip_sgd
    assert _parse(['--device', 'cpu'], tmp_path).eval_graph is False
    monkeypatch.setattr(gossip_sgd, 'finalize_args', lambda args, adpsgd=False: args)
    for flag in (['--eval_graph'], ['--eval_graph', 'True']):
        for extra in ([], ['--overlap', 'True'], ['--push_sum', 'False']):
            args = _parse(['--device', 'cuda', '--cuda_graph', 'True'] + flag + extra, tmp_path)
            assert args.eval_graph is True
    assert _parse(['--device', 'cuda', '--eval_graph', 'False'], tmp_path).eval_graph is False


@pytest.mark.parametrize('extra,what', [
    (['--all_reduce', 'True', '--graph_type', '-1', '--cuda_graph', 'True'], '--all_reduce'),
    (['--fused', 'False', '--cuda_graph', 'True'], '--fused False'),
    ([], '--cuda_graph False'),
    (['--cuda_graph', 'True', '--transport', 'c10d'], '--transport c10d'),
    (['--cuda_graph', 'True', '--device', 'cpu'], '--device cpu'),
])
def test_cli_rejects_eval_graph_without_the_captured_trainer(tmp_path, extra, what):
    with pytest.raises(ValueError, match='--eval_graph is not supported with %s' % what):
        _parse(['--eval_graph', 'True'] + extra, tmp_path)


def test_help_documents_the_flag(tmp_path, capsys):
    with pytest.raises(SystemExit):
        _parse(['--help'], tmp_path)
    text = ' '.join(capsys.readouterr().out.split())
    assert '--eval_graph' in text and 'GossipTrainer.evaluate' in text


def test_eval_accumulate_rejects_cpu_tensors():
    from stochastic_gradient_push_b200.ops import fused_loss
    acc = torch.zeros(4, dtype=torch.int64)
    with pytest.raises(ValueError, match='eval_accumulate needs'):
        fused_loss.eval_accumulate(torch.zeros(4, 10), torch.zeros(4, dtype=torch.int64), acc)


def test_eval_accumulator_layout():
    from stochastic_gradient_push_b200.ops import fused_loss
    acc = fused_loss.eval_accumulator('cpu')
    assert acc.dtype == torch.int64 and acc.shape == (4,) and int(acc.abs().sum()) == 0
    acc[:1].view(torch.float64).fill_(2.5)                 # the loss sum is fp64 bits in word 0
    assert float(acc[:1].view(torch.float64)) == 2.5


def test_bindings_exist():
    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    assert callable(C.conv1x1_bn_eval) and callable(C.xent_eval_accumulate)
