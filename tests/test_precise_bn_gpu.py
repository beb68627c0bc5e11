"""GossipTrainer.update_bn (precise BatchNorm statistics) on the GPU:

* the accumulate mode of both statistics finalize kernels (``bn_forward`` / ``conv1x1_bn_forward`` with
  ``acc``): outputs and coefficients bit-identical to the training call, ``acc`` gaining exactly what a
  momentum-1 call from zeroed buffers writes, running buffers and ``num_batches_tracked`` untouched, on the
  ResNet-50 shapes and forced small grids;
* end to end on ResNet-50 (fp32 and the bf16 twin, graphs on and off) against the momentum-1 oracle, bit for
  bit, replayed without a new capture; the launch count of one batch;
* no side effects on training (local, loop-back SGP and OSGP), the EMA, an evaluation graph captured
  before, and a command-line run with all three validations."""
import functools
import os
import subprocess
import sys

import pytest
import torch

from stochastic_gradient_push_b200.ops import native
from stochastic_gradient_push_b200.ops.fused_bn import FusedBatchNormAct2d, eval_bn_gemm

from test_conv1x1_scale_gpu import GRID_SHAPES, RESNET50_SHAPES
from test_gdp_loopback_gpu import _in_threads
from test_trainer_evaluate_gpu import _Block, _block_data, _data, _same_metrics, _trainer

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF16 = torch.bfloat16
DTYPES = {'f32': torch.float32, 'bf16': BF16}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def deterministic_cudnn():
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev


@pytest.fixture(scope='module')
def C():
    return native.load()


# ---------------------------------------------------------------------------------------------------- #
# the finalize kernels' accumulate mode
# ---------------------------------------------------------------------------------------------------- #
def _bn_state(N, g):
    gamma = torch.rand(N, device=DEV, generator=g) + 0.5
    beta = torch.randn(N, device=DEV, generator=g) * 0.2
    rm = torch.randn(N, device=DEV, generator=g) * 0.3
    rv = torch.rand(N, device=DEV, generator=g) + 0.5
    nbt = torch.full((), 5, dtype=torch.int64, device=DEV)
    acc = torch.randn(2 * N, device=DEV, dtype=torch.float64, generator=g)
    return gamma, beta, rm, rv, nbt, acc


def _check_accumulate(call, N, g):
    """call(rm, rv, nbt, momentum, acc) -> outputs; against the training call and a momentum-1 call"""
    gamma, beta, rm, rv, nbt, acc0 = _bn_state(N, g)
    train = call(gamma, beta, rm.clone(), rv.clone(), nbt.clone(), 0.1, None)
    zm, zv, znbt = torch.zeros_like(rm), torch.zeros_like(rv), nbt.clone()
    call(gamma, beta, zm, zv, znbt, 1.0, None)
    rm1, rv1, nbt1, acc = rm.clone(), rv.clone(), nbt.clone(), acc0.clone()
    got = call(gamma, beta, rm1, rv1, nbt1, 0.1, acc)
    torch.cuda.synchronize()
    assert len(got) == len(train)
    for a, b in zip(got, train):
        assert torch.equal(a, b)                            # outputs and mean / invstd / scale / shift
    assert torch.equal(rm1, rm) and torch.equal(rv1, rv) and int(nbt1) == 5
    assert torch.equal(acc, acc0 + torch.cat([zm, zv]).double())
    return acc


@pytest.mark.parametrize('dtype', list(DTYPES))
def test_bn_forward_accumulate_mode(C, dtype):
    # every ResNet-50 BatchNorm width at batch 8, and the stem's
    for (M, N) in [(M // 256 * 8, N) for (M, N, _) in RESNET50_SHAPES] + [(8 * 112 * 112, 64)]:
        g = torch.Generator(device=DEV).manual_seed(M + N)
        x = (torch.randn(M, N, device=DEV, generator=g) * 2 + 1).to(DTYPES[dtype])
        r = torch.randn(M, N, device=DEV, generator=g).to(DTYPES[dtype])
        for relu, res in ((False, None), (True, None), (True, r)):
            _check_accumulate(lambda gm, bt, rm, rv, nbt, mom, acc: C.bn_forward(
                x, res, gm, bt, rm, rv, nbt, True, mom, 1e-5, relu, acc), N, g)


def test_bn_forward_rejects_a_bad_accumulator(C):
    x = torch.randn(64, 16, device=DEV)
    gamma, beta, rm, rv, nbt, acc = _bn_state(16, torch.Generator(device=DEV).manual_seed(0))
    for bad in (acc[:16], acc.float(), acc.cpu()):
        with pytest.raises(RuntimeError, match='acc must be a contiguous fp64'):
            C.bn_forward(x, None, gamma, beta, rm, rv, nbt, True, 0.1, 1e-5, False, bad)
    with pytest.raises(RuntimeError, match='acc needs training mode'):
        C.bn_forward(x, None, gamma, beta, rm, rv, nbt, False, 0.1, 1e-5, False, acc)


@pytest.mark.parametrize('dtype', list(DTYPES))
def test_conv1x1_bn_forward_accumulate_mode(C, dtype):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cases = [((M // 256 * 8, N, K), 0) for (M, N, K) in RESNET50_SHAPES]
    cases += [(shape, n) for shape in GRID_SHAPES for n in (1, 3, 8)]
    cases += [((M, N, K), sms) for (M, N, K) in RESNET50_SHAPES[:4]]           # batch 256
    for (M, N, K), num_sms in cases:
        g = torch.Generator(device=DEV).manual_seed(M + N + K + num_sms)
        dt = DTYPES[dtype]
        x = torch.randn(M, K, device=DEV, generator=g).to(dt)
        w = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(dt)
        r = torch.randn(M, N, device=DEV, generator=g).to(dt)
        for relu, res in ((True, None), (True, r), (False, None)):
            _check_accumulate(lambda gm, bt, rm, rv, nbt, mom, acc: C.conv1x1_bn_forward(
                x, w, res, gm, bt, rm, rv, nbt, mom, 1e-5, relu, num_sms=num_sms, acc=acc), N, g)


def test_commit_kernel_divides_in_fp64_and_rounds_once(C):
    g = torch.Generator(device=DEV).manual_seed(3)
    sizes = [64, 8, 2048, 256, 24] * 250                 # 1250 layers: two launches
    flat = torch.randn(2 * sum(sizes), device=DEV, dtype=torch.float64, generator=g) * 1e3
    accs = list(flat.split([2 * c for c in sizes]))
    rms = [torch.empty(c, device=DEV) for c in sizes]
    rvs = [torch.empty(c, device=DEV) for c in sizes]
    c0 = C.launch_count()
    C.bn_stats_commit(accs, rms, rvs, 7)
    assert C.launch_count() - c0 == 2
    for a, m, v, c in zip(accs, rms, rvs, sizes):
        assert torch.equal(m, (a[:c] / 7).float()) and torch.equal(v, (a[c:] / 7).float())


# ---------------------------------------------------------------------------------------------------- #
# end to end
# ---------------------------------------------------------------------------------------------------- #
def _net(tr):
    twin = tr.model._twin
    return twin[0] if twin else tr.model.module


def _bns(tr):
    return [m for m in _net(tr).modules() if isinstance(m, FusedBatchNormAct2d)]


def _input(tr, x):
    dt = BF16 if tr.model._twin else torch.float32
    return x.to(DEV).to(dt).contiguous(memory_format=torch.channels_last)


def oracle(tr, batches):
    """one eager train-mode forward per batch of the trainer's network with every BN's running buffers
    zeroed and momentum 1 (so they hold exactly that batch's statistics), summed in fp64 on the host in
    batch order, / K, rounded to fp32.  Leaves the running buffers, momentum and num_batches_tracked of the
    network as they were."""
    net, bns = _net(tr), _bns(tr)
    saved = [(m.running_mean.clone(), m.running_var.clone(), m.num_batches_tracked.clone(), m.momentum)
             for m in bns]
    mode = net.training
    sums = [(torch.zeros(m.num_features, dtype=torch.float64), torch.zeros(m.num_features, dtype=torch.float64))
            for m in bns]
    net.train()
    for x, _ in batches:
        for m in bns:
            m.running_mean.zero_()
            m.running_var.zero_()
            m.momentum = 1.0
        with torch.no_grad(), tr._eval_autocast():
            net(_input(tr, x))
        sums = [(sm + m.running_mean.cpu().double(), sv + m.running_var.cpu().double())
                for (sm, sv), m in zip(sums, bns)]
    net.train(mode)
    for m, (rm, rv, nbt, mom) in zip(bns, saved):
        m.running_mean.copy_(rm)
        m.running_var.copy_(rv)
        m.num_batches_tracked.copy_(nbt)
        m.momentum = mom
    k = len(batches)
    return [((sm / k).float(), (sv / k).float()) for sm, sv in sums]


def _stats(tr):
    return [(m.running_mean.clone(), m.running_var.clone()) for m in _bns(tr)]


def _assert_stats(got, want):
    assert len(got) == len(want)
    for i, ((a, b), (c, d)) in enumerate(zip(got, want)):
        assert torch.equal(a.cpu(), c.cpu()) and torch.equal(b.cpu(), d.cpu()), i


@pytest.mark.parametrize('use_graph', [True, False], ids=['graph', 'eager'])
@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_update_bn_equals_the_oracle(twin, use_graph, deterministic_cudnn):
    tr = _trainer(twin=twin, use_graph=use_graph, lr=0.02)
    for s in range(3):                                    # weights and statistics away from their init
        tr.step(*_data(16, s))
    tr.finish()
    params = tr.model.arena.flat.clone()
    nbt = [int(m.num_batches_tracked) for m in _bns(tr)]
    mode = tr.model.module.training
    batches = [_data(16, 20), _data(16, 21), _data(6, 22)]           # two shapes, a partial batch last
    assert tr.update_bn(batches) == 3
    first = _stats(tr)
    assert len(first) == 53
    if use_graph:
        graphs = {k: s.bn_graph for k, s in tr._eval_slots.items()}
        assert len(graphs) == 2 and all(g is not None for g in graphs.values())
    assert tr.update_bn(iter(batches)) == 3               # replayed: same bits, nothing captured again
    _assert_stats(_stats(tr), first)
    if use_graph:
        assert {k: s.bn_graph for k, s in tr._eval_slots.items()} == graphs
    assert torch.equal(tr.model.arena.flat, params)
    assert [int(m.num_batches_tracked) for m in _bns(tr)] == nbt
    assert tr.model.module.training == mode and _net(tr).training == mode
    _assert_stats(first, oracle(tr, batches))
    # launches per batch: those of one eager no-grad train-mode forward
    C = tr.engine.C
    net = _net(tr)
    net.train()
    c0 = C.launch_count()
    with torch.no_grad(), tr._eval_autocast():
        net(_input(tr, batches[0][0]))
    assert tr.update_bn_launches_per_batch == C.launch_count() - c0 > 100
    # K = 0: nothing changes
    before = _stats(tr)
    assert tr.update_bn([]) == 0
    _assert_stats(_stats(tr), before)


def test_update_bn_does_not_disturb_training_local(deterministic_cudnn):
    """train k -> update_bn -> train k: arena, momentum, step count, num_batches_tracked and metrics equal
    2k plain steps, bit for bit (captured training and update_bn graphs in one pool)"""
    k = 3
    batches = [_block_data(16, 20 + s) for s in range(2 * k)]
    extra = [_block_data(16, 40), _block_data(7, 41)]
    refs = []
    for _ in range(2):                                  # the premise: training is reproducible
        ref = _trainer(net_fn=_Block)
        for b in batches:
            ref.step(*b)
        ref.finish()
        refs.append(ref)
    _equal(_train_state(refs[0]), _train_state(refs[1]))
    ref = refs[0]
    tr = _trainer(net_fn=_Block)
    for b in batches[:k]:
        tr.step(*b)
    assert tr.graph is not None
    torch.cuda.synchronize()
    before = tr.static_out.clone()
    assert tr.update_bn(extra) == 2
    _assert_stats(_stats(tr), oracle(tr, extra))
    assert torch.equal(tr.static_out, before)
    for b in batches[k:]:
        tr.step(*b)
    tr.finish()
    assert tr.engine.steps == ref.engine.steps
    _equal(_train_state(tr), _train_state(ref))
    _same_metrics(tr.metrics_ring[:2 * k], ref.metrics_ring[:2 * k])


def _train_state(tr):
    nbt = [m.num_batches_tracked.clone() for m in _bns(tr)]
    return [tr.model.arena.flat.clone(), tr.opt.momentum_flat[torch.float32].clone()] + nbt


def _equal(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), i


@pytest.mark.parametrize('algo', ['sgp', 'osgp'])
def test_update_bn_does_not_disturb_training_loopback(algo, deterministic_cudnn):
    """2 loop-back ranks, eager steps, captured update_bn; against a finish()-only run"""
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    overlap = algo == 'osgp'
    k = 2
    data = [[_block_data(8, 60 + 10 * r + s) for s in range(2 * k)] for r in range(2)]
    extra = [_block_data(8, 90), _block_data(3, 91)]

    def run(update, tag):
        lw = LocalWorld(2)
        trs = [_trainer(world=lw, rank=r, overlap=overlap, warmup=10 ** 6, name='pbn_%s_%s' % (algo, tag),
                        net_fn=_Block) for r in range(2)]
        after = None
        for s in range(2 * k):
            if s == k:
                torch.cuda.synchronize()
                for tr in trs:
                    if update:
                        assert tr.update_bn(extra) == 2
                    else:
                        tr.finish()
                if update:
                    after = [_stats(tr) for tr in trs]
                    for tr, st in zip(trs, after):
                        _assert_stats(st, oracle(tr, extra))
            _in_threads([functools.partial(trs[r].step, *data[r][s]) for r in range(2)])
            torch.cuda.synchronize()
        for tr in trs:
            tr.finish()
        return [(_train_state(tr), tr.metrics_ring[:2 * k].clone(), tr.engine.steps) for tr in trs]

    plain = run(False, 'b')
    for (sa, ma, na), (sb, mb, nb) in zip(run(False, 'c'), plain):      # the premise: reproducible
        _equal(sa, sb)
        _same_metrics(ma, mb)
        assert na == nb
    for (sa, ma, na), (sb, mb, nb) in zip(run(True, 'a'), plain):
        _equal(sa, sb)
        _same_metrics(ma, mb)
        assert na == nb


def test_update_bn_inside_ema_applied(deterministic_cudnn):
    tr = _trainer(ema_decay=0.5)
    for s in range(4):
        tr.step(*_data(16, 70 + s))
    batches = [_data(16, 80), _data(16, 81), _data(5, 82)]
    tr.update_bn(batches)                                   # captures both shapes
    graphs = {k: s.bn_graph for k, s in tr._eval_slots.items()}
    tr.finish()
    model_before = [tr.model.arena.flat.clone()] + [b.clone() for b in tr.model.module.buffers()]
    ema_before = tr.ema.ema.clone()
    with tr.ema.applied():
        assert tr.update_bn(batches) == 3
        inside = _stats(tr)
    assert {k: s.bn_graph for k, s in tr._eval_slots.items()} == graphs     # nothing captured again
    _equal([tr.model.arena.flat] + list(tr.model.module.buffers()), model_before)
    assert torch.equal(tr.ema.ema, ema_before)
    # a model loaded with the EMA state, its statistics recomputed by a trainer of its own
    ref = _trainer(lr=0.0, seed=12)
    ref.model.module.load_state_dict(tr.ema.state_dict()['state_dict'], strict=False)
    ref.update_bn(batches)
    _assert_stats(inside, _stats(ref))


def test_evaluation_graph_reads_the_new_statistics(deterministic_cudnn):
    tr = _trainer(lr=0.02)
    for s in range(3):
        tr.step(*_data(16, s))
    val = [_data(16, 50)]
    tr.evaluate(val)                                        # captured with the training statistics
    old = tr.eval_out.clone()
    tr.update_bn([_data(16, 30), _data(16, 31)])
    tr.evaluate(val)
    net = tr.model.module
    net.eval()
    with torch.no_grad(), eval_bn_gemm():
        want = net(_input(tr, val[0][0]))
    net.train()
    assert torch.equal(tr.eval_out, want)
    assert not torch.equal(old, want)


# ---------------------------------------------------------------------------------------------------- #
# command line
# ---------------------------------------------------------------------------------------------------- #
def test_cli_recomputes_the_statistics_before_every_validation(tmp_path, master_port):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '1',
           '--master-addr', '127.0.0.1', '--master-port', str(master_port), os.path.join(ROOT, 'gossip_sgd.py'),
           '--model', 'tiny', '--num_classes', '10', '--image_size', '32', '--synthetic', 'True',
           '--synthetic_len', '128', '--batch_size', '16', '--verbose', 'False', '--print_freq', '2',
           '--num_dataloader_workers', '0', '--lr', '0.05', '--push_sum', 'True', '--graph_type', '5',
           '--num_epochs', '2', '--num_itr_ignore', '0', '--cuda_graph', 'True', '--eval_graph', 'True',
           '--precise_bn_batches', '2', '--model_ema_decay', '0.9', '--validate_average', 'True',
           '--checkpoint_dir', str(tmp_path) + '/']
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    text = out.stdout
    assert text.count('precise BN: statistics from 2 training batches') == 2
    assert text.count('precise BN: EMA statistics from 2 training batches') == 2
    assert text.count('precise BN: average-model statistics from 2 training batches') == 2
    assert text.count(' * Prec@1') >= 4                     # rank model and average model, per epoch
    assert text.count(' * EMA Prec@1') == 2
    assert text.count('average-model Prec@1') == 2
    ck = torch.load(str(tmp_path / 'checkpoint_r0_n1.pth.tar'), map_location='cpu', weights_only=False)
    sd = ck['state_dict']['state_dict']
    assert all(torch.isfinite(v).all() for k, v in sd.items() if 'running_' in k)
