"""Single-GPU flagship path: smoke(), AR comparator at world 1, trainer on ResNet-50."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_graft_smoke():
    import __graft_entry__ as ge
    ge.smoke()


def test_trainer_resnet50_loss_decreases_world1():
    import stochastic_gradient_push_b200 as sgp
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    net = models.init_imagenet_in_1hr(models.resnet50()).to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1),
                               rank=0, world_size=1, heartbeat_timeout=20)
    opt = FusedGossipSGD(model, lr=0.02, momentum=0.9, weight_decay=1e-4, nesterov=True)
    tr = GossipTrainer(model, opt, use_cuda_graph=True, warmup_iters=2)
    x = torch.randn(8, 3, 96, 96).pin_memory()
    y = torch.randint(0, 1000, (8,)).pin_memory()
    slots = [tr.step(x, y) for _ in range(12)]
    tr.finish()
    losses = [float(tr.loss_ring[s]) for s in slots]
    assert tr.graph is not None                    # captured
    assert losses[-1] < losses[0]                  # memorises the fixed batch
    assert all(l == l for l in losses)


def test_trainer_fp32_tf32_path_matches_library_path(monkeypatch):
    """The precision-matched flagship step (fp32 activations / weights, TF32 wgmma 1x1 GEMMs with
    fused statistics + skip gradient, TF32 stem kernels, fused loss + accuracy) against the same
    step with every convolution on the library (cuDNN TF32): same losses within TF32 noise, both
    memorise a fixed batch, metrics ring carries [loss, prec@1, prec@5]."""
    import stochastic_gradient_push_b200 as sgp
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.ops import fused_bn
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    x = torch.randn(8, 3, 96, 96, generator=torch.Generator().manual_seed(5)).pin_memory()
    y = torch.randint(0, 1000, (8,), generator=torch.Generator().manual_seed(6)).pin_memory()
    runs = []
    for own in (True, False):
        monkeypatch.setattr(fused_bn, 'USE_TCGEN05_CONV1X1', own)
        monkeypatch.setattr(fused_bn, 'USE_STEM_KERNELS', own)
        torch.manual_seed(0)
        net = models.init_imagenet_in_1hr(models.resnet50()).to(dev).to(memory_format=torch.channels_last)
        model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1),
                                   rank=0, world_size=1, heartbeat_timeout=20)
        opt = FusedGossipSGD(model, lr=0.02, momentum=0.9, weight_decay=1e-4, nesterov=True)
        tr = GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=True, warmup_iters=2)
        slots = [tr.step(x, y) for _ in range(10)]
        tr.finish()
        rows = [tr.metrics_ring[s].tolist() for s in slots]
        assert tr.graph is not None and tr.own_launches_per_step > 100
        runs.append(rows)
    got, want = runs
    for (l1, a1, b1), (l2, a2, b2) in zip(got[:4], want[:4]):
        assert abs(l1 - l2) < 2e-2 * max(1.0, abs(l2)), (got, want)
    for rows in runs:
        assert rows[-1][0] < rows[0][0]
        assert all(0.0 <= r[1] <= r[2] <= 100.0 for r in rows)
    assert got[-1][1] >= 50.0          # the fixed batch of 8 is (mostly) memorised: prec@1 is live


def test_allreduce_world1_matches_torch_sgd():
    from stochastic_gradient_push_b200.parallel.allreduce import AllReduceDataParallel
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(64, 64), torch.nn.ReLU(), torch.nn.Linear(64, 8)).to(dev)
    import copy
    ref = copy.deepcopy(net)
    ar = AllReduceDataParallel(net, rank=0, world_size=1)
    opt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True)
    ar.set_hyper(0.1, 0.9, 1e-4, True)
    for _ in range(4):
        x = torch.randn(16, 64, device=dev)
        ar(x).square().mean().backward()
        ar.allreduce_step()
        opt.zero_grad()
        ref(x).square().mean().backward()
        opt.step()
    torch.cuda.synchronize()
    ar.check()
    for p, q in zip(net.parameters(), ref.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize('fused', [False, True])
def test_single_process_multi_replica_mode_matches_one_big_batch(fused):
    """reference launch mode (one process, several GPUs; gossip/distributed.py:87-99, 253-276,
    523-549): replicas on device_ids, scatter -> parallel_apply -> gather, the replicas' flat
    gradients summed into the master's by ONE P2P kernel.  With two replicas (both on cuda:0 when
    only one GPU is visible) the parameter trajectory must equal plain training on the whole
    batch (sum of per-replica sum-losses == whole-batch sum-loss)."""
    import copy
    import stochastic_gradient_push_b200 as sgp
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    ids = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Tanh(), torch.nn.Linear(32, 4)).to(dev)
    ref = copy.deepcopy(net)
    model = GossipDataParallel(net, device_ids=ids, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1),
                               rank=0, world_size=1, heartbeat_timeout=20)
    assert len(model._module_copies) == 2
    if fused:
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
    else:
        opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
    g = torch.Generator(device='cuda').manual_seed(1)
    for _ in range(5):
        x = torch.randn(24, 16, device=dev, generator=g)
        y = torch.randn(24, 4, device=dev, generator=g)
        out = model(x)
        assert out.shape == (24, 4) and out.device == dev
        (((out - y) ** 2).sum() / x.shape[0]).backward()      # (a stable step size: sum / batch)
        opt.step()
        opt.zero_grad(set_to_none=False) if not fused else opt.zero_grad()
        model.transfer_params()
        model._query_gossip_queue()
        model._flush_pending()
        (((ref(x) - y) ** 2).sum() / x.shape[0]).backward()
        ropt.step()
        ropt.zero_grad()
    torch.cuda.synchronize()
    for p, q in zip(net.parameters(), ref.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-5)
    # the replica was refreshed from the master at the last forward and has its own arena
    assert model._replica_arenas[1][0].flat.device.index == ids[1]


def _train_tiny(compute_dtype, amp, steps=6, graph=False):
    import stochastic_gradient_push_b200 as sgp
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    torch.manual_seed(3)
    net = models.TinyConvNet(width=32).to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0,
                               world_size=1, heartbeat_timeout=20, compute_dtype=compute_dtype)
    opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
    tr = GossipTrainer(model, opt, amp_dtype=amp, use_cuda_graph=graph, warmup_iters=2)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(32, 3, 32, 32, generator=g).pin_memory()
    y = torch.randint(0, 10, (32,), generator=g).pin_memory()
    slots = [tr.step(x, y) for _ in range(steps)]
    tr.finish()
    return model, [float(tr.loss_ring[s]) for s in slots]


@pytest.mark.parametrize('graph', [False, True])
def test_bf16_shadow_twin_tracks_the_autocast_path(graph):
    m_twin, l_twin = _train_tiny(torch.bfloat16, torch.bfloat16, graph=graph)
    m_auto, l_auto = _train_tiny(None, torch.bfloat16, graph=graph)
    assert m_twin.compute_module is not m_twin.module and m_auto.compute_module is m_auto.module
    # the shadow is exactly the bf16 rounding of the fp32 master arena, every step
    torch.testing.assert_close(m_twin.compute_shadow.float(), m_twin.arena.flat.bfloat16().float(),
                               rtol=0, atol=0)
    # BN parameters of the twin ARE the master tensors; running statistics are shared
    import torch.nn as nn
    for a, b in zip(m_twin.compute_module.modules(), m_twin.module.modules()):
        if isinstance(a, nn.BatchNorm2d):
            assert a.weight.data_ptr() == b.weight.data_ptr()
            assert a.running_mean.data_ptr() == b.running_mean.data_ptr()
    assert l_twin[-1] < l_twin[0]
    for lt, la in zip(l_twin, l_auto):
        assert abs(lt - la) < 0.05 * max(1.0, abs(la))
    rel = (m_twin.arena.flat - m_auto.arena.flat).norm() / m_auto.arena.flat.norm()
    assert rel.item() < 2e-2
