"""A residual block's last BatchNorm backward reduction folded into the next block's conv1 dgrad
GEMM (MODE 3 of csrc/conv1x1_kernels.cu), the 1-bit ReLU mask it reads, and the autograd hand-off
between the two ops (ops/fused_bn.py), against the stand-alone reduce path."""
import pytest
import torch
import torch.nn as nn

from stochastic_gradient_push_b200.ops import fused_bn, native

pytestmark = pytest.mark.gpu

# ResNet-50 conv1 dgrad (N = C_in, K = width) at a small ragged M; (2048, 512) fp32 keeps W non-resident
DGRAD_NK = [(256, 64), (256, 128), (512, 128), (512, 256), (1024, 256), (1024, 512), (2048, 512)]


def _unpack(mask, M, N):
    bits = (mask.view(M, N // 8, 1) >> torch.arange(8, device=mask.device, dtype=torch.uint8)) & 1
    return bits.view(M, N).bool()


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('M', [1000, 4224])
def test_apply_mask_matches_output_sign(dtype, M):
    C = native.load()
    K, N = 64, 256
    g = torch.Generator(device='cuda').manual_seed(M)
    x = torch.randn(M, K, device='cuda', generator=g).to(dtype)
    w = (torch.randn(N, K, device='cuda', generator=g) * K ** -0.5).to(dtype)
    r = torch.randn(M, N, device='cuda', generator=g).to(dtype)
    gamma = torch.rand(N, device='cuda') + 0.5
    beta = torch.randn(N, device='cuda') * 0.1
    mask = torch.empty(M, N // 8, dtype=torch.uint8, device='cuda')
    _, out, _ = C.conv1x1_bn_forward(x, w, r, gamma, beta, None, None, None, 0.1, 1e-5, True, mask)
    torch.cuda.synchronize()
    assert torch.equal(_unpack(mask, M, N), out > 0)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('N,K', DGRAD_NK)
def test_mode3_matches_composition(dtype, N, K):
    """dz = mask ? dY.W + R : 0 equals the MODE 2 output masked, bit for bit; the per-channel sums
    sum(dz) and sum(dz * xhat) match fp64 sums of that dz."""
    C = native.load()
    M = 1000
    g = torch.Generator(device='cuda').manual_seed(N + K)
    x = torch.randn(M, K, device='cuda', generator=g).to(dtype)
    wt = (torch.randn(N, K, device='cuda', generator=g) * K ** -0.5).to(dtype)
    r = torch.randn(M, N, device='cuda', generator=g).to(dtype)
    bn_x = (torch.randn(M, N, device='cuda', generator=g) * 2 + 1).to(dtype)
    coef = torch.empty(4, N, device='cuda')
    coef[0] = bn_x.float().mean(0)
    coef[1] = (bn_x.float().var(0, unbiased=False) + 1e-5).rsqrt()
    coef[2:] = 1.0
    mask = torch.randint(0, 256, (M, N // 8), dtype=torch.uint8, device='cuda', generator=g)
    dz, partial = C.conv1x1_dgrad_bn_reduce(x, wt, r, bn_x, coef, mask)
    v = C.conv1x1_forward(x, wt, False, r)
    torch.cuda.synchronize()
    keep = _unpack(mask, M, N)
    assert torch.equal(dz, torch.where(keep, v, torch.zeros_like(v)))
    assert partial.shape[1:] == (2, N)
    d = dz.double()
    xhat = (bn_x.double() - coef[0].double()) * coef[1].double()
    s, q = d.sum(0), (d * xhat).sum(0)
    sp, qp = partial.double().sum(0)
    torch.testing.assert_close(sp, s, rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(qp, q, rtol=1e-4, atol=1e-3)


def _chain(cin, specs, dtype, seed=5):
    from stochastic_gradient_push_b200.models.resnet import Bottleneck, _conv1x1, _BN
    torch.manual_seed(seed)
    blocks = []
    for width, stride in specs:
        ds = None
        if stride != 1 or cin != 4 * width:
            ds = nn.Sequential(_conv1x1(cin, 4 * width, stride), _BN(4 * width))
        blocks.append(Bottleneck(cin, width, stride, ds))
        cin = 4 * width
    net = nn.Sequential(*blocks).cuda().to(memory_format=torch.channels_last)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.1)
    if dtype == torch.bfloat16:
        for m in net.modules():
            if isinstance(m, nn.Conv2d):
                m.to(torch.bfloat16)
    return net


def _run(monkeypatch, fuse, specs, dtype, hook_at=None):
    monkeypatch.setattr(fused_bn, 'USE_BN_BWD_FUSE', fuse)
    C = native.load()
    calls = []
    orig = C.conv1x1_dgrad_bn_reduce
    monkeypatch.setattr(C, 'conv1x1_dgrad_bn_reduce', lambda *a: calls.append(1) or orig(*a))
    net = _chain(256, specs, dtype)
    g = torch.Generator(device='cuda').manual_seed(2)
    x0 = torch.randn(4, 256, 14, 14, device='cuda', generator=g).to(dtype) \
        .contiguous(memory_format=torch.channels_last).requires_grad_(True)
    h = x0 * 1                             # non-leaf block input, as inside the network
    seen = []
    for i, blk in enumerate(net):
        h = blk(h)
        if i == hook_at:
            h.register_hook(lambda grad: seen.append(grad.float().clone()))
    dy = torch.randn(h.shape, device='cuda', generator=g).to(dtype).contiguous(memory_format=torch.channels_last)
    h.backward(dy)
    torch.cuda.synchronize()
    monkeypatch.setattr(C, 'conv1x1_dgrad_bn_reduce', orig)
    return dict(y=h.detach().float(), dx=x0.grad.float(), calls=len(calls), seen=seen,
                grads={n: p.grad.float() for n, p in net.named_parameters()})


CHAINS = [[(64, 1), (128, 1)],                  # two blocks, the second with a stride-1 downsample
          [(64, 1), (128, 2), (128, 1)]]        # three blocks across a stride-2 downsample


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('specs', CHAINS)
def test_block_chain_matches_unfused(monkeypatch, dtype, specs):
    """Fused hand-off vs SGP_B200_BN_BWD_FUSE=0: output, input gradient and every parameter gradient."""
    got = _run(monkeypatch, True, specs, dtype)
    want = _run(monkeypatch, False, specs, dtype)
    assert got['calls'] == len(specs) - 1 and want['calls'] == 0
    assert torch.equal(got['y'], want['y'])
    tol = 1e-3 if dtype == torch.float32 else 2e-2
    rel = (got['dx'] - want['dx']).norm().item() / want['dx'].norm().item()
    assert rel < tol, rel
    for n in want['grads']:
        rel = (got['grads'][n] - want['grads'][n]).norm().item() / (want['grads'][n].norm().item() + 1e-6)
        assert rel < tol, (n, rel)


def test_hook_on_block_output_disables_fusion(monkeypatch):
    """A hook on the middle block's output must see the full (pre-mask) gradient, as without fusion."""
    specs = CHAINS[1]
    got = _run(monkeypatch, True, specs, torch.float32, hook_at=1)
    want = _run(monkeypatch, False, specs, torch.float32, hook_at=1)
    assert got['calls'] == 1                            # block 0 -> 1 still fused, block 1 -> 2 not
    assert len(got['seen']) == len(want['seen']) == 1
    torch.testing.assert_close(got['seen'][0], want['seen'][0], rtol=1e-4, atol=1e-5)
    rel = (got['dx'] - want['dx']).norm().item() / want['dx'].norm().item()
    assert rel < 1e-3, rel
