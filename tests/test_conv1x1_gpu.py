"""wgmma 1x1-convolution GEMM with fused BatchNorm statistics (csrc/conv1x1_kernels.cu)
vs plain PyTorch fp32 references of the same ops."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from stochastic_gradient_push_b200.ops import fused_bn, native
from stochastic_gradient_push_b200.ops.fused_bn import FusedBatchNormAct2d, conv_bn_act

pytestmark = pytest.mark.gpu

# (M, K, N): one tile / ragged last tile / several k-blocks / every BLOCK_N / more n-blocks than
# m-tiles / resident-W with 2 store slabs / ResNet-50 layer shapes at a small batch / K % 64 != 0
GEMM_SHAPES = [(128, 64, 64), (677, 64, 64), (1000, 256, 128), (4096, 128, 256), (3000, 512, 512),
               (130, 192, 1024), (4224, 256, 256), (2000, 1024, 64), (25088, 64, 256), (6272, 1024, 256), (1568, 2048, 512), (40000, 72, 192)]


def _mats(M, K, N, x_mean=0.0, dtype=torch.bfloat16):
    g = torch.Generator(device='cuda').manual_seed(M + K + N)
    x = (torch.randn(M, K, device='cuda', generator=g) + x_mean).to(dtype)
    w = (torch.randn(N, K, device='cuda', generator=g) * K ** -0.5).to(dtype)
    return x, w


def _tf32(t):
    """what kind::tf32 sees of an fp32 operand: the top 19 bits (sign, 8 exponent, 10 mantissa)"""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


# fp32 operands (K % 4 == 0 suffices: 16-byte rows), TF32 tensor-core math, fp32 output
GEMM_SHAPES_F32 = GEMM_SHAPES + [(515, 36, 64), (300, 100, 128)]


@pytest.mark.parametrize('M,K,N', GEMM_SHAPES_F32)
def test_tf32_gemm_matches_fp32_matmul(M, K, N):
    """kind::tf32 path: against an fp64 matmul of the tf32-truncated operands (tight) and of the
    full fp32 operands (TF32-level tolerance, the precision of the reference's cuDNN convs)."""
    C = native.load()
    x, w = _mats(M, K, N, dtype=torch.float32)
    assert C.conv1x1_can_fuse(x, w)
    y = C.conv1x1_forward(x, w)
    torch.cuda.synchronize()
    assert y.shape == (M, N) and y.dtype == torch.float32
    exact = (_tf32(x).double() @ _tf32(w).double().t()).float()
    torch.testing.assert_close(y, exact, rtol=2e-5, atol=2e-5 * K ** 0.5)
    want = (x.double() @ w.double().t()).float()
    torch.testing.assert_close(y, want, rtol=5e-3, atol=5e-3)


@pytest.mark.parametrize('M,K,N', GEMM_SHAPES_F32)
@pytest.mark.parametrize('x_mean', [0.0, 3.0])
def test_tf32_fused_statistics_match_two_pass(M, K, N, x_mean):
    C = native.load()
    x, w = _mats(M, K, N, x_mean, dtype=torch.float32)
    if x_mean:
        w = w + 0.05
    gamma = torch.rand(N, device='cuda') + 0.5
    beta = torch.randn(N, device='cuda') * 0.1
    rm, rv = torch.zeros(N, device='cuda'), torch.ones(N, device='cuda')
    nbt = torch.zeros((), dtype=torch.long, device='cuda')
    yraw, out, coef = C.conv1x1_bn_forward(x, w, None, gamma, beta, rm, rv, nbt, 0.1, 1e-5, True)
    torch.cuda.synchronize()
    assert yraw.dtype == torch.float32 and out.dtype == torch.float32
    exact = (_tf32(x).double() @ _tf32(w).double().t())
    torch.testing.assert_close(yraw.double(), exact, rtol=2e-5, atol=2e-5 * K ** 0.5 * max(1.0, x_mean * 4))
    yd = yraw.double()
    mean, var = yd.mean(0), yd.var(0, unbiased=False)
    torch.testing.assert_close(coef[0].double(), mean, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(coef[1].double(), (var + 1e-5).rsqrt(), rtol=2e-4, atol=1e-5)
    want = F.relu(F.batch_norm(yraw, None, None, gamma, beta, True, 0.1, 1e-5))
    torch.testing.assert_close(out, want, rtol=1e-3, atol=1e-3)
    assert int(nbt) == 1
    torch.testing.assert_close(rm.double(), 0.1 * mean, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize('M,K,N', GEMM_SHAPES_F32)
def test_tf32_gemm_residual_epilogue(M, K, N):
    C = native.load()
    x, w = _mats(M, K, N, dtype=torch.float32)
    g = torch.Generator(device='cuda').manual_seed(7)
    r = torch.randn(M, N, device='cuda', generator=g) * 2
    y = C.conv1x1_forward(x, w, False, r)
    torch.cuda.synchronize()
    exact = (_tf32(x).double() @ _tf32(w).double().t() + r.double()).float()
    torch.testing.assert_close(y, exact, rtol=2e-5, atol=2e-5 * K ** 0.5)


@pytest.mark.parametrize('M,K,N', GEMM_SHAPES)
def test_gemm_matches_fp32_matmul(M, K, N):
    C = native.load()
    x, w = _mats(M, K, N)
    assert C.conv1x1_can_fuse(x, w)
    y = C.conv1x1_forward(x, w)
    torch.cuda.synchronize()
    want = x.float() @ w.float().t()
    assert y.shape == (M, N) and y.dtype == torch.bfloat16
    torch.testing.assert_close(y.float(), want, rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize('M,K,N', GEMM_SHAPES)
@pytest.mark.parametrize('x_mean', [0.0, 3.0])
def test_fused_statistics_match_two_pass(M, K, N, x_mean):
    """mean / invstd from the epilogue partials == two-pass fp32 statistics of the bf16 output;
    x_mean=3 gives outputs whose |mean| is several standard deviations (cancellation check)."""
    C = native.load()
    x, w = _mats(M, K, N, x_mean)
    if x_mean:
        w = (w.float() + 0.05).to(torch.bfloat16)
    gamma = torch.rand(N, device='cuda') + 0.5
    beta = torch.randn(N, device='cuda') * 0.1
    rm, rv = torch.zeros(N, device='cuda'), torch.ones(N, device='cuda')
    nbt = torch.zeros((), dtype=torch.long, device='cuda')
    yraw, out, coef = C.conv1x1_bn_forward(x, w, None, gamma, beta, rm, rv, nbt, 0.1, 1e-5, True)
    torch.cuda.synchronize()
    yf = yraw.float()
    torch.testing.assert_close(yf, x.float() @ w.float().t(), rtol=1e-2, atol=1e-2 * max(1.0, x_mean * 4))
    mean = yf.mean(0)
    var = yf.var(0, unbiased=False)
    torch.testing.assert_close(coef[0], mean, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(coef[1], (var + 1e-5).rsqrt(), rtol=2e-4, atol=1e-5)
    want = F.relu(F.batch_norm(yf, None, None, gamma, beta, True, 0.1, 1e-5))
    bad = (out.float() - want).abs() > 2e-2 + 2e-2 * want.abs()
    assert bad.float().mean().item() < 2e-5
    assert int(nbt) == 1
    torch.testing.assert_close(rm, 0.1 * mean, rtol=1e-4, atol=1e-5)
    if M > 1:
        torch.testing.assert_close(rv, 0.9 + 0.1 * var * M / (M - 1), rtol=2e-4, atol=1e-5)


@pytest.mark.parametrize('M,K,N', GEMM_SHAPES)
def test_gemm_residual_epilogue(M, K, N):
    """y = x . w^T + r with the sum formed in fp32 before the single bf16 rounding."""
    C = native.load()
    x, w = _mats(M, K, N)
    g = torch.Generator(device='cuda').manual_seed(7)
    r = (torch.randn(M, N, device='cuda', generator=g) * 2).to(torch.bfloat16)
    y = C.conv1x1_forward(x, w, False, r)
    torch.cuda.synchronize()
    want = x.float() @ w.float().t() + r.float()
    torch.testing.assert_close(y.float(), want, rtol=1e-2, atol=2e-2)
    # strictly better than rounding twice would allow on average
    twice = (x.float() @ w.float().t()).to(torch.bfloat16).float() + r.float()
    assert (y.float() - want).abs().mean() <= (twice.to(torch.bfloat16).float() - want).abs().mean() * 1.05


def _block(cin, cout, seed):
    torch.manual_seed(seed)
    conv = nn.Conv2d(cin, cout, 1, bias=False).cuda().to(memory_format=torch.channels_last)
    bn = FusedBatchNormAct2d(cout).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.1)
    return conv, bn


@pytest.mark.parametrize('shape,cout', [((8, 64, 14, 14), 256), ((4, 256, 7, 9), 64), ((2, 512, 5, 5), 2048)])
@pytest.mark.parametrize('add', [False, True])
@pytest.mark.parametrize('bf16_weights', [True, False])
def test_conv_bn_act_matches_unfused_path(monkeypatch, shape, cout, add, bf16_weights):
    """Forward, input / weight / BN gradients and running statistics of the fused op vs
    library convolution + stand-alone fused BN (the path it replaces)."""
    results = []
    for use in (True, False):
        monkeypatch.setattr(fused_bn, 'USE_TCGEN05_CONV1X1', use)
        conv, bn = _block(shape[1], cout, seed=3)
        if bf16_weights:
            conv = conv.to(torch.bfloat16)
        g = torch.Generator(device='cuda').manual_seed(11)
        x = torch.randn(shape, device='cuda', generator=g).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last).requires_grad_(True)
        res = None
        if add:
            res = torch.randn((shape[0], cout) + shape[2:], device='cuda', generator=g).to(torch.bfloat16) \
                .contiguous(memory_format=torch.channels_last).requires_grad_(True)
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=not bf16_weights):
            y = conv_bn_act(conv, bn, x, residual=res, relu=True)
        dy = torch.randn(y.shape, device='cuda', generator=g).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last)
        y.backward(dy)
        torch.cuda.synchronize()
        results.append(dict(y=y.detach().float(), dx=x.grad.float(), dw=conv.weight.grad.float(),
                            dg=bn.weight.grad.clone(), db=bn.bias.grad.clone(),
                            dres=None if res is None else res.grad.float(),
                            rm=bn.running_mean.clone(), rv=bn.running_var.clone(),
                            nbt=int(bn.num_batches_tracked)))
    got, want = results
    assert got['nbt'] == want['nbt'] == 1
    for key, tol in (('y', 3e-2), ('dx', 3e-2), ('dres', 3e-2)):
        if want[key] is None:
            continue
        bad = (got[key] - want[key]).abs() > tol + tol * want[key].abs()
        assert bad.float().mean().item() < 1e-3, key
    for key in ('dw', 'dg', 'db'):
        scale = want[key].abs().max().item() + 1e-6
        assert (got[key] - want[key]).abs().max().item() < 3e-2 * scale, key
    torch.testing.assert_close(got['rm'], want['rm'], rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(got['rv'], want['rv'], rtol=1e-3, atol=1e-3)


def test_unsupported_inputs_fall_back(monkeypatch):
    """stride-2 / 3x3 / eval-mode / NCHW inputs must take the library path, not fail."""
    monkeypatch.setattr(fused_bn, 'USE_TCGEN05_CONV1X1', True)
    torch.manual_seed(0)
    x = torch.randn(2, 64, 8, 8, device='cuda').to(torch.bfloat16)
    for conv in (nn.Conv2d(64, 128, 1, 2, bias=False), nn.Conv2d(64, 128, 3, 1, 1, bias=False)):
        conv = conv.cuda().to(torch.bfloat16)
        bn = FusedBatchNormAct2d(128).cuda()
        y = conv_bn_act(conv, bn, x.contiguous(memory_format=torch.channels_last), relu=True)
        assert y.shape[1] == 128
    conv, bn = _block(64, 128, 0)
    conv = conv.to(torch.bfloat16)
    y = conv_bn_act(conv, bn, x, relu=True)          # NCHW input
    assert y.shape == (2, 128, 8, 8)
    bn.eval()
    y = conv_bn_act(conv, bn, x.contiguous(memory_format=torch.channels_last), relu=True)
    assert y.shape == (2, 128, 8, 8)


@pytest.mark.parametrize('cin,width,hw', [(256, 64, 14), (512, 128, 7)])
def test_fp32_bottleneck_matches_library_path(monkeypatch, cin, width, hw):
    """fp32 activations / weights (the precision-matched flagship path): a bottleneck through the
    TF32 wgmma GEMMs (statistics + skip gradient fused) and through library TF32 convolutions +
    the stand-alone fused BN, both measured against the SAME block evaluated in fp64.  TF32
    rounding flips ReLU masks of near-zero activations, so two TF32 paths differ element-wise;
    what must hold is that ours is as close to the fp64 truth as the library path is."""
    import copy
    from stochastic_gradient_push_b200.models.resnet import Bottleneck
    torch.manual_seed(5)
    blk0 = Bottleneck(cin, width, 1, None).cuda().to(memory_format=torch.channels_last)
    with torch.no_grad():
        for m in blk0.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.1)
    g = torch.Generator(device='cuda').manual_seed(2)
    xin = torch.randn(8, cin, hw, hw, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(8, 4 * width, hw, hw, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)

    def run(mode):
        blk = copy.deepcopy(blk0)
        x0 = xin.clone()
        d = dy
        if mode == 'fp64':
            blk, x0, d = blk.double(), x0.double(), dy.double()
            monkeypatch.setattr(fused_bn, 'FORCE_REFERENCE', True)
        else:
            monkeypatch.setattr(fused_bn, 'FORCE_REFERENCE', False)
            monkeypatch.setattr(fused_bn, 'USE_TCGEN05_CONV1X1', mode == 'ours')
        x0.requires_grad_(True)
        y = blk(x0 * 1)
        y.backward(d)
        torch.cuda.synchronize()
        out = dict(y=y.detach().double(), dx=x0.grad.double())
        out.update({n: p.grad.double() for n, p in blk.named_parameters()})
        return out

    truth, ours, lib = run('fp64'), run('ours'), run('lib')
    monkeypatch.setattr(fused_bn, 'FORCE_REFERENCE', False)
    for key in truth:
        scale = truth[key].norm().item() + 1e-12
        e_ours = (ours[key] - truth[key]).norm().item() / scale
        e_lib = (lib[key] - truth[key]).norm().item() / scale
        assert e_ours < max(3.0 * e_lib, 2e-3), (key, e_ours, e_lib)
        assert e_ours < 6e-2, (key, e_ours)     # (TF32 noise through three BatchNorm backward passes: ~2.7e-2 on dx)


@pytest.mark.parametrize('cin,width,hw', [(256, 64, 14), (64, 64, 9), (512, 128, 7)])
@pytest.mark.parametrize('downsample', [False, True])
def test_bottleneck_split_backward_matches_unfused(monkeypatch, cin, width, hw, downsample):
    """A whole bottleneck block (conv1 dgrad absorbs the skip gradient) vs the library path:
    outputs, input gradient and every parameter gradient."""
    from stochastic_gradient_push_b200.models.resnet import Bottleneck, _conv1x1, _BN
    results = []
    for use in (True, False):
        monkeypatch.setattr(fused_bn, 'USE_TCGEN05_CONV1X1', use)
        torch.manual_seed(5)
        ds = None
        if downsample or cin != 4 * width:
            ds = nn.Sequential(_conv1x1(cin, 4 * width), _BN(4 * width))
        blk = Bottleneck(cin, width, 1, ds).cuda().to(memory_format=torch.channels_last)
        for m in blk.modules():
            if isinstance(m, nn.Conv2d):
                m.to(torch.bfloat16)
        with torch.no_grad():
            for m in blk.modules():
                if isinstance(m, nn.BatchNorm2d):
                    m.weight.uniform_(0.5, 1.5)
                    m.bias.normal_(0, 0.1)
        g = torch.Generator(device='cuda').manual_seed(2)
        x0 = torch.randn(8, cin, hw, hw, device='cuda', generator=g).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last).requires_grad_(True)
        x = x0 * 1                      # non-leaf block input, as inside the network
        y = blk(x)
        dy = torch.randn(y.shape, device='cuda', generator=g).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last)
        y.backward(dy)
        torch.cuda.synchronize()
        results.append(dict(y=y.detach().float(), dx=x0.grad.float(),
                            grads={n: p.grad.float() for n, p in blk.named_parameters()}))
    got, want = results
    for key in ('y', 'dx'):
        bad = (got[key] - want[key]).abs() > 5e-2 + 5e-2 * want[key].abs()
        assert bad.float().mean().item() < 2e-3, key
    # a ReLU mask that flips on a 1-ulp difference moves one channel's gamma gradient by a whole
    # term at these tiny batch sizes, so parameter gradients are compared in relative L2 norm
    for n in want['grads']:
        rel = (got['grads'][n] - want['grads'][n]).norm().item() / (want['grads'][n].norm().item() + 1e-6)
        assert rel < 3e-2, (n, rel)
