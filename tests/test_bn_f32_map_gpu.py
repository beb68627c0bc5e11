"""fp32 BatchNorm kernels: the split channel map (a thread owns channels [4cv, 4cv+4) and
[C/2+4cv, C/2+4cv+4)) against the consecutive map (8 consecutive channels per thread).  A
channel's rows and their order are the same under both maps, so every output -- y, the ReLU
mask, the statistics and reduction partials, running statistics, dx, dz, grad gamma and grad
beta -- must be bit-identical.  Plus the split map's composition against fp64."""
import pytest
import torch
import torch.nn.functional as F

from stochastic_gradient_push_b200.ops import native
from stochastic_gradient_push_b200.ops.fused_bn import bn_f32_map, fused_bn_act

pytestmark = pytest.mark.gpu

CHANNELS = (24, 64, 256, 2048)


def rows_per_cta(C):
    return 256 // (C // 8)


def row_counts(C):
    """an M that is a multiple of the rows per CTA, one that is not (C = 2048 has one row per
    CTA, so there it is not a multiple of the grid's row stride instead), and one large enough
    for the largest grid to loop"""
    rpi = rows_per_cta(C)
    n = max(4096 // (C // 8 * rpi), 3) * rpi * 7
    return (n, n + 5 if rpi > 1 else n * 4 + 5, rpi * 132 * 16 * 3 + 3)


@pytest.fixture(scope='module')
def C_ext():
    if not torch.cuda.is_available() or not native.available():
        pytest.skip('needs the sm_90a extension and a GPU')
    return native.load()


def inputs(M, C, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    mk = lambda: torch.randn(M, C, device='cuda', generator=g)        # noqa: E731
    x = mk() * 2 + 0.5
    coef = torch.stack([x.mean(0), x.var(0).add(1e-5).rsqrt(),
                        torch.rand(C, device='cuda', generator=g) + 0.5,
                        torch.randn(C, device='cuda', generator=g) * 0.5]).contiguous()
    c23 = (torch.randn(2, C, device='cuda', generator=g) * 0.1).contiguous()
    return x, mk(), mk(), coef, c23


def both_maps(fn):
    outs = []
    for split in (False, True):
        with bn_f32_map(split):
            outs.append(fn())
    torch.cuda.synchronize()
    return outs


def assert_bitwise(a, b, what):
    if isinstance(a, (list, tuple)):
        for i, (u, v) in enumerate(zip(a, b)):
            assert_bitwise(u, v, '%s[%d]' % (what, i))
        return
    if a is None:
        return
    assert a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride(), what
    if a.dtype == torch.float32:        # bit patterns: tells -0.0 from 0.0 and compares NaNs
        a, b = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    assert torch.equal(a, b), what


def test_switch_round_trip(C_ext):
    cur = C_ext.bn_f32_map()
    with bn_f32_map(False):
        assert C_ext.bn_f32_map() == 0
        with bn_f32_map(True):
            assert C_ext.bn_f32_map() == 1
        assert C_ext.bn_f32_map() == 0
    assert C_ext.bn_f32_map() == cur


@pytest.mark.parametrize('C', CHANNELS)
def test_stats_partials_bitwise(C_ext, C):
    for M in row_counts(C):
        x = inputs(M, C, 1)[0]
        a, b = both_maps(lambda: C_ext.bn_kernel_stats(x))
        # rows [0, G): (sum, sum of squares) per CTA; row G: the shift K in [G][0] ([G][1] is not written)
        assert_bitwise(a[:-1], b[:-1], 'stats partial M=%d' % M)
        assert_bitwise(a[-1, 0], b[-1, 0], 'stats shift row M=%d' % M)


@pytest.mark.parametrize('C', CHANNELS)
@pytest.mark.parametrize('variant', ['plain', 'relu', 'add', 'add+relu', 'add+relu+mask'])
def test_apply_bitwise(C_ext, C, variant):
    if variant == 'add+relu+mask' and C % 16:
        pytest.skip('the mask needs C % 16 == 0 (test_mask_refuses_odd_pairs)')
    for M in row_counts(C):
        x, r, _, coef, _ = inputs(M, C, 2)
        add, relu = 'add' in variant, 'relu' in variant
        masks = []

        def run():
            mask = torch.full((M, C // 8), 0xA5, dtype=torch.uint8, device='cuda') if 'mask' in variant else None
            masks.append(mask)
            return C_ext.bn_kernel_apply(x, r if add else None, coef, relu, mask)
        a, b = both_maps(run)
        assert_bitwise(a, b, 'y M=%d' % M)
        if masks[0] is not None:
            assert_bitwise(masks[0], masks[1], 'mask M=%d' % M)
            bits = ((a > 0).view(M, C // 8, 8).long() << torch.arange(8, device='cuda')).sum(-1)
            assert torch.equal(masks[1].long(), bits), 'mask bit i of byte j is channel 8j+i'


def test_mask_refuses_odd_pairs(C_ext):
    M, C = 850, 24                      # C / 8 = 3 lanes per row: no lane pairs
    x, r, _, coef, _ = inputs(M, C, 3)
    mask = torch.empty(M, C // 8, dtype=torch.uint8, device='cuda')
    with bn_f32_map(True), pytest.raises(RuntimeError):
        C_ext.bn_kernel_apply(x, r, coef, True, mask)
    with bn_f32_map(False):
        C_ext.bn_kernel_apply(x, r, coef, True, mask)
    torch.cuda.synchronize()


@pytest.mark.parametrize('C', CHANNELS)
@pytest.mark.parametrize('mode', [0, 1, 2])
def test_reduce_bitwise(C_ext, C, mode):
    for M in row_counts(C):
        x, dy, y, coef, _ = inputs(M, C, 4)
        a, b = both_maps(lambda: C_ext.bn_kernel_reduce(mode, dy, x, y if mode == 2 else None, coef))
        assert_bitwise(a[0], b[0], 'reduce partial M=%d' % M)
        if mode == 2:
            assert_bitwise(a[1], b[1], 'dz M=%d' % M)


@pytest.mark.parametrize('C', CHANNELS)
@pytest.mark.parametrize('mode', [0, 1])
def test_dx_bitwise(C_ext, C, mode):
    for M in row_counts(C):
        x, dz, _, coef, c23 = inputs(M, C, 5)
        a, b = both_maps(lambda: C_ext.bn_kernel_dx(mode, dz, x, coef, c23))
        assert_bitwise(a, b, 'dx M=%d' % M)


def _layer(M, C, seed, residual, relu, dtype=torch.float32):
    g = torch.Generator(device='cuda').manual_seed(seed)
    N, H = M // 5, 5
    x = (torch.randn(N, C, H, 1, device='cuda', generator=g) * 3 + 1).to(dtype)
    x = x.contiguous(memory_format=torch.channels_last)
    res = torch.randn_like(x).contiguous(memory_format=torch.channels_last) if residual else None
    w = (torch.rand(C, device='cuda', generator=g) + 0.5).to(dtype)
    b = (torch.randn(C, device='cuda', generator=g) * 0.2).to(dtype)
    dy = torch.randn_like(x).contiguous(memory_format=torch.channels_last)
    return x, res, w, b, dy


def _fused_step(x, res, w, b, dy, relu, ref=False):
    x = x.clone().requires_grad_(True)
    res = res.clone().requires_grad_(True) if res is not None else None
    w = w.clone().requires_grad_(True)
    b = b.clone().requires_grad_(True)
    C = x.shape[1]
    rm = torch.zeros(C, device='cuda', dtype=x.dtype)
    rv = torch.ones(C, device='cuda', dtype=x.dtype)
    nbt = torch.zeros((), dtype=torch.long, device='cuda')
    if ref:
        y = F.batch_norm(x, rm, rv, w, b, True, 0.1, 1e-5)
        y = y + res if res is not None else y
        y = F.relu(y) if relu else y
    else:
        y = fused_bn_act(x, w, b, rm, rv, nbt, residual=res, relu=relu)
    grads = torch.autograd.grad(y, [t for t in (x, res, w, b) if t is not None], dy)
    return [y.detach(), rm, rv] + list(grads)


@pytest.mark.parametrize('C', CHANNELS)
@pytest.mark.parametrize('residual,relu', [(False, False), (False, True), (True, True)])
def test_layer_bitwise(C_ext, C, residual, relu):
    """forward + backward through fused_bn_act: y, running stats, dx, dz, grad gamma, grad beta"""
    M = 5 * rows_per_cta(C) * 41
    args = _layer(M, C, 6, residual, relu)
    a, b = both_maps(lambda: _fused_step(*args, relu))
    assert_bitwise(a, b, 'layer C=%d' % C)


@pytest.mark.parametrize('C', CHANNELS)
@pytest.mark.parametrize('residual,relu', [(False, True), (True, True)])
def test_split_map_matches_fp64(C_ext, C, residual, relu):
    M = 5 * rows_per_cta(C) * 41
    args = _layer(M, C, 7, residual, relu)
    with bn_f32_map(True):
        got = _fused_step(*args, relu)
    ref = _fused_step(*[t.double() if t is not None else None for t in args], relu, ref=True)
    names = ['y', 'running_mean', 'running_var', 'dx'] + (['dz'] if residual else []) + ['grad_gamma', 'grad_beta']
    for name, u, v in zip(names, got, ref):
        # ReLU boundary flips between an fp32 and an fp64 pre-activation are rare; compare elementwise
        # with a relative tolerance and allow a vanishing fraction of flipped elements
        # (a flip moves a per-channel sum: at most one channel may miss)
        err = (u.double() - v).abs()
        tol = 1e-4 * (v.abs() + v.abs().mean() + 1e-6)
        nbad = int((err > tol).sum().item())
        assert nbad <= (u.numel() // 10000 if u.numel() > C else 1), (name, nbad, err.max().item())
