"""Host-side launch plans of the MODE 3 GEMM (conv1 dgrad + skip gradient + the previous block's
BatchNorm backward reduction, csrc/conv1x1_kernels.cu).  Pure host logic -- runs without a GPU."""
import pytest

from stochastic_gradient_push_b200.ops import native

SMEM_LIMIT = 227 * 1024
A_BYTES = 128 * 64 * 2
SLAB = 2048

# ResNet-50 conv1 dgrad at batch 256: dX[M, Cin] = dY1[M, width] . W1  ->  (M, N = Cin, K = width)
CONV1_DGRAD_SHAPES = [
    (802816, 256, 64),                          # layer1
    (802816, 256, 128), (200704, 512, 128),     # layer2 (block 0 reads layer1's 56x56 output)
    (200704, 512, 256), (50176, 1024, 256),     # layer3
    (50176, 1024, 512), (12544, 2048, 512),     # layer4
]


@pytest.fixture(scope='module')
def C():
    try:
        return native.load()
    except Exception as e:      # no compiler on this host
        pytest.skip('native extension unavailable: %s' % e)


@pytest.mark.parametrize('f32', [False, True])
def test_bn_reduce_plans_fit(C, f32):
    for M, N, K in CONV1_DGRAD_SHAPES:
        p = C.conv1x1_plan(M, N, K, 132, True, f32, bn_reduce=True)
        bn = p['block_n']
        assert bn in (64, 128) and N % bn == 0, (M, N, K, p)       # no 256-wide MODE 3 instantiation
        assert p['store_slabs'] == 2 and 2 <= p['stages'] <= 8, (M, N, K, p)
        k_blocks = -(-K // (32 if f32 else 64))
        stage = A_BYTES + (0 if p['resident_w'] else bn * 128)
        want = 1024 + 512 + (k_blocks * bn * 128 if p['resident_w'] else 0) + p['stages'] * stage \
            + 8 * 2 * SLAB + 8 * 2 * SLAB                               # store slabs + bn_x slabs
        assert p['smem_bytes'] == want <= SMEM_LIMIT, (M, N, K, p)
        assert p['partial_rows'] == p['ctas_per_n']
        assert p['grid'] >= 128, (M, N, K, p)


def test_bn_reduce_plan_sweep(C):
    for M in (1, 129, 5000, 100000):
        for N in (64, 192, 256, 1024, 2048):
            for K in (8, 64, 256, 1000, 2048):
                for f32 in (False, True):
                    p = C.conv1x1_plan(M, N, K, 132, True, f32, bn_reduce=True)
                    assert p['block_n'] <= 128 and p['stages'] >= 2 and p['smem_bytes'] <= SMEM_LIMIT
