"""Host-side launch planning of the wgmma 1x1-conv GEMM (csrc/conv1x1_kernels.cu): tile
width, persistent grid, shared-memory budget.  Pure host logic -- runs without a GPU."""
import itertools

import pytest

from stochastic_gradient_push_b200.ops import native

SMEM_LIMIT = 227 * 1024
A_BYTES = 128 * 64 * 2
SLAB = 2048                 # one warp's store slab: 16 rows x 128 B

RESNET50_SHAPES = [  # (M, N, K) at batch 256
    (802816, 64, 64), (802816, 256, 64), (802816, 64, 256), (802816, 128, 256),
    (200704, 512, 128), (200704, 128, 512), (200704, 256, 512),
    (50176, 1024, 256), (50176, 256, 1024), (50176, 512, 1024),
    (12544, 2048, 512), (12544, 512, 2048),
]


@pytest.fixture(scope='module')
def C():
    try:
        return native.load()
    except Exception as e:      # no compiler on this host
        pytest.skip('native extension unavailable: %s' % e)


def _check(C, M, N, K, sms, residual, f32=False):
    p = C.conv1x1_plan(M, N, K, sms, residual, f32)
    bn = p['block_n']
    assert bn in (64, 128, 256) and N % bn == 0
    n_blocks = N // bn
    m_tiles = -(-M // 128)
    assert p['grid'] == n_blocks * p['ctas_per_n']
    assert 1 <= p['ctas_per_n'] <= m_tiles              # every CTA owns at least one row tile
    assert p['grid'] <= max(sms, n_blocks)              # one persistent CTA per SM
    assert p['partial_rows'] == p['ctas_per_n']         # one merged statistics row per CTA
    assert 2 <= p['stages'] <= 8
    assert p['store_slabs'] in (1, 2)
    if residual:
        assert p['store_slabs'] == 2                    # residual slabs are double-buffered
    k_blocks = -(-K // (32 if f32 else 64))     # a k-block is one 128-byte swizzle row
    b_bytes = bn * 128
    stage = A_BYTES + (0 if p['resident_w'] else b_bytes)
    want = 1024 + 512 + (k_blocks * b_bytes if p['resident_w'] else 0) + p['stages'] * stage \
        + 8 * p['store_slabs'] * SLAB
    assert p['smem_bytes'] == want <= SMEM_LIMIT
    if p['resident_w']:
        assert p['stages'] >= 3
    return p


@pytest.mark.parametrize('residual', [False, True])
def test_resnet50_layer_plans(C, residual):
    for M, N, K in RESNET50_SHAPES:
        p = _check(C, M, N, K, 132, residual)
        assert p['grid'] >= 128, (M, N, K, p)           # (almost) every SM busy at batch 256
    # the HBM-bound layers keep W resident and stream X through a deep ring
    p = C.conv1x1_plan(802816, 256, 64, 132, residual)
    assert p['resident_w'] and p['stages'] == 8 and p['block_n'] == 256
    # K = 2048 cannot be resident; a narrower tile shortens the critical path on the 7x7 maps
    p = C.conv1x1_plan(12544, 512, 2048, 132, residual)
    assert not p['resident_w'] and p['block_n'] == 128


def test_fp32_plans(C):
    """fp32 / TF32 operands: k-blocks of 32 elements; the tile width is narrowed until the CTA's W
    block stays resident when that is possible (fp32 W is twice as wide)."""
    for M, N, K in RESNET50_SHAPES:
        for residual in (False, True):
            p = _check(C, M, N, K, 132, residual, f32=True)
            assert p['grid'] >= 128, (M, N, K, p)
    p = C.conv1x1_plan(802816, 256, 64, 132, False, True)
    assert p['resident_w'] and p['block_n'] == 256          # 64 KB of W
    p = C.conv1x1_plan(50176, 1024, 256, 132, False, True)
    assert p['resident_w'] and p['block_n'] == 128          # 256-wide would be 256 KB
    for M, N, K, sms, res in itertools.product((1, 129, 5000), (64, 192, 1024), (8, 36, 100, 1000),
                                               (132, 148), (False, True)):
        _check(C, M, N, K, sms, res, f32=True)
    with pytest.raises(RuntimeError):
        C.conv1x1_plan(128, 64, 10, 132, False, True)        # 40-byte rows


def test_plan_invariants_over_a_shape_sweep(C):
    for M, N, K, sms, res in itertools.product(
            (1, 127, 128, 129, 5000, 100000), (64, 128, 192, 256, 320, 1024, 4096),
            (8, 64, 72, 256, 1000, 4096), (4, 132, 148, 160), (False, True)):
        _check(C, M, N, K, sms, res)


def test_unsupported_shapes_are_rejected(C):
    for M, N, K in ((128, 48, 64), (128, 64, 12), (0, 64, 64), (2 ** 31, 64, 64)):
        with pytest.raises(RuntimeError):
            C.conv1x1_plan(M, N, K)
