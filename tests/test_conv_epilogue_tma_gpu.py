"""Shared-memory epilogue of conv_tc_kernel (TMA-loaded addend and mask, TMA-stored results; the default where the tile geometry
allows it) against the register epilogue (mode bit 27), bit for bit: over the case lists of test_conv_epilogue_gpu.py, at row
lengths 16 to 256, through both stride-2 data-gradient classes and the upsample-folded forward, at geometries that must fall back
to the register epilogue, and at the production shapes of the 256x256 configuration."""
import pytest
import torch

from council_gan_b200.ops import ACT_NONE, ACT_RELU, ACT_LRELU
from test_conv_epilogue_gpu import FWD, DGRAD, WIDE, rnd

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
REG = 1 << 27  # every conv_tc_kernel launch on the register epilogue


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    o = CudaOps(DEV)
    yield o
    o.set_tensor_core_mode(1)


def both(ops, fn, wide=0):
    """fn() under the default and under bit 27 (same N tile rule): (default, register epilogue)"""
    out = []
    try:
        for mode in ((7 | wide) if wide else 1, 7 | wide | REG):
            ops.set_tensor_core_mode(mode)
            r = fn()
            torch.cuda.synchronize()
            out.append(tuple(t.clone() for t in (r if isinstance(r, tuple) else (r,))))
    finally:
        ops.set_tensor_core_mode(1)
    return out


def same(new, old, what):
    for i, (a, b) in enumerate(zip(new, old)):
        assert torch.equal(a, b), '%s output %d: max |diff| %.3e' % (what, i, (a - b).abs().max().item())


# (name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups) as FWD: row lengths Q 16..256 and the fall-back geometry Q = 12
FWD_Q = [
    ('q16_bn128', 2, 2, 1, 16, 16, 32, 128, 3, 1, 1, False),
    ('q32_bn64', 2, 2, 1, 32, 32, 32, 64, 3, 1, 1, False),
    ('q64_bn128', 1, 1, 1, 64, 64, 64, 128, 3, 1, 1, False),
    ('q128_bn256', 1, 1, 1, 8, 128, 32, 256, 3, 1, 1, False),
    ('q256_1x1_bn64', 1, 1, 1, 4, 256, 32, 64, 1, 1, 0, False),
    ('q128_s2_bn256', 1, 1, 1, 64, 256, 64, 256, 4, 2, 1, False),
    ('ups_q64_bn128', 2, 2, 1, 64, 64, 64, 128, 3, 1, 1, True),
    ('ups_q16_bn256', 1, 1, 2, 16, 16, 32, 256, 3, 1, 1, True),
    ('q12_fallback', 2, 2, 2, 12, 12, 64, 64, 3, 1, 1, False),
]


@pytest.mark.parametrize('case', FWD + FWD_Q, ids=[c[0] for c in FWD + FWD_Q])
@pytest.mark.parametrize('wide', [0, WIDE], ids=['fill', 'wide'])
def test_fwd_vs_register_epilogue(ops, case, wide):
    name, G, Gx, B, H, W, Cin, Cout, K, s, pad, ups = case
    x = rnd(Gx, B, H, W, Cin, seed=1)
    w = rnd(G, Cout, K, K, Cin, seed=2, scale=0.1)
    b = rnd(G, Cout, seed=3)
    for act in (ACT_NONE, ACT_RELU, ACT_LRELU):
        for bias in (b, None):
            new, old = both(ops, lambda: ops.conv_fwd(x, w, bias, s, pad, ups=ups, act=act, slope=0.2), wide)
            same(new, old, '%s act%d bias=%s' % (name, act, bias is not None))
    if Cout >= 32:
        new, old = both(ops, lambda: ops.conv_fwd_stats(x, w, s, pad, ups=ups), wide)
        same(new, old, name + ' stats')


# (name, G, B, H, W, Cin, Cout, K, stride, pad) as DGRAD: row lengths 16..256 of both strides and the fall-back Q = 12
DGRAD_Q = [
    ('s1_q256_bn64', 1, 1, 4, 256, 64, 64, 3, 1, 1),
    ('s1_q64_bn128', 1, 2, 64, 64, 128, 32, 3, 1, 1),
    ('s2_q128_bn128', 1, 1, 16, 256, 128, 64, 4, 2, 1),
    ('s2_q16_bn256', 1, 2, 32, 32, 256, 64, 4, 2, 1),
    ('s2_q12_fallback', 1, 2, 24, 24, 64, 64, 4, 2, 1),
    ('s1_q12_fallback', 2, 1, 12, 12, 64, 64, 3, 1, 1),
]


@pytest.mark.parametrize('case', DGRAD + DGRAD_Q, ids=[c[0] for c in DGRAD + DGRAD_Q])
@pytest.mark.parametrize('wide', [0, WIDE], ids=['fill', 'wide'])
def test_dgrad_vs_register_epilogue(ops, case, wide):
    name, G, B, H, W, Cin, Cout, K, s, pad = case
    Ho, Wo = (H + 2 * pad - K) // s + 1, (W + 2 * pad - K) // s + 1
    xs = (G, B, H, W, Cin)
    w = rnd(G, Cout, K, K, Cin, seed=2, scale=0.1)
    dy = rnd(G, B, Ho, Wo, Cout, seed=4)
    add = rnd(*xs, seed=5)
    msk = rnd(*xs, seed=6)
    for addend, mask, slope in ((None, None, 0.0), (add, None, 0.0), (None, msk, 0.0), (None, msk, 0.2), (add, msk, 0.2)):
        new, old = both(ops, lambda: ops.conv_dgrad(dy, w, xs, s, pad, addend=addend, mask_src=mask, mask_slope=slope), wide)
        same(new, old, '%s addend=%s mask=%s slope %.1f' % (name, addend is not None, mask is not None, slope))


def test_production_shapes_vs_register_epilogue(ops):
    """The generator's residual layer (3x3 256->256 at 64x64: statistics forward, addend data gradient) and a council
    discriminator layer (4x4 s2 64->128 at 128x128 in: bias + LeakyReLU forward, masked data gradient), council of 4, 8 images."""
    G, B = 4, 8
    xs = (G, B, 64, 64, 256)
    x = rnd(*xs, seed=1)
    w = rnd(G, 256, 3, 3, 256, seed=2, scale=0.05)
    new, old = both(ops, lambda: ops.conv_fwd_stats(x, w, 1, 1))
    same(new, old, 'residual forward + statistics')
    dy = rnd(G, B, 64, 64, 256, seed=4)
    new, old = both(ops, lambda: ops.conv_dgrad(dy, w, xs, 1, 1, addend=x))
    same(new, old, 'residual dgrad + addend')
    del x, w, dy, new, old
    xs = (G, B, 128, 128, 64)
    x = rnd(*xs, seed=1)
    w = rnd(G, 128, 4, 4, 64, seed=2, scale=0.05)
    b = rnd(G, 128, seed=3)
    new, old = both(ops, lambda: ops.conv_fwd(x, w, b, 2, 1, act=ACT_LRELU, slope=0.2))
    same(new, old, 'discriminator forward + bias + LeakyReLU')
    dy = rnd(*new[0].shape, seed=4)
    new, old = both(ops, lambda: ops.conv_dgrad(dy, w, xs, 2, 1, mask_src=x, mask_slope=0.2))
    same(new, old, 'discriminator masked dgrad')
