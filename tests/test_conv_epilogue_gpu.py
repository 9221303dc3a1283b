"""Epilogue of conv_tc_kernel: the batched epilogue and class-interleaved tile walk (default) against the previous epilogue and
walk (mode bit 26), bit for bit, across N tiles, epilogue operands, strides, the upsample-folded forward, shared inputs, row lengths
and a partial last tile; and the default against float64 torch at a production shape."""
import pytest
import torch

from ops_torch import TorchOps
from council_gan_b200.ops import ACT_NONE, ACT_RELU, ACT_LRELU

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
OLD = 7 | (1 << 26)  # every tensor-core path, previous conv_tc_kernel epilogue and tile walk
WIDE = 1 << 23       # widest N tile even where the launch has fewer tiles than SMs


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    o = CudaOps(DEV)
    yield o
    o.set_tensor_core_mode(1)


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def both(ops, fn, wide):
    """fn() under the default and under bit 26 (same N tile rule): (new, old)"""
    out = []
    try:
        for mode in ((7 | wide) if wide else 1, OLD | wide):
            ops.set_tensor_core_mode(mode)
            r = fn()
            torch.cuda.synchronize()
            out.append(r if isinstance(r, tuple) else (r,))
    finally:
        ops.set_tensor_core_mode(1)
    return out


def same(new, old, what):
    for i, (a, b) in enumerate(zip(new, old)):
        assert torch.equal(a, b), '%s output %d: max |diff| %.3e' % (what, i, (a - b).abs().max().item())


# (name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups): forward input H x W
FWD = [
    ('q16_bn64', 2, 2, 2, 16, 16, 64, 64, 3, 1, 1, False),
    ('q32_bn128', 2, 2, 2, 32, 32, 64, 128, 3, 1, 1, False),
    ('q64_bn256', 2, 2, 1, 64, 64, 32, 256, 3, 1, 1, False),
    ('q128_s2_bn128', 2, 2, 1, 256, 256, 32, 128, 4, 2, 1, False),
    ('q256_bn64', 1, 1, 1, 8, 256, 32, 64, 3, 1, 1, False),
    ('cout512_bn256', 2, 2, 2, 16, 16, 64, 512, 3, 1, 1, False),
    ('shared_input', 3, 1, 2, 32, 32, 64, 128, 3, 1, 1, False),
    ('ups_q32', 2, 2, 2, 16, 16, 128, 64, 3, 1, 1, True),
    ('ups_bn256', 2, 2, 1, 16, 16, 64, 256, 3, 1, 1, True),
    ('partial_tile', 2, 2, 1, 12, 12, 64, 128, 3, 1, 1, False),
    ('narrow_out_bn16', 2, 2, 2, 16, 16, 64, 12, 3, 1, 1, False),
]


@pytest.mark.parametrize('case', FWD, ids=[c[0] for c in FWD])
@pytest.mark.parametrize('wide', [0, WIDE], ids=['fill', 'wide'])
def test_fwd_bitwise(ops, case, wide):
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


# (name, G, B, H, W, Cin, Cout, K, stride, pad): forward input H x W, whose gradient is computed
DGRAD = [
    ('s1_q16_bn64', 2, 2, 16, 16, 64, 64, 3, 1, 1),
    ('s1_q32_bn128', 2, 2, 32, 32, 128, 64, 3, 1, 1),
    ('s1_q64_bn256', 2, 1, 64, 64, 256, 32, 3, 1, 1),
    ('s1_q128_bn256', 1, 1, 8, 128, 256, 64, 3, 1, 1),
    ('s2_q16_bn64', 2, 2, 32, 32, 64, 128, 4, 2, 1),
    ('s2_q32_bn128', 2, 2, 64, 64, 128, 256, 4, 2, 1),
    ('s2_q64_bn256', 2, 1, 128, 128, 256, 64, 4, 2, 1),
    ('s2_q256_bn64', 1, 1, 16, 512, 64, 64, 4, 2, 1),
    ('partial_tile', 2, 1, 12, 12, 128, 64, 3, 1, 1),
    ('narrow_in_bn16', 2, 2, 16, 16, 8, 64, 3, 1, 1),
]


@pytest.mark.parametrize('case', DGRAD, ids=[c[0] for c in DGRAD])
@pytest.mark.parametrize('wide', [0, WIDE], ids=['fill', 'wide'])
def test_dgrad_bitwise(ops, case, wide):
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


def test_production_shapes_vs_fp64(ops):
    """The generator's residual-addend data gradient (3x3 256->256, 64x64, council of 4, 8 images) and a discriminator's masked
    stride-2 data gradient and LeakyReLU+bias forward (4x4 s2 64->128, 128x128 in, council of 4, 8 images) against float64 torch,
    at the TF32 tolerance of tests/test_kernels_gpu.py."""
    ref = TorchOps(DEV, torch.float64)
    d = lambda t: None if t is None else t.double()

    def check(got, want, what):
        err = (got.double() - want).abs().max().item()
        mag = want.abs().max().item()
        assert err <= 4e-3 * mag, '%s: max err %.3e vs magnitude %.3e' % (what, err, mag)

    G, B = 4, 8
    xs = (G, B, 64, 64, 256)
    w = rnd(G, 256, 3, 3, 256, seed=2, scale=0.05)
    dy = rnd(G, B, 64, 64, 256, seed=4)
    add = rnd(*xs, seed=5)
    dx = ops.conv_dgrad(dy, w, xs, 1, 1, addend=add)
    check(dx, ref.conv_dgrad(d(dy), d(w), xs, 1, 1, addend=d(add)), 'residual dgrad + addend')
    del dy, add, dx
    xs = (G, B, 128, 128, 64)
    x = rnd(*xs, seed=1)
    w = rnd(G, 128, 4, 4, 64, seed=2, scale=0.05)
    b = rnd(G, 128, seed=3)
    y = ops.conv_fwd(x, w, b, 2, 1, act=ACT_LRELU, slope=0.2)
    check(y, ref.conv_fwd(d(x), d(w), d(b), 2, 1, act=ACT_LRELU, slope=0.2), 'discriminator forward + bias + LeakyReLU')
    dy = rnd(*y.shape, seed=4)
    dx = ops.conv_dgrad(dy, w, xs, 2, 1, mask_src=x, mask_slope=0.2)
    check(dx, ref.conv_dgrad(d(dy), d(w), xs, 2, 1, mask_src=d(x), mask_slope=0.2), 'discriminator masked dgrad')
