"""Weight gradient of stride-1 KxK convolutions on the TMA-fed kernel (wgrad_tma_kernel) against float64 torch, against the
previous tensor-core kernel (mode bit 25: bit-identical where a 32-pixel chunk is one row segment, Wo % 32 == 0), run-to-run
determinism and the workspace size it reports."""
import ctypes as C

import pytest
import torch

from ops_torch import TorchOps

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
OLD_WGRAD = 7 | (1 << 25)  # every tensor-core path, stride-1 weight gradients on wgrad_tc_kernel
TOL = 4e-3                  # TF32 operands, fp32 accumulation: relative to the magnitude of the result


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    o = CudaOps(DEV)
    yield o
    o.set_tensor_core_mode(1)


@pytest.fixture(scope='module')
def ref():
    return TorchOps(DEV, torch.float64)


def rnd(*shape, seed=0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV)


# (name, G, Gx, B, H, W, Cin, Cout, K, pad)
CASES = [
    ('c256_o256_32x32', 2, 2, 2, 32, 32, 256, 256, 3, 1),
    ('c256_o128', 2, 2, 2, 32, 32, 256, 128, 3, 1),
    ('c128_o256', 2, 2, 2, 32, 32, 128, 256, 3, 1),
    ('c64_o64_shared_input', 3, 1, 2, 32, 32, 64, 64, 3, 1),
    ('w48_odd_h', 2, 2, 2, 17, 48, 128, 128, 3, 1),
    ('w40_odd_h', 2, 2, 1, 13, 40, 128, 64, 3, 1),
    ('pad0_valid', 2, 2, 2, 34, 50, 64, 128, 3, 0),
    ('k5_pad2', 2, 2, 2, 32, 32, 64, 64, 5, 2),
    ('c96_o160_partial_tiles', 2, 2, 2, 32, 32, 96, 160, 3, 1),
    ('many_splits_g1_b8_64x64', 1, 1, 8, 64, 64, 128, 128, 3, 1),
]


def wgrad(ops, x, dy, G, Cout, K, Cin, pad):
    dw = torch.full((G, Cout, K, K, Cin), float('nan'), device=DEV)  # every element must be written
    ops.conv_wgrad(x, dy, dw, None, 1, pad)
    return dw


def check(got, want, what):
    err = (got.double() - want).abs().max().item()
    mag = want.abs().max().item() + 1e-30
    assert err <= TOL * mag, '%s: max err %.3e vs magnitude %.3e' % (what, err, mag)


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_wgrad_tma_vs_fp64(ops, ref, case):
    name, G, Gx, B, H, W, Cin, Cout, K, pad = case
    Ho, Wo = H + 2 * pad - K + 1, W + 2 * pad - K + 1
    x = rnd(Gx, B, H, W, Cin, seed=1)
    dy = rnd(G, B, Ho, Wo, Cout, seed=2)
    want = torch.zeros(G, Cout, K, K, Cin, dtype=torch.float64, device=DEV)
    ref.conv_wgrad(x.double(), dy.double(), want, None, 1, pad)
    results = {}
    for mode in (1, OLD_WGRAD):
        ops.set_tensor_core_mode(mode)
        try:
            n0 = ops.launch_count()
            dw = wgrad(ops, x, dy, G, Cout, K, Cin, pad)
            torch.cuda.synchronize()
            results[mode] = (dw, ops.launch_count() - n0)
        finally:
            ops.set_tensor_core_mode(1)
        check(dw, want, '%s mode %#x' % (name, mode))
    # the new path launches a transpose before the GEMM: a different launch count proves bit 25 selects another kernel
    assert results[1][1] != results[OLD_WGRAD][1], (name, results[1][1], results[OLD_WGRAD][1])
    if Wo % 32 == 0:  # same operands, splits and k-step order as wgrad_tc_kernel
        assert torch.equal(results[1][0], results[OLD_WGRAD][0]), '%s: differs from wgrad_tc_kernel' % name


def test_wgrad_tma_production_shape(ops, ref):
    """The 3x3 256->256 residual convolutions of the 256x256 configuration: council of 4, batch 8, 64x64 maps, per member."""
    G, B, H, W, C = 4, 8, 64, 64, 256
    x = rnd(G, B, H, W, C, seed=3)
    dy = rnd(G, B, H, W, C, seed=4)
    dw = wgrad(ops, x, dy, G, C, 3, C, 1)
    ops.set_tensor_core_mode(OLD_WGRAD)
    try:
        old = wgrad(ops, x, dy, G, C, 3, C, 1)
    finally:
        ops.set_tensor_core_mode(1)
    assert torch.equal(dw, old), 'production shape: differs from wgrad_tc_kernel'
    for g in range(G):
        want = torch.zeros(1, C, 3, 3, C, dtype=torch.float64, device=DEV)
        ref.conv_wgrad(x[g:g + 1].double(), dy[g:g + 1].double(), want, None, 1, 1)
        check(dw[g:g + 1], want, 'member %d' % g)


def test_wgrad_tma_deterministic(ops):
    G, B, H, W, C = 2, 8, 64, 64, 128
    x = rnd(G, B, H, W, C, seed=5)
    dy = rnd(G, B, H, W, C, seed=6)
    a = wgrad(ops, x, dy, G, C, 3, C, 1)
    b = wgrad(ops, x, dy, G, C, 3, C, 1)
    assert torch.equal(a, b), 'weight gradient must be run-to-run deterministic'


def test_wgrad_tma_workspace(ops):
    from council_gan_b200.ops import ConvGeom
    G, B, H, W, Cin, Cout = 2, 2, 32, 32, 256, 128
    x = rnd(G, B, H, W, Cin, seed=7)
    dy = rnd(G, B, H, W, Cout, seed=8)
    dw = torch.empty(G, Cout, 3, 3, Cin, device=DEV)
    g = ConvGeom(G, G, B, H, W, Cin, H, W, Cout, 3, 3, 1, 1, 0)
    need = int(ops.lib.cg_conv_workspace_bytes(C.byref(g), 2))
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream

    def call(nbytes):
        return ops.lib.cg_conv_wgrad(C.byref(g), x.data_ptr(), dy.data_ptr(), dw.data_ptr(), None, ws.data_ptr(), nbytes, stream)

    assert call(need - 1) == -2  # CG_ERR_WORKSPACE
    assert call(need) == 0, ops.lib.cg_last_error().decode()
    torch.cuda.synchronize()
    want = torch.zeros(G, Cout, 3, 3, Cin, dtype=torch.float64, device=DEV)
    TorchOps(DEV, torch.float64).conv_wgrad(x.double(), dy.double(), want, None, 1, 1)
    check(dw, want, 'direct call')
