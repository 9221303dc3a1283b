"""Weight gradient on the TMA-fed kernel (wgrad_tma_kernel) for stride-2 layers, read through the parity view of x, and for maps
narrower than 32 pixels, whose 32-pixel chunks are several whole rows.  Same checks as test_wgrad_tma_gpu.py: float64 torch,
bitwise equality with the previous tensor-core kernel (mode bit 25) wherever a chunk is 32 consecutive pixels, the routing bit,
and the workspace size."""
import ctypes as C

import pytest
import torch

from test_wgrad_tma_gpu import DEV, OLD_WGRAD, check, ops, ref, rnd  # noqa: F401  (ops, ref: fixtures)

pytestmark = pytest.mark.gpu

# (name, G, Gx, B, H, W, Cin, Cout, K, stride, pad)
CASES = [
    ('s2_c64_o128', 2, 2, 2, 64, 64, 64, 128, 4, 2, 1),
    ('s2_c128_o256', 2, 2, 2, 64, 64, 128, 256, 4, 2, 1),
    ('s2_c256_o512_wo16_shared_input', 2, 1, 2, 32, 32, 256, 512, 4, 2, 1),
    ('s2_c128_o256_wo8_shared_input', 3, 1, 4, 16, 16, 128, 256, 4, 2, 1),
    ('s2_c96_o160_partial_tiles', 2, 2, 2, 64, 64, 96, 160, 4, 2, 1),
    ('s2_c96_o160_wo16_partial_tiles', 2, 2, 2, 32, 32, 96, 160, 4, 2, 1),
    ('s2_c64_o96_partial_n_tile', 2, 2, 2, 64, 64, 64, 96, 4, 2, 1),
    ('s2_k3_pad1', 2, 2, 2, 64, 64, 64, 64, 3, 2, 1),
    ('s2_wo48_partial_chunks_odd_ho', 2, 2, 2, 34, 96, 64, 128, 4, 2, 1),
    ('s1_wo16', 2, 2, 4, 16, 16, 128, 128, 3, 1, 1),
    ('s1_wo8_k5_pad2', 2, 2, 8, 8, 8, 64, 64, 5, 1, 2),
]


def out_size(n, K, stride, pad):
    return (n + 2 * pad - K) // stride + 1


def whole_chunks(Ho, Wo):
    """a 32-pixel chunk is 32 consecutive pixels of dy: one row segment, or 32 / Wo whole rows"""
    return Wo % 32 == 0 or (Wo < 32 and 32 % Wo == 0 and Ho * Wo % 32 == 0)


def wgrad(ops, x, dy, G, Cout, K, Cin, stride, pad):
    dw = torch.full((G, Cout, K, K, Cin), float('nan'), device=DEV)  # every element must be written
    ops.conv_wgrad(x, dy, dw, None, stride, pad)
    return dw


def both_modes(ops, x, dy, G, Cout, K, Cin, stride, pad):
    """{mode: (dw, launches)} for the default kernel selection and with bit 25"""
    results = {}
    for mode in (1, OLD_WGRAD):
        ops.set_tensor_core_mode(mode)
        try:
            n0 = ops.launch_count()
            dw = wgrad(ops, x, dy, G, Cout, K, Cin, stride, pad)
            torch.cuda.synchronize()
            results[mode] = (dw, ops.launch_count() - n0)
        finally:
            ops.set_tensor_core_mode(1)
    return results


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_wgrad_tma_stride2_vs_fp64(ops, ref, case):
    name, G, Gx, B, H, W, Cin, Cout, K, stride, pad = case
    Ho, Wo = out_size(H, K, stride, pad), out_size(W, K, stride, pad)
    x = rnd(Gx, B, H, W, Cin, seed=1)
    dy = rnd(G, B, Ho, Wo, Cout, seed=2)
    want = torch.zeros(G, Cout, K, K, Cin, dtype=torch.float64, device=DEV)
    ref.conv_wgrad(x.double(), dy.double(), want, None, stride, pad)
    results = both_modes(ops, x, dy, G, Cout, K, Cin, stride, pad)
    for mode, (dw, _) in results.items():
        check(dw, want, '%s mode %#x' % (name, mode))
    # the new path launches a transpose before the GEMM: a different launch count proves bit 25 selects another kernel
    assert results[1][1] != results[OLD_WGRAD][1], (name, results[1][1], results[OLD_WGRAD][1])
    if whole_chunks(Ho, Wo):  # same operands, splits and k-step order as wgrad_tc_kernel
        assert torch.equal(results[1][0], results[OLD_WGRAD][0]), '%s: differs from wgrad_tc_kernel' % name


@pytest.mark.parametrize('H,W', [(33, 64), (64, 33)], ids=['odd_h', 'odd_w'])
def test_wgrad_stride2_odd_size_stays_on_old_kernel(ops, ref, H, W):
    """the parity view needs even H and W: such layers keep wgrad_tc_kernel in both modes"""
    G, B, Cin, Cout, K, stride, pad = 2, 2, 64, 128, 4, 2, 1
    Ho, Wo = out_size(H, K, stride, pad), out_size(W, K, stride, pad)
    x = rnd(G, B, H, W, Cin, seed=3)
    dy = rnd(G, B, Ho, Wo, Cout, seed=4)
    want = torch.zeros(G, Cout, K, K, Cin, dtype=torch.float64, device=DEV)
    ref.conv_wgrad(x.double(), dy.double(), want, None, stride, pad)
    results = both_modes(ops, x, dy, G, Cout, K, Cin, stride, pad)
    check(results[1][0], want, 'odd size %dx%d' % (H, W))
    assert results[1][1] == results[OLD_WGRAD][1], (results[1][1], results[OLD_WGRAD][1])
    assert torch.equal(results[1][0], results[OLD_WGRAD][0])


def test_wgrad_tma_council_dis_production_shape(ops):
    """The largest stride-2 weight gradient of the 256x256 configuration: the council discriminator's 4x4 64->128 layer on
    256x256 inputs, council of 4, 40 images per member (real, own fake and the peers' fakes of a batch of 8)."""
    G, B, H, W, Cin, Cout = 4, 40, 256, 256, 64, 128
    Ho, Wo = H // 2, W // 2
    x = rnd(G, B, H, W, Cin, seed=5)
    dy = rnd(G, B, Ho, Wo, Cout, seed=6)
    results = both_modes(ops, x, dy, G, Cout, 4, Cin, 2, 1)
    assert results[1][1] != results[OLD_WGRAD][1]
    assert torch.equal(results[1][0], results[OLD_WGRAD][0]), 'production shape: differs from wgrad_tc_kernel'
    # the workspace holds the channel-major copy of dy
    assert ops._ws.numel() >= G * B * Ho * Wo * Cout * 4, ops._ws.numel()


@pytest.mark.parametrize('H', [32, 64], ids=['wo16_whole_rows', 'wo32'])
def test_wgrad_tma_stride2_workspace(ops, H):
    from council_gan_b200.ops import ConvGeom
    G, B, Cin, Cout = 2, 2, 256, 128
    Ho = H // 2
    x = rnd(G, B, H, H, Cin, seed=7)
    dy = rnd(G, B, Ho, Ho, Cout, seed=8)
    dw = torch.empty(G, Cout, 4, 4, Cin, device=DEV)
    g = ConvGeom(G, G, B, H, H, Cin, Ho, Ho, Cout, 4, 4, 2, 1, 0)
    need = int(ops.lib.cg_conv_workspace_bytes(C.byref(g), 2))
    assert need >= G * B * Ho * Ho * Cout * 4  # at least the copy of dy
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream

    def call(nbytes):
        return ops.lib.cg_conv_wgrad(C.byref(g), x.data_ptr(), dy.data_ptr(), dw.data_ptr(), None, ws.data_ptr(), nbytes, stream)

    assert call(need - 1) == -2  # CG_ERR_WORKSPACE
    assert call(need) == 0, ops.lib.cg_last_error().decode()
    torch.cuda.synchronize()
    want = torch.zeros(G, Cout, 4, 4, Cin, dtype=torch.float64, device=DEV)
    from ops_torch import TorchOps
    TorchOps(DEV, torch.float64).conv_wgrad(x.double(), dy.double(), want, None, 2, 1)
    check(dw, want, 'direct call')
