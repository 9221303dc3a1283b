"""Per-kernel parity: every C-ABI op (through ctypes, council_gan_b200.ops.CudaOps) against the plain
PyTorch reference of the same op (tests/ops_torch.py) evaluated in float64 on the same device.

Tolerances: the SIMT kernels compute in exact fp32 -> 2e-5 relative to the tensor's max magnitude.
The tensor-core path (TF32 operands, fp32 accumulate) is compared at 3e-3 (10-bit mantissa operands).
"""
import pytest
import torch

from ops_torch import TorchOps

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    return CudaOps(DEV)


@pytest.fixture(scope='module')
def ref():
    return TorchOps(DEV, torch.float64)


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def d(t):
    return None if t is None else t.double()


def check(got, want, tol=2e-5, what=''):
    want = want.to(torch.float64)
    err = (got.double() - want).abs().max().item()
    mag = want.abs().max().item() + 1e-30
    assert err <= tol * mag + 1e-7, '%s: max err %.3e vs magnitude %.3e' % (what, err, mag)


# (name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups)
CONV_CASES = [
    ('enc0_7x7_img', 2, 1, 2, 16, 16, 4, 64, 7, 1, 3, False),
    ('enc1_4x4s2', 2, 2, 2, 16, 16, 64, 128, 4, 2, 1, False),
    ('res_3x3', 2, 2, 1, 8, 8, 256, 256, 3, 1, 1, False),
    ('up_3x3_ups', 2, 2, 2, 8, 8, 128, 64, 3, 1, 1, True),
    ('head_1x1', 2, 2, 2, 16, 16, 64, 64, 1, 1, 0, False),
    ('head_1x1_12', 2, 2, 2, 16, 16, 64, 12, 1, 1, 0, False),
    ('dis0_4x4s2_img', 3, 3, 2, 16, 16, 4, 64, 4, 2, 1, False),
    ('disc0_3x3_pair', 2, 2, 3, 12, 12, 8, 64, 3, 1, 1, False),
    ('dis_out_1x1', 2, 2, 4, 4, 4, 512, 1, 1, 1, 0, False),
    ('mlp_linear', 2, 1, 3, 1, 1, 64, 256, 1, 1, 0, False),
    ('mlp_linear_big', 2, 2, 3, 1, 1, 256, 5888, 1, 1, 0, False),
    ('mlp_linear_big_b8', 4, 4, 8, 1, 1, 256, 5888, 1, 1, 0, False),
    ('dis_out_1x1_b32', 4, 4, 32, 32, 32, 512, 1, 1, 1, 0, False),
    ('dis_out_1x1_c256_odd', 3, 3, 5, 7, 9, 256, 1, 1, 1, 0, False),
    ('odd_sizes', 1, 1, 1, 10, 14, 8, 20, 3, 1, 1, False),
    # shapes that qualify for the tensor-core path (>= 128 output pixels per member)
    ('tc_res_3x3_256', 2, 2, 2, 16, 16, 256, 256, 3, 1, 1, False),
    ('tc_down_4x4s2_64_128', 2, 2, 2, 32, 32, 64, 128, 4, 2, 1, False),
    ('tc_down_4x4s2_256_512', 2, 2, 3, 16, 16, 256, 512, 4, 2, 1, False),
    ('tc_up_3x3_128_64', 2, 2, 1, 32, 32, 128, 64, 3, 1, 1, False),
    ('tc_dc_1x1_512_512', 3, 3, 4, 8, 8, 512, 512, 1, 1, 0, False),
    ('tc_shared_input', 3, 1, 2, 16, 16, 64, 64, 3, 1, 1, False),
    ('tc_partial_tiles', 2, 2, 3, 12, 20, 64, 128, 3, 1, 1, False),
    # 256-wide tiles with partial pixel tiles (640 / 720 px), dgrad classes of a stride-2 layer
    ('tc_pair_half_tile', 2, 2, 5, 8, 16, 64, 256, 3, 1, 1, False),
    ('tc_pair_partial', 2, 2, 3, 12, 20, 32, 512, 3, 1, 1, False),
    ('tc_pair_dgrad_s2', 2, 2, 2, 32, 32, 256, 64, 4, 2, 1, False),
    # weight gradient with 256 output channels; 64- and 192-channel inputs (one full / one partial 64-channel tile per tap)
    ('tc_pair_wgrad_c64_o256', 2, 2, 2, 16, 16, 64, 256, 3, 1, 1, False),
    ('tc_pair_wgrad_c192_o256', 1, 1, 2, 16, 16, 192, 256, 3, 1, 1, False),
    # weight gradient with <= 64 output channels: 128 / 96 / 32 input channels (full and partial 64-channel tiles)
    ('tc_xm_wgrad_c128_o64', 2, 2, 2, 16, 16, 128, 64, 3, 1, 1, False),
    ('tc_xm_wgrad_1x1_c96_o64', 2, 1, 2, 16, 16, 96, 64, 1, 1, 0, False),
    ('tc_xm_wgrad_4x4s2_c32_o32', 2, 2, 2, 32, 32, 32, 32, 4, 2, 1, False),
    # image-side layers on the explicit-patch path (im2col -> 1x1 tensor-core GEMM)
    ('patch_disc0_3x3_pair', 2, 2, 2, 16, 16, 8, 64, 3, 1, 1, False),
    ('patch_dis0_4x4s2_img', 2, 2, 4, 16, 16, 4, 64, 4, 2, 1, False),
    ('patch_enc0_7x7_shared', 3, 1, 2, 16, 16, 4, 64, 7, 1, 3, False),
    # image-side layers on larger maps: several tiles per CTA, image borders inside tiles
    ('img_disc0_3x3_pair_multi', 3, 3, 5, 32, 32, 8, 64, 3, 1, 1, False),
    ('img_dis0_4x4s2_rect', 2, 2, 3, 32, 64, 4, 64, 4, 2, 1, False),
]


@pytest.mark.parametrize('case', CONV_CASES, ids=[c[0] for c in CONV_CASES])
@pytest.mark.parametrize('tc', [0, 1, 7 | 32 | 64 | (1 << 16), 7 | (1 << 17), 7 | (1 << 19), 7 | (1 << 20), 7 | (1 << 21), 7 | (1 << 22), 7 | (1 << 23)])
def test_conv_fwd_dgrad_wgrad(ops, ref, case, tc):
    """tc = 0: SIMT fp32; 1: the default tensor-core dispatch; the other masks add switch bits to the full mask (see
    cg_set_tensor_core_mode in include/council_b200.h: 1<<22 programmatic dependent launch, 1<<23 widest N tile even on small maps --
    the default narrows the tile when a launch has fewer tiles than SMs, which these test shapes do, so tc=1 exercises the narrowed
    tiles and this one the wide; bits the library ignores must leave every result unchanged).  Every mode runs on every
    geometry: whichever kernels a mode selects for a layer, the results must hold."""
    name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups = case
    ops.set_tensor_core_mode(tc)
    tol = 2e-5 if tc == 0 else 4e-3
    try:
        x = rnd(Gx, B, H, W, Cin, seed=1)
        w = rnd(G, Cout, K, K, Cin, seed=2, scale=0.1)
        b = rnd(G, Cout, seed=3)
        pre = ref.conv_fwd(d(x), d(w), d(b), stride, pad, ups=ups, act=0)
        pre_mag = pre.abs().max().item()
        for act in (0, 1, 2, 3):
            y = ops.conv_fwd(x, w, b, stride, pad, ups=ups, act=act, slope=0.2)
            want = ref.conv_fwd(d(x), d(w), d(b), stride, pad, ups=ups, act=act, slope=0.2)
            # every activation is 1-Lipschitz: the error budget is that of the pre-activation
            err = (y.double() - want).abs().max().item()
            assert err <= tol * pre_mag + 1e-7, '%s fwd act%d: max err %.3e vs pre-activation magnitude %.3e' % (name, act, err, pre_mag)
        y = ops.conv_fwd(x, w, None, stride, pad, ups=ups)
        check(y, ref.conv_fwd(d(x), d(w), None, stride, pad, ups=ups), tol, name + ' fwd nobias')
        dy = rnd(*y.shape, seed=4)
        xs = (G, B, H, W, Cin)
        add = rnd(*xs, seed=5)
        msk = rnd(*xs, seed=6)
        dx = ops.conv_dgrad(dy, w, xs, stride, pad, ups=ups)
        check(dx, ref.conv_dgrad(d(dy), d(w), xs, stride, pad, ups=ups), tol, name + ' dgrad')
        dx = ops.conv_dgrad(dy, w, xs, stride, pad, ups=ups, addend=add, mask_src=msk, mask_slope=0.2)
        check(dx, ref.conv_dgrad(d(dy), d(w), xs, stride, pad, ups=ups, addend=d(add), mask_src=d(msk), mask_slope=0.2),
              tol, name + ' dgrad+addend+mask')
        dw, db = torch.full_like(w, 7.0), torch.full_like(b, 7.0)
        ops.conv_wgrad(x, dy, dw, db, stride, pad, ups=ups)
        rw, rb = torch.zeros_like(w, dtype=torch.float64), torch.zeros_like(b, dtype=torch.float64)
        ref.conv_wgrad(d(x), d(dy), rw, rb, stride, pad, ups=ups)
        check(dw, rw, tol, name + ' wgrad')
        check(db, rb, tol, name + ' bias grad')
    finally:
        ops.set_tensor_core_mode(1)


STATS_CASES = [
    # name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups
    ('stats_res_3x3_256', 2, 2, 2, 16, 16, 256, 256, 3, 1, 1, False),
    ('stats_down_4x4s2', 2, 2, 2, 32, 32, 64, 128, 4, 2, 1, False),
    ('stats_up_classes', 2, 2, 2, 16, 16, 128, 64, 3, 1, 1, True),
    ('stats_first_7x7_patch', 2, 1, 2, 16, 16, 4, 64, 7, 1, 3, False),
    ('stats_small_map_simt', 2, 2, 1, 8, 8, 256, 256, 3, 1, 1, False),
    # statistics epilogue on 256- and 128-wide tiles, the production residual-block shape
    ('stats_pair_128_wide', 2, 2, 2, 32, 32, 128, 128, 3, 1, 1, False),
    ('stats_pair_down_128_256', 2, 2, 2, 32, 32, 128, 256, 4, 2, 1, False),
    ('stats_prod_res_3x3_256', 4, 4, 8, 64, 64, 256, 256, 3, 1, 1, False),
]


@pytest.mark.parametrize('case', STATS_CASES, ids=[c[0] for c in STATS_CASES])
@pytest.mark.parametrize('tc', [0, 1])
def test_conv_fwd_stats(ops, ref, case, tc):
    """conv + fused instance-norm statistics (tensor-core epilogue) vs conv followed by a separate statistics pass."""
    name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups = case
    ops.set_tensor_core_mode(tc)
    try:
        x = rnd(Gx, B, H, W, Cin, seed=11) + 0.3
        w = rnd(G, Cout, K, K, Cin, seed=12, scale=0.1)
        y, mean, rstd = ops.conv_fwd_stats(x, w, stride, pad, ups=ups)
        ry, rm, rr = ref.conv_fwd_stats(d(x), d(w), stride, pad, ups=ups)
        tol = 2e-5 if tc == 0 else 4e-3
        check(y, ry, tol, name + ' y')
        # statistics must describe the y that was actually produced (TF32 or fp32), to fp32 accuracy
        m2 = y.double().mean(dim=(2, 3))
        v2 = y.double().var(dim=(2, 3), unbiased=False)
        check(mean, m2, 2e-5, name + ' mean of own output')
        check(rstd, 1.0 / torch.sqrt(v2 + 1e-5), 5e-5, name + ' rstd of own output')
        check(mean, rm, tol * 4, name + ' mean vs fp64 reference')
    finally:
        ops.set_tensor_core_mode(1)


def test_conv_wgrad_split_k_large(ops, ref):
    """Many pixels, few output tiles -> split-K with the deterministic two-phase reduction."""
    x = rnd(1, 2, 64, 64, 8, seed=1)
    dy = rnd(2, 2, 64, 64, 16, seed=2)
    dw = ops.empty(2, 16, 3, 3, 8)
    db = ops.empty(2, 16)
    ops.conv_wgrad(x, dy, dw, db, 1, 1)
    dw2 = torch.empty_like(dw)
    ops.conv_wgrad(x, dy, dw2, None, 1, 1)
    assert torch.equal(dw, dw2), 'wgrad must be run-to-run deterministic'
    rw, rb = torch.zeros_like(dw, dtype=torch.float64), torch.zeros_like(db, dtype=torch.float64)
    ref.conv_wgrad(d(x), d(dy), rw, rb, 1, 1)
    check(dw, rw, 2e-5, 'wgrad split-K')
    check(db, rb, 2e-5, 'bias grad')


@pytest.mark.parametrize('C', [64, 128, 256])
@pytest.mark.parametrize('adain_on,res_on,act,ups', [(False, False, 1, False), (True, True, 0, False),
                                                     (True, False, 1, True), (False, True, 0, False)])
def test_norm_fwd_bwd(ops, ref, C, adain_on, res_on, act, ups):
    G, B, H, W = 2, 2, 12, 10
    y = rnd(G, B, H, W, C, seed=1, scale=2.0) + 0.5
    P = 4 * C + 16
    off = 8
    adain = rnd(G, B, P, seed=2) if adain_on else None
    res = rnd(G, B, H, W, C, seed=3) if res_on else None
    mean, rstd = ops.in_stats(y)
    rm, rr = ref.in_stats(d(y))
    check(mean, rm, 2e-5, 'mean')
    check(rstd, rr, 2e-5, 'rstd')
    z = ops.norm_act_fwd(y, mean, rstd, adain, off, res, act, ups)
    check(z, ref.norm_act_fwd(d(y), rm, rr, d(adain), off, d(res), act, ups), 3e-5, 'norm fwd')
    dz = rnd(*z.shape, seed=4)
    d_adain = ops.zeros(G, B, P) if adain_on else None
    dy = ops.norm_act_bwd(dz, y, mean, rstd, adain, off, act, ups, d_adain)
    r_dad = torch.zeros(G, B, P, dtype=torch.float64, device=DEV) if adain_on else None
    rdy = ref.norm_act_bwd(d(dz), d(y), rm, rr, d(adain), off, act, ups, r_dad)
    check(dy, rdy, 1e-4, 'norm bwd dy')
    if adain_on:
        check(d_adain, r_dad, 1e-4, 'norm bwd d_adain')


def test_mask_head(ops, ref):
    G, B, H, W = 2, 2, 9, 7
    h = torch.tanh(rnd(G, B, H, W, 12, seed=1, scale=0.3))
    x_in = rnd(1, B, H, W, 4, seed=2)
    x_in[..., 3] = 0
    xf, mask = ops.mask_head_fwd(h, x_in)
    rxf, rmask = ref.mask_head_fwd(d(h), d(x_in))
    check(xf, rxf, 2e-5, 'x_fake')
    check(mask, rmask, 2e-5, 'mask')
    assert float(xf[..., 3].abs().max()) == 0 and float(mask[..., 3].abs().max()) == 0
    dxf, dm = rnd(G, B, H, W, 4, seed=3), rnd(G, B, H, W, 4, seed=4)
    for dmask in (None, dm):
        got = ops.mask_head_bwd(h, x_in, dxf, dmask)
        want = ref.mask_head_bwd(d(h), d(x_in), d(dxf), d(dmask))
        check(got, want, 5e-5, 'mask head bwd')


@pytest.mark.parametrize('shape', [(2, 2, 16, 16), (4, 8, 256, 256), (3, 1, 8, 48)])
@pytest.mark.parametrize('adain_on', [True, False])
def test_head_fused(ops, ref, shape, adain_on):
    """cg_head_fused (AdaIN + ReLU -> 1x1 -> 1x1 -> 1x1 tanh -> mask compositing in one wgmma kernel) against the float64
    composition of the separate ops, and against the separate CUDA ops it replaces."""
    G, B, H, W = shape
    y = rnd(G, B, H, W, 64, seed=1, scale=1.5) + 0.2
    P, off = 4 * 64 + 8, 4
    adain = rnd(G, B, P, seed=2) if adain_on else None
    w1, w2 = rnd(G, 64, 1, 1, 64, seed=3, scale=0.15), rnd(G, 64, 1, 1, 64, seed=4, scale=0.15)
    w3 = rnd(G, 12, 1, 1, 64, seed=5, scale=0.1)
    b1, b2, b3 = rnd(G, 64, seed=6, scale=0.1), rnd(G, 64, seed=7, scale=0.1), rnd(G, 12, seed=8, scale=0.1)
    x_in = rnd(1, B, H, W, 4, seed=9)
    x_in[..., 3] = 0
    mean, rstd = ops.in_stats(y)
    xf, mask = ops.head_fused(y, mean, rstd, adain, off, w1, b1, w2, b2, w3, b3, x_in)
    rxf, rmask = ref.head_fused(d(y), d(mean), d(rstd), d(adain), off, d(w1), d(b1), d(w2), d(b2), d(w3), d(b3), d(x_in))
    # three chained TF32 GEMMs feeding tanh(10 tanh(.)): compare at the TF32 tolerance on O(1) outputs
    assert (xf.double() - rxf).abs().max().item() < 2e-2 and (xf.double() - rxf).abs().mean().item() < 1e-3
    assert (mask.double() - rmask).abs().max().item() < 2e-2 and (mask.double() - rmask).abs().mean().item() < 1e-3
    assert float(xf[..., 3].abs().max()) == 0 and float(mask[..., 3].abs().max()) == 0
    # the separate tensor-core kernels round the same way: much tighter agreement
    z = ops.norm_act_fwd(y, mean, rstd, adain, off, None, 1, False)
    z = ops.conv_fwd(ops.conv_fwd(z, w1, b1, 1, 0, act=1), w2, b2, 1, 0, act=1)
    sxf, smask = ops.mask_head_fwd(ops.conv_fwd(z, w3, b3, 1, 0, act=3), x_in)
    assert (xf - sxf).abs().mean().item() < 2e-4 and (mask - smask).abs().mean().item() < 2e-4


def test_image_helpers(ops, ref):
    G, B, H, W = 2, 3, 8, 12
    x = rnd(G, B, H, W, 8, seed=1)
    check(ops.avgpool_fwd(x), ref.avgpool_fwd(d(x)), 2e-5, 'avgpool fwd')
    dy = rnd(G, B, H // 2, W // 2, 8, seed=2)
    for acc in (False, True):
        dx = rnd(G, B, H, W, 4, seed=3)
        rdx = d(dx).clone()
        ops.avgpool_bwd(dy, dx, 4, acc)
        ref.avgpool_bwd(d(dy), rdx, 4, acc)
        check(dx, rdx, 2e-5, 'avgpool bwd acc=%s' % acc)
    dst, src = rnd(G, B, H, W, 4, seed=4), rnd(G, B, H, W, 8, seed=5)
    rdst = d(dst).clone()
    ops.acc_slice(dst, src, 4)
    ref.acc_slice(rdst, d(src), 4)
    check(dst, rdst, 1e-6, 'acc_slice')
    pool = rnd(5, H, W, 4, seed=6)
    idx = torch.tensor([[0, 4, 2, 2, 1, 3], [3, 3, 0, 1, 4, 2]], dtype=torch.int32, device=DEV)
    x_in = rnd(1, 3, H, W, 4, seed=7)
    for xi in (None, x_in):
        got = ops.gather_images(pool, idx, xi, 2, 6)
        want = ref.gather_images(d(pool), idx, d(xi), 2, 6)
        assert torch.equal(got.double(), want)
    # two pools without torch.cat: slots < 3 read pool_a, the rest pool_b
    pool_a, pool_b = pool[:3].contiguous(), pool[3:].contiguous()
    for xi in (None, x_in):
        got = ops.gather_images((pool_a, pool_b), idx, xi, 2, 6)
        assert torch.equal(got.double(), ref.gather_images(d(pool), idx, d(xi), 2, 6))
    # host -> device staging: one pinned buffer, views keep dtype / shape / contents
    a, b = torch.randn(1, 3, 1, 1, 64), torch.arange(24, dtype=torch.int32).reshape(2, 12)
    for _ in range(10):  # more rounds than ring slots: buffers are reused safely
        da, db = ops.stage([a, b])
        assert da.is_cuda and da.dtype == torch.float32 and db.dtype == torch.int32
        assert torch.equal(da.cpu(), a) and torch.equal(db.cpu(), b)
    img = rnd(3, 3, H, W, seed=8)
    nhwc = ops.nchw_to_nhwc(img, 4)
    assert torch.equal(nhwc.double(), ref.nchw_to_nhwc(d(img), 4))
    assert torch.equal(ops.nhwc_to_nchw(nhwc, 3), img)


def test_losses(ops, ref):
    G, nseg, B, h, w = 3, 3, 2, 5, 4
    out = rnd(G, nseg * B, h, w, 1, seed=1)
    targets = torch.tensor([0.0, 1.0, 1.0], device=DEV)
    weights = torch.tensor([[2.0, 0.5, 0.5], [1.0, 1.0, 0.25], [0.5, 2.0, 3.0]], device=DEV)
    loss = torch.full((G,), 3.0, device=DEV)
    rloss = loss.double().clone()
    for acc in (False, True):
        sums = ops.lsgan_fwd(out, targets, weights, nseg, loss, acc)
        rs = ref.lsgan_fwd(d(out), d(targets), d(weights), nseg, rloss, acc)
        check(sums, rs, 2e-5, 'lsgan sums')
        check(loss, rloss, 2e-5, 'lsgan loss')
    coef = rnd(G, nseg, seed=2)
    check(ops.lsgan_bwd(out, targets, coef, nseg), ref.lsgan_bwd(d(out), d(targets), d(coef), nseg), 2e-5, 'lsgan bwd')
    mask = torch.sigmoid(rnd(G, 2, 11, 9, 4, seed=3, scale=3.0))
    mask[..., 3] = 0
    check(ops.focus_fwd(mask, 0.5, 0.01), ref.focus_fwd(d(mask), 0.5, 0.01), 5e-5, 'focus sums')
    fc = rnd(G, 3, seed=4)
    check(ops.focus_bwd(mask, fc, 0.5, 0.01), ref.focus_bwd(d(mask), d(fc), 0.5, 0.01), 5e-5, 'focus bwd')
    fc[:, 2] = 0  # TV off (male2female config)
    check(ops.focus_bwd(mask, fc, 0.5, 0.01), ref.focus_bwd(d(mask), d(fc), 0.5, 0.01), 5e-5, 'focus bwd no tv')


def test_fused_losses(ops, ref):
    """cg_lsgan_fused / cg_gen_loss_fwd / cg_gen_loss_bwd (csrc/losses.cu) against their plain restatement in float64:
    loss values, every gradient, the published values and the history rings, over the gating combinations."""
    G, B = 3, 2
    outs = [rnd(G, 3 * B, 5, 4, 1, seed=1), rnd(G, 3 * B, 3, 2, 1, seed=2)]
    wrows = [[2.0, 0.5, 0.5], [1.0, 1.0, 0.25], [0.5, 2.0, 3.0]]
    tot, plain = torch.full((G,), 3.0, device=DEV), torch.zeros(G, device=DEV)
    rtot, rplain = tot.double().clone(), plain.double().clone()
    for acc in (False, True):
        douts = ops.lsgan_fused(outs, 3, [0.0, 1.0, 1.0], wrows, 0.5, 0.25, tot, acc, plain)
        rd = ref.lsgan_fused([d(o) for o in outs], 3, [0.0, 1.0, 1.0], wrows, 0.5, 0.25, rtot, acc, rplain)
        check(tot, rtot, 2e-5, 'lsgan_fused total acc=%s' % acc)
        check(plain, rplain, 2e-5, 'lsgan_fused plain')
        for a, b in zip(douts, rd):
            check(a, b, 2e-5, 'lsgan_fused grad')
    mask = torch.sigmoid(rnd(G, B, 11, 9, 4, seed=3, scale=3.0))
    mask[..., 3] = 0
    adv = [rnd(G, B, 4, 4, 1, seed=4), rnd(G, B, 2, 2, 1, seed=5)]
    cl = [rnd(G, B, 6, 6, 1, seed=6), rnd(G, B, 3, 3, 1, seed=7)]
    hist = 5
    combos = [dict(gan_on=1, council_on=1, focus_on=1, matching=1, small_abs=0, small_square=1, wtv=0.0),
              dict(gan_on=1, council_on=1, focus_on=1, matching=1, small_abs=1, small_square=1, wtv=2.2),
              dict(gan_on=1, council_on=0, focus_on=0, matching=1, small_abs=0, small_square=1, wtv=0.0),
              dict(gan_on=1, council_on=1, focus_on=0, matching=0, small_abs=0, small_square=1, wtv=0.0),
              dict(gan_on=0, council_on=1, focus_on=1, matching=1, small_abs=0, small_square=1, wtv=0.0)]
    for ci, c in enumerate(combos):
        a_in = adv if c['gan_on'] else []
        c_in = cl if c['council_on'] else []
        m_in = mask if c['focus_on'] else None
        scal, rscal = ops.empty(G, 6), torch.zeros(G, 6, dtype=torch.float64, device=DEV)
        d_adv = ops.gen_loss_fwd(a_in, c_in, m_in, 0.5, 0.01, 24.0 / 2, scal)
        r_adv = ref.gen_loss_fwd([d(o) for o in a_in], [d(o) for o in c_in], d(m_in), 0.5, 0.01, 24.0 / 2, rscal)
        check(scal, rscal, 5e-5, 'gen_loss_fwd scal combo %d' % ci)
        for a, b in zip(d_adv, r_adv):
            check(a, b, 2e-5, 'adv grad')
        hg = (torch.rand(G, hist + 1, dtype=torch.float64) + 0.5).to(DEV)
        hc = (torch.rand(G, hist + 1, dtype=torch.float64) + 0.5).to(DEV)
        rhg, rhc = hg.clone(), hc.clone()
        hp = dict(world=2, hist_size=hist, head_gan=4, head_council=2, gan_w=24.0, council_w=4.0, w01=0.5, wtot=57.0,
                  numel=float(2 * B * 3 * 11 * 9), **c)
        for acc in (False, True):  # accumulate: the second direction adds to the double-precision total kept by the first call
            total, pub = torch.full((G,), 9.0, device=DEV), ops.empty(G, 8)
            rtotal, rpub = total.double().clone(), torch.zeros(G, 8, dtype=torch.float64, device=DEV)
            d_cl, d_mask = ops.gen_loss_bwd(c_in, m_in, 0.5, 0.01, scal, hp, hg, hc, total, acc, pub, c['focus_on'] == 1)
            r_cl, r_mask = ref.gen_loss_bwd([d(o) for o in c_in], d(m_in), 0.5, 0.01, scal.double(), hp, rhg, rhc, rtotal, acc, rpub,
                                            c['focus_on'] == 1)
            check(total, rtotal, 2e-6, 'total combo %d acc %s' % (ci, acc))
            check(pub, rpub, 2e-6, 'published values combo %d' % ci)
            for a, b in zip(d_cl, r_cl):
                check(a, b, 2e-5, 'council map grad')
            if c['focus_on']:
                check(d_mask, r_mask, 5e-5, 'mask grad combo %d' % ci)
            else:
                assert d_mask is None
            # the kernel stores the float32-rounded loss (like the reference's history); the float64 restatement does not round
            assert torch.allclose(hg, rhg, rtol=0, atol=1e-6) and torch.allclose(hc, rhc, rtol=0, atol=1e-6), 'history rings'
    # the scratch buffer is left clean: a second identical call gives identical results
    t1, t2 = ops.empty(G), ops.empty(G)
    ops.lsgan_fused(outs, 3, [0.0, 1.0, 1.0], wrows, 1.0, 1.0, t1, False)
    ops.lsgan_fused(outs, 3, [0.0, 1.0, 1.0], wrows, 1.0, 1.0, t2, False)
    assert torch.equal(t1, t2)


def test_tensor_map_cache(ops):
    """TMA descriptors are cached by (pointer, geometry): the second identical launch encodes nothing."""
    x = rnd(2, 2, 16, 16, 64, seed=1)
    w = rnd(2, 64, 3, 3, 64, seed=2, scale=0.1)
    y1 = ops.conv_fwd(x, w, None, 1, 1)
    s1 = ops.tensor_map_cache_stats()
    y2 = ops.conv_fwd(x, w, None, 1, 1)
    s2 = ops.tensor_map_cache_stats()
    assert torch.equal(y1, y2)
    assert s2['hits'] > s1['hits'] and s2['misses'] == s1['misses']


def test_adam(ops, ref):
    n = 100003
    p, g = rnd(n, seed=1), rnd(n, seed=2, scale=0.01)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    rp, rm, rv = d(p).clone(), d(m).clone(), d(v).clone()
    for step in (1, 2, 3):
        ops.adam_step(p, g, m, v, 1e-4, 0.5, 0.999, 1e-8, 1e-4, step)
        ref.adam_step(rp, d(g), rm, rv, 1e-4, 0.5, 0.999, 1e-8, 1e-4, step)
    assert (p.double() - rp).abs().max().item() < 1e-6  # a few fp32 ulps of |p| ~ 1.5 over three steps
    check(m, rm, 2e-5, 'exp_avg')
    check(v, rv, 2e-5, 'exp_avg_sq')


# ---- size-independent properties at the BASELINE sizes (256x256, council of 4, batch 8) ------------------
def test_full_size_adjoint_identities(ops):
    """<conv(x), dy> == <x, dgrad(dy)> == <w, wgrad(x, dy)> for the dominant 3x3 256->256 layer at the
    male2female B=8 shape (G=4, 64x64 maps), and instance-norm output statistics."""
    G, B, H, W, C = 4, 8, 64, 64, 256
    x = rnd(G, B, H, W, C, seed=1)
    w = rnd(G, C, 3, 3, C, seed=2, scale=0.02)
    dy = rnd(G, B, H, W, C, seed=3)
    y = ops.conv_fwd(x, w, None, 1, 1)
    dx = ops.conv_dgrad(dy, w, x.shape, 1, 1)
    dw = ops.empty(*w.shape)
    ops.conv_wgrad(x, dy, dw, None, 1, 1)
    a = (y.double() * dy.double()).sum().item()
    b = (x.double() * dx.double()).sum().item()
    c = (w.double() * dw.double()).sum().item()
    assert abs(a - b) <= 2e-3 * abs(a) and abs(a - c) <= 2e-3 * abs(a), (a, b, c)
    mean, rstd = ops.in_stats(y)
    z = ops.norm_act_fwd(y, mean, rstd, None, 0, None, 0, False)
    zm = z.double().mean(dim=(2, 3))
    zv = z.double().var(dim=(2, 3), unbiased=False)
    assert zm.abs().max().item() < 1e-4 and (zv - 1).abs().max().item() < 1e-3


# ---- every distinct production geometry of BASELINE configs[1] (male2female 256x256, council 4, batch 8; the council
# discriminator sees (1+U)*B = 32 images per member) against the float64 reference of the same convolution ----------------
PROD_CASES = [
    # name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups, check dgrad/wgrad
    ('prod_e0_7x7_img', 4, 1, 8, 256, 256, 4, 64, 7, 1, 3, False, True),
    ('prod_e1_4x4s2_64_128', 4, 4, 8, 256, 256, 64, 128, 4, 2, 1, False, True),
    ('prod_e2_4x4s2_128_256', 4, 4, 8, 128, 128, 128, 256, 4, 2, 1, False, True),
    ('prod_res_3x3_256', 4, 4, 8, 64, 64, 256, 256, 3, 1, 1, False, True),
    ('prod_u1_3x3_256_128_folded_ups', 4, 4, 8, 64, 64, 256, 128, 3, 1, 1, True, False),
    ('prod_u1_3x3_256_128', 4, 4, 8, 128, 128, 256, 128, 3, 1, 1, False, True),
    ('prod_u2_3x3_128_128', 4, 4, 8, 128, 128, 128, 128, 3, 1, 1, False, True),
    ('prod_u3_3x3_128_64_folded_ups', 4, 4, 8, 128, 128, 128, 64, 3, 1, 1, True, False),
    ('prod_u3_3x3_128_64', 4, 4, 8, 256, 256, 128, 64, 3, 1, 1, False, True),
    ('prod_u4_3x3_64_64', 4, 4, 8, 256, 256, 64, 64, 3, 1, 1, False, True),
    ('prod_h_1x1_64_64', 4, 4, 8, 256, 256, 64, 64, 1, 1, 0, False, True),
    ('prod_h3_1x1_64_12', 4, 4, 8, 256, 256, 64, 12, 1, 1, 0, False, True),
    ('prod_d0_4x4s2_img_b16', 4, 4, 16, 256, 256, 4, 64, 4, 2, 1, False, True),
    ('prod_d3_4x4s2_256_512_b16', 4, 4, 16, 32, 32, 256, 512, 4, 2, 1, False, True),
    ('prod_dc0_3x3_pair_b32', 4, 4, 32, 256, 256, 8, 64, 3, 1, 1, False, True),
    ('prod_dc1_4x4s2_64_128_b32', 4, 4, 32, 256, 256, 64, 128, 4, 2, 1, False, True),
    ('prod_dc2_4x4s2_128_256_b32', 4, 4, 32, 128, 128, 128, 256, 4, 2, 1, False, True),
    ('prod_dc3_4x4s2_256_512_b32', 4, 4, 32, 64, 64, 256, 512, 4, 2, 1, False, True),
    ('prod_dc4_1x1_512_512_b32', 4, 4, 32, 32, 32, 512, 512, 1, 1, 0, False, True),
]


@pytest.mark.parametrize('case', PROD_CASES, ids=[c[0] for c in PROD_CASES])
def test_production_geometry_vs_fp64(ops, ref, case):
    """Forward, data gradient and weight gradient of the default (tensor-core) dispatch at the exact shapes the bench runs,
    against float64 torch, at the TF32 tolerance (4e-3 of the tensor's magnitude)."""
    name, G, Gx, B, H, W, Cin, Cout, K, stride, pad, ups, bwd = case
    tol = 4e-3
    x = rnd(Gx, B, H, W, Cin, seed=21)
    w = rnd(G, Cout, K, K, Cin, seed=22, scale=1.0 / (K * K * Cin) ** 0.5)
    y = ops.conv_fwd(x, w, None, stride, pad, ups=ups)
    dy = rnd(*y.shape, seed=23) if bwd else None
    xs = (G, B, H, W, Cin)
    dx = ops.conv_dgrad(dy, w, xs, stride, pad) if bwd else None
    dw = torch.empty_like(w)
    if bwd:
        ops.conv_wgrad(x, dy, dw, None, stride, pad)
    # float64 reference one member at a time (memory)
    for g in range(G):
        xg = d(x[g if Gx > 1 else 0:(g if Gx > 1 else 0) + 1])
        wg = d(w[g:g + 1])
        check(y[g:g + 1], ref.conv_fwd(xg, wg, None, stride, pad, ups=ups), tol, '%s fwd member %d' % (name, g))
        if bwd:
            dyg = d(dy[g:g + 1])
            check(dx[g:g + 1], ref.conv_dgrad(dyg, wg, (1, B, H, W, Cin), stride, pad), tol, '%s dgrad member %d' % (name, g))
            rw = torch.zeros_like(wg)
            ref.conv_wgrad(xg, dyg, rw, None, stride, pad)
            check(dw[g:g + 1], rw, tol, '%s wgrad member %d' % (name, g))
        del xg, wg
        torch.cuda.empty_cache()
