"""vgg_w on the GPU: the preprocessing and max-pool kernels against torch (bit for bit) and float64 autograd (exact routing, ties, all-zero
windows, odd sizes), the loss kernel against float64 autograd, the whole frozen VGG-16 (relu5_3 and its input gradient) against a float64
torch Vgg16 on the synthetic weights, the training step against the unmodified reference's numbers (tests/golden/*_vgg*.json), and the
launch list of an update with the term on."""
import pytest
import torch
import torch.nn.functional as F

from common import close, load_golden, setup_case
from test_trainer_recon_cpu import golden_records, n_iters
from test_trainer_vgg_cpu import CASES, LISTS, published, run
from vgg_oracle import POOL_AFTER, VGG_LAYERS, synth_vgg16, vgg16, vgg_preprocess, write_vgg16

pytestmark = pytest.mark.gpu

U_TF32 = 2.0 ** -11  # unit roundoff of a TF32 operand (10 explicit mantissa bits)


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    return CudaOps('cuda:0')


def _nchw(x):
    G, B, H, W, C = x.shape
    return x.reshape(G * B, H, W, C).permute(0, 3, 1, 2)


def test_preprocess_bit_exact(ops):
    gen = torch.Generator().manual_seed(1)
    x = (torch.rand(1, 3, 37, 29, 4, generator=gen) * 2 - 1).cuda()
    x[..., 3] = 7.0  # junk in lane 3 must not leak
    y = ops.vgg_preprocess(x)
    want = vgg_preprocess(_nchw(x)[:, :3].contiguous()).permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    assert torch.equal(y[..., :3].reshape(want.shape), want) and float(y[..., 3].abs().max()) == 0
    d = torch.randn(1, 3, 37, 29, 4, generator=gen).cuda()
    dx = torch.full_like(x, 0.25)
    ops.vgg_preprocess_bwd(d, dx, accumulate=True)
    torch.cuda.synchronize()
    assert torch.equal(dx[..., :3], 0.25 + 127.5 * d[..., [2, 1, 0]]) and torch.equal(dx[..., 3], torch.full_like(dx[..., 3], 0.25))
    ops.vgg_preprocess_bwd(d, dx, accumulate=False)
    torch.cuda.synchronize()
    assert torch.equal(dx[..., :3], 127.5 * d[..., [2, 1, 0]]) and float(dx[..., 3].abs().max()) == 0


def _relu_with_ties(shape, seed):
    """ReLU outputs on a coarse grid: many ties inside windows and many all-zero windows"""
    gen = torch.Generator().manual_seed(seed)
    return torch.relu(torch.randint(-3, 3, shape, generator=gen).float() * 0.5).cuda()


@pytest.mark.parametrize('B,H,W,C', [(2, 7, 9, 4), (1, 17, 17, 64), (3, 32, 32, 128), (2, 2, 2, 512)])
def test_maxpool_forward_and_backward_exact(ops, B, H, W, C):
    x = _relu_with_ties((1, B, H, W, C), seed=H * W + C)
    y = ops.maxpool2x2_fwd(x)
    dy = torch.randn(1, B, H // 2, W // 2, C, generator=torch.Generator().manual_seed(3)).cuda()
    dx = ops.maxpool2x2_bwd(dy, x)
    torch.cuda.synchronize()
    assert torch.equal(_nchw(y), F.max_pool2d(_nchw(x), 2, 2))
    x64 = x.double().requires_grad_(True)
    g, = torch.autograd.grad(F.max_pool2d(_nchw(x64), 2, 2), x64, _nchw(dy.double()))
    want = (g * (x64 > 0)).float()
    assert torch.equal(dx, want)
    assert (x == 0).any() and float(dx[..., :2 * (H // 2), :2 * (W // 2), :].ne(0).float().mean()) < 0.25
    if H % 2:
        assert float(dx[:, :, -1].abs().max()) == 0
    if W % 2:
        assert float(dx[:, :, :, -1].abs().max()) == 0


@pytest.mark.parametrize('N,B,h,w', [(2, 2, 8, 8), (4, 1, 5, 3), (1, 3, 32, 32)])
def test_loss_kernel_matches_float64(ops, N, B, h, w):
    gen = torch.Generator().manual_seed(N * 100 + h)
    C = 512
    R = 2 * N * B
    f = torch.relu(torch.randn(1, R, h, w, C, generator=gen)).cuda()
    t = torch.relu(torch.randn(1, 2 * B, h, w, C, generator=gen)).cuda()
    coef = 0.7 / (B * C * h * w)
    sums = ops.empty(2, N)
    d_pre = ops.vgg_loss(f, t, B, N * B, coef, sums)
    torch.cuda.synchronize()
    tgt = torch.tensor([(r // (N * B)) * B + r % B for r in range(R)])
    f64 = f.double().requires_grad_(True)
    d = F.instance_norm(_nchw(f64), eps=1e-5) - F.instance_norm(_nchw(t.double())[tgt], eps=1e-5)
    per_row = (d ** 2).sum(dim=(1, 2, 3))
    g, = torch.autograd.grad(coef * per_row.sum(), f64)
    want_sums = per_row.detach().reshape(2 * N, B).sum(-1)
    assert torch.allclose(sums.double().view(-1), want_sums, rtol=2e-5)
    want = g * (f > 0)
    rel = ((d_pre.double() - want).norm() / want.norm()).item()
    assert rel < 1e-4, rel
    assert float(d_pre[f == 0].abs().max()) == 0


def _dgrad64(sd64, saved, d_pre, x_nchw_shape):
    """float64 data gradient of the VGG with the ReLU masks and max-pool windows of the product's own saved activations: what is left
    is the rounding of the 13 data-gradient convolutions"""
    d = _nchw(d_pre.double())
    for li in range(len(VGG_LAYERS) - 1, -1, -1):
        w = sd64[VGG_LAYERS[li][0] + '.weight']
        if li == 0:
            return torch.nn.grad.conv2d_input(x_nchw_shape, w, d, padding=1)
        prev = _nchw(saved[li - 1].double())
        if VGG_LAYERS[li - 1][0] in POOL_AFTER:
            p = prev.clone().requires_grad_(True)
            pooled = F.max_pool2d(p, 2, 2)
            d = torch.nn.grad.conv2d_input(pooled.shape, w, d, padding=1)
            d, = torch.autograd.grad(pooled, p, d)
        else:
            d = torch.nn.grad.conv2d_input(prev.shape, w, d, padding=1)
        d = d * (prev > 0)


@pytest.mark.parametrize('H,W', [(36, 44), (64, 64)])
def test_vgg_matches_float64(ops, H, W, tmp_path):
    from council_gan_b200.networks import Vgg16
    sd = synth_vgg16(16)
    write_vgg16(sd, str(tmp_path))
    net = Vgg16(ops).load(str(tmp_path))
    gen = torch.Generator().manual_seed(H)
    img = (torch.rand(1, 2, H, W, 4, generator=gen) * 2 - 1).cuda()
    img[..., 3] = 0
    x = ops.vgg_preprocess(img)
    saved = []
    f = net.forward(x, saved)
    d_f = torch.randn(f.shape, generator=gen).cuda()
    d_pre = (d_f * (f > 0)).contiguous()
    dx = net.backward(d_pre, x.shape, saved)
    torch.cuda.synchronize()
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    x64 = _nchw(x.double())[:, :3].contiguous()
    f64 = vgg16(sd64, x64)
    g64 = _dgrad64(sd64, saved, d_pre, x64.shape)
    # TF32 rounds both operands of every product to 10 mantissa bits (unit roundoff u = 2^-11), so one layer's output is off by at
    # most sqrt(2) u in relative L2, and the error grows at most linearly through the 13 layers of either pass.  The gradient is taken
    # with the product's own ReLU masks and max-pool windows: float64 masks would differ wherever a pre-activation or a window tie lies
    # within rounding distance, and such flips are not rounding error of the gradient.
    tol = 13 * 2 ** 0.5 * U_TF32
    rel_f = ((_nchw(f.double()) - f64).norm() / f64.norm()).item()
    rel_g = ((_nchw(dx.double())[:, :3] - g64).norm() / g64.norm()).item()
    assert rel_f < tol, ('relu5_3', rel_f, tol)
    assert rel_g < tol, ('d(input)', rel_g, tol)
    assert tuple(f.shape) == (1, 2, H // 8, W // 8, 512) and float(dx[..., 3].abs().max()) == 0


def _run_gpu(gold, vgg_dir, tc, on_iter=None):
    from council_gan_b200.ops import CudaOps
    cops = CudaOps('cuda:0')
    cops.set_tensor_core_mode(tc)
    try:
        tr, hp = run(gold, vgg_dir, ops=cops, on_iter=on_iter)
        torch.cuda.synchronize()
    finally:
        cops.set_tensor_core_mode(1)
    return tr, hp


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('tc', [0, 1])
def test_iteration_matches_golden(case, tc, tmp_path):
    """the loss gates of test_trainer_recon_x_gpu, on every iteration of the case"""
    gold = load_golden(case)
    log = []
    tr, hp = _run_gpu(gold, tmp_path, tc, on_iter=lambda k, t: log.append(([float(v) for v in t.loss_dis_total_s],
                                                                           [float(v) for v in t.loss_gen_total_s], published(t))))
    assert len(log) == n_iters(gold)
    for k, (rec, (dis, gen, lists)) in enumerate(zip(golden_records(gold), log)):
        rtol = ([1e-3, 3e-3, 3e-2] if tc == 0 else [2e-3, 2e-2, 6e-2])[k]
        for i in range(tr.council_size):
            assert close(dis[i], rec['loss_dis_total'][i], rtol), ('dis', k, i)
            assert close(gen[i], rec['loss_gen_total'][i], rtol), ('gen', k, i, gen[i], rec['loss_gen_total'][i])
        # the VGG terms compare instance-normalised features of translations that carry the generator's fp32 / TF32 noise: 2.3e-3
        # from the reference in the first step with TF32, 3.2e-3 in the second in exact fp32; the totals above stay the tight gate
        rtol_lists = max(rtol, [5e-3, 1e-2, 5e-2][k])
        for key in LISTS:
            assert len(lists[key]) == len(rec[key]), key
            for g, r in zip(lists[key], rec[key]):
                assert close(g, r, rtol_lists, 1e-6), (key, k, g, r)


def _kernels(prof):
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and not e.name.lower().startswith(('memcpy', 'memset'))]


def test_update_with_term_on_launches_no_pytorch_kernels(tmp_path):
    from torch.profiler import ProfilerActivity, profile
    from council_gan_b200 import Council_Trainer
    gold = load_golden('glasses64_n2_b2_vgg')
    hp, _, x_a, x_b = setup_case(gold)
    write_vgg16(synth_vgg16(gold['vgg_seed']), str(tmp_path))
    hp['vgg_model_path'] = str(tmp_path)
    tr = Council_Trainer(hp, 'cuda:0')
    tr.dis_update(x_a, x_b, hp)
    tr.gen_update(x_a, x_b, hp, gold['iteration'])  # warm: workspaces, caches
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.gen_update(x_a, x_b, hp, gold['iteration'] + 1)
        torch.cuda.synchronize()
    kernels = _kernels(prof)
    assert any('vgg_loss' in n for n in kernels) and any('maxpool2x2_bwd' in n for n in kernels)
    foreign = [n for n in kernels if 'at::' in n or 'native' in n or 'cublas' in n.lower() or 'cudnn' in n.lower()]
    assert not foreign, sorted(set(foreign))


def test_vgg_convolutions_run_on_tensor_cores(ops, tmp_path):
    """every 3x3 layer with Cin >= 64 runs on the tensor-core kernel (conv_tc_kernel), forward and data gradient, at the smallest stacked
    batch of the fixture cases (2 directions x 2 members x 2 images at 64 x 64: relu5_3 at 8 x 8).  Each call is made twice on the same
    inputs, with the tensor-core path on (mode 1) and in the exact-fp32 SIMT mode (mode 0): a layer that fell back to conv_*_simt_kernel
    would give the SIMT kernel's bits in both, so the results must differ, and by no more than one layer's TF32 rounding (sqrt(2) u).
    The kernel choice is a host-side function of the geometry, so this is decided without a profiler, whose kernel records of a short
    session are not reliably delivered."""
    from council_gan_b200.networks import Vgg16
    write_vgg16(synth_vgg16(16), str(tmp_path))
    net = Vgg16(ops).load(str(tmp_path))
    gen = torch.Generator().manual_seed(5)
    x = ops.vgg_preprocess((torch.rand(1, 8, 64, 64, 4, generator=gen) * 2 - 1).cuda())
    saved = []
    net.forward(x, saved)
    torch.cuda.synchronize()
    checked = 0
    for li, s in enumerate(net.specs):
        if s.cin < 64:
            continue
        inp = saved[li - 1]
        if net.specs[li - 1].key in net.POOL_AFTER:
            inp = ops.maxpool2x2_fwd(inp)
        w, b = net.bank.p(s.wname), net.bank.p(s.bname)
        dy = torch.randn(saved[li].shape, generator=gen).cuda()
        out = {}
        for mode in (1, 0):
            ops.set_tensor_core_mode(mode)
            try:
                out[mode] = (ops.conv_fwd(inp, w, b, 1, 1, act=1), ops.conv_dgrad(dy, w, inp.shape, 1, 1))
                torch.cuda.synchronize()
            finally:
                ops.set_tensor_core_mode(1)
        for k, what in enumerate(('forward', 'data gradient')):
            tc, simt = out[1][k].double(), out[0][k].double()
            rel = ((tc - simt).norm() / simt.norm()).item()
            assert 0 < rel < 2 ** 0.5 * U_TF32, (s.key, what, rel)
            checked += 1
    assert checked == 24
