"""pad_type: reflect on the GPU: cg_reflect_pad against torch's ReflectionPad2d (and nearest upsample) bit for bit, cg_reflect_pad_bwd
against float64 autograd, the training step against the oracle and the unmodified reference's numbers (tests/golden/*_reflect*.json),
sample() against the oracle, and the zero path running neither kernel."""
import pytest
import torch

import council_oracle as co
from common import close, load_golden, setup_case
from pad_oracle import padding
from test_trainer_gpu import _run_cuda_iters, run_cuda
from test_trainer_host_cpu import compare_with_oracle, load_states
from test_trainer_pad_cpu import CASES, TorchOps, run
from test_trainer_recon_cpu import compare
from test_trainer_recon_x_cpu import LISTS, published

pytestmark = pytest.mark.gpu

SHAPES = [  # (Gx, B, H, W, C, p)
    (1, 2, 8, 7, 4, 1), (2, 1, 9, 13, 8, 3), (3, 2, 16, 15, 64, 1), (2, 2, 5, 9, 256, 3), (1, 1, 4, 4, 64, 3), (4, 1, 33, 31, 8, 1)]


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    return CudaOps('cuda:0')


def _x(shape, seed):
    Gx, B, H, W, C, _ = shape
    return torch.randn(Gx, B, H, W, C, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('ups', [False, True])
def test_reflect_pad_bit_identical(ops, shape, ups):
    """ReflectionPad2d (of the nearest x2 upsample with ups): stacked and shared (Gx = 1) inputs, odd widths, C from 4 to 256"""
    p = shape[-1]
    if not ups and p >= min(shape[2], shape[3]):
        pytest.skip('the map is not larger than the pad')
    x = _x(shape, seed=sum(shape))
    got = ops.reflect_pad(x, p, ups)
    torch.cuda.synchronize()
    assert torch.equal(got, TorchOps('cuda').reflect_pad(x, p, ups))


@pytest.mark.parametrize('shape', SHAPES + [(2, 1, 3, 3, 4, 2)])  # the last: a pixel copied to up to 9 padded positions
@pytest.mark.parametrize('extra', ['none', 'addend', 'relu', 'lrelu+addend'])
def test_reflect_pad_bwd_matches_float64(ops, shape, extra):
    Gx, B, H, W, C, p = shape
    if p >= min(H, W):
        pytest.skip('the map is not larger than the pad')
    gen = torch.Generator().manual_seed(H * W + C)
    dxp = torch.randn(Gx, B, H + 2 * p, W + 2 * p, C, generator=gen).cuda()
    addend = torch.randn(Gx, B, H, W, C, generator=gen).cuda() if 'addend' in extra else None
    mask = torch.randn(Gx, B, H, W, C, generator=gen).cuda() if extra != 'none' and extra != 'addend' else None
    slope = 0.2 if extra.startswith('lrelu') else 0.0
    got = ops.reflect_pad_bwd(dxp, p, addend=addend, mask_src=mask, mask_slope=slope)
    torch.cuda.synchronize()
    t64 = TorchOps('cuda', torch.float64)
    want = t64.reflect_pad_bwd(dxp.double(), p, None if addend is None else addend.double(), None if mask is None else mask.double(),
                               slope)
    # at most 9 float32 additions (10 with the addend): rounding bounded by the size of the terms
    scale = dxp.abs().max().item() * (1 if addend is None else 2)
    assert (got.double() - want).abs().max().item() <= 10 * 2 ** -24 * 4 * scale
    if mask is not None and slope == 0:
        assert torch.all(got[mask <= 0] == 0)


def test_pad_not_smaller_than_map_refused(ops):
    x = torch.randn(1, 1, 3, 5, 4, device='cuda')
    for p, ups in ((3, False), (6, True)):
        with pytest.raises(RuntimeError, match='pad'):
            ops.reflect_pad(x, p, ups)
    with pytest.raises(RuntimeError, match='pad'):
        ops.reflect_pad_bwd(torch.randn(1, 1, 9, 11, 4, device='cuda'), 3)
    ops.reflect_pad(x, 5, True)  # 5 < 6: allowed on the upsampled map


def _align_dead_betas(tr, orc):
    """Under generator reflect the AdaIN beta of each residual block's second layer (no activation) has a zero gradient: its shift is
    constant over the map, the reflect padding of every following convolution keeps it constant, and the instance norm after that
    convolution removes it.  Adam's first step moves those parameters by lr * sign(rounding noise), differently on the two sides, so
    the parameter comparison takes them (the MLP's output rows that produce them) from the oracle."""
    tr.synchronize()
    for d in orc.dirs:
        net = tr._nets['gen_' + d]
        if not net.reflect:
            continue
        for i in range(tr.council_size):
            ref = orc.P['gen_' + d][i]
            for blk in net.dec_res:
                o, c = net.adain_off[blk[1].key], blk[1].cout
                net.bank.p('mlp.model.2.fc.bias')[i][o:o + c].copy_(ref['mlp.model.2.fc.bias'][o:o + c].detach())
                net.bank.p('mlp.model.2.fc.weight')[i][o:o + c].copy_(ref['mlp.model.2.fc.weight'][o:o + c].detach().reshape(c, 1, 1, -1))


@pytest.mark.parametrize('case', [c for c in CASES if 'iter3' not in c])
@pytest.mark.parametrize('tc', [0, 1])
def test_iteration_matches_oracle_and_golden(case, tc):
    """the gates of test_trainer_gpu.check_iteration, against the oracle with the case's padding"""
    gold = load_golden(case)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    orc, hp = run(gold, torch.float32)
    tr, _ = run_cuda(gold, tc)
    N = tr.council_size
    # the reconstruction case under TF32: test_trainer_recon_x_gpu's first-iteration gate (its generator totals land 1.0e-3 off)
    rtol = 2e-3 if tc == 1 and hp['do_a2b'] and hp['do_b2a'] else 1e-3
    for i in range(N):
        assert close(float(tr.loss_dis_total_s[i]), gold['loss_dis_total'][i], rtol), ('dis', i)
        assert close(float(tr.loss_gen_total_s[i]), gold['loss_gen_total'][i], rtol), ('gen', i)
        if gold['dis_council_ran']:
            assert close(float(tr.loss_dis_council_total_s[i]), gold['loss_dis_council_total'][i], rtol), ('disc', i)
    if hp['do_a2b'] and hp['do_b2a']:
        got = published(tr)
        for k in LISTS:
            for g, w in zip(got[k], gold[k]):
                assert close(g, w, rtol, 1e-6), (k, g, w)
    for d in orc.dirs:
        for i in range(N):
            xf = tr.ops.nhwc_to_nchw(tr._last_fw[d]['x_fake'][i], 3).cpu()
            mae = (xf - orc.x_fake_gen[d][i].detach()).abs().mean().item()
            assert mae < (2e-4 if tc == 0 else 3e-3), ('pixel MAE', d, i, mae)
    _align_dead_betas(tr, orc)
    if hp['do_a2b'] and hp['do_b2a']:  # the reconstruction terms train the style encoder: test_trainer_recon_x_gpu's comparison
        if tc == 0:
            compare(tr, orc, hp, rtol_loss=1e-3, grad_rel_l2=5e-2, flip_frac=0.05)
    elif tc == 0:
        compare_with_oracle(tr, orc, hp, rtol_loss=1e-3, grad_rel_l2=3e-2, flip_frac=0.03, min_cos=0.999)
    else:
        compare_with_oracle(tr, orc, hp, rtol_loss=1e-3, grad_rel_l2=1.0, flip_frac=0.2, shallow_only=True)


@pytest.mark.parametrize('tc', [0, 1])
def test_three_iterations(tc):
    """both networks reflect, council flip 2 on / 1 off, StepLR step 2"""
    gold = load_golden('glasses64_n3_b2_reflect_iter3')
    log = []
    _run_cuda_iters(gold, tc, 3, lambda k, t: log.append(([float(v) for v in t.loss_dis_total_s], [float(v) for v in t.loss_gen_total_s])))
    tol = [1e-3, 3e-3, 2e-2] if tc == 0 else [1e-3, 1e-2, 5e-2]
    for k, (dis, gen) in enumerate(log):
        rec = gold['iters'][k]
        for g, r in zip(dis + gen, rec['loss_dis_total'] + rec['loss_gen_total']):
            assert close(g, r, tol[k], 1e-6), (k, g, r)


@pytest.mark.parametrize('tc', [0, 1])
def test_sample_matches_oracle(tc):
    """sample() under reflect: the no-grad decoder reads the upsampled, padded map from cg_reflect_pad(ups) instead of folding the
    upsample into the convolution"""
    from council_gan_b200 import Council_Trainer
    gold = load_golden('glasses64_n2_b2_reflect_recon')
    hp, states, x_a, x_b = setup_case(gold)
    tr = Council_Trainer(hp, 'cuda:0')
    load_states(tr, states)
    tr.ops.set_tensor_core_mode(tc)
    try:
        s = torch.randn(x_a.size(0), hp['gen']['style_dim'], 1, 1, generator=torch.Generator().manual_seed(3))
        out = tr.sample(x_a, x_b, s_a=s, s_b=s, return_mask=False)
        torch.cuda.synchronize()
    finally:
        tr.ops.set_tensor_core_mode(1)
    with padding(hp), torch.no_grad():
        for d, x, (_, second, first, _) in (('a2b', x_a, out[:4]), ('b2a', x_b, out[4:])):
            for i in range(tr.council_size):
                p = states['gen_' + d][i]
                c = co.content_encode(p, hp, x)
                for got, st in ((first, s), (second, co.style_encode(p, hp, x))):
                    want, _ = co.decode(p, hp, c, st, x)
                    mae = (got[i::tr.council_size].cpu() - want).abs().mean().item()
                    assert mae < (2e-5 if tc == 0 else 3e-3), (d, i, mae)


@pytest.mark.parametrize('case', ['glasses64_n2_b2_both', 'm2f64_n4_b2'])
def test_kernels_never_called_when_zero(case):
    """pad_type zero (the shipped configs): neither padding kernel runs in training or sampling"""
    from council_gan_b200 import Council_Trainer
    from council_gan_b200.ops import CudaOps

    def boom(*a, **k):
        raise AssertionError('a reflection-padding kernel was called with pad_type zero')
    gold = load_golden(case)
    hp, _, x_a, x_b = setup_case(gold)
    assert hp['gen']['pad_type'] == hp['dis']['pad_type'] == 'zero'
    tr = Council_Trainer(hp, 'cuda:0')
    saved = CudaOps.reflect_pad, CudaOps.reflect_pad_bwd
    CudaOps.reflect_pad = CudaOps.reflect_pad_bwd = boom
    try:
        tr.dis_update(x_a, x_b, hp)
        tr.dis_council_update(x_a, x_b, hp)
        tr.gen_update(x_a, x_b, hp, gold['iteration'])
        tr.sample(x_a, x_b)
    finally:
        CudaOps.reflect_pad, CudaOps.reflect_pad_bwd = saved
    torch.cuda.synchronize()
