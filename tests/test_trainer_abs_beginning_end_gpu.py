"""abs_beginning_end on the GPU: the two kernels of csrc/losses.cu (cg_abs_beginning_end_fwd / _bwd) against float64 torch, the
training step against the oracle and the unmodified reference's numbers (tests/golden/*_abs*.json), and the off path."""
import pytest
import torch

from common import close, load_golden
from test_trainer_abs_beginning_end_cpu import published, run, setup_inputs
from test_trainer_gpu import _run_cuda_iters, run_cuda
from test_trainer_host_cpu import compare_with_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    return CudaOps('cuda:0')


def _inputs(G, B, H, W, kind, seed):
    """x_fake [G,B,H,W,4], x [1,B,H,W,4] (lane 3 carries junk that must be ignored)."""
    gen = torch.Generator().manual_seed(seed)
    q = lambda t: torch.round(t * 1024) / 1024  # multiples of 2^-10: x + d and x_fake - x are exact in float32
    x = q(torch.rand(1, B, H, W, 4, generator=gen) * 2 - 1)
    if kind == 'tie':  # |d| in {0, 1}: sum |d| == sum d^2 exactly -> L2
        d = torch.randint(-1, 2, (G, B, H, W, 4), generator=gen).float()
    elif kind == 'zero':  # x_fake == x bit for bit (a saturated mask): value 0, gradient sign(0) = 0
        d = torch.zeros(G, B, H, W, 4)
    else:
        scale = {'l1': 0.5, 'l2': 3.0}[kind]
        d = q((torch.rand(G, B, H, W, 4, generator=gen) * 2 - 1) * scale)
        d[:, :, 1::3, ::2] = 0  # exact zeros inside a live branch
    return (x + d).cuda(), x.cuda()


def _expect(x_fake, x, weights):
    d = (x_fake.double() - x.double())[..., :3]
    G = d.shape[0]
    numel = d[0].numel()
    s1, s2 = d.abs().reshape(G, -1).sum(-1), (d * d).reshape(G, -1).sum(-1)
    l1, l2 = s1 / numel, s2 / numel
    use_l1 = l1 > l2
    val = torch.where(use_l1, l1, l2)
    w = torch.tensor(weights, dtype=torch.float64, device=d.device)
    coef = (w / numel).view(G, 1, 1, 1, 1)
    grad = torch.where(use_l1.view(G, 1, 1, 1, 1), coef * torch.sign(d), coef * 2 * d)
    return s1, s2, val, w * val, grad, use_l1


def _prime_total(ops, G, base):
    """gen_loss_bwd with only the adversarial term on: total[g] = base[g] and the direction accumulator holds it."""
    scal = torch.zeros(G, 6, device='cuda')
    scal[:, 0] = base
    hp = {'world': 1, 'hist_size': 1, 'head_gan': 0, 'head_council': 0, 'gan_on': 1, 'council_on': 0, 'focus_on': 0, 'matching': 0,
          'small_abs': 0, 'small_square': 0, 'gan_w': 1.0, 'council_w': 0.0, 'w01': 0.0, 'wtot': 0.0, 'wtv': 0.0, 'numel': 1.0}
    ring = torch.ones(G, 2, dtype=torch.float64, device='cuda')
    total, pub = ops.empty(G), ops.empty(G, 8)
    ops.gen_loss_bwd([], None, 0.5, 0.01, scal, hp, ring, ring.clone(), total, False, pub, False)
    return total


SHAPES = [(1, 1, 1, 1), (2, 2, 7, 5), (3, 1, 33, 17), (4, 2, 64, 64), (8, 1, 45, 77), (8, 3, 64, 96)]


@pytest.mark.parametrize('kind', ['l1', 'l2', 'tie', 'zero'])
@pytest.mark.parametrize('shape', SHAPES)
def test_kernels_match_float64(ops, shape, kind):
    G, B, H, W = shape
    x_fake, x = _inputs(G, B, H, W, kind, seed=G * 1000 + H)
    weights = [0.0 if g == G - 1 and G > 2 else 0.25 * (g + 1) for g in range(G)]  # the last member's gate closed
    s1, s2, val, wval, grad, use_l1 = _expect(x_fake, x, weights)
    if kind in ('l1', 'l2'):
        assert bool((use_l1 == (kind == 'l1')).all())
    sums = ops.empty(G, 2)
    ops.abs_beginning_end_fwd(x_fake, x, sums)
    assert torch.allclose(sums[:, 0].double(), s1, rtol=2e-6, atol=1e-6) and torch.allclose(sums[:, 1].double(), s2, rtol=2e-6, atol=1e-6)
    if kind == 'tie':
        assert torch.equal(sums[:, 0], sums[:, 1])
    base = torch.arange(1, G + 1, dtype=torch.float32, device='cuda') * 0.75
    total = _prime_total(ops, G, base)
    d_x0 = torch.randn(G, B, H, W, 4, device='cuda')
    d_x, pub = d_x0.clone(), ops.empty(G)
    ops.abs_beginning_end_bwd(x_fake, x, sums, 3 * B * H * W, weights, total, pub, d_x)
    torch.cuda.synchronize()
    assert torch.allclose(pub.double(), val, rtol=2e-6, atol=1e-7)
    assert torch.allclose(total.double(), base.double() + wval, rtol=2e-6, atol=1e-6)
    assert torch.equal(d_x[..., 3], d_x0[..., 3])
    assert torch.allclose(d_x[..., :3].double(), d_x0[..., :3].double() + grad, rtol=1e-6, atol=1e-7)
    for g, w in enumerate(weights):
        if w == 0:
            assert torch.equal(d_x[g], d_x0[g]) and float(total[g]) == float(base[g])
    if kind == 'zero':
        assert float(pub.abs().max()) == 0 and torch.equal(d_x, d_x0)


def test_kernels_global_numel_and_member_limit(ops):
    """pass 2 takes the sums and numel of the GLOBAL minibatch (data parallel); G above the member limit is refused."""
    G, B, H, W = 2, 2, 16, 16
    x_fake, x = _inputs(G, B, H, W, 'l1', seed=5)
    sums = ops.empty(G, 2)
    ops.abs_beginning_end_fwd(x_fake, x, sums)
    sums *= 2  # as if a second rank had contributed the same sums
    total, pub, d_x = _prime_total(ops, G, torch.zeros(G, device='cuda')), ops.empty(G), torch.zeros(G, B, H, W, 4, device='cuda')
    ops.abs_beginning_end_bwd(x_fake, x, sums, 2 * 3 * B * H * W, [1.0, 2.0], total, pub, d_x)
    _, _, val, wval, grad, _ = _expect(x_fake, x, [1.0, 2.0])
    assert torch.allclose(pub.double(), val, rtol=2e-6) and torch.allclose(total.double(), wval, rtol=2e-6)
    assert torch.allclose(d_x[..., :3].double(), grad / 2, rtol=1e-6, atol=1e-8)
    x9, xs = _inputs(9, 1, 4, 4, 'l1', seed=1)
    with pytest.raises(RuntimeError):
        ops.abs_beginning_end_fwd(x9, xs, ops.empty(9, 2))


def _check_published(tr, rec, rtol):
    a, b, w = published(tr)
    for got, key in ((a, 'loss_gen_beginning_end_a_ab'), (b, 'loss_gen_beginning_end_b_ba')):
        assert len(got) == len(rec[key]), (key, got, rec[key])
        for g, r in zip(got, rec[key]):
            assert close(g, r, rtol, 1e-6), (key, g, r)
    assert w == rec['abs_beginning_end_w_conf']


@pytest.mark.parametrize('case', ['glasses64_n2_b2_abs', 'anime64_n3_b2_abs', 'glasses64_n2_b2_both_abs'])
@pytest.mark.parametrize('tc', [0, 1])
def test_iteration_matches_oracle_and_golden(case, tc):
    """the gates of test_trainer_gpu.check_iteration, against the oracle extended with the term"""
    gold = load_golden(case)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    orc, hp = run(gold, torch.float32)
    tr, _ = run_cuda(gold, tc)
    d0 = orc.dirs[0]
    N = tr.council_size
    for i in range(N):
        assert close(float(tr.loss_dis_total_s[i]), gold['loss_dis_total'][i], 1e-3), ('dis', i)
        assert close(float(tr.loss_gen_total_s[i]), gold['loss_gen_total'][i], 1e-3), ('gen', i)
        if gold['dis_council_ran']:
            assert close(float(tr.loss_dis_council_total_s[i]), gold['loss_dis_council_total'][i], 1e-3), ('disc', i)
    for i in range(N):
        xf = tr.ops.nhwc_to_nchw(tr._last_fw[d0]['x_fake'][i], 3).cpu()
        mae = (xf - orc.x_fake_gen[d0][i].detach()).abs().mean().item()
        assert mae < (2e-4 if tc == 0 else 3e-3), ('pixel MAE', i, mae)
    if tc == 0:
        compare_with_oracle(tr, orc, hp, rtol_loss=1e-3, grad_rel_l2=3e-2, flip_frac=0.03, min_cos=0.999)
    else:
        no_focus = case == 'anime64_n3_b2_abs'  # focus weights 0: gradient direction asserted, as check_iteration does
        compare_with_oracle(tr, orc, hp, rtol_loss=1e-3, grad_rel_l2=1.0, flip_frac=0.2, min_cos=0.98 if no_focus else None,
                            shallow_only=True)
    _check_published(tr, gold, 1e-3)


@pytest.mark.parametrize('tc', [0, 1])
def test_l2_branch_iteration_matches_golden(tc):
    """inputs of +-3 (the fixture's input_scale): the L2 branch, against the reference's numbers"""
    from council_gan_b200 import Council_Trainer
    import council_oracle as co
    from test_trainer_host_cpu import load_states
    gold = load_golden('glasses64_n2_b2_abs_l2')
    hp, states, x_a, x_b = setup_inputs(gold)
    co.seed_all(hp['random_seed'])
    tr = Council_Trainer(hp, 'cuda:0')
    tr.ops.set_tensor_core_mode(tc)
    load_states(tr, states)
    co.seed_all(gold['rng_seed'])
    tr.dis_update(x_a, x_b, hp)
    tr.dis_council_update(x_a, x_b, hp)
    tr.gen_update(x_a, x_b, hp, gold['iteration'])
    torch.cuda.synchronize()
    tr.ops.set_tensor_core_mode(1)
    # TF32: inputs of +-3 triple the absolute rounding error of the image-side layers, and the L2 branch doubles the relative
    # error of x_fake - x (the tensor-core run lands 1.0e-3 from the reference on member 0's total)
    rtol = 1e-3 if tc == 0 else 2e-3
    for i in range(tr.council_size):
        assert close(float(tr.loss_dis_total_s[i]), gold['loss_dis_total'][i], 1e-3), ('dis', i)
        assert close(float(tr.loss_gen_total_s[i]), gold['loss_gen_total'][i], rtol), ('gen', i)
    _check_published(tr, gold, rtol)


@pytest.mark.parametrize('tc', [0, 1])
def test_decay_across_iterations(tc):
    """the weight crosses 0.005 in the third call: member 0 only, then the term stays off"""
    gold = load_golden('glasses64_n2_b2_abs_decay')
    log = []
    _run_cuda_iters(gold, tc, 4, lambda k, t: log.append((published(t), [float(v) for v in t.loss_gen_total_s])))
    tol = [1e-3, 3e-3, 2e-2, 2e-2] if tc == 0 else [1e-3, 1e-2, 5e-2, 5e-2]
    for k, ((a, b, w), gen) in enumerate(log):
        rec = gold['iters'][k]
        assert len(a) == len(rec['loss_gen_beginning_end_a_ab']) == [2, 2, 1, 0][k] and b == [0.0] * len(a)
        assert w == rec['abs_beginning_end_w_conf']
        for g, r in zip(a + gen, rec['loss_gen_beginning_end_a_ab'] + rec['loss_gen_total']):
            assert close(g, r, tol[k]), (k, g, r)


def test_ops_never_called_when_off():
    """abs_beginning_end 0 (every shipped config), and a term whose weight has decayed: no launch of either kernel"""
    from council_gan_b200 import Council_Trainer
    from council_gan_b200.ops import CudaOps

    def boom(*a, **k):
        raise AssertionError('abs_beginning_end kernel called while the term is off')
    for case, it in (('glasses64_n2_b2_early', None), ('glasses64_n2_b2_abs_decay', 9)):
        gold = load_golden(case)
        hp, _, x_a, x_b = setup_inputs(gold)
        tr = Council_Trainer(hp, 'cuda:0')
        if it is not None:
            tr.abs_beginning_end_w_conf = 0.5 ** 8  # the state after the crossing call
        saved = CudaOps.abs_beginning_end_fwd, CudaOps.abs_beginning_end_bwd
        CudaOps.abs_beginning_end_fwd = CudaOps.abs_beginning_end_bwd = boom
        try:
            tr.dis_update(x_a, x_b, hp)
            tr.gen_update(x_a, x_b, hp, it or gold['iteration'])
        finally:
            CudaOps.abs_beginning_end_fwd, CudaOps.abs_beginning_end_bwd = saved
        torch.cuda.synchronize()
        if it is None:
            assert not hasattr(tr, 'loss_gen_beginning_end_a_ab_s')
        else:
            assert tr.loss_gen_beginning_end_a_ab_s == [] and tr.loss_gen_beginning_end_b_ba_s == []
