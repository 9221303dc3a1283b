"""council_abs_w on the GPU: the two kernels of csrc/losses.cu (cg_council_abs_fwd / _bwd) against float64 torch, the training step
against the oracle and the unmodified reference's numbers (tests/golden/*_council_abs*.json), the off path, and a trainer without
council discriminators (council_w 0)."""
import os
import random

import pytest
import torch

from common import close, load_golden, setup_case
from test_trainer_council_abs_cpu import ITER3, published, run
from test_trainer_gpu import _run_cuda_iters, run_cuda
from test_trainer_host_cpu import compare_with_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    return CudaOps('cuda:0')


def _peers(G, seed):
    """another member for each g; for G > 2 member 0 is the peer of several members"""
    gen = random.Random(seed)
    return [(g + 1) % G if g == 0 else (0 if g % 2 else gen.choice([k for k in range(G) if k != g])) for g in range(G)]


def _inputs(G, B, H, W, seed, same=()):
    """x_fake [G,B,H,W,4] on multiples of 2^-10 (differences exact in float32) with junk in lane 3 and exact zeros of d; members
    in `same` are copies of their peer's image"""
    gen = torch.Generator().manual_seed(seed)
    x = torch.round((torch.rand(G, B, H, W, 4, generator=gen) * 2 - 1) * 1024) / 1024
    x[..., 3] = 1e6 * torch.rand(G, B, H, W, generator=gen)
    x[1:, :, 1::3, ::2] = x[0, :, 1::3, ::2]
    for g, p in same:
        x[g] = x[p]
    return x.cuda()


def _expect(x_fake, peers, gray, w, numel_scale=1):
    x = x_fake.double()[..., :3]
    xp = x[peers]
    d = x.sum(-1) - xp.sum(-1) if gray else x - xp
    G = d.shape[0]
    sums = d.abs().reshape(G, -1).sum(-1)
    numel = d[0].numel() * numel_scale
    grad = torch.sign(d) * (w / numel)
    return sums, w * sums * numel_scale / numel, grad.unsqueeze(-1).expand(*x.shape) if gray else grad


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


SHAPES = [(2, 1, 1, 1), (2, 2, 7, 5), (3, 1, 33, 17), (4, 2, 64, 64), (5, 3, 9, 130), (8, 1, 45, 77), (8, 3, 64, 96)]


@pytest.mark.parametrize('gray', [False, True])
@pytest.mark.parametrize('shape', SHAPES)
def test_kernels_match_float64(ops, shape, gray):
    G, B, H, W = shape
    peers = _peers(G, seed=G + H)
    same = [(G - 1, peers[G - 1])] if G > 2 else []  # an identical pair: value and gradient exactly 0
    x_fake = _inputs(G, B, H, W, seed=G * 1000 + H, same=same)
    w = 1.5
    sums_want, term, grad = _expect(x_fake, peers, gray, w)
    sums = ops.empty(G)
    ops.council_abs_fwd(x_fake, peers, gray, sums)
    assert torch.allclose(sums.double(), sums_want, rtol=2e-6, atol=1e-6)
    base = torch.arange(1, G + 1, dtype=torch.float32, device='cuda') * 0.75
    total = _prime_total(ops, G, base)
    d_x0 = torch.randn(G, B, H, W, 4, device='cuda')
    d_x, pub = d_x0.clone(), ops.empty(G)
    numel = (1 if gray else 3) * B * H * W
    ops.council_abs_bwd(x_fake, peers, gray, sums, numel, w, total, pub, d_x)
    torch.cuda.synchronize()
    assert torch.allclose(pub.double(), term, rtol=2e-6, atol=1e-7)
    assert torch.allclose(total.double(), base.double() + term, rtol=2e-6, atol=1e-6)
    assert torch.equal(d_x[..., 3], d_x0[..., 3])  # lane 3 untouched
    assert torch.allclose(d_x[..., :3].double(), d_x0[..., :3].double() + grad, rtol=1e-6, atol=1e-7)
    for g, _ in same:
        assert float(sums[g]) == 0 and float(pub[g]) == 0 and torch.equal(d_x[g], d_x0[g])


def test_kernels_global_numel_and_refusals(ops):
    """pass 2 takes the sums and numel of the GLOBAL minibatch (data parallel); bad member counts and peers are refused"""
    G, B, H, W = 4, 2, 16, 16
    peers = [1, 0, 0, 0]
    x_fake = _inputs(G, B, H, W, seed=5)
    for gray in (False, True):
        sums = ops.empty(G)
        ops.council_abs_fwd(x_fake, peers, gray, sums)
        sums *= 2  # as if a second rank had contributed the same sums
        total, pub, d_x = _prime_total(ops, G, torch.zeros(G, device='cuda')), ops.empty(G), torch.zeros(G, B, H, W, 4, device='cuda')
        ops.council_abs_bwd(x_fake, peers, gray, sums, 2 * (1 if gray else 3) * B * H * W, 2.0, total, pub, d_x)
        _, term, grad = _expect(x_fake, peers, gray, 2.0, numel_scale=2)
        assert torch.allclose(pub.double(), term, rtol=2e-6) and torch.allclose(total.double(), term, rtol=2e-6)
        assert torch.allclose(d_x[..., :3].double(), grad, rtol=1e-6, atol=1e-8)
    x9 = _inputs(9, 1, 4, 4, seed=1)
    for x, bad in ((x9, [1, 0, 0, 0, 0, 0, 0, 0, 0]), (x_fake[:1].contiguous(), [0]), (x_fake, [1, 1, 0, 0]), (x_fake, [1, 0, 4, 0]),
                   (x_fake, [1, 0, -1, 0])):
        with pytest.raises(RuntimeError):
            ops.council_abs_fwd(x, bad, False, ops.empty(x.shape[0]))
        with pytest.raises(RuntimeError):
            ops.council_abs_bwd(x, bad, False, ops.zeros(x.shape[0]), 48.0, 1.0, ops.zeros(x.shape[0]), ops.empty(x.shape[0]),
                                torch.zeros_like(x))


def _check_published(tr, rec, rtol):
    ab, ba, _ = published(tr)
    for got, key in ((ab, 'council_loss_ab'), (ba, 'council_loss_ba')):
        assert len(got) == len(rec[key]), (key, got, rec[key])
        for g, r in zip(got, rec[key]):
            assert close(g, r, rtol, 1e-6), (key, g, r)
    assert tr.peers_drawn == rec['peers']


def _wrap_gen_update(fn):
    """run fn with Council_Trainer.gen_update recording the peers it draws in `peers_drawn`"""
    from council_gan_b200 import Council_Trainer
    init = Council_Trainer.gen_update

    def gen_update(self, *a, **k):
        choice, drawn = random.choice, []

        def record(seq):
            j = choice(seq)
            drawn.append(j)
            return j
        random.choice = record
        try:
            return init(self, *a, **k)
        finally:
            random.choice = choice
            self.peers_drawn = drawn
    Council_Trainer.gen_update = gen_update
    try:
        return fn()
    finally:
        Council_Trainer.gen_update = init


@pytest.mark.parametrize('case', ['glasses64_n2_b2_council_abs', 'm2f64_n4_b2_council_abs_nodc', 'anime64_n3_b2_council_abs_gray',
                                  'glasses64_n2_b2_council_abs_early'])
@pytest.mark.parametrize('tc', [0, 1])
def test_iteration_matches_oracle_and_golden(case, tc):
    """the gates of test_trainer_gpu.check_iteration, against the oracle extended with the term"""
    gold = load_golden(case)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    orc, hp = run(gold, torch.float32)
    tr, _ = _wrap_gen_update(lambda: run_cuda(gold, tc))
    N = tr.council_size
    for i in range(N):
        assert close(float(tr.loss_dis_total_s[i]), gold['loss_dis_total'][i], 1e-3), ('dis', i)
        assert close(float(tr.loss_gen_total_s[i]), gold['loss_gen_total'][i], 1e-3), ('gen', i)
        if gold['dis_council_ran']:
            assert close(float(tr.loss_dis_council_total_s[i]), gold['loss_dis_council_total'][i], 1e-3), ('disc', i)
    for d in orc.dirs:
        for i in range(N):
            xf = tr.ops.nhwc_to_nchw(tr._last_fw[d]['x_fake'][i], 3).cpu()
            mae = (xf - orc.x_fake_gen[d][i].detach()).abs().mean().item()
            assert mae < (2e-4 if tc == 0 else 3e-3), ('pixel MAE', d, i, mae)
    if tc == 0:
        compare_with_oracle(tr, orc, hp, rtol_loss=1e-3, grad_rel_l2=3e-2, flip_frac=0.03, min_cos=0.999)
    else:
        compare_with_oracle(tr, orc, hp, rtol_loss=1e-3, grad_rel_l2=1.0, flip_frac=0.2, shallow_only=True)
    _check_published(tr, gold, 1e-3)


@pytest.mark.parametrize('tc', [0, 1])
def test_three_iterations_gate_and_random_stream(tc):
    """flip 2 on / 1 off: the term and dis_council_update's draws interleave in one `random` stream, then the gate closes"""
    gold = load_golden(ITER3)
    log = []
    _wrap_gen_update(lambda: _run_cuda_iters(gold, tc, 3, lambda k, t: log.append((published(t), [float(v) for v in t.loss_gen_total_s]))))
    tol = [1e-3, 3e-3, 2e-2] if tc == 0 else [1e-3, 1e-2, 5e-2]
    for k, ((ab, ba, peers), gen) in enumerate(log):
        rec = gold['iters'][k]
        assert peers == rec['peers'] and len(peers) == [3, 3, 0][k]
        for g, r in zip(ab + ba + gen, rec['council_loss_ab'] + rec['council_loss_ba'] + rec['loss_gen_total']):
            assert close(g, r, tol[k], 1e-6), (k, g, r)


@pytest.mark.parametrize('case', ['glasses64_n2_b2_early', 'glasses64_n2_b2_both', 'anime64_n3_b2', 'glasses64_n2_b2_council_abs_early'])
def test_ops_never_called_when_off(case):
    """council_abs_w 0 (the shipped configs) or the council gate closed: neither kernel runs and gen_update draws nothing"""
    from council_gan_b200 import Council_Trainer
    from council_gan_b200.ops import CudaOps

    def boom(*a, **k):
        raise AssertionError('council_abs kernel called while the term is off')
    gold = load_golden(case)
    hp, _, x_a, x_b = setup_case(gold)
    tr = Council_Trainer(hp, 'cuda:0')
    saved = CudaOps.council_abs_fwd, CudaOps.council_abs_bwd
    CudaOps.council_abs_fwd = CudaOps.council_abs_bwd = boom
    try:
        tr.dis_update(x_a, x_b, hp)
        before = random.getstate()
        tr.gen_update(x_a, x_b, hp, gold['iteration'])
        assert random.getstate() == before
    finally:
        CudaOps.council_abs_fwd, CudaOps.council_abs_bwd = saved
    torch.cuda.synchronize()


def test_trainer_without_council_discriminators(tmp_path):
    """council_w 0: no council-discriminator network, dis_council_update launches nothing, and save() writes no dis_council file or
    optimiser entry"""
    from council_gan_b200 import Council_Trainer
    gold = load_golden('m2f64_n4_b2_council_abs_nodc')
    hp, _, x_a, x_b = setup_case(gold)
    tr = Council_Trainer(hp, 'cuda:0')
    assert not tr.do_dis_council and not any(k.startswith('dis_council') for k in tr._nets)
    assert not hasattr(tr, 'dis_council_a2b_s') and not hasattr(tr, 'dis_council_b2a_s')
    tr.dis_update(x_a, x_b, hp)
    torch.cuda.synchronize()
    n0 = tr.ops.launch_count()
    tr.dis_council_update(x_a, x_b, hp)
    assert tr.ops.launch_count() == n0
    tr.gen_update(x_a, x_b, hp, gold['iteration'])
    tr.save(str(tmp_path), 0)
    files = os.listdir(tmp_path)
    assert files and not any('dis_council' in f for f in files)
    for i in range(tr.council_size):
        assert set(torch.load(os.path.join(tmp_path, 'optimizer_%d.pt' % i))) == {'gen', 'dis'}
