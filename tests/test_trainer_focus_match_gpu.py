"""Focus-loss matching (do_w_loss_matching_focus) on the GPU: cg_gen_loss_bwd with the matching on against its float64 restatement
(tests/test_trainer_focus_match_cpu.py) over random rings and heads, the training step against the unmodified reference's numbers
(tests/golden/*focus_match*.json), the switch as a no-op with the focus gate closed, and no extra launch."""
import pytest
import torch

from common import close, load_golden, setup_case
from test_trainer_focus_match_cpu import CASES, ITER3, TorchOps, check_focus, check_lists, record
from test_trainer_gpu import _run_cuda_iters, run_cuda

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    return CudaOps('cuda:0')


@pytest.mark.parametrize('G, B, H, W, hist', [(1, 1, 8, 8, 1), (3, 2, 17, 9, 2), (8, 2, 64, 64, 5), (5, 1, 33, 40, 40)])
@pytest.mark.parametrize('small', [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize('b2a', [False, True])
def test_gen_loss_bwd_matching_matches_float64(ops, G, B, H, W, hist, small, b2a):
    gen = torch.Generator().manual_seed(G * 1000 + H * 10 + hist + 7 * b2a + 3 * small[0])
    mask = torch.zeros(G, B, H, W, 4)
    mask[..., :3] = torch.rand(G, B, H, W, 3, generator=gen)
    mask[..., 3] = 1e6  # junk in lane 3
    cl = [torch.randn(G, 1, 5, 5, generator=gen).abs() + 0.5]
    numel = float(B * 3 * H * W)
    hp = {'world': 1, 'hist_size': hist, 'head_gan': int(torch.randint(0, hist + 1, (1,), generator=gen)),
          'head_council': int(torch.randint(0, hist + 1, (1,), generator=gen)), 'gan_on': 1, 'council_on': 1, 'focus_on': 1,
          'matching': 1, 'small_abs': int(small[0]), 'small_square': int(small[1]), 'gan_w': 24.0, 'council_w': 12.0, 'w01': 10.0,
          'wtot': 57.0, 'wtv': 2.2, 'numel': numel, 'focus_matching': 1,
          'head_focus': int(torch.randint(0, hist + 1, (1,), generator=gen)),
          'head_focus01': int(torch.randint(0, hist + 1, (1,), generator=gen))}
    rings = [torch.rand(G, hist + 1, generator=gen, dtype=torch.float64) + 0.2 for _ in range(4)]
    scal = torch.empty(G, 6)
    ref = TorchOps('cpu', torch.float32)
    ref.gen_loss_fwd([torch.randn(G, 1, 3, 3, generator=gen)], cl, mask, 0.5, 0.01, 1.0, scal)
    src = torch.zeros(G, 8)
    src[:, 3] = torch.rand(G, generator=gen) if b2a else 0
    want_rings = [r.clone() for r in rings]
    want_total, want_pub, want_w = torch.zeros(G), torch.zeros(G, 8), torch.zeros(G, 2)
    want_dcl, want_dm = ref.gen_loss_bwd(cl, mask, 0.5, 0.01, scal, hp, want_rings[0], want_rings[1], want_total, False, want_pub, True,
                                         hist_focus=want_rings[2], hist_focus01=want_rings[3], focus_src=src if b2a else None,
                                         focus_w=want_w)
    dev_rings = [r.cuda() for r in rings]
    total, pub, fw = ops.empty(G), ops.empty(G, 8), ops.empty(G, 2)
    d_cl, d_mask = ops.gen_loss_bwd([c.cuda() for c in cl], mask.cuda(), 0.5, 0.01, scal.cuda(), hp, dev_rings[0], dev_rings[1], total,
                                    False, pub, True, hist_focus=dev_rings[2], hist_focus01=dev_rings[3],
                                    focus_src=src.cuda() if b2a else None, focus_w=fw)
    torch.cuda.synchronize()
    for got, want in zip(dev_rings, want_rings):  # appends: float32 values, or the cross-direction source as it is
        assert torch.allclose(got.cpu(), want, rtol=1e-12, atol=0), (got, want)
    assert torch.allclose(fw.cpu().double(), want_w.double(), rtol=2e-6, atol=0)
    assert torch.allclose(pub.cpu(), want_pub, rtol=2e-6, atol=1e-7)
    assert torch.allclose(total.cpu(), want_total, rtol=2e-6, atol=1e-7)
    assert torch.allclose(d_cl[0].cpu(), want_dcl[0], rtol=2e-6, atol=1e-9)
    scale = want_dm.abs().max().item()
    assert (d_mask.cpu() - want_dm).abs().max().item() <= 2e-5 * scale
    assert torch.all(d_mask[..., 3] == 0)


def test_gen_loss_bwd_refuses_matching_without_rings(ops):
    G = 2
    mask = ops.zeros(G, 1, 4, 4, 4)
    hp = {'world': 1, 'hist_size': 2, 'focus_on': 1, 'w01': 1.0, 'wtot': 1.0, 'small_square': 1, 'numel': 48.0, 'focus_matching': 1}
    rings = torch.ones(G, 3, dtype=torch.float64, device='cuda')
    with pytest.raises(RuntimeError):
        ops.gen_loss_bwd([], mask, 0.5, 0.01, ops.zeros(G, 6), hp, rings, rings, ops.empty(G), False, ops.empty(G, 8), True,
                         hist_focus=rings.clone())
    with pytest.raises(RuntimeError):
        ops.gen_loss_bwd([], mask, 0.5, 0.01, ops.zeros(G, 6), dict(hp, head_focus=3), rings, rings, ops.empty(G), False,
                         ops.empty(G, 8), True, hist_focus=rings.clone(), hist_focus01=rings.clone())


@pytest.mark.parametrize('case', CASES)
def test_iteration_matches_golden(case):
    gold = load_golden(case)
    tr, _ = run_cuda(gold, 0)
    for i in range(tr.council_size):
        assert close(float(tr.loss_dis_total_s[i]), gold['loss_dis_total'][i], 1e-3), ('dis', i)
        assert close(float(tr.loss_gen_total_s[i]), gold['loss_gen_total'][i], 1e-3), ('gen', i)
    check_focus(record(tr)['dirs'], gold['focus'], 1e-3)


@pytest.mark.parametrize('case', ITER3)
def test_three_iterations_match_golden(case):
    """histories of 2 entries that wrap; with both directions b2a's mask-total history takes a2b's scaled term"""
    gold = load_golden(case)
    log = []
    _run_cuda_iters(gold, 0, 3, lambda k, t: log.append(record(t)))
    for k, got in enumerate(log):
        rec = gold['iters'][k]
        tol = [1e-3, 3e-3, 2e-2][k]
        check_lists(got['dis'], rec['loss_dis_total'], tol, 1e-6)
        check_lists(got['gen'], rec['loss_gen_total'], tol, 1e-6)
        # the zero-one histories sum 1 / (|m - 0.5| + 0.01) over masks near 0.5, which amplifies the fp32 noise Adam's steps carry:
        # measured 4.6e-3 in the second step and 2.5e-2 in the third
        check_focus(got['dirs'], rec['focus'], [1e-3, 1e-2, 5e-2][k])


def _step(hp_edit):
    from council_gan_b200 import Council_Trainer
    gold = load_golden('glasses64_n2_b2_focus_match_closed')
    hp, states, x_a, x_b = setup_case(gold)
    hp_edit(hp)
    import council_oracle as co
    from test_trainer_host_cpu import load_states
    co.seed_all(hp['random_seed'])
    tr = Council_Trainer(hp, 'cuda:0')
    load_states(tr, states)
    co.seed_all(gold['rng_seed'])
    tr.dis_update(x_a, x_b, hp)
    tr.dis_council_update(x_a, x_b, hp)
    n0 = tr.ops.launch_count()
    tr.gen_update(x_a, x_b, hp, hp['iteration'])
    n = tr.ops.launch_count() - n0
    tr.synchronize()
    torch.cuda.synchronize()
    return tr, n


def test_gate_closed_is_bit_identical():
    runs = []
    for on in (True, False):
        tr, _ = _step(lambda hp: hp['focus_loss'].update(do_w_loss_matching_focus=on))
        runs.append(([float(v) for v in tr.loss_gen_total_s], {k: n.bank.data.clone() for k, n in tr._nets.items()}))
    assert runs[0][0] == runs[1][0]
    for k, v in runs[0][1].items():
        assert torch.equal(v, runs[1][1][k]), k


def test_no_extra_launch():
    def edit(on):
        def f(hp):
            hp['iteration'] = 20001  # focus gate open
            hp['do_b2a'] = True
            hp['focus_loss']['do_w_loss_matching_focus'] = on
        return f
    counts = [_step(edit(on))[1] for on in (True, False)]
    assert counts[0] == counts[1], counts
