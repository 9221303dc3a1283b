"""do_Dis_only_gray, useRandomGen and useRandomDis on the GPU: the three kernels of csrc/pointwise.cu (cg_gather_images_gray,
cg_gray_fold, cg_gather_members) against float64 torch, the training step against the oracle and the unmodified reference's numbers
(tests/golden/*gray*.json, *random_pairing*.json, *dis_options*.json), and the off path."""
import ctypes as C

import numpy as np
import pytest
import torch

from common import close, load_golden, setup_case
from make_golden_dis_options import with_draws
from test_trainer_dis_options_cpu import CASES, ITER3, _record, run
from test_trainer_gpu import _run_cuda_iters, run_cuda
from test_trainer_host_cpu import compare_with_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    from council_gan_b200.ops import CudaOps
    return CudaOps('cuda:0')


def _pools(S0, S1, H, W, seed):
    """two image pools [S,H,W,4] with junk in lane 3"""
    gen = torch.Generator().manual_seed(seed)
    p = torch.rand(S0 + S1, H, W, 4, generator=gen) * 2 - 1
    p[..., 3] = 1e6 * torch.rand(S0 + S1, H, W, generator=gen)
    return p[:S0].contiguous().cuda(), p[S0:].contiguous().cuda()


@pytest.mark.parametrize('shape', [(1, 1, 1, 1), (2, 2, 7, 5), (4, 4, 33, 17), (4, 16, 64, 64), (8, 6, 9, 130)])
def test_gather_images_gray_matches_float64(ops, shape):
    G, Bt, H, W = shape
    p0, p1 = _pools(3 * Bt, Bt, H, W, seed=G * 100 + H)
    gen = torch.Generator().manual_seed(H)
    idx = torch.randint(0, 4 * Bt, (G, Bt), generator=gen, dtype=torch.int32)  # slots in both pools, repeats included
    y = ops.gather_images_gray((p0, p1), idx.cuda(), G, Bt)
    pool = torch.cat((p0, p1)).double()[idx.long()]
    m = pool[..., :3].sum(-1) / 3
    assert torch.allclose(y[..., :3].double(), m.unsqueeze(-1).expand(*m.shape, 3), rtol=0, atol=3e-7)
    assert torch.equal(y[..., 0], y[..., 1]) and torch.equal(y[..., 0], y[..., 2])
    assert torch.all(y[..., 3] == 0)
    # the reference's float32 order: sum, then a true division
    want = (torch.cat((p0, p1))[idx.long().cuda()][..., :3].sum(-1) / 3)
    assert (y[..., 0] - want).abs().max().item() <= 1.2e-7 * max(1.0, want.abs().max().item())


def test_gather_images_gray_refuses_x_in(ops):
    p0, _ = _pools(2, 1, 4, 4, seed=1)
    idx = torch.zeros(1, 2, dtype=torch.int32, device='cuda')
    y = ops.empty(1, 2, 4, 4, 8)
    rc = ops.lib.cg_gather_images_gray(p0.data_ptr(), 2, None, idx.data_ptr(), p0.data_ptr(), y.data_ptr(), 1, 2, 2, 16,
                                       ops._stream())
    assert rc != 0 and b'x_in' in ops.lib.cg_last_error()


@pytest.mark.parametrize('shape', [(1, 1, 1, 1), (3, 2, 17, 9), (4, 8, 64, 64)])
def test_gray_fold_matches_float64(ops, shape):
    G, B, H, W = shape
    gen = torch.Generator().manual_seed(G + H)
    d0 = torch.randn(G, B, H, W, 4, generator=gen).cuda()
    d = d0.clone()
    ops.gray_fold(d)
    scale = d0[..., :3].abs().max().item()  # the sum may cancel: rounding is bounded by the size of its terms
    want = (d0[..., :3].double() / 3).sum(-1)
    assert torch.allclose(d[..., :3].double(), want.unsqueeze(-1).expand(*want.shape, 3), rtol=0, atol=2.4e-7 * scale)
    assert torch.equal(d[..., 3], d0[..., 3])  # lane 3 untouched
    # autograd of the reference's conversion, float32
    x = torch.zeros(G * B, 3, H, W, device='cuda', requires_grad=True)
    (torch.sum(x, 1).unsqueeze(1).repeat(1, 3, 1, 1) / 3).backward(d0[..., :3].permute(0, 1, 4, 2, 3).reshape(G * B, 3, H, W))
    g = x.grad.reshape(G, B, 3, H, W).permute(0, 1, 3, 4, 2)
    assert (d[..., :3] - g).abs().max().item() <= 2.4e-7 * scale


def _bank(ops, G, seed):
    """a discriminator-sized parameter bank: segment lengths that are and are not multiples of 4, junk between segments"""
    from council_gan_b200.networks import ParamBank
    entries = [('w%d' % k, shape) for k, shape in enumerate([(64, 4, 4, 4), (1,), (3,), (128, 4, 4, 64), (5, 7), (1, 1, 1, 512)])]
    src, dst = ParamBank(ops, G, entries, trainable=False), ParamBank(ops, G, entries, trainable=False)
    gen = torch.Generator().manual_seed(seed)
    src.data.copy_(torch.randn(src.total, generator=gen))
    dst.data.fill_(-7.0)
    return src, dst


@pytest.mark.parametrize('member_map', [[0], [1, 0], [0, 0, 0], [2, 3, 2, 3], [0, 3, 1, 0], [7, 0, 7, 3, 4, 5, 6, 1]])
def test_gather_members_matches_reference(ops, member_map):
    """repeats, self-pairs and members no one draws"""
    G = len(member_map)
    src, dst = _bank(ops, G, seed=G)
    ops.gather_members(src.data, dst.data, src.member_segments(), member_map)
    covered = torch.zeros(src.total, dtype=torch.bool, device='cuda')
    for name in src.table:
        assert torch.equal(dst.p(name), src.p(name)[member_map]), name
        off, _, n = src.table[name]
        covered[off:off + n] = True
    assert torch.all(dst.data[~covered] == -7.0)  # the padding between segments is not written


def test_gather_members_refusals(ops):
    src, dst = _bank(ops, 4, seed=1)
    segs = src.member_segments()
    for bad in ([0, 1, 2, 4], [0, -1, 0, 0]):
        with pytest.raises(RuntimeError):
            ops.gather_members(src.data, dst.data, segs, bad)
    src9, dst9 = _bank(ops, 9, seed=2)
    with pytest.raises(RuntimeError):
        ops.gather_members(src9.data, dst9.data, src9.member_segments(), list(range(9)))
    with pytest.raises(RuntimeError):
        ops.gather_members(src.data, dst.data, [(2, 3)], [0, 1, 2, 3])  # a segment start that is not 16-byte aligned
    with pytest.raises(RuntimeError):
        ops.gather_members(src.data, dst.data, segs * 11, [0, 1, 2, 3])  # more segments than the parameter struct holds
    n0 = (C.c_int64 * 1)(0)
    assert ops.lib.cg_gather_members(src.data.data_ptr(), dst.data.data_ptr(), n0, n0, 1, None, 4, ops._stream()) != 0


def _wrap_updates(fn):
    """run fn with Council_Trainer's dis_update / gen_update recording their numpy draws in `dis_draws` / `gen_draws`"""
    from council_gan_b200 import Council_Trainer
    init = Council_Trainer.dis_update, Council_Trainer.gen_update

    def dis_update(self, *a, **k):
        sink = [None]
        try:
            return with_draws(init[0], sink)(self, *a, **k)
        finally:
            self.dis_draws = sink[0]

    def gen_update(self, *a, **k):
        sink = [None]
        try:
            return with_draws(init[1], sink)(self, *a, **k)
        finally:
            self.gen_draws = sink[0]
    Council_Trainer.dis_update, Council_Trainer.gen_update = dis_update, gen_update
    try:
        return fn()
    finally:
        Council_Trainer.dis_update, Council_Trainer.gen_update = init


@pytest.mark.parametrize('case', CASES)
@pytest.mark.parametrize('tc', [0, 1])
def test_iteration_matches_oracle_and_golden(case, tc):
    """the gates of test_trainer_gpu.check_iteration, against the oracle extended with the switches"""
    gold = load_golden(case)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    orc, hp = run(gold, torch.float32)
    tr, _ = _wrap_updates(lambda: run_cuda(gold, tc))
    assert tr.dis_draws == gold['dis_draws'] == orc.dis_draws and tr.gen_draws == gold['gen_draws'] == orc.gen_draws
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


@pytest.mark.parametrize('tc', [0, 1])
def test_three_iterations_all_switches(tc):
    """both directions, all three switches, flip 2 on / 1 off: both updates' numpy draws interleave over the iterations while the loss
    histories evolve"""
    gold = load_golden(ITER3)
    log = []
    _wrap_updates(lambda: _run_cuda_iters(gold, tc, 3, lambda k, t: log.append(_record(t))))
    tol = [1e-3, 3e-3, 2e-2] if tc == 0 else [1e-3, 1e-2, 5e-2]
    for k, (dis, gen, dd, gd) in enumerate(log):
        rec = gold['iters'][k]
        assert dd == rec['dis_draws'] and gd == rec['gen_draws']
        for g, r in zip(dis + gen, rec['loss_dis_total'] + rec['loss_gen_total']):
            assert close(g, r, tol[k], 1e-6), (k, g, r)


@pytest.mark.parametrize('case', ['glasses64_n2_b2_early', 'glasses64_n2_b2_both', 'anime64_n3_b2', 'm2f64_n4_b2'])
def test_ops_never_called_when_off(case):
    """the switches off (the shipped configs): none of the three kernels runs and neither update draws from numpy"""
    from council_gan_b200 import Council_Trainer
    from council_gan_b200.ops import CudaOps

    def boom(*a, **k):
        raise AssertionError('a gray-scale / random-pairing kernel was called while the switches are off')
    gold = load_golden(case)
    hp, _, x_a, x_b = setup_case(gold)
    assert not (hp['dis']['do_Dis_only_gray'] or hp['dis']['useRandomGen'] or hp['gen']['useRandomDis'])
    tr = Council_Trainer(hp, 'cuda:0')
    saved = CudaOps.gather_images_gray, CudaOps.gray_fold, CudaOps.gather_members
    CudaOps.gather_images_gray = CudaOps.gray_fold = CudaOps.gather_members = boom
    try:
        before = np.random.get_state()
        tr.dis_update(x_a, x_b, hp)
        tr.dis_council_update(x_a, x_b, hp)
        tr.gen_update(x_a, x_b, hp, gold['iteration'])
        after = np.random.get_state()
        assert all(np.array_equal(a, b) for a, b in zip(before, after))
    finally:
        CudaOps.gather_images_gray, CudaOps.gray_fold, CudaOps.gather_members = saved
    torch.cuda.synchronize()
    assert tr._dis_pick == {}


def test_scratch_bank_is_allocated_once():
    """useRandomDis: one scratch bank per direction for the trainer's life, so its address (a key of the tensor-map cache) is stable"""
    gold = load_golden(ITER3)
    ptrs = []
    _wrap_updates(lambda: _run_cuda_iters(gold, 1, 2, lambda k, t: ptrs.append({d: b.data.data_ptr() for d, b in t._dis_pick.items()})))
    assert set(ptrs[0]) == {'a2b', 'b2a'} and ptrs[0] == ptrs[1]
