"""The image reconstruction term recon_x_w (trainer_council.py:339-345, 455-459) on the CPU: the oracle (oracle/recon_x_oracle.py)
against the unmodified reference's numbers (tests/golden/*_recon_x*.json, written by oracle/make_golden_recon_x.py), the product's
host logic against the oracle in fp64 through the torch test double (extended here with the two reconstruction-head ops), the
single-direction refusal, the off path, the style encoder's optimiser state in the checkpoint files, and data parallelism (gloo,
world 2)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import council_oracle as co
from common import close, load_golden, setup_case
from council_gan_b200.trainer_council import Council_Trainer
from recon_x_oracle import ReconXOracleTrainer
from test_trainer_host_cpu import _randn, _randn32, load_states
from test_trainer_recon_cpu import TorchOps as _TorchOps
from test_trainer_recon_cpu import check_lists, compare, golden_records, n_iters

CASES = ['glasses64_n2_b2_recon_x', 'glasses64_n2_b2_recon_xsc_iter3', 'anime64_n3_b2_recon_x_abs']
LISTS = ['loss_gen_recon_%s_%s' % (k, d) for k in ('x', 's', 'c') for d in ('a', 'b')]
RTOL = 2e-5  # as tests/test_oracle_golden.py: both sides are torch-CPU fp32


class TorchOps(_TorchOps):
    """The torch test double with the reconstruction-head ops of council_gan_b200.ops.CudaOps."""

    def recon_head_fwd(self, h, x_in, sums):
        im, _ = self._mask_head(h, x_in)
        sums.view(-1).copy_((im - x_in[..., :3]).abs().reshape(h.shape[0], -1).sum(-1))

    def recon_head_bwd(self, h, x_in, coef):
        im, _ = self._mask_head(h, x_in)
        d = coef * torch.sign(im - x_in[..., :3])
        return self.mask_head_bwd(h, x_in, torch.cat((d, torch.zeros_like(d[..., :1])), -1))


def published(tr):
    return {k: [float(v) for v in getattr(tr, k + '_s')] for k in LISTS}


def run(gold, dtype=torch.float32, ops=None, on_iter=None, inputs=None, hp_over=None):
    """The oracle (ops None) or the product on the test double, n_iters(gold) iterations as oracle/make_golden.py runs them."""
    hp, states, x_a, x_b = setup_case(gold)
    hp.update(hp_over or {})
    if inputs is not None:
        x_a, x_b = inputs
    if ops is None:
        states = {k: [{kk: vv.to(dtype) for kk, vv in sd.items()} for sd in lst] for k, lst in states.items()}
        x_a, x_b = x_a.to(dtype), x_b.to(dtype)
        tr = ReconXOracleTrainer(hp, states)
    else:
        co.seed_all(hp['random_seed'])
        tr = Council_Trainer(hp, str(ops.device), _ops=ops)
        load_states(tr, states)
    co.seed_all(gold['rng_seed'])
    torch.randn = _randn32(dtype if ops is None else torch.float32)
    try:
        for k in range(n_iters(gold)):
            hp['iteration'] = gold['iteration'] + k
            tr.dis_update(x_a, x_b, hp)
            if ops is None:
                tr.disc_ran = tr.dis_council_update(x_a, x_b, hp)
            else:
                tr.loss_dis_council_total_s = None
                tr.dis_council_update(x_a, x_b, hp)
            tr.gen_update(x_a, x_b, hp, hp['iteration'])
            if on_iter is not None:
                on_iter(k, tr)
            if n_iters(gold) > 1:
                tr.update_learning_rate()
    finally:
        torch.randn = _randn
    return tr, hp


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference_golden(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    log = []
    run(gold, torch.float32, on_iter=lambda k, tr: log.append(([float(v) for v in tr.loss_dis_total_s],
                                                              [float(v) for v in tr.loss_gen_total_s], published(tr))))
    assert len(log) == n_iters(gold)
    for k, (rec, (dis, gen, lists)) in enumerate(zip(golden_records(gold), log)):
        rtol = [RTOL, 1e-4, 1e-3][k]  # fp32 summation-order noise grows through Adam's sign-like first steps
        check_lists(dis, rec['loss_dis_total'], rtol)
        check_lists(gen, rec['loss_gen_total'], rtol)
        for key in LISTS:
            check_lists(lists[key], rec[key], rtol)


def test_fixtures_pin_what_they_are_for():
    x = load_golden('glasses64_n2_b2_recon_x')
    assert len(x['loss_gen_recon_x_a']) == 2 and x['loss_gen_recon_s_a'] == [] and x['loss_gen_recon_c_b'] == [] and x['dis_council_ran']
    style = [k for k in x['params'] if 'enc_style' in k]
    assert style and all('grad' in x['params'][k] for k in style)  # recon_x alone trains the style encoder
    assert [[len(r[k]) for k in LISTS] for r in load_golden('glasses64_n2_b2_recon_xsc_iter3')['iters']] == [[2] * 6] * 3
    anime = load_golden('anime64_n3_b2_recon_x_abs')
    assert len(anime['loss_gen_recon_x_b']) == 3 and anime['loss_gen_recon_s_a'] == []


@pytest.mark.parametrize('case', CASES)
def test_host_logic_exact_in_fp64(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    orc, hp = run(gold, torch.float64)
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64))
    # three iterations: fp64 rounding amplified through Adam's sign-like first steps and the sign() of the L1 gradients
    multi = n_iters(gold) > 1
    compare(tr, orc, hp, rtol_loss=1e-7, grad_rel_l2=1e-4 if multi else 1e-7, flip_frac=1e-3 if multi else 0.0)
    got, want = published(tr), published(orc)
    for k in ('loss_gen_recon_x_a', 'loss_gen_recon_x_b'):
        check_lists(got[k], want[k], 1e-7)


def test_single_direction_refused():
    gold = load_golden('glasses64_n2_b2_early')
    hp = setup_case(gold)[0]
    with pytest.raises(NotImplementedError, match='do_a2b and do_b2a'):
        Council_Trainer(dict(hp, recon_x_w=1), 'cpu', _ops=TorchOps('cpu'))
    tr = Council_Trainer(dict(hp, do_b2a=True), 'cpu', _ops=TorchOps('cpu'))  # built with recon_x_w 0: its style encoder is frozen
    x_a, x_b = setup_case(gold)[2:]
    with pytest.raises(NotImplementedError, match='recon_x_w'):
        tr.gen_update(x_a, x_b, dict(hp, do_b2a=True, recon_x_w=1), 0)


class _NoHeadOps(TorchOps):
    def recon_head_fwd(self, *a, **k):
        raise AssertionError('the reconstruction head ran while recon_x_w is 0')

    recon_head_bwd = recon_head_fwd


def test_term_off_publishes_nothing_new():
    tr, _ = run(load_golden('glasses64_n2_b2_both'), ops=_NoHeadOps('cpu'))
    assert not any(hasattr(tr, k + '_s') for k in LISTS)
    assert not tr._nets['gen_a2b'].sty_bank.trainable
    # another reconstruction term on: all six lists are published, recon_x's empty, and its head never runs
    tr, _ = run(load_golden('glasses64_n2_b2_recon_s'), ops=_NoHeadOps('cpu'))
    assert tr.loss_gen_recon_x_a_s == [] and tr.loss_gen_recon_x_b_s == [] and len(tr.loss_gen_recon_s_a_s) == 2


# ---- optimiser files ------------------------------------------------------------------------------------------------------------
def test_optimizer_file_style_entries_and_resume(tmp_path):
    gold = load_golden('glasses64_n2_b2_recon_x')
    tr, hp = run(dict(gold, n_iters=2), ops=TorchOps('cpu'))
    tr.save(str(tmp_path), 10)
    sd = torch.load(os.path.join(tmp_path, 'optimizer_0.pt'))['gen']
    plist = tr._opt_params('gen')
    style = [idx for idx, (net, spec, is_w) in enumerate(plist) if spec.key.startswith('enc_style')]
    assert style and all(idx in sd['state'] for idx in style)
    for idx in style:  # recon_x alone gave the style encoder its gradients: two Adam steps, non-zero moments
        ent = sd['state'][idx]
        net, spec, is_w = plist[idx]
        shape = tuple(tr.gen_a2b_s[0].state_dict()[spec.wname if is_w else spec.bname].shape)
        assert float(ent['step']) == 2.0 and tuple(ent['exp_avg'].shape) == shape and float(ent['exp_avg_sq'].abs().sum()) > 0
    co.seed_all(1)
    tr2 = Council_Trainer(dict(hp), 'cpu', _ops=TorchOps('cpu'))
    tr2.resume(str(tmp_path), dict(hp))
    for d in ('a2b', 'b2a'):
        a, b = tr._nets['gen_' + d].sty_bank, tr2._nets['gen_' + d].sty_bank
        assert b.step == a.step == 2 and torch.equal(a.exp_avg, b.exp_avg) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)


# ---- data parallel ------------------------------------------------------------------------------------------------------------
DP_CASE = 'glasses64_n2_b2_recon_xsc_iter3'


def _dp_run(x_a, x_b):
    gold = dict(load_golden(DP_CASE), n_iters=1)
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), inputs=(x_a, x_b))
    out = {'gen': [float(v) for v in tr.loss_gen_total_s], 'lists': published(tr)}
    tr.synchronize()
    for name, net in tr._nets.items():
        out['p_' + name] = net.bank.data.clone()
        if name.startswith('gen_'):
            out['sty_' + name] = net.sty_bank.data.clone()
            out['sty_m_' + name] = net.sty_bank.exp_avg.clone()
    return out


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dp_worker(rank, world, port, ret):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.set_num_threads(2)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    _, _, x_a, x_b = setup_case(load_golden(DP_CASE))
    b = x_a.size(0) // world
    out = _dp_run(x_a[rank * b:(rank + 1) * b], x_b[rank * b:(rank + 1) * b])
    if rank == 0:
        ret.update(out)
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one_rank_global_batch():
    torch.set_num_threads(4)
    _, _, x_a, x_b = setup_case(load_golden(DP_CASE))
    single = _dp_run(x_a, x_b)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dp_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    ret = dict(ret)
    for a, b in zip(single['gen'], ret['gen']):
        assert close(a, b, 1e-7, 0.0), ('gen', a, b)
    for k in LISTS:
        assert len(single['lists'][k]) == len(ret['lists'][k]) == 2, k
        for a, b in zip(single['lists'][k], ret['lists'][k]):
            assert close(a, b, 1e-7, 0.0), (k, a, b)
    for k, v in single.items():
        if k.startswith(('p_', 'sty_')):
            diff = (v - ret[k]).abs().max().item()
            assert diff < 1e-7, (k, diff)
