"""The discriminator-side switches do_Dis_only_gray, useRandomGen and useRandomDis (trainer_council.py:499-510, 736-765) on the CPU:
the oracle (oracle/dis_options_oracle.py) against the unmodified reference's numbers and numpy draws (tests/golden/*gray*.json,
*random_pairing*.json, *dis_options*.json, written by oracle/make_golden_dis_options.py), the product's host logic against the oracle
in fp64 through the torch test double (extended here with the switches' ops), the numpy stream left alone when the switches are off
or gan_w is 0, and data parallelism (gloo, world 2)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import council_oracle as co
from common import close, load_golden, setup_case
from council_gan_b200.trainer_council import Council_Trainer
from dis_options_oracle import DisOptionsOracleTrainer
from make_golden_dis_options import with_draws
from ops_torch import TorchOps as _TorchOps
from test_trainer_host_cpu import _randn, _randn32, compare_with_oracle, load_states


class TorchOps(_TorchOps):
    """The torch test double with the ops of council_gan_b200.ops.CudaOps that the three switches use."""

    def gather_images_gray(self, pools, idx, G, Bt):
        y = self.gather_images(pools, idx, None, G, Bt)
        m = (y[..., 0] + y[..., 1] + y[..., 2]) / 3
        out = torch.zeros_like(y)
        out[..., :3] = m.unsqueeze(-1)
        return out

    def gray_fold(self, d_x):
        d_x[..., :3] = (d_x[..., 0] / 3 + d_x[..., 1] / 3 + d_x[..., 2] / 3).unsqueeze(-1)

    def gather_members(self, src, dst, segments, member_map):
        G = len(member_map)
        for off, n in segments:
            dst[off:off + G * n].view(G, n).copy_(src[off:off + G * n].view(G, n)[list(member_map)])


CASES = ['glasses64_n2_b2_gray', 'anime64_n3_b2_gray', 'm2f64_n4_b2_random_pairing']
ITER3 = 'glasses64_n3_b2_dis_options_iter3'
RTOL = 2e-5  # as tests/test_oracle_golden.py: both sides are torch-CPU fp32


def golden_records(gold):
    return gold['iters'] if 'iters' in gold else [gold]


def set_nested(hp, overrides):
    for k, v in (overrides or {}).items():
        d = hp
        ks = k.split('.')
        for kk in ks[:-1]:
            d = d[kk]
        d[ks[-1]] = v


def run(gold, dtype=torch.float32, ops=None, on_iter=None, inputs=None, overrides=None, n_iters=None):
    """The oracle (ops None) or the product on the test double, as oracle/make_golden.py runs the reference.  Both record the numpy
    draws of each update in `dis_draws` / `gen_draws`."""
    hp, states, x_a, x_b = setup_case(gold)
    set_nested(hp, overrides)
    if inputs is not None:
        x_a, x_b = inputs
    if ops is None:
        states = {k: [{kk: vv.to(dtype) for kk, vv in sd.items()} for sd in lst] for k, lst in states.items()}
        x_a, x_b = x_a.to(dtype), x_b.to(dtype)
        tr = DisOptionsOracleTrainer(hp, states)
    else:
        co.seed_all(hp['random_seed'])
        tr = Council_Trainer(hp, str(ops.device), _ops=ops)
        load_states(tr, states)
    co.seed_all(gold['rng_seed'])
    torch.randn = _randn32(dtype if ops is None else torch.float32)
    n = len(golden_records(gold)) if n_iters is None else n_iters
    try:
        for k in range(n):
            hp['iteration'] = gold['iteration'] + k
            if ops is None:
                tr.dis_update(x_a, x_b, hp)
                tr.disc_ran = tr.dis_council_update(x_a, x_b, hp)
                tr.gen_update(x_a, x_b, hp, hp['iteration'])
            else:
                dis_draws, gen_draws = [None], [None]
                with_draws(tr.dis_update, dis_draws)(x_a, x_b, hp)
                tr.loss_dis_council_total_s = None
                tr.dis_council_update(x_a, x_b, hp)
                with_draws(tr.gen_update, gen_draws)(x_a, x_b, hp, hp['iteration'])
                tr.dis_draws, tr.gen_draws = dis_draws[0], gen_draws[0]
            if on_iter is not None:
                on_iter(k, tr)
            if n > 1:
                tr.update_learning_rate()
    finally:
        torch.randn = _randn
    return tr, hp


def check_lists(got, want, rtol, atol=1e-7):
    assert len(got) == len(want), (got, want)
    for g, w in zip(got, want):
        assert close(g, w, rtol, atol), (g, w)


def _record(tr):
    return ([float(v) for v in tr.loss_dis_total_s], [float(v) for v in tr.loss_gen_total_s], list(tr.dis_draws), list(tr.gen_draws))


@pytest.mark.parametrize('case', CASES + [ITER3])
def test_oracle_matches_reference_golden(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    log = []
    run(gold, torch.float32, on_iter=lambda k, tr: log.append(_record(tr)))
    for k, (rec, (dis, gen, dd, gd)) in enumerate(zip(golden_records(gold), log)):
        # later iterations: fp32 summation-order noise grows through Adam's sign-like first steps; in the third, the reference run with
        # 3 threads instead of 8 moves its own generator losses by 1.5e-3
        rtol = [RTOL, 1e-4, 5e-3][k]
        check_lists(dis, rec['loss_dis_total'], rtol)
        check_lists(gen, rec['loss_gen_total'], rtol)
        assert dd == rec['dis_draws'] and gd == rec['gen_draws']


def test_fixtures_pin_what_they_are_for():
    for case in CASES[:2]:  # gray scale alone draws nothing
        gold = load_golden(case)
        assert gold['dis_draws'] == gold['gen_draws'] == [] and gold['dis_council_ran']
    rp = load_golden('m2f64_n4_b2_random_pairing')
    # self-pairs (member 0 draws 0), members sharing a discriminator / generator, and discriminators no member uses
    assert rp['dis_draws'] == [0, 3, 1, 0] and rp['gen_draws'] == [2, 3, 2, 3]
    it3 = load_golden(ITER3)
    assert [len(r['dis_draws']) for r in it3['iters']] == [3, 3, 3] and [len(r['gen_draws']) for r in it3['iters']] == [3, 3, 3]
    assert [r['dis_council_ran'] for r in it3['iters']] == [True, True, False]


@pytest.mark.parametrize('case', CASES + [ITER3])
def test_host_logic_exact_in_fp64(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    olog, plog = [], []
    orc, hp = run(gold, torch.float64, on_iter=lambda k, t: olog.append(_record(t)))
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), on_iter=lambda k, t: plog.append(_record(t)))
    for k, (o, p, rec) in enumerate(zip(olog, plog, golden_records(gold))):
        rtol = 1e-9 if k == 0 else 1e-6  # later iterations: fp64 rounding amplified through Adam's first steps
        check_lists(p[0], o[0], rtol)
        check_lists(p[1], o[1], rtol)
        assert p[2] == o[2] == rec['dis_draws'] and p[3] == o[3] == rec['gen_draws']
    # three iterations: fp64 rounding amplified by ~1e5 per iteration through the mask head; the first content layer of the third
    # iteration is 1.2e-4 off while the losses agree to 1e-7
    multi = len(golden_records(gold)) > 1
    compare_with_oracle(tr, orc, hp, rtol_loss=1e-7, grad_rel_l2=1e-3 if multi else 1e-7, flip_frac=1e-3 if multi else 0.0)


def test_random_dis_with_gan_w_zero_draws_nothing():
    """useRandomDis is read only while gan_w != 0 (trainer_council.py:498-501): gen_update then leaves numpy's stream alone"""
    gold = load_golden('m2f64_n4_b2_random_pairing')
    hp, states, x_a, x_b = setup_case(gold)
    hp['gan_w'] = 0
    hp['dis']['useRandomGen'] = False
    tr = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    load_states(tr, states)
    tr.dis_update(x_a, x_b, hp)
    before = np.random.get_state()
    tr.gen_update(x_a, x_b, hp, gold['iteration'])
    after = np.random.get_state()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert tr._dis_pick == {}


@pytest.mark.parametrize('case', ['glasses64_n2_b2_both', 'anime64_n3_b2'])
def test_off_path_leaves_numpy_untouched(case):
    """the switches off (the shipped configs): neither update draws from numpy and no scratch bank is made"""
    gold = load_golden(case)
    hp, states, x_a, x_b = setup_case(gold)
    tr = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    load_states(tr, states)
    before = np.random.get_state()
    tr.dis_update(x_a, x_b, hp)
    tr.dis_council_update(x_a, x_b, hp)
    tr.gen_update(x_a, x_b, hp, gold['iteration'])
    after = np.random.get_state()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert tr._dis_pick == {}


# ---- data parallel ------------------------------------------------------------------------------------------------------------
DP_CASE = ITER3


def _dp_run(x_a, x_b):
    gold = load_golden(DP_CASE)
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), inputs=(x_a, x_b), n_iters=1)
    out = {'dis': [float(v) for v in tr.loss_dis_total_s], 'gen': [float(v) for v in tr.loss_gen_total_s],
           'draws': (tr.dis_draws, tr.gen_draws)}
    tr.synchronize()
    for name, net in tr._nets.items():
        out['p_' + name] = net.bank.data.clone()
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
    ret[rank] = out['draws']
    if rank == 0:
        ret.update({k: v for k, v in out.items() if k != 'draws'})
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one_rank_global_batch():
    """all three switches, both directions: every rank draws the same members from numpy, and the step equals one rank's on the
    global minibatch"""
    torch.set_num_threads(4)
    _, _, x_a, x_b = setup_case(load_golden(DP_CASE))
    single = _dp_run(x_a, x_b)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dp_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    ret = dict(ret)
    assert ret[0] == ret[1] == single['draws']
    for k in ('dis', 'gen'):
        for a, b in zip(single[k], ret[k]):
            assert abs(a - b) <= 1e-7 * abs(a), (k, a, b)
    for k, v in single.items():
        if k.startswith('p_'):
            diff = (v - ret[k]).abs().max().item()
            assert diff < 1e-7, (k, diff)
