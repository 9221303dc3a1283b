"""council_abs_w (trainer_council.py:224-228, 595-619), the council loss without a discriminator, on the CPU: the oracle
(oracle/council_abs_oracle.py) against the unmodified reference's numbers and drawn peers (tests/golden/*_council_abs*.json, written by
oracle/make_golden_council_abs.py), the product's host logic against the oracle in fp64 through the torch test double (extended here
with the term's ops), the swapped published lists, the single-direction refusal and data parallelism (gloo, world 2)."""
import os
import random
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import council_oracle as co
from common import close, config_for, load_golden, setup_case
from council_abs_oracle import CouncilAbsOracleTrainer
from council_gan_b200.trainer_council import Council_Trainer
from make_golden_council_abs import _with_peers
from ops_torch import TorchOps as _TorchOps
from test_trainer_host_cpu import _randn, _randn32, compare_with_oracle, load_states


class TorchOps(_TorchOps):
    """The torch test double with the council_abs_w ops of council_gan_b200.ops.CudaOps."""

    @staticmethod
    def _council_abs_d(x_fake, peers, gray):
        x, xp = x_fake[..., :3], x_fake[list(peers)][..., :3]
        return x.sum(-1) - xp.sum(-1) if gray else x - xp

    def council_abs_fwd(self, x_fake, peers, gray, sums):
        sums.copy_(self._council_abs_d(x_fake, peers, gray).abs().flatten(1).sum(1))

    def council_abs_bwd(self, x_fake, peers, gray, sums, numel, w, total, pub, d_x):
        """Restatement of csrc/losses.cu council_abs_bwd_kernel: the direction totals share gen_loss_bwd's float64 accumulator."""
        sc = sums.detach().double().cpu()
        for g in range(x_fake.shape[0]):
            term = w * float(sc[g]) / numel
            pub[g] = term
            self._tot64[g] += term
            total[g] = self._tot64[g]
        s = torch.sign(self._council_abs_d(x_fake, peers, gray)) * (w / numel)
        d_x[..., :3] += s.unsqueeze(-1) if gray else s

    def add_column(self, dst, k, src):
        dst[:, k] += src


CASES = ['glasses64_n2_b2_council_abs', 'm2f64_n4_b2_council_abs_nodc', 'anime64_n3_b2_council_abs_gray',
         'glasses64_n2_b2_council_abs_early']
ITER3 = 'glasses64_n3_b2_council_abs_iter3'
RTOL = 2e-5  # as tests/test_oracle_golden.py: both sides are torch-CPU fp32


def n_iters(gold):
    return gold.get('n_iters', 1)


def golden_records(gold):
    return gold['iters'] if 'iters' in gold else [gold]


def run(gold, dtype=torch.float32, ops=None, on_iter=None, inputs=None, overrides=None):
    """The oracle (ops None) or the product on the test double, n_iters(gold) iterations as oracle/make_golden.py runs them.  The
    product records the peers its gen_update draws in `peers_drawn`."""
    hp, states, x_a, x_b = setup_case(gold)
    hp.update(overrides or {})
    if inputs is not None:
        x_a, x_b = inputs
    if ops is None:
        states = {k: [{kk: vv.to(dtype) for kk, vv in sd.items()} for sd in lst] for k, lst in states.items()}
        x_a, x_b = x_a.to(dtype), x_b.to(dtype)
        tr = CouncilAbsOracleTrainer(hp, states)
    else:
        co.seed_all(hp['random_seed'])
        tr = Council_Trainer(hp, str(ops.device), _ops=ops)
        load_states(tr, states)
        tr.gen_update = _with_peers(tr)
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


def published(tr):
    """(council_loss_ab, council_loss_ba, drawn peers) of either trainer, as floats / ints."""
    if isinstance(tr, CouncilAbsOracleTrainer):
        ab, ba, peers = tr.council_loss_s['a2b'], tr.council_loss_s['b2a'], tr.peers
    else:
        ab, ba, peers = tr.council_loss_ab_s, tr.council_loss_ba_s, tr.peers_drawn
    return [float(v) for v in ab], [float(v) for v in ba], list(peers)


def check_lists(got, want, rtol, atol=1e-7):
    assert len(got) == len(want), (got, want)
    for g, w in zip(got, want):
        assert close(g, w, rtol, atol), (g, w)


@pytest.mark.parametrize('case', CASES + [ITER3])
def test_oracle_matches_reference_golden(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    log = []

    def grab(k, tr):
        log.append(([float(v) for v in tr.loss_dis_total_s], [float(v) for v in tr.loss_gen_total_s], published(tr)))
    run(gold, torch.float32, on_iter=grab)
    for k, (rec, (dis, gen, (ab, ba, peers))) in enumerate(zip(golden_records(gold), log)):
        rtol = [RTOL, 1e-4, 1e-3][k]  # later iterations: fp32 summation-order noise grows through Adam's sign-like first steps
        check_lists(dis, rec['loss_dis_total'], rtol)
        check_lists(gen, rec['loss_gen_total'], rtol)
        check_lists(ab, rec['council_loss_ab'], rtol)
        check_lists(ba, rec['council_loss_ba'], rtol)
        assert peers == rec['peers']


def test_fixtures_pin_what_they_are_for():
    both = load_golden('glasses64_n2_b2_council_abs')
    assert both['dis_council_ran'] and both['peers'] == [1, 0]  # council discriminators and the single-candidate draw
    nodc = load_golden('m2f64_n4_b2_council_abs_nodc')
    assert not nodc['dis_council_ran'] and len(set(nodc['peers'])) > 1
    assert [len(r['peers']) for r in load_golden(ITER3)['iters']] == [3, 3, 0]  # the gate closes in the third iteration
    assert [r['dis_council_ran'] for r in load_golden(ITER3)['iters']] == [True, True, False]
    early = load_golden('glasses64_n2_b2_council_abs_early')
    assert early['peers'] == [] and early['council_loss_ab'] == [0.0, 0.0]


def test_published_lists_take_the_other_directions_term():
    """council_loss_ab_s[i] holds the b2a abs term and council_loss_ba_s[i] the a2b one (trainer_council.py:616-619); with
    council_w 0 nothing else is in them"""
    gold = load_golden('m2f64_n4_b2_council_abs_nodc')
    tr, hp = run(gold, ops=TorchOps('cpu', torch.float64))
    w = hp['council_abs_w']
    for name, other in (('council_loss_ab_s', 'b2a'), ('council_loss_ba_s', 'a2b')):
        x = tr._last_fw[other]['x_fake'][..., :3]
        want = [w * float((x[i] - x[j]).abs().mean()) for i, j in enumerate(tr.peers_drawn)]
        own = tr._last_fw['a2b' if other == 'b2a' else 'b2a']['x_fake'][..., :3]
        assert all(abs(w * float((own[i] - own[j]).abs().mean()) - v) > 1e-3 for i, (j, v) in enumerate(zip(tr.peers_drawn, want)))
        check_lists([float(v) for v in getattr(tr, name)], want, 1e-12)


@pytest.mark.parametrize('case', CASES + [ITER3])
def test_host_logic_exact_in_fp64(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    olog, plog = [], []
    orc, hp = run(gold, torch.float64, on_iter=lambda k, t: olog.append(published(t)))
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), on_iter=lambda k, t: plog.append(published(t)))
    for k, ((oab, oba, op), (pab, pba, pp), rec) in enumerate(zip(olog, plog, golden_records(gold))):
        rtol = 1e-9 if k == 0 else 1e-6  # later iterations: fp64 rounding amplified through Adam's first steps
        check_lists(pab, oab, rtol)
        check_lists(pba, oba, rtol)
        assert pp == op == rec['peers']
    # three iterations (the term is off in the third): fp64 rounding amplified by ~1e5 per iteration through the mask head, here with
    # three members and both directions
    grad_tol = 1e-7 if n_iters(gold) == 1 else 1e-4
    compare_with_oracle(tr, orc, hp, rtol_loss=1e-7, grad_rel_l2=grad_tol, flip_frac=0.0 if n_iters(gold) == 1 else 1e-3)
    if not plog[-1][2]:  # gate closed: the int 0 of the reference
        assert all(type(v) is int and v == 0 for v in tr.council_loss_ab_s + tr.council_loss_ba_s)


def test_single_direction_raises():
    for cfg in ('glasses', 'selfie2anime'):
        hp = config_for(cfg)
        with pytest.raises(NotImplementedError, match='do_a2b and do_b2a'):
            Council_Trainer(dict(hp, council_abs_w=1), 'cpu', _ops=TorchOps('cpu'))


@pytest.mark.parametrize('case', ['glasses64_n2_b2_both', 'glasses64_n2_b2_council_abs_early'])
def test_off_path_leaves_random_untouched(case):
    """term off (the shipped configs) or gate closed: gen_update draws nothing from `random`, and nothing new is published"""
    gold = load_golden(case)
    hp, states, x_a, x_b = setup_case(gold)
    tr = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    load_states(tr, states)
    tr.dis_update(x_a, x_b, hp)
    before = random.getstate()
    tr.gen_update(x_a, x_b, hp, gold['iteration'])
    assert random.getstate() == before


# ---- data parallel ------------------------------------------------------------------------------------------------------------
DP_CASE = 'm2f64_n4_b2_council_abs_nodc'


def _dp_run(x_a, x_b, gray):
    gold = load_golden(DP_CASE)
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), inputs=(x_a, x_b), overrides={'council_abs_gray_scale': gray})
    ab, ba, peers = published(tr)
    out = {'gen': [float(v) for v in tr.loss_gen_total_s], 'ab': ab, 'ba': ba, 'peers': peers}
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


def _dp_worker(rank, world, port, gray, ret):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.set_num_threads(2)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    _, _, x_a, x_b = setup_case(load_golden(DP_CASE))
    b = x_a.size(0) // world
    out = _dp_run(x_a[rank * b:(rank + 1) * b], x_b[rank * b:(rank + 1) * b], gray)
    ret[rank] = out['peers']
    if rank == 0:
        ret.update({k: v for k, v in out.items() if k != 'peers'})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('gray', [False, True])
def test_two_ranks_equal_one_rank_global_batch(gray):
    """Every rank draws the same peers; the sums ride in the scalar all-reduce and the mean is over the GLOBAL minibatch."""
    torch.set_num_threads(4)
    _, _, x_a, x_b = setup_case(load_golden(DP_CASE))
    single = _dp_run(x_a, x_b, gray)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dp_worker, args=(2, _free_port(), gray, ret), nprocs=2, join=True)
    ret = dict(ret)
    assert ret[0] == ret[1] == single['peers']
    for k in ('gen', 'ab', 'ba'):
        for a, b in zip(single[k], ret[k]):
            assert abs(a - b) <= 1e-7 * abs(a), (k, a, b)
    for k, v in single.items():
        if k.startswith('p_'):
            diff = (v - ret[k]).abs().max().item()
            assert diff < 1e-7, (k, diff)
