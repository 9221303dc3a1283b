"""abs_beginning_end (trainer_council.py:210-215, 477-495), the input-to-output pixel loss with a decaying weight, on the CPU:
the oracle (oracle/abs_beginning_end_oracle.py) against the unmodified reference's numbers (tests/golden/*_abs*.json, written by
oracle/make_golden_abs.py), the product's host logic against the oracle in fp64 through the torch test double (extended here with
the term's two ops), the gate state machine, and data parallelism (gloo, world 2)."""
import os
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import council_oracle as co
from abs_beginning_end_oracle import AbsBeginningEndOracleTrainer
from common import close, load_golden, setup_case
from council_gan_b200.trainer_council import Council_Trainer
from ops_torch import TorchOps as _TorchOps
from test_trainer_host_cpu import _randn, _randn32, compare_with_oracle, load_states


class TorchOps(_TorchOps):
    """The torch test double with the two abs_beginning_end ops of council_gan_b200.ops.CudaOps."""

    def abs_beginning_end_fwd(self, x_fake, x, sums):
        d = x_fake[..., :3] - x[..., :3]
        sums[:, 0] = d.abs().sum(dim=(1, 2, 3, 4))
        sums[:, 1] = (d * d).sum(dim=(1, 2, 3, 4))

    def abs_beginning_end_bwd(self, x_fake, x, sums, numel, weights, total, pub, d_x):
        """Restatement of csrc/losses.cu abs_be_bwd_kernel: the direction totals share gen_loss_bwd's float64 accumulator."""
        sc = sums.detach().double().cpu()
        for g, w in enumerate(weights):
            l1, l2 = float(sc[g, 0]) / numel, float(sc[g, 1]) / numel
            use_l1 = l1 > l2  # a tie picks L2
            val = l1 if use_l1 else l2
            pub[g] = val
            if w == 0:
                continue
            self._tot64[g] += w * val
            total[g] = self._tot64[g]
            d = x_fake[g, ..., :3] - x[0, ..., :3]
            d_x[g, ..., :3] += (w / numel) * (torch.sign(d) if use_l1 else 2.0 * d)

SINGLE = ['glasses64_n2_b2_abs', 'anime64_n3_b2_abs', 'glasses64_n2_b2_both_abs', 'glasses64_n2_b2_abs_l2']
DECAY = 'glasses64_n2_b2_abs_decay'
RTOL = 2e-5  # as tests/test_oracle_golden.py: both sides are torch-CPU fp32


def setup_inputs(gold):
    hp, states, x_a, x_b = setup_case(gold)
    s = gold.get('input_scale', 1)
    return hp, states, x_a * s, x_b * s


def n_iters(gold):
    return gold.get('n_iters', 1)


def run(gold, dtype=torch.float32, ops=None, on_iter=None, inputs=None):
    """The oracle (ops None) or the product on the test double, n_iters(gold) iterations as oracle/make_golden.py runs them."""
    hp, states, x_a, x_b = setup_inputs(gold)
    if inputs is not None:
        x_a, x_b = inputs
    if ops is None:
        states = {k: [{kk: vv.to(dtype) for kk, vv in sd.items()} for sd in lst] for k, lst in states.items()}
        x_a, x_b = x_a.to(dtype), x_b.to(dtype)
        tr = AbsBeginningEndOracleTrainer(hp, states)
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


def published(tr):
    """(a_ab list, b_ba list, weight) of either trainer, as floats."""
    if isinstance(tr, AbsBeginningEndOracleTrainer):
        a, b = tr.loss_gen_beginning_end_s['a2b'], tr.loss_gen_beginning_end_s['b2a']
    else:
        a, b = tr.loss_gen_beginning_end_a_ab_s, tr.loss_gen_beginning_end_b_ba_s
    return [float(v) for v in a], [float(v) for v in b], float(tr.abs_beginning_end_w_conf)


def golden_records(gold):
    return gold['iters'] if 'iters' in gold else [gold]


def check_lists(got, want, rtol, atol=1e-7):
    assert len(got) == len(want), (got, want)
    for g, w in zip(got, want):
        assert close(g, w, rtol, atol), (g, w)


@pytest.mark.parametrize('case', SINGLE + [DECAY])
def test_oracle_matches_reference_golden(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    log = []

    def grab(k, tr):
        log.append(([float(v) for v in tr.loss_dis_total_s], [float(v) for v in tr.loss_gen_total_s], published(tr)))
    run(gold, torch.float32, on_iter=grab)
    for k, (rec, (dis, gen, (a, b, w))) in enumerate(zip(golden_records(gold), log)):
        # later iterations of the decay case: fp32 summation-order noise grows through Adam's sign-like first steps (the fp64
        # oracle is 8e-5 away from the fp32 reference by the third iteration)
        rtol = [RTOL, 1e-4, 1e-3, 1e-3][k]
        check_lists(dis, rec['loss_dis_total'], rtol)
        check_lists(gen, rec['loss_gen_total'], rtol)
        check_lists(a, rec['loss_gen_beginning_end_a_ab'], rtol)
        check_lists(b, rec['loss_gen_beginning_end_b_ba'], rtol)
        assert w == rec['abs_beginning_end_w_conf']


def test_fixtures_pin_what_they_are_for():
    l2 = load_golden('glasses64_n2_b2_abs_l2')
    tr, _ = run(l2)
    x_a = setup_inputs(l2)[2]
    assert any(float((xf - x_a).pow(2).mean()) > float((xf - x_a).abs().mean()) for xf in tr.x_fake_gen['a2b'])  # L2 is taken
    plain = load_golden('glasses64_n2_b2_abs')
    assert plain['dis_council_ran'] and plain['loss_gen_mask_zero_one'] and plain['council_loss']  # council + focus gates open
    assert load_golden('anime64_n3_b2_abs')['loss_gen_beginning_end_a_ab'] == [0.0] * 3
    assert [len(r['loss_gen_beginning_end_a_ab']) for r in load_golden(DECAY)['iters']] == [2, 2, 1, 0]


@pytest.mark.parametrize('case', SINGLE + [DECAY])
def test_host_logic_exact_in_fp64(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    olog, plog = [], []
    orc, hp = run(gold, torch.float64, on_iter=lambda k, t: olog.append(published(t)))
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), on_iter=lambda k, t: plog.append(published(t)))
    for (oa, ob, ow), (pa, pb, pw) in zip(olog, plog):
        check_lists(pa, oa, 1e-7)  # published as fp32 tensors
        check_lists(pb, ob, 1e-7)
        assert pw == ow
    # four iterations of the decay case: fp64 rounding amplified through Adam's sign-like first steps (as the iter3 test)
    grad_tol = 1e-7 if n_iters(gold) == 1 else 1e-5
    compare_with_oracle(tr, orc, hp, rtol_loss=1e-7, grad_rel_l2=grad_tol, flip_frac=0.0 if n_iters(gold) == 1 else 1e-3)
    if not hp['do_a2b']:
        assert all(type(v) is int and v == 0 for v in tr.loss_gen_beginning_end_a_ab_s)


def test_gate_state_machine():
    """Member 0 is gated by the previous call's weight, the others by this call's; at or below 0.005 the term stays off."""
    def gate(hp, N, its):
        t = types.SimpleNamespace(council_size=N, abs_beginning_end_w_conf=hp['abs_beginning_end'])
        out = []
        for it in its:
            ws = Council_Trainer._abs_beginning_end_weights(t, hp, it)
            out.append((None if ws is None else len(ws), t.abs_beginning_end_w_conf))
        return out
    hp = {'abs_beginning_end': 1, 'abs_beginning_end_less_by': 0.5, 'abs_beginning_end_minimume': 0}
    assert gate(hp, 3, [6, 7, 8, 9, 10, 0]) == [(3, 0.5 ** 6), (3, 0.5 ** 7), (1, 0.5 ** 8), (0, 0.5 ** 8), (0, 0.5 ** 8), (0, 0.5 ** 8)]
    assert gate(dict(hp, abs_beginning_end_minimume=0.01), 2, [6, 20, 1000]) == [(2, 2 ** -6), (2, 0.01), (2, 0.01)]
    assert gate(dict(hp, abs_beginning_end=0), 2, [0, 1]) == [(None, 0), (None, 0)]
    assert gate(dict(hp, abs_beginning_end=0.004), 2, [0]) == [(0, 0.004)]  # starts below the threshold: never entered
    assert gate(dict(hp, abs_beginning_end_less_by=0), 3, [1, 2]) == [(1, 0), (0, 0)]  # the weight may be 0 while member 0 is open


def test_published_lists_across_iterations_fp32_vs_reference():
    gold = load_golden(DECAY)
    log = []
    run(gold, ops=TorchOps('cpu'), on_iter=lambda k, t: log.append(published(t)))
    for k, ((a, b, w), rec) in enumerate(zip(log, gold['iters'])):
        # the tolerances of test_trainer_host_cpu's three-iteration check: the hand-written backward rounds differently from autograd
        check_lists(a, rec['loss_gen_beginning_end_a_ab'], [1e-4, 2e-3, 1e-2, 1e-2][k])
        assert b == [0.0] * len(a) and w == rec['abs_beginning_end_w_conf']


def test_term_off_publishes_nothing_new():
    gold = load_golden('glasses64_n2_b2_early')
    tr, _ = run(gold, ops=TorchOps('cpu'))
    assert not hasattr(tr, 'loss_gen_beginning_end_a_ab_s') and not hasattr(tr, 'loss_gen_beginning_end_b_ba_s')
    assert tr.abs_beginning_end_w_conf == 0


# ---- data parallel ------------------------------------------------------------------------------------------------------------
DP_CASE = 'glasses64_n2_b2_abs'
DP_SCALE = (0.3, 3.0)  # image 0 (rank 0's shard) keeps |d| < 1 -> L1 alone; image 1 (rank 1's) goes to L2 alone


def _dp_inputs():
    gold = load_golden(DP_CASE)
    _, _, x_a, x_b = setup_inputs(gold)
    s = torch.tensor(DP_SCALE).view(2, 1, 1, 1)
    return gold, x_a * s, x_b * s


def _dp_run(x_a, x_b):
    gold = load_golden(DP_CASE)
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), inputs=(x_a, x_b))
    out = {'gen': [float(v) for v in tr.loss_gen_total_s], 'be': published(tr)[0]}
    tr.synchronize()
    for name, net in tr._nets.items():
        out['p_' + name] = net.bank.data.clone()
    out['x_fake'] = tr._last_fw['a2b']['x_fake'].clone()
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
    _, x_a, x_b = _dp_inputs()
    b = x_a.size(0) // world
    out = _dp_run(x_a[rank * b:(rank + 1) * b], x_b[rank * b:(rank + 1) * b])
    if rank == 0:
        ret.update({k: v for k, v in out.items() if k != 'x_fake'})
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one_rank_global_batch():
    """The branch is chosen on the GLOBAL sums: each shard alone would choose differently for some member."""
    torch.set_num_threads(4)
    _, x_a, x_b = _dp_inputs()
    single = _dp_run(x_a, x_b)
    xf, x = single['x_fake'][..., :3], x_a.to(torch.float64).permute(0, 2, 3, 1)[None]
    d = xf - x
    shard_l1 = [[bool(d[g, b].abs().mean() > d[g, b].pow(2).mean()) for b in range(2)] for g in range(d.shape[0])]
    assert all(s[0] != s[1] for s in shard_l1), shard_l1  # the shards disagree, so one of them disagrees with the global choice
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dp_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    ret = dict(ret)
    for k in ('gen', 'be'):
        for a, b in zip(single[k], ret[k]):
            assert abs(a - b) <= 1e-7 * abs(a), (k, a, b)
    for k, v in single.items():
        if k.startswith('p_'):
            diff = (v - ret[k]).abs().max().item()
            assert diff < 1e-7, (k, diff)
