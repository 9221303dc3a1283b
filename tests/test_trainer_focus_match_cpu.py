"""Focus-loss matching (do_w_loss_matching_focus, trainer_council.py:398-410, 433-445) on the CPU: the oracle
(oracle/focus_match_oracle.py) against the unmodified reference's numbers, histories and ratios (tests/golden/*focus_match*.json,
written by oracle/make_golden_focus_match.py), the product's host logic against the oracle in fp64 through the torch test double
(extended here with a float64 restatement of the matching in gen_loss_bwd), the refused configurations, the switch as a no-op when
both focus weights are 0, and data parallelism (gloo, world 2)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import council_oracle as co
from common import close, load_golden, probe, setup_case
from council_gan_b200.trainer_council import Council_Trainer
from focus_match_oracle import FocusMatchOracleTrainer
from ops_torch import TorchOps as _TorchOps
from test_trainer_host_cpu import _randn, _randn32, compare_with_oracle, load_states


class TorchOps(_TorchOps):
    """The torch test double with cg_gen_loss_bwd's focus matching: a plain float64 restatement of gen_loss_bwd_kernel."""

    def gen_loss_bwd(self, cl_outs, mask, center, eps, scal, hp, hist_gan, hist_council, total, accumulate, pub, want_dmask, *,
                     hist_focus=None, hist_focus01=None, focus_src=None, focus_w=None):
        if not hp.get('focus_matching'):
            return super().gen_loss_bwd(cl_outs, mask, center, eps, scal, hp, hist_gan, hist_council, total, accumulate, pub,
                                        want_dmask)
        G = total.shape[0]
        R, n = hp['hist_size'] + 1, hp['hist_size']
        f32 = self.dtype == torch.float32

        def r32(v):  # the device keeps float32 loss values and float32 ratios; the fp64 oracle does not round
            return float(np.float32(v)) if f32 else float(v)

        def window(ring, g, head, k0=0):
            return [float(ring[g, (head + k) % R]) for k in range(k0, n)]

        sc = scal.detach().double().cpu().numpy()
        coef = np.zeros((G, 3))
        cdis = np.zeros(G)
        for g in range(G):
            adv, cl = sc[g, 0] / hp['world'], sc[g, 1] / hp['world']
            l01, msum, ltv = sc[g, 2] / hp['numel'], sc[g, 3] / hp['numel'], (sc[g, 4] + sc[g, 5]) / hp['numel']
            tot, ltot, w01m, wtm = 0.0, 0.0, 1.0, 1.0
            if hp['focus_on']:
                gan_before = sum(window(hist_gan, g, hp['head_gan'])) / n  # :402, read before this update's GAN append
                if hp['w01'] != 0:
                    app = r32(l01)
                    w01m = gan_before / ((sum(window(hist_focus01, g, hp['head_focus01'], 1)) + app) / n)
                    hist_focus01[g, (hp['head_focus01'] + n) % R] = app
                    l01 *= r32(w01m)
                    tot += hp['w01'] * l01
                    coef[g, 0] = hp['w01'] * r32(w01m) / hp['numel']
                if hp['wtv'] != 0:
                    tot += hp['wtv'] * ltv
                    coef[g, 2] = hp['wtv'] / hp['numel']
                if hp['wtot'] != 0:
                    if hp['small_abs']:
                        ltot += abs(msum)
                        coef[g, 1] += hp['wtot'] * np.sign(msum) / hp['numel']
                    if hp['small_square']:
                        ltot += msum ** 2
                        coef[g, 1] += hp['wtot'] * 2.0 * msum / hp['numel']
                    app = float(focus_src[g, 3]) if focus_src is not None else r32(ltot)  # :441 for b2a
                    wtm = gan_before / ((sum(window(hist_focus, g, hp['head_focus'], 1)) + app) / n)
                    hist_focus[g, (hp['head_focus'] + n) % R] = app
                    ltot *= r32(wtm)
                    coef[g, 1] *= r32(wtm)
                    tot += hp['wtot'] * ltot
            adv32 = r32(adv)
            if hp['gan_on'] and hp['matching']:
                mean_gan = (sum(window(hist_gan, g, hp['head_gan'], 1)) + adv32) / n
                hist_gan[g, (hp['head_gan'] + n) % R] = adv32
            else:
                mean_gan = sum(window(hist_gan, g, hp['head_gan'])) / n
            if hp['gan_on']:
                tot += hp['gan_w'] * adv
            w, closs = 1.0, 0.0
            if hp['council_on']:
                if hp['matching']:
                    cl32 = r32(cl)
                    mean_c = (sum(window(hist_council, g, hp['head_council'], 1)) + cl32) / n
                    hist_council[g, (hp['head_council'] + n) % R] = cl32
                    w = mean_gan / mean_c
                closs = cl * r32(w) * hp['council_w']
                tot += closs
                cdis[g] = w * hp['council_w']
            prev = self._tot64[g] if accumulate else 0.0
            self._tot64[g] = prev + tot
            total[g] = self._tot64[g]
            pub[g] = torch.tensor([tot, adv, l01, ltot, ltv, closs, w, cl], dtype=pub.dtype)
            if focus_w is not None:
                focus_w[g] = torch.tensor([w01m, wtm], dtype=focus_w.dtype)
        cl_douts = []
        for out in cl_outs:
            o = out.reshape(G, -1)
            cf = torch.tensor(cdis * 2.0 / (o.shape[-1] * hp['world']), dtype=self.dtype, device=self.device)
            cl_douts.append((cf[:, None] * (o - 1)).reshape(out.shape).contiguous())
        d_mask = None
        if want_dmask:
            d_mask = self.focus_bwd(mask, torch.tensor(coef, dtype=self.dtype, device=self.device), center, eps)
        return cl_douts, d_mask


CASES = ['glasses64_n2_b2_focus_match_abs_square', 'm2f64_n2_b2_focus_match_no01', 'glasses64_n2_b2_focus_match_gan0',
         'glasses64_n2_b2_focus_match_closed']
ITER3 = ['glasses64_n2_b2_focus_match_iter3', 'glasses64_n2_b2_focus_match_both_iter3']
KINDS = ('gan', 'council', 'focus', 'focus_zero_one')


def golden_records(gold):
    return gold['iters'] if 'iters' in gold else [gold]


def run(gold, dtype=torch.float32, ops=None, on_iter=None, inputs=None, n_iters=None, hp_edit=None):
    """The oracle (ops None) or the product on the test double, as oracle/make_golden.py runs the reference."""
    hp, states, x_a, x_b = setup_case(gold)
    if hp_edit is not None:
        hp_edit(hp)
    if inputs is not None:
        x_a, x_b = inputs
    if ops is None:
        states = {k: [{kk: vv.to(dtype) for kk, vv in sd.items()} for sd in lst] for k, lst in states.items()}
        x_a, x_b = x_a.to(dtype), x_b.to(dtype)
        tr = FocusMatchOracleTrainer(hp, states)
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
            tr.dis_update(x_a, x_b, hp)
            if ops is not None:
                tr.loss_dis_council_total_s = None
            tr.disc_ran = tr.dis_council_update(x_a, x_b, hp)
            tr.gen_update(x_a, x_b, hp, hp['iteration'])
            if on_iter is not None:
                on_iter(k, tr)
            if n > 1:
                tr.update_learning_rate()
    finally:
        torch.randn = _randn
    return tr, hp


def record(tr):
    """Losses, histories and focus ratios of one iteration, from the oracle or the product."""
    rec = {'dis': [float(v) for v in tr.loss_dis_total_s], 'gen': [float(v) for v in tr.loss_gen_total_s], 'dirs': {}}
    oracle = isinstance(tr, FocusMatchOracleTrainer)
    for d in (tr.dirs if oracle else tr._dirs):
        ab = 'ab' if d == 'a2b' else 'ba'
        if oracle:
            hist = {'gan': tr.hist_gan[d], 'council': tr.hist_council[d], 'focus': tr.hist_focus[d],
                    'focus_zero_one': tr.hist_focus_zero_one[d]}
            # the reference publishes the int 0 per member for a mask-total term that did not run (:384)
            r = {'loss_gen_mask_zero_one': tr.loss_gen_mask_zero_one_s[d], 'loss_gen_mask_total': tr.loss_gen_mask_total_s[d] or [0] * tr.N,
                 'w_match_focus': tr.w_match_focus[d], 'w_match_focus_zero_one': tr.w_match_focus_zero_one[d]}
        else:
            hist = {k: getattr(tr, 'los_hist_%s_%s_s' % (k, d)) for k in KINDS}
            r = {'loss_gen_mask_zero_one': getattr(tr, 'loss_gen_mask_zero_one_%s_s' % ab),
                 'loss_gen_mask_total': getattr(tr, 'loss_gen_mask_total_%s_s' % ab),
                 'w_match_focus': tr.__dict__.get('w_match_focus_%s_conf' % d, 1),
                 'w_match_focus_zero_one': tr.__dict__.get('w_match_focus_zero_one_%s_conf' % d, 1)}
        rec['dirs'][d] = {'hist': {k: [[float(v) for v in h] for h in hist[k]] for k in KINDS},
                          'loss_gen_mask_zero_one': [float(v) for v in r['loss_gen_mask_zero_one']],
                          'loss_gen_mask_total': [float(v) for v in r['loss_gen_mask_total']],
                          'w_match_focus': float(r['w_match_focus']), 'w_match_focus_zero_one': float(r['w_match_focus_zero_one'])}
    return rec


def check_lists(got, want, rtol, atol=1e-7, what=''):
    assert len(got) == len(want), (what, got, want)
    for g, w in zip(got, want):
        assert close(g, w, rtol, atol), (what, g, w)


def check_focus(got, want, rtol):
    """got: record(); want: a golden iteration record's 'focus' or another record's 'dirs'"""
    assert set(got) == set(want)
    for d, w in want.items():
        g = got[d]
        for k in KINDS:
            assert len(g['hist'][k]) == len(w['hist'][k])
            for hg, hw in zip(g['hist'][k], w['hist'][k]):
                check_lists(hg, hw, rtol, what=(d, k))
        for k in ('loss_gen_mask_zero_one', 'loss_gen_mask_total'):
            check_lists(g[k], w[k], rtol, what=(d, k))
        for k in ('w_match_focus', 'w_match_focus_zero_one'):
            assert close(g[k], w[k], rtol, 1e-7), (d, k, g[k], w[k])


def test_fixtures_pin_what_they_are_for():
    it3 = load_golden(ITER3[0])
    hist = [r['focus']['a2b']['hist'] for r in it3['iters']]
    # histories of 2 entries: after the second iteration no initial 1 is left (the rings have wrapped)
    assert all(v != 1.0 for k in ('focus', 'focus_zero_one') for h in hist[1][k] for v in h)
    both = load_golden(ITER3[1])
    for r in both['iters']:
        # b2a's mask-total history ends with a2b's scaled term (:441)
        assert [h[-1] for h in r['focus']['b2a']['hist']['focus']] == r['focus']['a2b']['loss_gen_mask_total']
    assert both['iters'][-1]['focus']['a2b']['w_match'] != 1.0  # council matching live
    assert load_golden('m2f64_n2_b2_focus_match_no01')['focus']['a2b']['loss_gen_mask_zero_one'] == []
    gan0 = load_golden('glasses64_n2_b2_focus_match_gan0')['focus']['a2b']
    assert all(v == 1.0 for h in gan0['hist']['gan'] for v in h)
    closed = load_golden('glasses64_n2_b2_focus_match_closed')['focus']['a2b']
    assert closed['w_match_focus'] == closed['w_match_focus_zero_one'] == 1.0
    assert all(v == 1.0 for k in ('focus', 'focus_zero_one') for h in closed['hist'][k] for v in h)


def _check_params(orc, gold, hp):
    d0 = orc.dirs[0]
    for key, rec in gold['params'].items():
        head, i, name = key.split('.', 2)
        fam_d = head if head.endswith(('_a2b', '_b2a')) else '%s_%s' % (head, d0)
        got = probe(orc.P[fam_d][int(i)][name])
        for f in ('mean', 'absmean', 'l2'):
            assert close(got[f], rec['post'][f], 1e-4, 1e-9), (key, f, got[f], rec['post'][f])
        for a, b in zip(got['samples'], rec['post']['samples']):  # Adam moves every weight by ~lr per step
            assert abs(a - b) <= 2.1 * hp['lr'] + 1e-6, (key, a, b)


@pytest.mark.parametrize('case', CASES + ITER3)
def test_oracle_matches_reference_golden(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    log = []
    orc, hp = run(gold, torch.float32, on_iter=lambda k, tr: log.append(record(tr)))
    for k, (rec, got) in enumerate(zip(golden_records(gold), log)):
        rtol = [2e-5, 1e-4, 5e-3][k]  # fp32 summation-order noise grows through Adam's first steps
        check_lists(got['dis'], rec['loss_dis_total'], rtol, what='dis')
        check_lists(got['gen'], rec['loss_gen_total'], rtol, what='gen')
        # sum 1 / (|m - 0.5| + 0.01) over masks near 0.5 amplifies that noise: the zero-one histories move 1.2e-4 in the second iteration
        check_focus(got['dirs'], rec['focus'], [2e-5, 1e-3, 1e-2][k])
    if len(log) == 1:  # over three steps the focus terms' fp32 noise moves the parameters by a fraction of lr: losses and histories pin those
        _check_params(orc, gold, hp)


@pytest.mark.parametrize('case', CASES + ITER3)
def test_host_logic_exact_in_fp64(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    olog, plog = [], []
    orc, hp = run(gold, torch.float64, on_iter=lambda k, t: olog.append(record(t)))
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64), on_iter=lambda k, t: plog.append(record(t)))
    for k, (o, p) in enumerate(zip(olog, plog)):
        rtol = 1e-9 if k == 0 else 1e-6  # later iterations: fp64 rounding amplified through Adam's first steps
        check_lists(p['dis'], o['dis'], rtol)
        check_lists(p['gen'], o['gen'], rtol)
        check_focus(p['dirs'], o['dirs'], 1e-9 if k == 0 else 1e-5)  # the zero-one term amplifies that rounding further
    multi = len(golden_records(gold)) > 1
    compare_with_oracle(tr, orc, hp, rtol_loss=1e-7, grad_rel_l2=3e-3 if multi else 1e-7, flip_frac=1e-3 if multi else 0.0)


def _focus_on(**kw):
    def edit(hp):
        hp['focus_loss']['do_w_loss_matching_focus'] = True
        for k, v in kw.items():
            hp[k] = v
    return edit


@pytest.mark.parametrize('edit', [dict(mask_total_w=0), dict(do_a2b=False, do_b2a=True)])
def test_refused_where_the_reference_fails(edit):
    """mask_total_w 0 with a zero-one weight (AttributeError at :435) and b2a without a2b (IndexError at :441): refused at construction
    and in every update"""
    gold = load_golden('glasses64_n2_b2_focus_match_abs_square')
    hp, states, x_a, x_b = setup_case(gold)
    with pytest.raises(NotImplementedError, match='do_w_loss_matching_focus'):
        Council_Trainer(dict(hp, **edit, focus_loss=dict(hp['focus_loss'])), 'cpu', _ops=TorchOps('cpu'))
    # built with the switch off, then updated with it on
    off = dict(hp, **edit)
    off['focus_loss'] = dict(hp['focus_loss'], do_w_loss_matching_focus=False)
    tr = Council_Trainer(off, 'cpu', _ops=TorchOps('cpu'))
    on = dict(off, focus_loss=dict(off['focus_loss'], do_w_loss_matching_focus=True))
    for update in (tr.dis_update, tr.gen_update):
        with pytest.raises(NotImplementedError, match='do_w_loss_matching_focus'):
            update(x_a, x_b, on)


def test_allowed_when_both_focus_weights_are_zero():
    gold = load_golden('anime64_n3_b2')
    hp, _, _, _ = setup_case(gold)
    assert hp['mask_zero_or_one_w'] == hp['mask_total_w'] == 0 and not hp['do_a2b']
    hp['focus_loss']['do_w_loss_matching_focus'] = True
    Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))


def _params(tr):
    tr.synchronize()
    return {name: net.bank.data.clone() for name, net in tr._nets.items()}


@pytest.mark.parametrize('case, edit', [('anime64_n3_b2', _focus_on()),  # selfie2anime, b2a only: both focus weights 0
                                        ('glasses64_n2_b2_focus_match_closed', None)])  # the focus gate closed
def test_switch_is_a_no_op_without_an_open_focus_term(case, edit):
    """bit-identical losses and parameters with the switch on and off"""
    gold = load_golden(case)
    torch.set_num_threads(4)

    def off(hp):
        if edit is not None:
            edit(hp)
        hp['focus_loss']['do_w_loss_matching_focus'] = False
    runs = []
    for e in (edit or _focus_on(), off):
        tr, _ = run(gold, ops=_TorchOps('cpu'), hp_edit=e, n_iters=1)
        runs.append(([float(v) for v in tr.loss_gen_total_s], [float(v) for v in tr.loss_dis_total_s], _params(tr)))
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    for k, v in runs[0][2].items():
        assert torch.equal(v, runs[1][2][k]), k


# ---- data parallel ------------------------------------------------------------------------------------------------------------
DP_CASE = ITER3[1]


def _dp_run(x_a, x_b):
    gold = load_golden(DP_CASE)
    out = {}

    def grab(k, t):
        out.setdefault('rec', []).append(record(t))
        if k == 0:  # the parameters after the first step (the second one amplifies fp64 rounding through Adam's sign-like steps)
            out.update({'p_' + name: v for name, v in _params(t).items()})
    run(gold, ops=TorchOps('cpu', torch.float64), inputs=(x_a, x_b), n_iters=2, on_iter=grab)
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
    ret[rank] = out['rec']
    if rank == 0:
        ret.update({k: v for k, v in out.items() if k != 'rec'})
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one_rank_global_batch():
    """both directions, two iterations (the rings wrap): every rank derives the same histories and ratios, and the step equals one
    rank's on the global minibatch"""
    torch.set_num_threads(4)
    _, _, x_a, x_b = setup_case(load_golden(DP_CASE))
    single = _dp_run(x_a, x_b)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_dp_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    ret = dict(ret)
    for k, rec in enumerate(single['rec']):
        for r in (ret[0][k], ret[1][k]):
            check_lists(r['dis'], rec['dis'], 1e-7)
            check_lists(r['gen'], rec['gen'], 1e-7)
            check_focus(r['dirs'], rec['dirs'], 1e-7)
    for k, v in single.items():
        if k.startswith('p_'):
            diff = (v - ret[k]).abs().max().item()
            assert diff < 1e-7, (k, diff)
