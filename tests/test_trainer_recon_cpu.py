"""The latent reconstruction terms recon_c_w / recon_s_w (trainer_council.py:359-369, 460-469) on the CPU: the oracle
(oracle/recon_oracle.py) against the unmodified reference's numbers (tests/golden/*_recon*.json, written by
oracle/make_golden_recon.py), the product's host logic against the oracle in fp64 through the torch test double (extended here
with the new ops), the single-direction refusal, the style encoder's optimiser state in the checkpoint files, and data parallelism
(gloo, world 2)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import council_oracle as co
from common import close, load_golden, setup_case
from council_gan_b200.trainer_council import Council_Trainer
from recon_oracle import ReconOracleTrainer
from test_trainer_abs_beginning_end_cpu import TorchOps as _TorchOps
from test_trainer_host_cpu import _randn, _randn32, load_states


class TorchOps(_TorchOps):
    """The torch test double with the ops of the latent reconstruction (council_gan_b200.ops.CudaOps)."""

    def add_(self, dst, src):
        dst.view(-1).add_(src.reshape(-1))

    def global_avgpool_fwd(self, h):
        return h.mean(dim=(2, 3), keepdim=True).contiguous()

    def global_avgpool_bwd(self, dy, h, relu_gate=True):
        dh = (dy / (h.shape[2] * h.shape[3])).expand_as(h)
        return (torch.where(h > 0, dh, torch.zeros_like(dh)) if relu_gate else dh).contiguous()

    def latent_l1(self, a, b, sums, coef, da=None, db=None, accumulate=False):
        G = a.shape[0]
        d = a - (b.expand_as(a) if b.shape[0] == 1 else b)
        sums.view(-1).copy_(d.abs().reshape(G, -1).sum(-1))
        g = coef * torch.sign(d)
        for t, v in ((da, g), (db, -g)):
            if t is not None:
                t.copy_(t + v if accumulate else v)

    def recon_finalize(self, sums, numel, weights, total, pub):
        """Restatement of csrc/losses.cu recon_finalize_kernel: the member totals share gen_loss_bwd's float64 accumulator."""
        sc = sums.detach().double().cpu()
        for k, (n, w) in enumerate(zip(numel, weights)):
            for g in range(sums.shape[1]):
                val = float(sc[k, g]) / n
                pub[k, g] = val
                if w != 0:
                    self._tot64[g] += w * val
                    total[g] = self._tot64[g]


CASES = ['glasses64_n2_b2_recon_c', 'glasses64_n2_b2_recon_s', 'glasses64_n2_b2_recon_iter3', 'anime64_n3_b2_recon_abs']
LISTS = ['loss_gen_recon_%s_%s' % (k, d) for k in ('s', 'c') for d in ('a', 'b')]
RTOL = 2e-5  # as tests/test_oracle_golden.py: both sides are torch-CPU fp32


def n_iters(gold):
    return gold.get('n_iters', 1)


def run(gold, dtype=torch.float32, ops=None, on_iter=None, inputs=None, hp_over=None):
    """The oracle (ops None) or the product on the test double, n_iters(gold) iterations as oracle/make_golden.py runs them."""
    hp, states, x_a, x_b = setup_case(gold)
    hp.update(hp_over or {})
    if inputs is not None:
        x_a, x_b = inputs
    if ops is None:
        states = {k: [{kk: vv.to(dtype) for kk, vv in sd.items()} for sd in lst] for k, lst in states.items()}
        x_a, x_b = x_a.to(dtype), x_b.to(dtype)
        tr = ReconOracleTrainer(hp, states)
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
    return {k: [float(v) for v in getattr(tr, k + '_s')] for k in LISTS}


def golden_records(gold):
    return gold['iters'] if 'iters' in gold else [gold]


def check_lists(got, want, rtol, atol=1e-7):
    assert len(got) == len(want), (got, want)
    for g, w in zip(got, want):
        assert close(g, w, rtol, atol), (g, w)


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference_golden(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    log = []
    run(gold, torch.float32, on_iter=lambda k, tr: log.append(([float(v) for v in tr.loss_dis_total_s],
                                                              [float(v) for v in tr.loss_gen_total_s], published(tr))))
    for k, (rec, (dis, gen, lists)) in enumerate(zip(golden_records(gold), log)):
        rtol = [RTOL, 1e-4, 1e-3][k]  # fp32 summation-order noise grows through Adam's sign-like first steps
        check_lists(dis, rec['loss_dis_total'], rtol)
        check_lists(gen, rec['loss_gen_total'], rtol)
        for key in LISTS:
            check_lists(lists[key], rec[key], rtol)


def test_fixtures_pin_what_they_are_for():
    c, s = load_golden('glasses64_n2_b2_recon_c'), load_golden('glasses64_n2_b2_recon_s')
    assert c['loss_gen_recon_s_a'] == [] and len(c['loss_gen_recon_c_a']) == 2 and c['dis_council_ran']
    assert s['loss_gen_recon_c_b'] == [] and len(s['loss_gen_recon_s_b']) == 2
    style = [k for k in s['params'] if 'enc_style' in k]
    assert style and all('grad' in s['params'][k] for k in style)  # recon_s trains the style encoder ...
    assert not any('grad' in v for k, v in c['params'].items() if 'enc_style' in k)  # ... recon_c does not
    assert [len(r['loss_gen_recon_s_a']) for r in load_golden('glasses64_n2_b2_recon_iter3')['iters']] == [2, 2, 2]
    assert len(load_golden('anime64_n3_b2_recon_abs')['loss_gen_recon_c_b']) == 3


def compare(tr, orc, hp, rtol_loss, grad_rel_l2, flip_frac):
    """Losses, the four lists, every generator gradient (relative L2, style encoder included) and every post-step parameter."""
    for i in range(tr.council_size):
        assert close(float(tr.loss_dis_total_s[i]), float(orc.loss_dis_total_s[i]), rtol_loss), ('dis', i)
        assert close(float(tr.loss_gen_total_s[i]), float(orc.loss_gen_total_s[i]), rtol_loss), ('gen', i)
    got, want = published(tr), published(orc)
    for k in LISTS:
        check_lists(got[k], want[k], rtol_loss)
    tr.synchronize()
    for name in orc.P:
        fam = name.rsplit('_', 1)[0]
        net = tr._nets[name]
        dead = getattr(net, 'dead_bias', set())
        for i in range(tr.council_size):
            sd = getattr(tr, name + '_s')[i].state_dict()
            for spec in net._specs():
                for key, is_w in ((spec.wname, True), (spec.bname, False)):
                    if key in dead:
                        continue
                    ref = orc.P[name][i][key].detach()
                    diff = (sd[key].cpu().to(ref.dtype) - ref).abs()
                    assert (diff > 0.5 * hp['lr']).double().mean().item() <= flip_frac, (name, i, key)
                    og = orc.P[name][i][key].grad
                    if fam != 'gen':
                        continue
                    bank = net._bank_of(key)
                    if og is None:  # the style encoder without recon_s: never stepped
                        assert not bank.trainable or bank.step == 0, key
                        assert torch.equal(sd[key].cpu().to(ref.dtype), ref), key
                        continue
                    g = bank.g(key)[i]
                    g = (spec.export_weight(g) if is_w else g).cpu().to(og.dtype)
                    rel = ((g - og).norm() / (og.norm() + 1e-30)).item()
                    assert rel <= grad_rel_l2, (name, i, key, rel)


@pytest.mark.parametrize('case', CASES)
def test_host_logic_exact_in_fp64(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    orc, hp = run(gold, torch.float64)
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64))
    # three iterations: fp64 rounding amplified through Adam's sign-like first steps and the sign() of the L1 gradients
    multi = n_iters(gold) > 1
    compare(tr, orc, hp, rtol_loss=1e-7, grad_rel_l2=1e-4 if multi else 1e-7, flip_frac=1e-3 if multi else 0.0)


def test_single_direction_refused():
    gold = load_golden('glasses64_n2_b2_early')
    hp = setup_case(gold)[0]
    for key in ('recon_c_w', 'recon_s_w'):
        with pytest.raises(NotImplementedError, match='do_a2b and do_b2a'):
            Council_Trainer(dict(hp, **{key: 1}), 'cpu', _ops=TorchOps('cpu'))
    tr = Council_Trainer(dict(hp, do_b2a=True), 'cpu', _ops=TorchOps('cpu'))  # built with recon_s_w 0: its style encoder is frozen
    x_a, x_b = setup_case(gold)[2:]
    with pytest.raises(NotImplementedError, match='recon_s_w'):
        tr.gen_update(x_a, x_b, dict(hp, do_b2a=True, recon_s_w=1), 0)


def test_terms_off_publish_nothing_new():
    tr, _ = run(load_golden('glasses64_n2_b2_both'), ops=TorchOps('cpu'))
    assert not any(hasattr(tr, k + '_s') for k in LISTS)
    assert not tr._nets['gen_a2b'].sty_bank.trainable


# ---- optimiser files ------------------------------------------------------------------------------------------------------------
def test_optimizer_file_style_entries_and_resume(tmp_path):
    gold = load_golden('glasses64_n2_b2_recon_s')
    tr, hp = run(dict(gold, n_iters=2), ops=TorchOps('cpu'))
    tr.save(str(tmp_path), 10)
    sd = torch.load(os.path.join(tmp_path, 'optimizer_0.pt'))['gen']
    # torch.optim.Adam over the reference's per-member parameter list (:152-179), stepped twice with every parameter holding a
    # gradient, as recon_s gives the style encoder one (the dead biases get exact zeros from the reference's autograd, not None)
    plist = tr._opt_params('gen')
    params = [torch.zeros(1, requires_grad=True) for _ in plist]
    opt = torch.optim.Adam(params, lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), weight_decay=hp['weight_decay'])
    for p in params:
        p.grad = torch.ones(1)
    opt.step()
    opt.step()
    want = opt.state_dict()
    assert sd['param_groups'][0]['params'] == want['param_groups'][0]['params']
    style = [idx for idx, (net, spec, is_w) in enumerate(plist) if spec.key.startswith('enc_style')]
    assert style and set(sd['state']) - set(want['state']) == set()
    for idx in style:  # the reference's order: the style encoder first in each generator
        ent = sd['state'][idx]
        assert set(ent) == set(want['state'][idx]) and float(ent['step']) == 2.0
        net, spec, is_w = plist[idx]
        shape = tuple(getattr(tr, 'gen_a2b_s')[0].state_dict()[spec.wname if is_w else spec.bname].shape)
        assert tuple(ent['exp_avg'].shape) == shape and float(ent['exp_avg_sq'].abs().sum()) > 0
    # round trip: a fresh trainer resumes the same moments and step counts and writes the same file
    hp2 = dict(hp)
    co.seed_all(1)
    tr2 = Council_Trainer(hp2, 'cpu', _ops=TorchOps('cpu'))
    tr2.resume(str(tmp_path), hp2)
    for d in ('a2b', 'b2a'):
        a, b = tr._nets['gen_' + d].sty_bank, tr2._nets['gen_' + d].sty_bank
        assert b.step == a.step == 2 and torch.equal(a.exp_avg, b.exp_avg) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)
    out2 = tmp_path / 'again'
    out2.mkdir()
    tr2.save(str(out2), 10)
    sd2 = torch.load(os.path.join(out2, 'optimizer_0.pt'))['gen']
    assert set(sd2['state']) == set(sd['state'])
    for idx in sd['state']:
        for k in ('exp_avg', 'exp_avg_sq', 'step'):
            assert torch.equal(sd2['state'][idx][k], sd['state'][idx][k]), (idx, k)


def test_resume_checkpoint_written_with_term_off(tmp_path):
    gold = load_golden('glasses64_n2_b2_recon_s')
    off, hp = run(gold, ops=TorchOps('cpu'), hp_over={'recon_s_w': 0})
    off.save(str(tmp_path), 10)
    assert not any(idx for idx, (n, s, w) in enumerate(off._opt_params('gen'))
                   if s.key.startswith('enc_style') and idx in torch.load(os.path.join(tmp_path, 'optimizer_0.pt'))['gen']['state'])
    on, hp_on = run(gold, ops=TorchOps('cpu'))  # style moments and step are non-zero here ...
    assert on._nets['gen_a2b'].sty_bank.step == 1
    on.resume(str(tmp_path), hp_on)  # ... and restart from zero with this checkpoint
    for d in ('a2b', 'b2a'):
        sb, gb = on._nets['gen_' + d].sty_bank, on._nets['gen_' + d].bank
        assert sb.step == 0 and float(sb.exp_avg.abs().sum()) == 0 and float(sb.exp_avg_sq.abs().sum()) == 0
        assert gb.step == off._nets['gen_' + d].bank.step


# ---- data parallel ------------------------------------------------------------------------------------------------------------
DP_CASE = 'glasses64_n2_b2_recon_iter3'


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
        assert abs(a - b) <= 1e-7 * abs(a), ('gen', a, b)
    for k in LISTS:
        for a, b in zip(single['lists'][k], ret['lists'][k]):
            assert abs(a - b) <= 1e-7 * abs(a), (k, a, b)
    for k, v in single.items():
        if k.startswith(('p_', 'sty_')):
            diff = (v - ret[k]).abs().max().item()
            assert diff < 1e-7, (k, diff)
