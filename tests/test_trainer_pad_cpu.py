"""pad_type: reflect (Conv2dBlock networks.py:463-520: nn.ReflectionPad2d, then a convolution with padding 0) on the CPU: the oracle
(council_oracle's blocks under oracle/pad_oracle.py) against the unmodified reference's numbers (tests/golden/*_reflect*.json, written by
oracle/make_golden_pad.py), the product's host logic against the oracle in fp64 through the torch test double (extended here with the
two padding ops), the zero path running neither op, the refusals, and the checkpoint files."""
import os

import pytest
import torch
import torch.nn.functional as F

import council_oracle as co
from common import config_for, load_golden, setup_case
from council_gan_b200.trainer_council import Council_Trainer
from pad_oracle import padding
from test_trainer_host_cpu import compare_with_oracle, load_states
from test_trainer_recon_cpu import check_lists, compare, golden_records, n_iters
from test_trainer_recon_x_cpu import LISTS, published
from test_trainer_recon_x_cpu import TorchOps as _TorchOps
from test_trainer_recon_x_cpu import run as _run

CASES = ['glasses64_n2_b2_reflect_gen', 'm2f64_n4_b2_reflect_dis', 'glasses64_n2_b2_reflect_recon', 'glasses64_n3_b2_reflect_iter3',
         'm2f256_n2_b1_reflect']
RTOL = 2e-5  # as tests/test_oracle_golden.py: both sides are torch-CPU fp32


class TorchOps(_TorchOps):
    """The torch test double with the reflection-padding ops of council_gan_b200.ops.CudaOps."""

    def reflect_pad(self, x, p, ups=False):
        G, B, H, W, Cc = x.shape
        t = x.reshape(G * B, H, W, Cc).permute(0, 3, 1, 2)
        if ups:
            t = F.interpolate(t, scale_factor=2)
        t = F.pad(t, (p, p, p, p), mode='reflect')
        return t.permute(0, 2, 3, 1).reshape(G, B, t.shape[2], t.shape[3], Cc).contiguous()

    def reflect_pad_bwd(self, dxp, p, addend=None, mask_src=None, mask_slope=0.0):
        G, B, Hp, Wp, Cc = dxp.shape
        x = torch.zeros(G, B, Hp - 2 * p, Wp - 2 * p, Cc, dtype=dxp.dtype, device=dxp.device, requires_grad=True)
        with torch.enable_grad():
            y = self.reflect_pad(x, p)
        dx, = torch.autograd.grad(y, x, dxp)
        if addend is not None:
            dx = dx + addend
        if mask_src is not None:
            dx = dx * torch.where(mask_src > 0, torch.ones_like(dx), torch.full_like(dx, mask_slope))
        return dx.contiguous()


def run(gold, dtype=torch.float32, ops=None, **kw):
    """test_trainer_recon_x_cpu.run (the oracle when ops is None, else the product on ops) with the oracle's blocks padded as the
    case's configuration says"""
    with padding(config_for(gold)):
        return _run(gold, dtype, ops, **kw)


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_reference_golden(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    log = []
    run(gold, torch.float32, on_iter=lambda k, tr: log.append(([float(v) for v in tr.loss_dis_total_s],
                                                              [float(v) for v in tr.loss_gen_total_s], published(tr))))
    assert len(log) == n_iters(gold)
    for k, (rec, (dis, gen, lists)) in enumerate(zip(golden_records(gold), log)):
        # fp32 summation-order noise grows through Adam's sign-like first steps and the focus loss on masks near 0.5 (as in
        # tests/test_oracle_golden.py); the council of three moves one generator total by 2.4e-4 in the second iteration
        rtol = [RTOL, 5e-4, 5e-3][k]
        check_lists(dis, rec['loss_dis_total'], rtol)
        check_lists(gen, rec['loss_gen_total'], rtol)
        for key in LISTS:
            check_lists(lists[key], rec[key], rtol)


def test_fixtures_pin_what_they_are_for():
    pads = {c: (config_for(load_golden(c))['gen']['pad_type'], config_for(load_golden(c))['dis']['pad_type']) for c in CASES}
    assert pads == {'glasses64_n2_b2_reflect_gen': ('reflect', 'zero'), 'm2f64_n4_b2_reflect_dis': ('zero', 'reflect'),
                    'glasses64_n2_b2_reflect_recon': ('reflect', 'reflect'), 'glasses64_n3_b2_reflect_iter3': ('reflect', 'reflect'),
                    'm2f256_n2_b1_reflect': ('reflect', 'reflect')}
    assert all(load_golden(c)['dis_council_ran'] for c in CASES if 'iter3' not in c)
    rec = load_golden('glasses64_n2_b2_reflect_recon')
    assert all(len(rec[k]) == 2 for k in LISTS)  # the style encoder and the re-encode passes run
    assert [r['dis_council_ran'] for r in load_golden('glasses64_n3_b2_reflect_iter3')['iters']] == [True, True, False]
    # the padding changes the numbers: the zero-padded fixture of the same geometry differs
    assert load_golden('m2f256_n2_b1_reflect')['loss_gen_total'] != load_golden('m2f256_n2_b1')['loss_gen_total']


@pytest.mark.parametrize('case', CASES)
def test_host_logic_exact_in_fp64(case):
    gold = load_golden(case)
    torch.set_num_threads(8)
    orc, hp = run(gold, torch.float64)
    tr, _ = run(gold, ops=TorchOps('cpu', torch.float64))
    # three iterations: fp64 rounding amplified through Adam's sign-like first steps and the focus loss
    multi = n_iters(gold) > 1
    # the reconstruction lists (and their comparison) exist with both directions only
    check = compare if hp['do_a2b'] and hp['do_b2a'] else compare_with_oracle
    check(tr, orc, hp, rtol_loss=1e-7, grad_rel_l2=1e-3 if multi else 1e-7, flip_frac=1e-3 if multi else 0.0)


def test_sample_matches_oracle():
    """sample() (no-grad encode / decode: the upsample goes into the padding pass instead of the convolution) under reflect"""
    gold = load_golden('glasses64_n2_b2_reflect_recon')
    hp, states, x_a, x_b = setup_case(gold)
    tr = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu', torch.float64))
    load_states(tr, states)
    s = torch.randn(x_a.size(0), hp['gen']['style_dim'], 1, 1, generator=torch.Generator().manual_seed(3))
    out = tr.sample(x_a, x_b, s_a=s, s_b=s, return_mask=False)
    with padding(hp), torch.no_grad():
        for d, x, (_, second, first, _) in (('a2b', x_a, out[:4]), ('b2a', x_b, out[4:])):
            for i in range(tr.council_size):
                p = {k: v.double() for k, v in states['gen_' + d][i].items()}
                c = co.content_encode(p, hp, x.double())
                want, _ = co.decode(p, hp, c, s.double(), x.double())
                own, _ = co.decode(p, hp, c, co.style_encode(p, hp, x.double()), x.double())
                assert torch.allclose(first[i::tr.council_size].double(), want, rtol=0, atol=1e-9), (d, i)
                assert torch.allclose(second[i::tr.council_size].double(), own, rtol=0, atol=1e-9), (d, i)


class _Spy(TorchOps):
    def reflect_pad(self, *a, **k):
        raise AssertionError('reflect_pad ran with pad_type zero')

    reflect_pad_bwd = reflect_pad


@pytest.mark.parametrize('case', ['glasses64_n2_b2_recon_xsc_iter3', 'm2f64_n4_b2'])
def test_zero_runs_no_pad_op(case):
    """pad_type zero (the shipped configs): neither padding op runs in training or sampling"""
    gold = load_golden(case)
    hp, states, x_a, x_b = setup_case(gold)
    assert hp['gen']['pad_type'] == hp['dis']['pad_type'] == 'zero'
    tr = Council_Trainer(hp, 'cpu', _ops=_Spy('cpu'))
    load_states(tr, states)
    tr.dis_update(x_a, x_b, hp)
    tr.dis_council_update(x_a, x_b, hp)
    tr.gen_update(x_a, x_b, hp, gold['iteration'])
    tr.sample(x_a, x_b, return_mask=False)


@pytest.mark.parametrize('net', ['gen', 'dis'])
@pytest.mark.parametrize('pad_type', ['replicate', 'circular'])
def test_other_pad_types_refused(net, pad_type):
    hp = config_for('glasses')
    hp[net]['pad_type'] = pad_type
    with pytest.raises(AssertionError):
        Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))


@pytest.mark.parametrize('net', ['gen', 'dis'])
def test_map_smaller_than_pad_raises(net):
    """ReflectionPad2d needs the pad to be smaller than the padded dimension (the generator's 2x2 content map under its pad-1 residual
    blocks at 8x8 images; the discriminator's last 4x4 stride-2 layers on 1x1 maps)"""
    gold = load_golden('glasses64_n2_b2_reflect_gen')
    hp, states, _, _ = setup_case(gold)
    hp['gen']['pad_type'], hp['dis']['pad_type'] = ('reflect', 'zero') if net == 'gen' else ('zero', 'reflect')
    tr = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    load_states(tr, states)
    x_a, x_b = co.synth_inputs(2, 4 if net == 'gen' else 16, seed=1)
    with pytest.raises(RuntimeError):
        tr.dis_update(x_a, x_b, hp)


def test_save_resume_round_trip(tmp_path):
    """reflect changes no parameter name: the checkpoint files and keys are those of zero padding, and resume() restores every bank"""
    gold = dict(load_golden('glasses64_n2_b2_reflect_recon'))
    out = {}
    for pad in ('zero', 'reflect'):
        tr, hp = _run(gold, ops=TorchOps('cpu'), hp_over={'gen': dict(config_for(gold)['gen'], pad_type=pad),
                                                           'dis': dict(config_for(gold)['dis'], pad_type=pad)})
        d = tmp_path / pad
        d.mkdir()
        tr.save(str(d), 10)
        out[pad] = {f: {k: (sorted(v.keys()) if isinstance(v, dict) else None) for k, v in torch.load(d / f).items()}
                    for f in sorted(os.listdir(d))}
    assert out['zero'] == out['reflect']
    tr2 = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    assert tr2.resume(str(tmp_path / 'reflect'), hp) == 11
    tr.synchronize()
    for name, net in tr._nets.items():
        for a, b in zip(net._banks(), tr2._nets[name]._banks()):
            assert torch.equal(a.data, b.data), name
