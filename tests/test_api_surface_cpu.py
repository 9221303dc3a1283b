"""Reference API surface beyond the three updates (SURVEY.md section 8f): checkpoint files, resume, sample(),
update_learning_rate, unsupported-path errors.  CPU, torch test double for the op-set."""
import os

import pytest
import torch

import council_oracle as co
from common import config_for, load_golden, setup_case
from council_gan_b200.trainer_council import Council_Trainer
from ops_torch import TorchOps
from test_trainer_host_cpu import load_states


def make(gold_name='glasses64_n2_b2_early'):
    gold = load_golden(gold_name)
    hp, states, x_a, x_b = setup_case(gold)
    co.seed_all(3)
    tr = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    load_states(tr, states)
    return tr, hp, states, x_a, x_b


def test_checkpoint_files_and_resume(tmp_path):
    tr, hp, states, x_a, x_b = make()
    co.seed_all(5)
    tr.dis_update(x_a, x_b, hp)
    tr.gen_update(x_a, x_b, hp, hp['iteration'])
    tr.save(str(tmp_path), 41)
    names = sorted(os.listdir(tmp_path))
    # reference naming: {a2b,b2a}_{gen,dis,dis_council}_{i}_{iter+1:08d}.pt + optimizer_{i}.pt  (trainer_council.py:969-992)
    for i in range(2):
        for fam in ('gen', 'dis', 'dis_council'):
            assert 'a2b_%s_%d_%08d.pt' % (fam, i, 42) in names
        assert 'optimizer_%d.pt' % i in names
    sd = torch.load(os.path.join(tmp_path, 'a2b_gen_0_%08d.pt' % 42))['a2b']
    ref_keys = [k[:-4] if k.endswith('#buf') else k for k, _ in co.gen_param_shapes(hp)]
    assert list(sd.keys()) == ref_keys
    for (k, shape), kk in zip(co.gen_param_shapes(hp), ref_keys):
        assert tuple(sd[kk].shape) == tuple(shape), kk
    # resume into a fresh trainer: parameters, Adam moments and the iteration come back
    co.seed_all(9)
    tr2 = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    it = tr2.resume(str(tmp_path), hp)
    assert it == 42
    for name, net in tr._nets.items():
        assert torch.equal(net.bank.data, tr2._nets[name].bank.data), name
        assert torch.equal(net.bank.exp_avg, tr2._nets[name].bank.exp_avg), name
        assert net.bank.step == tr2._nets[name].bank.step
    # the next update is identical
    co.seed_all(6)
    tr.dis_update(x_a, x_b, hp)
    co.seed_all(6)
    tr2.dis_update(x_a, x_b, hp)
    assert torch.equal(tr._nets['dis_a2b'].bank.data, tr2._nets['dis_a2b'].bank.data)


def test_sample_and_lr_schedule():
    tr, hp, states, x_a, x_b = make()
    out = tr.sample(x_a, x_b)
    assert len(out) == 8 and out[4] is None  # a2b only: (x_a, mask, x_ab1, x_ab2, None, None, None, None)
    n = x_a.size(0) * tr.council_size
    assert out[0].shape == (n, 3, 64, 64) and out[1].shape == (n, 3, 64, 64) and out[2].shape == out[3].shape == (n, 3, 64, 64)
    assert float(out[1].min()) >= 0 and float(out[1].max()) <= 1  # masks
    # StepLR(step_size, gamma): lr halves after step_size scheduler steps (utils.py:392-400)
    hp2 = dict(hp, step_size=3, gamma=0.5)
    tr3 = Council_Trainer(hp2, 'cpu', _ops=TorchOps('cpu'))
    lrs = []
    for _ in range(7):
        lrs.append(tr3._lr('gen'))
        tr3.update_learning_rate()
    assert lrs == [hp['lr']] * 3 + [hp['lr'] * 0.5] * 3 + [hp['lr'] * 0.25]


def test_unsupported_paths_raise():
    hp = config_for('glasses')
    for key in ('recon_x_w', 'vgg_w', 'council_abs_w'):
        with pytest.raises(NotImplementedError):
            Council_Trainer(dict(hp, **{key: 1}), 'cpu', _ops=TorchOps('cpu'))
    bad = dict(hp, dis=dict(hp['dis'], gan_type='nsgan'))
    with pytest.raises(AssertionError):
        Council_Trainer(bad, 'cpu', _ops=TorchOps('cpu'))
    tr = Council_Trainer(dict(hp, council=dict(hp['council'], council_size=2)), 'cpu', _ops=TorchOps('cpu'))
    with pytest.raises(NotImplementedError):
        tr.forward(torch.zeros(1, 3, 64, 64))


def test_gating_before_start_iterations():
    """dis_council_update is a no-op before council_start_at_iter; N<=1 prints the reference's message."""
    tr, hp, states, x_a, x_b = make()
    before = tr._nets['dis_council_a2b'].bank.data.clone()
    tr.loss_dis_council_total_s = 'untouched'
    tr.dis_council_update(x_a, x_b, hp)  # iteration 100 < 10000
    assert tr.loss_dis_council_total_s == 'untouched'
    assert torch.equal(before, tr._nets['dis_council_a2b'].bank.data)


def test_optimizer_file_is_torch_adam_state_dict(tmp_path):
    """optimizer_{i}.pt holds {'gen','dis','dis_council': torch.optim.Adam.state_dict()} like the reference (:988-992): a real
    torch.optim.Adam over reference-shaped parameters must load it, moment shapes must be the OIHW parameter shapes, and a
    reference-written file must round-trip through resume() into our flat moment buffers."""
    tr, hp, states, x_a, x_b = make()
    co.seed_all(5)
    tr.dis_update(x_a, x_b, hp)
    tr.gen_update(x_a, x_b, hp, hp['iteration'])
    tr.save(str(tmp_path), 9)
    opt = torch.load(os.path.join(tmp_path, 'optimizer_1.pt'))
    assert set(opt) == {'gen', 'dis', 'dis_council'}
    shapes = {'gen': [s for k, s in co.gen_param_shapes(hp) if not k.endswith('#buf')],
              'dis': [s for _, s in co.dis_param_shapes(hp, False)], 'dis_council': [s for _, s in co.dis_param_shapes(hp, True)]}
    for fam in ('gen', 'dis'):
        params = [torch.zeros(s, requires_grad=True) for s in shapes[fam]]
        adam = torch.optim.Adam(params, lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), weight_decay=hp['weight_decay'])
        adam.load_state_dict(opt[fam])  # raises on a layout mismatch
        st = adam.state_dict()['state']
        assert len(st) > 0
        for idx, ent in st.items():
            assert tuple(ent['exp_avg'].shape) == tuple(shapes[fam][idx]), (fam, idx)
            assert float(ent['step']) == 1.0
        if fam == 'gen':  # the style encoder never receives a gradient: no state entries, like the reference
            n_style = sum(1 for k, _ in co.gen_param_shapes(hp) if k.startswith('enc_style'))
            assert all(idx >= n_style for idx in st)
    # a file written by torch.optim.Adam itself (what the reference saves) comes back through resume()
    params = [torch.randn(s).requires_grad_(True) for s in shapes['dis']]
    adam = torch.optim.Adam(params, lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), weight_decay=hp['weight_decay'])
    for p in params:
        p.grad = torch.randn_like(p)
    adam.step()
    adam.step()
    ref_sd = adam.state_dict()
    full = torch.load(os.path.join(tmp_path, 'optimizer_0.pt'))
    full['dis'] = ref_sd
    torch.save(full, os.path.join(tmp_path, 'optimizer_0.pt'))
    tr2 = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    tr2.resume(str(tmp_path), hp)
    assert tr2._nets['dis_a2b'].bank.step == 2
    back = tr2._opt_state_dict('dis', 0)['state']
    for idx, ent in ref_sd['state'].items():
        assert torch.equal(back[idx]['exp_avg'], ent['exp_avg']) and torch.equal(back[idx]['exp_avg_sq'], ent['exp_avg_sq']), idx


def test_image_cache_misses_on_a_new_tensor():
    """The three updates of one iteration share one upload; a NEW host tensor (even with equal contents, even at the address of
    a freed one) is always uploaded again -- bench.py's e2e leg relies on it."""
    tr, hp, states, x_a, x_b = make()
    m0 = tr.img_cache_misses
    tr._img(x_a)
    tr._img(x_b)
    tr._img(x_a)
    assert tr.img_cache_misses - m0 == 2
    x_c = x_a.clone()
    tr._img(x_c)
    assert tr.img_cache_misses - m0 == 3
    x_a.add_(1.0)  # in-place change of a cached tensor bumps its version
    tr._img(x_a)
    assert tr.img_cache_misses - m0 == 4


def test_batched_sample_equals_member_api():
    """sample() runs all members / images as one stacked pass; row (i * M + j) must equal member j's own encode/decode of image i."""
    tr, hp, states, x_a, x_b = make()
    torch.manual_seed(11)
    out = tr.sample(x_a, x_b, council_member_to_sample_vec=[1, 0])
    torch.manual_seed(11)
    s2 = torch.randn(x_a.size(0), hp['gen']['style_dim'], 1, 1)
    row = 0
    for i in range(x_a.size(0)):
        xi = x_a[i:i + 1]
        for j in (1, 0):
            g = tr.gen_a2b_s[j]
            c, _ = g.encode(xi)
            o1, m1 = g.decode(c, tr.s_b[i:i + 1], xi, return_mask=True)
            o2 = g.decode(c, s2[i:i + 1], xi)
            # batch-1 and stacked convolutions sum in different orders on CPU; the mask head is tanh(10 h): fp32 noise x10
            assert torch.allclose(out[0][row], xi[0]) and (out[1][row] - m1[0]).abs().max() < 2e-3
            assert (out[2][row] - o1[0]).abs().max() < 2e-3 and (out[3][row] - o2[0]).abs().max() < 2e-3
            row += 1
    rec = tr.sample(x_a, x_b, return_mask=False)  # second entry = reconstruction with each member's own style code
    c, s_fake = tr.gen_a2b_s[1].encode(x_a[0:1])
    assert (rec[1][1] - tr.gen_a2b_s[1].decode(c, s_fake, x_a[0:1])[0]).abs().max() < 2e-3


def test_weight_init_statistics():
    """weights_init (utils.py:402-422): kaiming fan_in normal for generators, N(0, 0.02) for both discriminators, zero biases."""
    import math
    tr, hp, states, x_a, x_b = make()
    co.seed_all(1)
    tr2 = Council_Trainer(hp, 'cpu', _ops=TorchOps('cpu'))
    sd = tr2.gen_a2b_s[0].state_dict()
    w = sd['enc_content.model.3.model.0.model.0.conv.weight']  # 256 x 256 x 3 x 3
    assert abs(w.std().item() / math.sqrt(2.0 / (w.shape[1] * 9)) - 1) < 0.02 and abs(w.mean().item()) < 1e-3
    w = sd['mlp.model.1.fc.weight']
    assert abs(w.std().item() / math.sqrt(2.0 / w.shape[1]) - 1) < 0.03
    assert all(float(v.abs().max()) == 0 for k, v in sd.items() if k.endswith('.bias'))
    for net in (tr2.dis_a2b_s[1], tr2.dis_council_a2b_s[0]):
        sdd = net.state_dict()
        w = sdd['cnns.0.2.conv.weight']
        assert abs(w.std().item() / 0.02 - 1) < 0.02 and abs(w.mean().item()) < 2e-4
        assert all(float(v.abs().max()) == 0 for k, v in sdd.items() if k.endswith('.bias'))
    a, b = tr2.gen_a2b_s[0].state_dict(), tr2.gen_a2b_s[1].state_dict()
    assert not torch.equal(a['dec.model.2.conv.weight'], b['dec.model.2.conv.weight'])  # members are initialised independently


def test_update_pins_the_stream_and_picks_pdl_by_batch_size():
    """host logic of the launch path: an update resolves the stream once (ops.pin_stream / unpin_stream around the call, also when it
    raises) and turns programmatic dependent launch on only for small batches."""
    from council_gan_b200 import trainer_council as tc

    class FakeOps:
        def __init__(self):
            self._stream_cached, self.log = None, []

        def pin_stream(self):
            self._stream_cached = 1
            self.log.append('pin')

        def unpin_stream(self):
            self._stream_cached = None
            self.log.append('unpin')

        def set_pdl(self, on):
            self.log.append(('pdl', bool(on)))

    class T:
        def __init__(self):
            self.ops = FakeOps()

        @tc._pinned
        def update(self, x, fail=False):
            assert self.ops._stream_cached == 1
            if fail:
                raise ValueError('boom')
            return self.nested(x)

        @tc._pinned
        def nested(self, x):  # an update called from inside another one does not unpin
            return 'ok'

    t = T()
    assert t.update(torch.zeros(1, 3, 128, 128)) == 'ok'
    assert t.ops.log == ['pin', ('pdl', True), 'unpin'] and t.ops._stream_cached is None
    t.ops.log.clear()
    t.update(torch.zeros(8, 3, 256, 256))
    assert t.ops.log == ['pin', ('pdl', False), 'unpin']
    t.ops.log.clear()
    t.update(torch.zeros(1, 2, 64, 64, tc.IMG_C))  # channels-last device batch [1, B, H, W, lanes]
    assert t.ops.log[1] == ('pdl', True)
    t.ops.log.clear()
    with pytest.raises(ValueError):
        t.update(torch.zeros(1, 3, 64, 64), fail=True)
    assert t.ops.log[-1] == 'unpin' and t.ops._stream_cached is None
