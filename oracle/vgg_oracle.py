"""CPU oracle of the perceptual loss vgg_w  --  TEST INFRASTRUCTURE ONLY.

Extends ``recon_x_oracle.ReconXOracleTrainer`` (the oracle trainer with abs_beginning_end, recon_x_w, recon_c_w and recon_s_w) with the
reference's domain-invariant perceptual loss, trainer_council.py:531-538 and compute_vgg_loss :636-641: each member's translation and
its source image through vgg_preprocess (utils.py:380-390) and the frozen Vgg16 up to relu5_3 (networks.py:573-622), compared after
nn.InstanceNorm2d(512) (:121) by the mean squared error.  The translations take the gradient, the targets and the VGG weights none.
Also the seeded synthetic VGG-16 weights the fixtures are made with (``synth_vgg16``: the real ones are 59 MB and not redistributable
here) and their file layout (``write_vgg16``).  Pinned against the unmodified reference by ``oracle/make_golden_vgg.py``
(tests/golden/*_vgg*.json).  Like the base oracle it is the checker, never the product.
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.nn.functional as F

import council_oracle as co
from abs_beginning_end_oracle import recon_v2_color
from recon_oracle import recon_criterion
from recon_x_oracle import ReconXOracleTrainer

VGG_LAYERS = [('conv1_1', 3, 64), ('conv1_2', 64, 64), ('conv2_1', 64, 128), ('conv2_2', 128, 128), ('conv3_1', 128, 256),
              ('conv3_2', 256, 256), ('conv3_3', 256, 256), ('conv4_1', 256, 512), ('conv4_2', 512, 512), ('conv4_3', 512, 512),
              ('conv5_1', 512, 512), ('conv5_2', 512, 512), ('conv5_3', 512, 512)]
POOL_AFTER = ('conv1_2', 'conv2_2', 'conv3_3')


def synth_vgg16(seed):
    """A Vgg16 state_dict (keys conv{1_1..5_3}.{weight,bias}, float32): kaiming-normal fan-in weights, std sqrt(2 / (9 cin)), and
    biases N(0, 0.01^2), drawn layer by layer (weight, then bias) from one CPU generator seeded with `seed`."""
    gen = torch.Generator().manual_seed(seed)
    sd = {}
    for k, cin, cout in VGG_LAYERS:
        sd[k + '.weight'] = torch.randn(cout, cin, 3, 3, generator=gen) * float(np.sqrt(2.0 / (9 * cin)))
        sd[k + '.bias'] = torch.randn(cout, generator=gen) * 0.01
    return sd


def write_vgg16(sd, vgg_model_path):
    """Write sd where load_vgg16 (utils.py:350-366) reads it for hp['vgg_model_path'] = vgg_model_path -> the file's path"""
    d = os.path.join(vgg_model_path, 'models')
    os.makedirs(d, exist_ok=True)
    path = os.path.join(d, 'vgg16.weight')
    torch.save(sd, path)
    return path


def vgg_preprocess(x):
    """utils.py:380-390 on NCHW RGB in [-1, 1]"""
    r, g, b = torch.chunk(x, 3, dim=1)
    x = torch.cat((b, g, r), dim=1)
    x = (x + 1) * 255 * 0.5
    mean = torch.tensor([103.939, 116.779, 123.680], dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return x - mean


def vgg16(sd, x, keep=None):
    """Vgg16.forward (networks.py:594-622) -> relu5_3; keep (a list): every ReLU output"""
    h = x
    for k, _, _ in VGG_LAYERS:
        h = F.relu(F.conv2d(h, sd[k + '.weight'].to(h.dtype), sd[k + '.bias'].to(h.dtype), 1, 1))
        if keep is not None:
            keep.append(h)
        if k in POOL_AFTER:
            h = F.max_pool2d(h, kernel_size=2, stride=2)
    return h


def compute_vgg_loss(sd, img, target):
    """trainer_council.py:636-641 with nn.InstanceNorm2d(512, affine=False) (:121)"""
    f = vgg16(sd, vgg_preprocess(img))
    t = vgg16(sd, vgg_preprocess(target))
    return torch.mean((F.instance_norm(f, eps=1e-5) - F.instance_norm(t, eps=1e-5)) ** 2)


class VggOracleTrainer(ReconXOracleTrainer):
    """The oracle trainer with vgg_w > 0 allowed as well (both directions on); vgg_sd: the frozen Vgg16 state_dict.  Publishes the
    reference's ``loss_gen_vgg_{a,b}_s`` (one entry per member; [] while vgg_w is 0)."""

    def __init__(self, hp, states, vgg_sd=None):
        super().__init__(dict(hp, vgg_w=0), states)  # the base refuses the term; everything else is the same
        self.hp = hp
        assert hp['vgg_w'] >= 0, 'the reference fails with an AttributeError on a negative vgg_w (trainer_council.py:534)'
        assert hp['vgg_w'] == 0 or (hp['do_a2b'] and hp['do_b2a']), \
            'the reference fails with an IndexError on a single direction (trainer_council.py:534)'
        self.vgg = None if hp['vgg_w'] == 0 else {k: v.detach().clone() for k, v in vgg_sd.items()}

    # -- gen_update: ReconXOracleTrainer.gen_update with the term of :531-538 at the end of loop 1 --------------------------------
    def gen_update(self, x_a, x_b, hp, iterations=0):  # trainer_council.py:280-634, ReconXOracleTrainer.gen_update + :531-538
        assert not hp['gen']['useRandomDis'] and not hp['dis']['do_Dis_only_gray']
        assert not hp['focus_loss']['do_w_loss_matching_focus']
        fl = hp['focus_loss']
        for o in self.gen_opt:
            o.zero_grad()
        s_a = torch.randn(x_a.size(0), self.style_dim, 1, 1).to(x_a.device)  # :284-285 both always drawn, a then b
        s_b = torch.randn(x_b.size(0), self.style_dim, 1, 1).to(x_b.device)
        s = {'a2b': s_b, 'b2a': s_a}
        focus_on = hp['iteration'] > fl['focus_loss_start_at_iter'] and \
            (hp['mask_zero_or_one_w'] != 0 or hp['mask_total_w'] != 0)  # :390
        recon_on = hp['recon_s_w'] != 0 or hp['recon_c_w'] != 0
        self.loss_gen_total_s = []
        self.loss_gen_adv_s = {d: [] for d in self.dirs}
        self.loss_gen_mask_zero_one_s = {d: [] for d in self.dirs}
        self.loss_gen_mask_total_s = {d: [] for d in self.dirs}
        self.loss_gen_mask_TV_s = {d: [] for d in self.dirs}
        self.council_loss_s = {d: [] for d in self.dirs}
        self.loss_gen_beginning_end_s = {'a2b': [], 'b2a': []}
        self.loss_gen_recon_x_a_s, self.loss_gen_recon_x_b_s = [], []  # :308-309
        self.loss_gen_recon_s_a_s, self.loss_gen_recon_s_b_s = [], []
        self.loss_gen_recon_c_a_s, self.loss_gen_recon_c_b_s = [], []
        self.loss_gen_vgg_a_s, self.loss_gen_vgg_b_s = [], []  # :320-321
        self.x_fake_gen = {d: [] for d in self.dirs}
        self.mask_gen = {d: [] for d in self.dirs}
        totals = []
        for i in range(self.N):  # loop 1, :328-538
            total = 0
            content, style = {}, {}
            for d in self.dirs:
                g = self.P['gen_' + d][i]
                src = self._src(d, x_a, x_b)
                content[d] = co.content_encode(g, hp, src)
                if hp['recon_x_w'] != 0:  # :331-337: the member's own style code of its source image
                    style[d] = co.style_encode(g, hp, src)
            if hp['recon_x_w'] != 0:  # :339-345: decoded by the OTHER direction's generator; its mask takes no loss
                x_a_recon, _ = co.decode(self.P['gen_b2a'][i], hp, content['a2b'], style['a2b'], x_a)
                x_b_recon, _ = co.decode(self.P['gen_a2b'][i], hp, content['b2a'], style['b2a'], x_b)
            for d in self.dirs:  # :347-357
                g = self.P['gen_' + d][i]
                src = self._src(d, x_a, x_b)
                xf, mask = co.decode(g, hp, content[d], s[d], src)
                self.x_fake_gen[d].append(xf)
                self.mask_gen[d].append(mask)
            if recon_on:  # :359-369: x_ba through gen_a2b, x_ab through gen_b2a
                ga, gb = self.P['gen_a2b'][i], self.P['gen_b2a'][i]
                x_ab, x_ba = self.x_fake_gen['a2b'][i], self.x_fake_gen['b2a'][i]
                c_b_recon, s_a_recon = co.content_encode(ga, hp, x_ba), co.style_encode(ga, hp, x_ba)
                c_a_recon, s_b_recon = co.content_encode(gb, hp, x_ab), co.style_encode(gb, hp, x_ab)
            if focus_on:
                for d in self.dirs:
                    mask = self.mask_gen[d][i]
                    if hp['mask_zero_or_one_w'] != 0:  # :392-415
                        l01 = co.mask_zero_one(mask, fl['mask_zero_or_one_center'], fl['mask_zero_or_one_epsilon'])
                        self.loss_gen_mask_zero_one_s[d].append(l01)
                        total = total + hp['mask_zero_or_one_w'] * l01
                    if hp['mask_tv_w'] != 0:  # :425-431 (added to the total before the mask_total term)
                        ltv = co.mask_tv(mask)
                        self.loss_gen_mask_TV_s[d].append(ltv)
                        total = total + hp['mask_tv_w'] * ltv
                    if hp['mask_total_w'] != 0:  # :418-422, :447-451
                        lt = co.mask_small(mask, fl['mask_small_use_abs'], fl['mask_small_use_square'])
                        self.loss_gen_mask_total_s[d].append(lt)
                        total = total + hp['mask_total_w'] * lt
            if hp['recon_x_w'] != 0:  # :455-459
                self.loss_gen_recon_x_a_s.append(recon_criterion(x_a_recon, x_a))
                self.loss_gen_recon_x_b_s.append(recon_criterion(x_b_recon, x_b))
                total = total + hp['recon_x_w'] * (self.loss_gen_recon_x_a_s[i] + self.loss_gen_recon_x_b_s[i])
            if hp['recon_s_w'] != 0:  # :460-464
                self.loss_gen_recon_s_a_s.append(recon_criterion(s_a_recon, s_a))
                self.loss_gen_recon_s_b_s.append(recon_criterion(s_b_recon, s_b))
                total = total + hp['recon_s_w'] * (self.loss_gen_recon_s_a_s[i] + self.loss_gen_recon_s_b_s[i])
            if hp['recon_c_w'] != 0:  # :465-469, the targets c_a / c_b are not detached
                self.loss_gen_recon_c_a_s.append(recon_criterion(c_a_recon, content['a2b']))
                self.loss_gen_recon_c_b_s.append(recon_criterion(c_b_recon, content['b2a']))
                total = total + hp['recon_c_w'] * (self.loss_gen_recon_c_a_s[i] + self.loss_gen_recon_c_b_s[i])
            if hp['abs_beginning_end'] != 0 and self.abs_beginning_end_w_conf > 0.005:  # :477-495
                be = {}
                for d in self.DIRS:  # the int 0 for an inactive direction
                    be[d] = recon_v2_color(self.x_fake_gen[d][i], self._src(d, x_a, x_b)) if d in self.dirs else 0
                    self.loss_gen_beginning_end_s[d].append(be[d])
                self.abs_beginning_end_w_conf = max(hp['abs_beginning_end'] * hp['abs_beginning_end_less_by'] ** iterations,
                                                    hp['abs_beginning_end_minimume'])
                for d in self.dirs:
                    total = total + self.abs_beginning_end_w_conf * be[d]
            if hp['gan_w'] != 0:  # :497-529
                for d in self.dirs:
                    adv = co.lsgan_gen_loss(co.ms_dis(self.P['dis_' + d][i], hp, self.x_fake_gen[d][i]))
                    self.loss_gen_adv_s[d].append(adv)
                    if hp['do_w_loss_matching']:
                        self.hist_gan[d][i].append(adv.detach().cpu().numpy())
                        self.hist_gan[d][i].popleft()
                    total = total + hp['gan_w'] * adv
            if hp['vgg_w'] != 0:  # :531-538: x_ba against x_b, x_ab against x_a
                self.loss_gen_vgg_a_s.append(compute_vgg_loss(self.vgg, self.x_fake_gen['b2a'][i], x_b))
                self.loss_gen_vgg_b_s.append(compute_vgg_loss(self.vgg, self.x_fake_gen['a2b'][i], x_a))
                total = total + hp['vgg_w'] * (self.loss_gen_vgg_a_s[i] + self.loss_gen_vgg_b_s[i])
            totals.append(total)
        do_council = self._council_active(hp, for_gen=True)
        self.w_match = {d: 1 for d in self.dirs}
        for i in range(self.N):  # loop 2, :558-634
            total = totals[i]
            if (hp['council_w'] != 0) and do_council and self.N > 1:
                for d in self.dirs:
                    src = self._src(d, x_a, x_b)
                    cl = co.lsgan_gen_loss(co.ms_dis_council(self.P['dis_council_' + d][i], hp, self.x_fake_gen[d][i], src))
                    if hp['do_w_loss_matching']:  # :576-586
                        self.hist_council[d][i].append(cl.detach().cpu().numpy())
                        self.hist_council[d][i].popleft()
                        self.w_match[d] = np.mean(self.hist_gan[d][i]) / np.mean(self.hist_council[d][i])
                        cl = cl * self.w_match[d]
                    cl = cl * hp['council_w']
                    self.council_loss_s[d].append(cl)
                    total = total + cl
            self.loss_gen_total_s.append(total)
            total.backward()
            self.gen_opt[i].step()
        # reference leaves stale grads on D/DC that the next dis_update zeroes (:738-739, :803-804)
        for fam in ('dis', 'dis_council'):
            for d in self.dirs:
                for sd in self.P.get('%s_%s' % (fam, d), []):
                    for v in sd.values():
                        v.grad = None
