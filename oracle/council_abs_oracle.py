"""CPU oracle of the council abs loss council_abs_w  --  TEST INFRASTRUCTURE ONLY.

Extends ``council_oracle.OracleTrainer`` (plain PyTorch, CPU, autograd) with the reference's discriminator-free council term,
trainer_council.py:224-228 (criteria) and :595-619 (the term in loop 2 of gen_update): member i's translation against the detached
translation of one peer drawn with ``random.choice``, in colour or on channel sums (council_abs_gray_scale), weighted by council_abs_w.
Each direction's term joins the OTHER direction's published council loss (:616-619); the member total gets both.  Pinned against the
unmodified reference by ``oracle/make_golden_council_abs.py`` (tests/golden/*_council_abs*.json).  Like the base oracle it is the
checker, never the product.
"""
from __future__ import annotations

import random

import numpy as np
import torch

import council_oracle as co


def council_abs_color(x, target):
    """council_basic_criterion_with_color trainer_council.py:227-228"""
    return torch.mean(torch.abs(x - target))


def council_abs_gray(x, target):
    """council_basic_criterion_gray_scale trainer_council.py:224-225"""
    return torch.mean(torch.abs(torch.sum(x, 1) - torch.sum(target, 1)))


class CouncilAbsOracleTrainer(co.OracleTrainer):
    """OracleTrainer with council_abs_w allowed (both directions on).  Publishes ``council_loss_s`` = {'a2b': [...], 'b2a': [...]}, the
    reference's council_loss_ab_s / council_loss_ba_s (one entry per member, the int 0 while the gate is closed), and ``peers``, the
    members drawn by gen_update."""

    def __init__(self, hp, states):
        super().__init__(dict(hp, council_abs_w=0), states)  # the base refuses the term; everything else is the same
        self.hp = hp
        assert hp['council_abs_w'] == 0 or (hp['do_a2b'] and hp['do_b2a']), \
            'the reference fails with an AttributeError on a single direction (trainer_council.py:617-619)'

    # -- gen_update  trainer_council.py:280-634: council_oracle.OracleTrainer.gen_update with the term of :595-619 in loop 2 ---------
    def gen_update(self, x_a, x_b, hp, iterations=0):
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
        self.loss_gen_total_s = []
        self.loss_gen_adv_s = {d: [] for d in self.dirs}
        self.loss_gen_mask_zero_one_s = {d: [] for d in self.dirs}
        self.loss_gen_mask_total_s = {d: [] for d in self.dirs}
        self.loss_gen_mask_TV_s = {d: [] for d in self.dirs}
        self.council_loss_s = {d: [] for d in self.dirs}
        self.peers = []
        self.x_fake_gen = {d: [] for d in self.dirs}
        self.mask_gen = {d: [] for d in self.dirs}
        totals = []
        for i in range(self.N):  # loop 1, :328-538
            total = 0
            for d in self.dirs:
                g = self.P['gen_' + d][i]
                src = self._src(d, x_a, x_b)
                cc = co.content_encode(g, hp, src)
                xf, mask = co.decode(g, hp, cc, s[d], src)
                self.x_fake_gen[d].append(xf)
                self.mask_gen[d].append(mask)
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
            if hp['gan_w'] != 0:  # :497-529
                for d in self.dirs:
                    adv = co.lsgan_gen_loss(co.ms_dis(self.P['dis_' + d][i], hp, self.x_fake_gen[d][i]))
                    self.loss_gen_adv_s[d].append(adv)
                    if hp['do_w_loss_matching']:
                        self.hist_gan[d][i].append(adv.detach().cpu().numpy())
                        self.hist_gan[d][i].popleft()
                    total = total + hp['gan_w'] * adv
            totals.append(total)
        do_council = self._council_active(hp, for_gen=True)
        self.w_match = {d: 1 for d in self.dirs}
        crit = council_abs_gray if hp['council_abs_gray_scale'] else council_abs_color
        for i in range(self.N):  # loop 2, :558-634
            total = totals[i]
            if (hp['council_w'] != 0 or hp['council_abs_w'] != 0) and do_council and self.N > 1:
                cl = {d: 0 for d in self.dirs}
                if self.do_dis_council:  # :567-593
                    for d in self.dirs:
                        src = self._src(d, x_a, x_b)
                        c = co.lsgan_gen_loss(co.ms_dis_council(self.P['dis_council_' + d][i], hp, self.x_fake_gen[d][i], src))
                        if hp['do_w_loss_matching']:  # :576-586
                            self.hist_council[d][i].append(c.detach().cpu().numpy())
                            self.hist_council[d][i].popleft()
                            self.w_match[d] = np.mean(self.hist_gan[d][i]) / np.mean(self.hist_council[d][i])
                            c = c * self.w_match[d]
                        cl[d] = cl[d] + c * hp['council_w']
                if hp['council_abs_w'] != 0:  # :595-619: one peer for both directions; the peer's image is detached
                    j = random.choice(list(range(0, i)) + list(range(i + 1, self.N)))
                    self.peers.append(j)
                    ab = {d: hp['council_abs_w'] * crit(self.x_fake_gen[d][i], self.x_fake_gen[d][j].detach()) for d in self.dirs}
                    cl['a2b'] = cl['a2b'] + ab['b2a']  # :616-619, sic: each list takes the other direction's term
                    cl['b2a'] = cl['b2a'] + ab['a2b']
                for d in self.dirs:  # :621-624
                    self.council_loss_s[d].append(cl[d])
                    total = total + cl[d]
            else:
                for d in self.dirs:
                    self.council_loss_s[d].append(0)
            self.loss_gen_total_s.append(total)
            total.backward()
            self.gen_opt[i].step()
        # reference leaves stale grads on D/DC that the next dis_update zeroes (:738-739, :803-804)
        for fam in ('dis', 'dis_council'):
            for d in self.dirs:
                for sd in self.P.get('%s_%s' % (fam, d), []):
                    for v in sd.values():
                        v.grad = None
