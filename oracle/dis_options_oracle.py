"""CPU oracle of the discriminator-side switches do_Dis_only_gray, useRandomGen and useRandomDis  --  TEST INFRASTRUCTURE ONLY.

Extends ``council_oracle.OracleTrainer`` (plain PyTorch, CPU, autograd) with the reference's three switches, in the reference's order:
  * do_Dis_only_gray (trainer_council.py:736-737, 761, 765 in dis_update; :504, 510 in gen_update): the non-council discriminator sees
    ``torch.sum(x, 1).unsqueeze(1).repeat(1, input_dim, 1, 1) / input_dim``; council discriminators keep seeing colour;
  * useRandomGen (:748-750): dis_update trains D_i on the translation of generator ``np.random.randint(N)``, one draw per member;
  * useRandomDis (:499-501): gen_update takes member i's adversarial loss from D_``np.random.randint(N)``, one draw per member while
    gan_w != 0; the loss history and w_match stay member i's.
The draws are kept in ``dis_draws`` / ``gen_draws``.  Pinned against the unmodified reference by
``oracle/make_golden_dis_options.py`` (tests/golden/*gray*.json, *random_pairing*.json, *dis_options*.json).  Like the base oracle it
is the checker, never the product.
"""
from __future__ import annotations

import numpy as np
import torch

import council_oracle as co


def gray(x, input_dim=3):
    """trainer_council.py:736 / 504: channel sum repeated over the channels, divided by input_dim"""
    return torch.sum(x, 1).unsqueeze(1).repeat(1, input_dim, 1, 1) / input_dim


class DisOptionsOracleTrainer(co.OracleTrainer):
    """OracleTrainer with do_Dis_only_gray, useRandomGen and useRandomDis allowed."""

    # -- dis_update  trainer_council.py:735-780 ------------------------------------------------
    def dis_update(self, x_a, x_b, hp):
        to_dis = gray if hp['dis']['do_Dis_only_gray'] else (lambda x: x)
        for o in self.dis_opt:
            o.zero_grad()
        s = {}
        if 'a2b' in self.dirs:  # :740-745, draw order a2b (s_b) then b2a (s_a)
            s['a2b'] = torch.randn(x_b.size(0), self.style_dim, 1, 1).to(x_b.device)
        if 'b2a' in self.dirs:
            s['b2a'] = torch.randn(x_a.size(0), self.style_dim, 1, 1).to(x_a.device)
        self.loss_dis_total_s = []
        self.loss_dis_s = {d: [] for d in self.dirs}
        self.dis_draws = []
        for i in range(self.N):
            i_gen = i
            if hp['dis']['useRandomGen']:  # :748-750
                i_gen = np.random.randint(self.N)
                self.dis_draws.append(i_gen)
            total = 0
            for d in self.dirs:
                g = self.P['gen_' + d][i_gen]
                src = self._src(d, x_a, x_b)
                with torch.no_grad():
                    c = co.content_encode(g, hp, src)
                    x_fake, _ = co.decode(g, hp, c, s[d], src)
                dp = self.P['dis_' + d][i]
                loss = co.lsgan_dis_loss(co.ms_dis(dp, hp, to_dis(x_fake)), co.ms_dis(dp, hp, to_dis(self._real(d, x_a, x_b))))
                self.loss_dis_s[d].append(loss)
                total = total + (hp['gan_w'] * loss if d == 'a2b' else loss)  # :775 / :777
            self.loss_dis_total_s.append(total)
            total.backward()
            self.dis_opt[i].step()

    # -- gen_update  trainer_council.py:280-634: council_oracle.OracleTrainer.gen_update with the switches of :499-510 in loop 1 -----
    def gen_update(self, x_a, x_b, hp, iterations=0):
        assert not hp['focus_loss']['do_w_loss_matching_focus']
        to_dis = gray if hp['dis']['do_Dis_only_gray'] else (lambda x: x)
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
        self.x_fake_gen = {d: [] for d in self.dirs}
        self.mask_gen = {d: [] for d in self.dirs}
        self.gen_draws = []
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
                i_dis = i
                if hp['gen']['useRandomDis']:  # :499-501
                    i_dis = np.random.randint(self.N)
                    self.gen_draws.append(i_dis)
                for d in self.dirs:
                    adv = co.lsgan_gen_loss(co.ms_dis(self.P['dis_' + d][i_dis], hp, to_dis(self.x_fake_gen[d][i])))
                    self.loss_gen_adv_s[d].append(adv)
                    if hp['do_w_loss_matching']:  # member i's history, whichever discriminator judged it
                        self.hist_gan[d][i].append(adv.detach().cpu().numpy())
                        self.hist_gan[d][i].popleft()
                    total = total + hp['gan_w'] * adv
            totals.append(total)
        do_council = self._council_active(hp, for_gen=True)
        self.w_match = {d: 1 for d in self.dirs}
        for i in range(self.N):  # loop 2, :558-634: the council discriminators see colour
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
