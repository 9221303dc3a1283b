"""CPU oracle of the image reconstruction term recon_x_w  --  TEST INFRASTRUCTURE ONLY.

Extends ``recon_oracle.ReconOracleTrainer`` (the oracle trainer with abs_beginning_end, recon_c_w and recon_s_w) with the
reference's within-domain decode, trainer_council.py:339-345 -- each source image decoded by the other direction's generator with
the member's own content and style codes, composited over the source -- and its loss, :455-459, added to the member total before
the latent terms.  Nothing is detached: the loss trains the other generator's decoder, head and MLP and this generator's content
and style encoders.  Pinned against the unmodified reference by ``oracle/make_golden_recon_x.py`` (tests/golden/*_recon_x*.json).
Like the base oracle it is the checker, never the product.
"""
from __future__ import annotations

import numpy as np
import torch

import council_oracle as co
from abs_beginning_end_oracle import recon_v2_color
from recon_oracle import ReconOracleTrainer, recon_criterion


class ReconXOracleTrainer(ReconOracleTrainer):
    """The oracle trainer with recon_x_w allowed as well (both directions on).  Publishes the reference's
    ``loss_gen_recon_{x,s,c}_{a,b}_s`` lists (unweighted, one entry per member; [] while a weight is 0)."""

    def __init__(self, hp, states):
        super().__init__(dict(hp, recon_x_w=0), states)  # the base refuses the term; everything else is the same
        self.hp = hp
        assert hp['recon_x_w'] == 0 or (hp['do_a2b'] and hp['do_b2a']), \
            'the reference fails with an IndexError on a single direction (trainer_council.py:344)'

    # -- gen_update: ReconOracleTrainer.gen_update with the within-domain decode of :339-345 and the term of :455-459 in loop 1 -----
    def gen_update(self, x_a, x_b, hp, iterations=0):  # trainer_council.py:280-634
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
