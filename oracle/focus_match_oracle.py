"""CPU oracle of focus-loss matching (do_w_loss_matching_focus)  --  TEST INFRASTRUCTURE ONLY.

Extends ``council_oracle.OracleTrainer`` (plain PyTorch, CPU, autograd) with the reference's focus matching
(trainer_council.py:398-410, 433-445), in the reference's order within member i:
  * zero-one term (mask_zero_or_one_w != 0), a2b then b2a: append the unscaled value to the zero-one history, then scale the term by
    mean(GAN history) / mean(zero-one history) -- the GAN history as it was BEFORE this member's GAN append (:497-529 runs later);
  * TV term, unmatched;
  * mask-total term, whenever the focus gate is open: a2b appends its unscaled term and scales it; b2a appends a2b's SCALED term
    (:441) and scales its own by its own ratio.
The ratios of the last member are kept in ``w_match_focus{,_zero_one}[d]``.  Pinned against the unmodified reference by
``oracle/make_golden_focus_match.py`` (tests/golden/*focus_match*.json).  Like the base oracle it is the checker, never the product.
"""
from __future__ import annotations

from collections import deque

import numpy as np
import torch

import council_oracle as co


class FocusMatchOracleTrainer(co.OracleTrainer):
    """OracleTrainer with do_w_loss_matching_focus allowed."""

    def __init__(self, hp, states):
        super().__init__(hp, states)
        hist = hp['loss_matching_hist_size']
        self.hist_focus = {d: [deque(np.ones(hist)) for _ in range(self.N)] for d in self.dirs}  # :73-92
        self.hist_focus_zero_one = {d: [deque(np.ones(hist)) for _ in range(self.N)] for d in self.dirs}
        self.w_match_focus = {d: 1 for d in self.dirs}  # :65-68
        self.w_match_focus_zero_one = {d: 1 for d in self.dirs}

    @staticmethod
    def _append(hist, v):
        hist.append(v.detach().cpu().numpy().copy())
        hist.popleft()

    # -- gen_update  trainer_council.py:280-634 --------------------------------------------------
    def gen_update(self, x_a, x_b, hp, iterations=0):
        assert not hp['gen']['useRandomDis'] and not hp['dis']['do_Dis_only_gray']
        fl = hp['focus_loss']
        match = bool(fl['do_w_loss_matching_focus'])
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
                if hp['mask_zero_or_one_w'] != 0:  # :392-415
                    for d in self.dirs:
                        l01 = co.mask_zero_one(self.mask_gen[d][i], fl['mask_zero_or_one_center'], fl['mask_zero_or_one_epsilon'])
                        if match:  # :398-410
                            self._append(self.hist_focus_zero_one[d][i], l01)
                            w = np.mean(self.hist_gan[d][i]) / np.mean(self.hist_focus_zero_one[d][i])
                            self.w_match_focus_zero_one[d] = w
                            l01 = l01 * w
                        self.loss_gen_mask_zero_one_s[d].append(l01)
                        total = total + hp['mask_zero_or_one_w'] * l01
                lts = {}
                if hp['mask_total_w'] != 0:  # :418-422
                    for d in self.dirs:
                        lts[d] = co.mask_small(self.mask_gen[d][i], fl['mask_small_use_abs'], fl['mask_small_use_square'])
                if hp['mask_tv_w'] != 0:  # :425-431
                    for d in self.dirs:
                        ltv = co.mask_tv(self.mask_gen[d][i])
                        self.loss_gen_mask_TV_s[d].append(ltv)
                        total = total + hp['mask_tv_w'] * ltv
                for d in self.dirs:  # :433-451
                    lt = lts.get(d)
                    if lt is None:
                        continue
                    if match:
                        self._append(self.hist_focus[d][i], lts['a2b'] if d == 'b2a' else lt)  # :441: b2a appends a2b's scaled term
                        w = np.mean(self.hist_gan[d][i]) / np.mean(self.hist_focus[d][i])
                        self.w_match_focus[d] = w
                        lt = lt * w
                        lts[d] = lt
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
        for i in range(self.N):  # loop 2, :558-634
            total = totals[i]
            if (hp['council_w'] != 0) and do_council and self.N > 1:
                for d in self.dirs:
                    src = self._src(d, x_a, x_b)
                    cl = co.lsgan_gen_loss(co.ms_dis_council(self.P['dis_council_' + d][i], hp, self.x_fake_gen[d][i], src))
                    if hp['do_w_loss_matching']:  # :576-586, the GAN history after this update's append
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
        for fam in ('dis', 'dis_council'):  # the reference's stale D / DC grads are zeroed by the next dis_update (:738-739, :803-804)
            for d in self.dirs:
                for sd in self.P.get('%s_%s' % (fam, d), []):
                    for v in sd.values():
                        v.grad = None
