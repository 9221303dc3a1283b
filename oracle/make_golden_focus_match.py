"""Golden fixtures of focus-loss matching (do_w_loss_matching_focus) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden.py`` (its reference import shims, synthetic parameters, inputs and fixture layout), for cases
with the switch on (trainer_council.py:398-410, 433-445).  On top of make_golden's record, every iteration also records, per active
direction, the published losses, the four focus / GAN histories after the update (``hist``) and the reference's ratio attributes
``w_match_focus_<d>_conf`` / ``w_match_focus_zero_one_<d>_conf`` (the last member's).  Runs in the build container only.

    python oracle/make_golden_focus_match.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mk  # noqa: E402

FOCUS = {'focus_loss.do_w_loss_matching_focus': True}

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # a2b, focus gate open, histories of 2 entries over 3 iterations: every ring wraps
    'glasses64_n2_b2_focus_match_iter3': ('glasses', dict(FOCUS, **{'council.council_size': 2, 'loss_matching_hist_size': 2}),
                                          64, 2, 20001, 3),
    # both directions with council matching: b2a's mask-total history takes a2b's scaled term, and the focus ratios read the GAN
    # history before this update's append while w_match reads it after
    'glasses64_n2_b2_focus_match_both_iter3': ('glasses', dict(FOCUS, do_b2a=True, **{'council.council_size': 2,
                                                                                       'loss_matching_hist_size': 2}), 64, 2, 20001, 3),
    # mask_small_use_abs and mask_small_use_square together
    'glasses64_n2_b2_focus_match_abs_square': ('glasses', dict(FOCUS, **{'council.council_size': 2, 'loss_matching_hist_size': 3,
                                                                         'focus_loss.mask_small_use_abs': True}), 64, 2, 20001),
    # no zero-one term: only the mask-total term is matched
    'm2f64_n2_b2_focus_match_no01': ('male2female', dict(FOCUS, mask_zero_or_one_w=0, **{'council.council_size': 2,
                                                                                         'loss_matching_hist_size': 3}), 64, 2, 60001),
    # gan_w 0: the GAN history never moves, the ratios are 1 / mean(focus history)
    'glasses64_n2_b2_focus_match_gan0': ('glasses', dict(FOCUS, gan_w=0, **{'council.council_size': 2, 'loss_matching_hist_size': 2}),
                                         64, 2, 20001),
    # the focus gate closed: the switch changes nothing
    'glasses64_n2_b2_focus_match_closed': ('glasses', dict(FOCUS, **{'council.council_size': 2, 'loss_matching_hist_size': 2}),
                                           64, 2, 100),
}


def _floats(hists):
    return [[float(v) for v in h] for h in hists]


def focus_record(tr, hp):
    """Per active direction: the published losses, the histories and the focus ratios."""
    out = {}
    for d in ('a2b', 'b2a'):
        if not hp['do_' + d]:
            continue
        rec = mk._dir_losses(tr, d)
        rec['hist'] = {kind: _floats(getattr(tr, 'los_hist_%s_%s_s' % (kind, d)))
                       for kind in ('gan', 'council', 'focus', 'focus_zero_one')}
        rec['w_match_focus'] = float(getattr(tr, 'w_match_focus_%s_conf' % d))
        rec['w_match_focus_zero_one'] = float(getattr(tr, 'w_match_focus_zero_one_%s_conf' % d))
        out[d] = rec
    return out


def run_case(Council_Trainer, case):
    """make_golden.run_case on this module's case, with the focus record of every iteration."""
    run_iteration = mk.run_iteration

    def run_iteration_rec(tr, hp, x_a, x_b, it):
        rec = run_iteration(tr, hp, x_a, x_b, it)
        return dict(rec, focus=focus_record(tr, hp))
    mk.CASES[case] = CASES[case]
    mk.run_iteration = run_iteration_rec
    try:
        return mk.run_case(Council_Trainer, case)
    finally:
        mk.run_iteration = run_iteration
        del mk.CASES[case]


def main():
    Council_Trainer = mk.import_reference()
    for case in sys.argv[1:] or list(CASES):
        out = run_case(Council_Trainer, case)
        with open(os.path.join(mk.ROOT, 'tests', 'golden', case + '.json'), 'w') as f:
            json.dump(out, f, indent=1)
        print(case, 'gen', out['loss_gen_total'], 'focus', {d: (r['w_match_focus'], r['w_match_focus_zero_one'])
                                                            for d, r in out['focus'].items()})


if __name__ == '__main__':
    main()
