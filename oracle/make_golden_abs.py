"""Golden fixtures of the abs_beginning_end term from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden.py`` (its reference import shims, synthetic parameters, inputs and fixture layout), for
cases with abs_beginning_end on (trainer_council.py:210-215, 477-495).  On top of make_golden's record, every iteration also
records what gen_update publishes about the term (loss_gen_beginning_end_a_ab / _b_ba, abs_beginning_end_w_conf), and a case
may scale the synthetic inputs (``input_scale`` in the fixture).  Runs in the build container only.

    python oracle/make_golden_abs.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import council_oracle as co  # noqa: E402
import make_golden as mk  # noqa: E402

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run, input scale)
CASES = {
    # a2b with the council and focus gates open; weight 0.9999 ** 20001 = 0.135
    'glasses64_n2_b2_abs': ('glasses', {'council.council_size': 2, 'abs_beginning_end': 1, 'abs_beginning_end_less_by': 0.9999,
                                        'abs_beginning_end_minimume': 0.01}, 64, 2, 20001, 1, 1),
    # b2a only: the a2b list holds the int 0 of the inactive direction; the weight sits on its minimum
    'anime64_n3_b2_abs': ('selfie2anime', {'council.council_size': 3, 'abs_beginning_end': 2, 'abs_beginning_end_less_by': 0.99,
                                           'abs_beginning_end_minimume': 0.1}, 64, 2, 2001, 1, 1),
    # both directions: the term of each direction joins the same member total
    'glasses64_n2_b2_both_abs': ('glasses', {'council.council_size': 2, 'do_b2a': True, 'abs_beginning_end': 1,
                                             'abs_beginning_end_less_by': 1, 'abs_beginning_end_minimume': 0}, 64, 2, 20001, 1, 1),
    # the weight 0.5 ** it crosses 0.005 at iteration 8: only member 0 gets the term in that call, nobody afterwards
    'glasses64_n2_b2_abs_decay': ('glasses', {'council.council_size': 2, 'abs_beginning_end': 1, 'abs_beginning_end_less_by': 0.5,
                                              'abs_beginning_end_minimume': 0}, 64, 2, 6, 4, 1),
    # inputs of +-3: |x_fake - x| mostly exceeds 1, so mean d^2 > mean |d| and the L2 branch is taken
    'glasses64_n2_b2_abs_l2': ('glasses', {'council.council_size': 2, 'abs_beginning_end': 1, 'abs_beginning_end_less_by': 1,
                                           'abs_beginning_end_minimume': 0}, 64, 2, 20001, 1, 3.0),
}


def _beginning_end(trainer):
    """What gen_update publishes about abs_beginning_end (trainer_council.py:477-495)."""
    return {'loss_gen_beginning_end_a_ab': [float(v) for v in trainer.loss_gen_beginning_end_a_ab_s],
            'loss_gen_beginning_end_b_ba': [float(v) for v in trainer.loss_gen_beginning_end_b_ba_s],
            'abs_beginning_end_w_conf': float(trainer.abs_beginning_end_w_conf)}


def run_case(Council_Trainer, case):
    """make_golden.run_case on this module's case, with the term's attributes recorded per iteration and the inputs scaled."""
    cfg, overrides, size, batch, iteration, n_iters, scale = CASES[case]
    run_iteration, synth_inputs = mk.run_iteration, co.synth_inputs
    mk.CASES[case] = (cfg, overrides, size, batch, iteration, n_iters)
    mk.run_iteration = lambda tr, hp, x_a, x_b, it: dict(run_iteration(tr, hp, x_a, x_b, it), **_beginning_end(tr))
    co.synth_inputs = lambda *a, **k: tuple(x * scale for x in synth_inputs(*a, **k))
    try:
        out = mk.run_case(Council_Trainer, case)
    finally:
        mk.run_iteration, co.synth_inputs = run_iteration, synth_inputs
        del mk.CASES[case]
    if scale != 1:
        out['input_scale'] = scale
    return out


def main():
    Council_Trainer = mk.import_reference()
    for case in sys.argv[1:] or list(CASES):
        out = run_case(Council_Trainer, case)
        with open(os.path.join(mk.ROOT, 'tests', 'golden', case + '.json'), 'w') as f:
            json.dump(out, f, indent=1)
        print(case, 'gen', out['loss_gen_total'], 'beginning_end', out['loss_gen_beginning_end_a_ab'], out['loss_gen_beginning_end_b_ba'])


if __name__ == '__main__':
    main()
