"""Golden fixtures of the council abs loss (council_abs_w) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden.py`` (its reference import shims, synthetic parameters, inputs and fixture layout), for cases
with council_abs_w on (trainer_council.py:224-228, 595-619; both directions).  On top of make_golden's record, every iteration also
records both published council lists (council_loss_ab / council_loss_ba) and the peers gen_update drew, taken by wrapping
``random.choice`` for the duration of that call.  Runs in the build container only.

    python oracle/make_golden_council_abs.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mk  # noqa: E402

BOTH = {'do_a2b': True, 'do_b2a': True}

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # council discriminators and the abs term together; N = 2: random.choice of a single candidate
    'glasses64_n2_b2_council_abs': ('glasses', dict(BOTH, **{'council.council_size': 2, 'council_abs_w': 1}), 64, 2, 20001, 1),
    # council_w 0: no council discriminator at all, dis_council_update returns at once; four members draw real random peers
    'm2f64_n4_b2_council_abs_nodc': ('male2female', dict(BOTH, council_w=0, council_abs_w=2), 64, 2, 60001, 1),
    # the gray-scale criterion: |sum_c x_i - sum_c x_j| over B x H x W
    'anime64_n3_b2_council_abs_gray': ('selfie2anime', dict(BOTH, **{'council.council_size': 3, 'council_abs_w': 1,
                                                                     'council_abs_gray_scale': True}), 64, 2, 2001, 1),
    # three iterations, council flip 2 on / 1 off, StepLR step 2: the gate closes in the third, and dis_council_update's draws
    # interleave with gen_update's in one `random` stream
    'glasses64_n3_b2_council_abs_iter3': ('glasses', dict(BOTH, **{'council.council_size': 3, 'council_abs_w': 1,
                                                                   'council.flipOnOff': True, 'council.flipOnOff_On_iteration': 2,
                                                                   'council.flipOnOff_Off_iteration': 1, 'step_size': 2}),
                                          64, 2, 20001, 3),
    # before council_start_at_iter: the gate is closed, nothing is drawn and the lists hold the int 0
    'glasses64_n2_b2_council_abs_early': ('glasses', dict(BOTH, **{'council.council_size': 2, 'council_abs_w': 1}), 64, 2, 100, 1),
}


def _council(trainer):
    """What gen_update publishes about the council terms (trainer_council.py:556-630)."""
    return {'council_loss_ab': [float(v) for v in trainer.council_loss_ab_s],
            'council_loss_ba': [float(v) for v in trainer.council_loss_ba_s]}


def _with_peers(trainer):
    """trainer.gen_update recording the members random.choice returns while it runs in `trainer.peers_drawn`."""
    gen_update = trainer.gen_update

    def wrapped(*args, **kwargs):
        choice, drawn = random.choice, []

        def record(seq):
            j = choice(seq)
            drawn.append(j)
            return j
        random.choice = record
        try:
            return gen_update(*args, **kwargs)
        finally:
            random.choice = choice
            trainer.peers_drawn = drawn
    return wrapped


def run_case(Council_Trainer, case):
    """make_golden.run_case on this module's case, with the council lists and the drawn peers recorded per iteration."""
    run_iteration = mk.run_iteration

    def run_iteration_rec(tr, hp, x_a, x_b, it):
        tr.gen_update = _with_peers(tr)
        rec = run_iteration(tr, hp, x_a, x_b, it)
        del tr.gen_update
        return dict(rec, peers=tr.peers_drawn, **_council(tr))
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
        print(case, 'gen', out['loss_gen_total'], 'ab', out['council_loss_ab'], 'ba', out['council_loss_ba'], 'peers', out['peers'])


if __name__ == '__main__':
    main()
