"""Golden fixtures of the discriminator-side switches (do_Dis_only_gray, useRandomGen, useRandomDis) from the UNMODIFIED reference  --
TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden.py`` (its reference import shims, synthetic parameters, inputs and fixture layout), for cases
with the switches on (trainer_council.py:499-510, 736-765).  On top of make_golden's record, every iteration also records the
``np.random.randint`` draws of dis_update (``dis_draws``) and of gen_update (``gen_draws``) separately, taken by wrapping
``np.random.randint`` for the duration of each call.  Runs in the build container only.

    python oracle/make_golden_dis_options.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mk  # noqa: E402

GRAY = {'dis.do_Dis_only_gray': True}
RANDOM = {'dis.useRandomGen': True, 'gen.useRandomDis': True}

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # a2b, every gate open: D sees gray in dis_update and gen_update, the council discriminators colour
    'glasses64_n2_b2_gray': ('glasses', dict(GRAY, **{'council.council_size': 2}), 64, 2, 20001),
    # b2a only: dis_update applies no gan_w on this branch (:777)
    'anime64_n3_b2_gray': ('selfie2anime', dict(GRAY, **{'council.council_size': 3}), 64, 2, 2001),
    # both random switches with loss matching on: self-pairs, shared and unused discriminators
    'm2f64_n4_b2_random_pairing': ('male2female', dict(RANDOM), 64, 2, 60001),
    # both directions, all three switches, council flip 2 on / 1 off and StepLR step 2: both updates' draws interleave over three
    # iterations while the loss histories evolve
    'glasses64_n3_b2_dis_options_iter3': ('glasses', dict(GRAY, do_b2a=True, **RANDOM, **{
        'council.council_size': 3, 'council.flipOnOff': True, 'council.flipOnOff_On_iteration': 2,
        'council.flipOnOff_Off_iteration': 1, 'step_size': 2}), 64, 2, 20001, 3),
}


def with_draws(fn, sink):
    """fn recording every np.random.randint result while it runs in the list sink[0] (a new list per call)."""
    def wrapped(*args, **kwargs):
        randint, drawn = np.random.randint, []

        def record(*a, **k):
            v = randint(*a, **k)
            drawn.append(int(v))
            return v
        np.random.randint = record
        try:
            return fn(*args, **kwargs)
        finally:
            np.random.randint = randint
            sink[0] = drawn
    return wrapped


def run_case(Council_Trainer, case):
    """make_golden.run_case on this module's case, with both updates' draws recorded per iteration."""
    run_iteration = mk.run_iteration

    def run_iteration_rec(tr, hp, x_a, x_b, it):
        dis_draws, gen_draws = [None], [None]
        tr.dis_update = with_draws(tr.dis_update, dis_draws)
        tr.gen_update = with_draws(tr.gen_update, gen_draws)
        rec = run_iteration(tr, hp, x_a, x_b, it)
        del tr.dis_update, tr.gen_update
        return dict(rec, dis_draws=dis_draws[0], gen_draws=gen_draws[0])
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
        print(case, 'dis', out['loss_dis_total'], 'gen', out['loss_gen_total'], 'draws', out['dis_draws'], out['gen_draws'])


if __name__ == '__main__':
    main()
