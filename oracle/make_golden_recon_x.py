"""Golden fixtures of the image reconstruction term (recon_x_w) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden_recon.py`` (make_golden's reference import shims, synthetic parameters, inputs and fixture
layout, with the style encoder probed), for cases with recon_x_w on (trainer_council.py:339-345, 455-459; both directions).  Every
iteration also records the six published lists loss_gen_recon_{x,s,c}_{a,b}.  Runs in the build container only.

    python oracle/make_golden_recon_x.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mk  # noqa: E402
import make_golden_recon as mkr  # noqa: E402

BOTH = mkr.BOTH

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # council and focus gates open; image reconstruction only: the style encoder is trained by recon_x alone
    'glasses64_n2_b2_recon_x': ('glasses', dict(BOTH, recon_x_w=1), 64, 2, 20001, 1),
    # all three reconstruction terms over three iterations: two style-encoder passes and two content gradients are summed, and the
    # style encoder's Adam state evolves
    'glasses64_n2_b2_recon_xsc_iter3': ('glasses', dict(BOTH, recon_x_w=1, recon_s_w=1, recon_c_w=1), 64, 2, 20001, 3),
    # council of three with abs_beginning_end on as well: every extra term shares the member totals' accumulator
    'anime64_n3_b2_recon_x_abs': ('selfie2anime', {'council.council_size': 3, 'do_a2b': True, 'recon_x_w': 3,
                                                   'abs_beginning_end': 2, 'abs_beginning_end_less_by': 0.99,
                                                   'abs_beginning_end_minimume': 0.1}, 64, 2, 2001, 1),
}


def _recon(trainer):
    """The six lists gen_update publishes about the reconstruction terms (trainer_council.py:308-313, 455-469)."""
    return {'loss_gen_recon_%s_%s' % (k, d): [float(v) for v in getattr(trainer, 'loss_gen_recon_%s_%s_s' % (k, d))]
            for k in ('x', 's', 'c') for d in ('a', 'b')}


def run_case(Council_Trainer, case):
    """make_golden_recon.run_case on this module's case, with the six lists recorded per iteration."""
    cases, recon = mkr.CASES, mkr._recon
    mkr.CASES, mkr._recon = dict(cases, **{case: CASES[case]}), _recon
    try:
        return mkr.run_case(Council_Trainer, case)
    finally:
        mkr.CASES, mkr._recon = cases, recon


def main():
    Council_Trainer = mk.import_reference()
    for case in sys.argv[1:] or list(CASES):
        out = run_case(Council_Trainer, case)
        with open(os.path.join(mk.ROOT, 'tests', 'golden', case + '.json'), 'w') as f:
            json.dump(out, f, indent=1)
        print(case, 'gen', out['loss_gen_total'], {k: v for k, v in out.items() if k.startswith('loss_gen_recon_x')})


if __name__ == '__main__':
    main()
