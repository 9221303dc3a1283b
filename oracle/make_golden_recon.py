"""Golden fixtures of the latent reconstruction terms (recon_c_w / recon_s_w) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden.py`` (its reference import shims, synthetic parameters, inputs and fixture layout), for cases
with recon_c_w and / or recon_s_w on (trainer_council.py:359-369, 460-469; both directions).  On top of make_golden's record, every
iteration also records the four published lists loss_gen_recon_{s,c}_{a,b}, and the style encoder is probed (post-step values and
gradients) next to make_golden's generator parameters.  Runs in the build container only.

    python oracle/make_golden_recon.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mk  # noqa: E402

STYLE_PROBES = ['enc_style.model.0.conv.weight', 'enc_style.model.4.conv.weight', 'enc_style.model.6.weight', 'enc_style.model.6.bias']
BOTH = {'council.council_size': 2, 'do_b2a': True}

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # council and focus gates open; content reconstruction only: the style encoder gets no gradient
    'glasses64_n2_b2_recon_c': ('glasses', dict(BOTH, recon_c_w=1), 64, 2, 20001, 1),
    # style reconstruction only: the one term that trains the style encoder
    'glasses64_n2_b2_recon_s': ('glasses', dict(BOTH, recon_s_w=1), 64, 2, 20001, 1),
    # both terms over three iterations: the style encoder's Adam state evolves
    'glasses64_n2_b2_recon_iter3': ('glasses', dict(BOTH, recon_c_w=1, recon_s_w=1), 64, 2, 20001, 3),
    # council of three with abs_beginning_end on as well: every extra term shares the member totals' accumulator
    'anime64_n3_b2_recon_abs': ('selfie2anime', {'council.council_size': 3, 'do_a2b': True, 'recon_c_w': 0.5, 'recon_s_w': 2,
                                                 'abs_beginning_end': 2, 'abs_beginning_end_less_by': 0.99,
                                                 'abs_beginning_end_minimume': 0.1}, 64, 2, 2001, 1),
}


def _recon(trainer):
    """The four lists gen_update publishes about the terms (trainer_council.py:310-313, 460-469)."""
    return {'loss_gen_recon_%s_%s' % (k, d): [float(v) for v in getattr(trainer, 'loss_gen_recon_%s_%s_s' % (k, d))]
            for k in ('s', 'c') for d in ('a', 'b')}


def run_case(Council_Trainer, case):
    """make_golden.run_case on this module's case, with the lists recorded per iteration and the style encoder probed."""
    run_iteration, probes = mk.run_iteration, list(mk.PROBE_PARAMS['gen'])
    mk.CASES[case] = CASES[case]
    mk.run_iteration = lambda tr, hp, x_a, x_b, it: dict(run_iteration(tr, hp, x_a, x_b, it), **_recon(tr))
    mk.PROBE_PARAMS['gen'] = probes + STYLE_PROBES
    try:
        return mk.run_case(Council_Trainer, case)
    finally:
        mk.run_iteration, mk.PROBE_PARAMS['gen'] = run_iteration, probes
        del mk.CASES[case]


def main():
    Council_Trainer = mk.import_reference()
    for case in sys.argv[1:] or list(CASES):
        out = run_case(Council_Trainer, case)
        with open(os.path.join(mk.ROOT, 'tests', 'golden', case + '.json'), 'w') as f:
            json.dump(out, f, indent=1)
        print(case, 'gen', out['loss_gen_total'], {k: v for k, v in out.items() if k.startswith('loss_gen_recon')})


if __name__ == '__main__':
    main()
