"""Golden fixtures of the discriminators' normalisation (dis.norm: in, ln) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden_dis_options.py`` (make_golden's reference import shims, synthetic parameters, inputs and
fixture layout; the np.random.randint draws of both updates recorded per iteration), for cases with ``dis.norm`` set to 'in' or
'ln' (MsImageDis / MsImageDisCouncil layers 1 .. n_layer-1, networks.py:40-44, 137-143).  Under 'ln' the synthetic states carry
each block's LayerNorm gamma / beta (dis_norm_oracle.synth_all_states).  The fixtures keep the published losses of every iteration
(and the draws) and drop make_golden's parameter and image probes (UNUSED below): tests/test_trainer_dis_norm_*.py compare the
post-step parameters with the oracle, which these losses pin to the reference.  Runs in the build container only.

    python oracle/make_golden_dis_norm.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import council_oracle as co  # noqa: E402
import dis_norm_oracle as dno  # noqa: E402
import make_golden as mk  # noqa: E402
import make_golden_dis_options as mkd  # noqa: E402

IN, LN = {'dis.norm': 'in'}, {'dis.norm': 'ln'}
ITER3 = {'council.flipOnOff': True, 'council.flipOnOff_On_iteration': 2, 'council.flipOnOff_Off_iteration': 1, 'step_size': 2,
         'loss_matching_hist_size': 2}
UNUSED = ('params', 'post_x_fake0', 'post_mask0')

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # a2b, every gate open: both discriminator families normalised (their second scale ends on 2x2 maps)
    'glasses64_n2_b2_dis_in': ('glasses', dict(IN, **{'council.council_size': 2}), 64, 2, 20001, 1),
    'glasses64_n2_b2_dis_ln': ('glasses', dict(LN, **{'council.council_size': 2}), 64, 2, 20001, 1),
    # three iterations with 2-entry loss histories, the council flip (2 on / 1 off) and StepLR step 2
    'glasses64_n2_b2_dis_in_iter3': ('glasses', dict(IN, **ITER3, **{'council.council_size': 2}), 64, 2, 20001, 3),
    'glasses64_n2_b2_dis_ln_iter3': ('glasses', dict(LN, **ITER3, **{'council.council_size': 2}), 64, 2, 20001, 3),
    # both directions
    'glasses64_n2_b2_dis_in_both': ('glasses', dict(IN, do_b2a=True, **{'council.council_size': 2}), 64, 2, 20001, 1),
    'glasses64_n2_b2_dis_ln_both': ('glasses', dict(LN, do_b2a=True, **{'council.council_size': 2}), 64, 2, 20001, 1),
    # b2a only (selfie2anime: no gan_w on the b2a branch of dis_update)
    'anime64_n3_b2_dis_ln': ('selfie2anime', dict(LN, **{'council.council_size': 3}), 64, 2, 2001, 1),
    # ln with randomly paired discriminators (gen_update draws the LN parameters with the rest) and gray discriminators
    'm2f64_n4_b2_dis_ln_gray_random': ('male2female', dict(LN, **mkd.GRAY, **mkd.RANDOM), 64, 2, 60001, 1),
    # in with reflection padding in the discriminators
    'm2f64_n4_b2_dis_in_reflect': ('male2female', dict(IN, **{'dis.pad_type': 'reflect'}), 64, 2, 60001, 1),
    # the benchmark's 256x256 geometry with batch 1 (LayerNorm's batch-1 branch)
    'm2f256_n2_b1_dis_ln': ('male2female', dict(LN, **{'council.council_size': 2}), 256, 1, 60001, 1),
}


def run_case(Council_Trainer, case):
    """make_golden_dis_options.run_case on this module's case, with the LayerNorm parameters in the synthetic states and without
    the UNUSED probes"""
    cases, synth = mkd.CASES, co.synth_all_states
    mkd.CASES = dict(cases, **{case: CASES[case]})
    co.synth_all_states = dno.synth_all_states
    try:
        out = mkd.run_case(Council_Trainer, case)
    finally:
        mkd.CASES, co.synth_all_states = cases, synth
    return {k: v for k, v in out.items() if k not in UNUSED}


def main():
    Council_Trainer = mk.import_reference()
    for case in sys.argv[1:] or list(CASES):
        out = run_case(Council_Trainer, case)
        with open(os.path.join(mk.ROOT, 'tests', 'golden', case + '.json'), 'w') as f:
            json.dump(out, f, indent=1)
        print(case, 'dis', out['loss_dis_total'], 'gen', out['loss_gen_total'])


if __name__ == '__main__':
    main()
