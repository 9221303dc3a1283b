"""Golden fixtures of pad_type: reflect from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden_recon_x.py`` (make_golden's reference import shims, synthetic parameters, inputs and fixture
layout, the style encoder probed, the six reconstruction lists recorded per iteration), for cases with ``gen.pad_type`` and / or
``dis.pad_type`` set to 'reflect' (Conv2dBlock, networks.py:463-520).  Parameter names and shapes do not depend on the padding, so
the synthetic parameters are those of the zero-padded cases.  Runs in the build container only.

    python oracle/make_golden_pad.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mk  # noqa: E402
import make_golden_recon_x as mkx  # noqa: E402

GEN = {'gen.pad_type': 'reflect'}
DIS = {'dis.pad_type': 'reflect'}
BOTH_PADS = dict(GEN, **DIS)

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # generator reflect (content encoder and decoder), discriminators zero, council and focus gates open
    'glasses64_n2_b2_reflect_gen': ('glasses', dict(GEN, **{'council.council_size': 2}), 64, 2, 20001, 1),
    # both discriminator families reflect (MsImageDis layer 0 on the image, MsImageDisCouncil layer 0 on the pair), generator zero
    'm2f64_n4_b2_reflect_dis': ('male2female', dict(DIS), 64, 2, 60001, 1),
    # both reflect, both directions, the three reconstruction terms: the style encoder and the re-encode passes
    'glasses64_n2_b2_reflect_recon': ('glasses', dict(BOTH_PADS, **mkx.BOTH, recon_x_w=1, recon_s_w=1, recon_c_w=1), 64, 2, 20001, 1),
    # both reflect, three iterations with the council flip live (2 on / 1 off) and StepLR step 2
    'glasses64_n3_b2_reflect_iter3': ('glasses', dict(BOTH_PADS, **{'council.council_size': 3, 'council.flipOnOff': True,
                                                                    'council.flipOnOff_On_iteration': 2,
                                                                    'council.flipOnOff_Off_iteration': 1, 'step_size': 2}),
                                      64, 2, 20001, 3),
    # both reflect at the benchmark's 256x256 geometry (council and batch reduced so the CPU reference finishes in seconds)
    'm2f256_n2_b1_reflect': ('male2female', dict(BOTH_PADS, **{'council.council_size': 2}), 256, 1, 60001, 1),
}


def run_case(Council_Trainer, case):
    """make_golden_recon_x.run_case on this module's case"""
    cases = mkx.CASES
    mkx.CASES = dict(cases, **{case: CASES[case]})
    try:
        return mkx.run_case(Council_Trainer, case)
    finally:
        mkx.CASES = cases


def main():
    Council_Trainer = mk.import_reference()
    for case in sys.argv[1:] or list(CASES):
        out = run_case(Council_Trainer, case)
        with open(os.path.join(mk.ROOT, 'tests', 'golden', case + '.json'), 'w') as f:
            json.dump(out, f, indent=1)
        print(case, 'dis', out['loss_dis_total'], 'gen', out['loss_gen_total'])


if __name__ == '__main__':
    main()
