"""Golden fixtures of the perceptual loss (vgg_w) from the UNMODIFIED reference  --  TEST INFRASTRUCTURE ONLY.

Same machinery as ``oracle/make_golden_recon.py`` (make_golden's reference import shims, synthetic parameters, inputs and fixture
layout, with the style encoder probed), for cases with vgg_w on (trainer_council.py:199-205, 531-538, 636-641; both directions).  The
frozen VGG-16 is ``vgg_oracle.synth_vgg16(VGG_SEED)``, written to a temporary vgg_model_path where the reference's load_vgg16
(utils.py:350-366) finds ``vgg16.weight`` and never reaches torchfile or its download.  Fixtures record the seed, not the weights.
Every iteration also records the six reconstruction lists and loss_gen_vgg_{a,b}.  Runs in the build container only.

    python oracle/make_golden_vgg.py            # regenerates every case in CASES
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mk  # noqa: E402
import make_golden_recon as mkr  # noqa: E402
import make_golden_recon_x as mkx  # noqa: E402
from vgg_oracle import synth_vgg16, write_vgg16  # noqa: E402

BOTH = mkr.BOTH
VGG_SEED = 16

# case name -> (config yaml, overrides, image size, batch, iteration, iterations run)
CASES = {
    # council and focus gates open, the perceptual loss alone
    'glasses64_n2_b2_vgg': ('glasses', dict(BOTH, vgg_w=1), 64, 2, 20001, 1),
    # three iterations: Adam carries the VGG gradient
    'glasses64_n2_b2_vgg_iter3': ('glasses', dict(BOTH, vgg_w=1), 64, 2, 20001, 3),
    # council of four with recon_x_w and abs_beginning_end: the member totals' shared accumulator and a d_x summed from four terms
    'm2f64_n4_b2_vgg_recon_x_abs': ('male2female', {'do_b2a': True, 'vgg_w': 0.5, 'recon_x_w': 1, 'abs_beginning_end': 2,
                                                    'abs_beginning_end_less_by': 0.99, 'abs_beginning_end_minimume': 0.1}, 64, 2, 60001, 1),
    # every VGG geometry of the headline resolution: conv1 at 256 x 256, relu5_3 at 32 x 32
    'm2f256_n2_b1_vgg': ('male2female', {'council.council_size': 2, 'do_b2a': True, 'vgg_w': 1}, 256, 1, 60001, 1),
}


def _lists(trainer):
    out = mkx._recon(trainer)
    out.update({'loss_gen_vgg_%s' % d: [float(v) for v in getattr(trainer, 'loss_gen_vgg_%s_s' % d)] for d in ('a', 'b')})
    return out


def run_case(Council_Trainer, case, vgg_model_path):
    """make_golden_recon.run_case on this module's case, with vgg_model_path set and the lists recorded per iteration."""
    cases, recon, load_config = mkr.CASES, mkr._recon, mk.load_config
    mkr.CASES, mkr._recon = dict(cases, **{case: CASES[case]}), _lists
    mk.load_config = lambda name, overrides: dict(load_config(name, overrides), vgg_model_path=vgg_model_path)
    try:
        out = mkr.run_case(Council_Trainer, case)
    finally:
        mkr.CASES, mkr._recon, mk.load_config = cases, recon, load_config
    out['vgg_seed'] = VGG_SEED
    return out


def main():
    Council_Trainer = mk.import_reference()
    with tempfile.TemporaryDirectory() as tmp:
        write_vgg16(synth_vgg16(VGG_SEED), tmp)
        for case in sys.argv[1:] or list(CASES):
            out = run_case(Council_Trainer, case, tmp)
            with open(os.path.join(mk.ROOT, 'tests', 'golden', case + '.json'), 'w') as f:
                json.dump(out, f, indent=1)
            print(case, 'gen', out['loss_gen_total'], {k: v for k, v in out.items() if k.startswith('loss_gen_vgg')})


if __name__ == '__main__':
    main()
