"""Cost of pad_type: reflect (Conv2dBlock networks.py:463-520) at male2female 256x256, council of 4, batch 8 (the benchmark's
configuration, a2b).

    python scripts/prof_pad.py [steps]

1. Every cg_reflect_pad / cg_reflect_pad_bwd launch of one training step with both networks on reflect, at the step's own layer shapes:
   CUDA events around each launch (ops.start_timing, the keys bench.py's roofline uses), us per launch, the HBM bytes each must move
   (input read once, output written once; the fold also reads its addend), the achieved rate and the floor that bytes / 3.35 TB/s
   (H100 SXM data sheet) implies.
2. The training step (dis_update, dis_council_update, gen_update), `steps` (default 5) steps per block, alternating 3x in one process
   after a warm-up step of each, for four trainers built with the same parameters: both networks zero, the generators reflect, the
   discriminators reflect, both reflect.  Step time, and peak working memory: the peak allocated during a block above what was
   allocated before it.
Prints the card's name, power limit and max SM clock beside the numbers."""
import copy
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from bench import load_hp, synth

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def with_pads(hp, gen, dis):
    h = copy.deepcopy(hp)
    h['gen']['pad_type'], h['dis']['pad_type'] = gen, dis
    return h


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    from council_gan_b200 import Council_Trainer
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    hp, N, B, size, it = load_hp('male2female_256_n4_b8')
    xa, xb = (t.cuda() for t in synth(B, size, 123))
    runs = (('zero', with_pads(hp, 'zero', 'zero')), ('gen reflect', with_pads(hp, 'reflect', 'zero')),
            ('dis reflect', with_pads(hp, 'zero', 'reflect')), ('both reflect', with_pads(hp, 'reflect', 'reflect')))
    trainers = {}
    for name, h in runs:
        torch.manual_seed(1)
        np.random.seed(1)
        trainers[name] = Council_Trainer(h, 'cuda:0')
    src = trainers['zero']
    for name, tr in trainers.items():  # the same parameters in all four
        for a, b in zip(src._nets.values(), tr._nets.values()):
            for ba, bb in zip(a._banks(), b._banks()):
                bb.data.copy_(ba.data)

    def step(tr, h):
        tr.dis_update(xa, xb, h)
        tr.dis_council_update(xa, xb, h)
        tr.gen_update(xa, xb, h, it)

    # ---- every padding launch of one step -------------------------------------------------------------------------------------------
    tr, h = trainers['both reflect'], runs[3][1]
    step(tr, h)
    tr.synchronize()
    torch.cuda.synchronize()
    tr.ops.start_timing()
    step(tr, h)
    tr.synchronize()
    rec = tr.ops.stop_timing()
    tot_ms = tot_floor = 0.0
    n_launch = 0
    for key in sorted(k for k in rec if 'reflect_pad' in k):
        ms, n, nbytes = rec[key]
        us = ms * 1e3 / n
        floor = nbytes / HBM_BYTES_PER_S * 1e6
        tot_ms, tot_floor, n_launch = tot_ms + ms, tot_floor + floor * n, n_launch + n
        print('%-52s x%-3d %8.1f us/launch  %7.1f MB  %5.2f TB/s  (floor %6.1f us)' % (key[4:], n, us, nbytes / 1e6, nbytes / us / 1e6,
                                                                                     floor))
    print('padding per step: %d launches, %.2f ms (floor %.2f ms at 3.35 TB/s)' % (n_launch, tot_ms, tot_floor / 1e3))

    # ---- the training step ------------------------------------------------------------------------------------------------------------
    def block(name, h, n):
        tr = trainers[name]
        tr.synchronize()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            step(tr, h)
        tr.synchronize()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n, (torch.cuda.max_memory_allocated() - base) / 2 ** 30

    for name, h in runs:
        block(name, h, 1)
    res = {name: [] for name, _ in runs}
    for _ in range(3):
        for name, h in runs:
            res[name].append(block(name, h, steps))
    base = sum(t for t, _ in res['zero']) / 3
    for name, _ in runs:
        mean = sum(t for t, _ in res[name]) / 3
        print('%-13s %s ms   %.1f images/s   %+.2f ms (%+.1f %%) vs zero   peak working memory %.2f GiB'
              % (name, '  '.join('%.2f' % t for t, _ in res[name]), B * 1e3 / mean, mean - base, 100 * (mean - base) / base,
                 max(m for _, m in res[name])))


if __name__ == '__main__':
    main()
