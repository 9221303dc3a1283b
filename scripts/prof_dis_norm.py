"""Cost of the discriminators' normalisation dis.norm in / ln (networks.py:40-44, 137-143, 659-686) at male2female 256x256, council of
4, batch 8 (the benchmark's configuration, a2b).

    python scripts/prof_dis_norm.py [steps]

1. Every normalisation launch the discriminators add to one training step, for 'in' and for 'ln', at the step's own layer shapes:
   CUDA events around each launch (ops.start_timing, the keys bench.py's roofline uses), us per launch, the HBM bytes each must move
   (hbm:in_stats and hbm:ln_stats read y once; the forward passes read y and write z; the backward passes read (y, dz) twice and
   write dy), the achieved rate and the floor that bytes / 3.35 TB/s (H100 SXM data sheet) implies.  Under 'in' the statistics of
   the tensor-core convolutions come from their epilogue (no hbm:in_stats launch).
2. The training step (dis_update, dis_council_update, gen_update), `steps` (default 5) steps per block, alternating 3x in one process
   after a warm-up step of each, for three trainers built with the same parameters: norm none, in, ln.  Step time, and peak working
   memory: the peak allocated during a block above what was allocated before it.
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


def with_norm(hp, norm):
    h = copy.deepcopy(hp)
    h['dis']['norm'] = norm
    return h


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    from council_gan_b200 import Council_Trainer
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    hp, N, B, size, it = load_hp('male2female_256_n4_b8')
    xa, xb = (t.cuda() for t in synth(B, size, 123))
    runs = (('none', with_norm(hp, 'none')), ('in', with_norm(hp, 'in')), ('ln', with_norm(hp, 'ln')))
    trainers = {}
    for name, h in runs:
        torch.manual_seed(1)
        np.random.seed(1)
        trainers[name] = Council_Trainer(h, 'cuda:0')
    src = trainers['none']
    for name, tr in trainers.items():  # the same conv parameters in all three (ln's gamma / beta keep their own init)
        for a, b in zip(src._nets.values(), tr._nets.values()):
            for ba, bb in zip(a._banks(), b._banks()):
                for k in ba.table:
                    bb._view(bb.data, k).copy_(ba._view(ba.data, k))

    def step(tr, h):
        tr.dis_update(xa, xb, h)
        tr.dis_council_update(xa, xb, h)
        tr.gen_update(xa, xb, h, it)

    # ---- every normalisation launch the discriminators add to one step ----------------------------------------------------------
    for name, h in runs[1:]:
        tr = trainers[name]
        step(tr, h)
        tr.synchronize()
        torch.cuda.synchronize()
        tr.ops.start_timing()
        step(tr, h)
        tr.synchronize()
        rec = tr.ops.stop_timing()
        # the discriminators' normalised maps have 128 / 256 / 512 channels; the generators' instance norms have 64 / 128 / 256 at
        # different sizes, so a key names a discriminator launch when the 'none' trainer has no such key
        tr0 = trainers['none']
        step(tr0, runs[0][1])
        tr0.synchronize()
        tr0.ops.start_timing()
        step(tr0, runs[0][1])
        tr0.synchronize()
        rec0 = tr0.ops.stop_timing()
        tot_ms = tot_floor = 0.0
        n_launch = 0
        print('-- dis.norm %s' % name)
        for key in sorted(k for k in rec if k.startswith('hbm:') and ('norm_act' in k or 'ln_' in k or 'in_stats' in k)):
            ms, n_all, nbytes = rec[key]
            n = n_all - (rec0[key][1] if key in rec0 else 0)  # the launches the discriminators' norm adds (same shape, same cost)
            if n <= 0:
                continue
            us = ms * 1e3 / n_all
            ms = us * n / 1e3
            floor = nbytes / HBM_BYTES_PER_S * 1e6
            tot_ms, tot_floor, n_launch = tot_ms + ms, tot_floor + floor * n, n_launch + n
            print('%-52s x%-3d %8.1f us/launch  %7.1f MB  %5.2f TB/s  (floor %6.1f us)' % (key[4:], n, us, nbytes / 1e6, nbytes / us / 1e6,
                                                                                         floor))
        print('normalisation per step: %d launches, %.2f ms (floor %.2f ms at 3.35 TB/s)' % (n_launch, tot_ms, tot_floor / 1e3))

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
    base = sum(t for t, _ in res['none']) / 3
    for name, _ in runs:
        mean = sum(t for t, _ in res[name]) / 3
        print('%-13s %s ms   %.1f images/s   %+.2f ms (%+.1f %%) vs none   peak working memory %.2f GiB'
              % (name, '  '.join('%.2f' % t for t, _ in res[name]), B * 1e3 / mean, mean - base, 100 * (mean - base) / base,
                 max(m for _, m in res[name])))


if __name__ == '__main__':
    main()
