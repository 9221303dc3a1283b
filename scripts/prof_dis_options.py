"""Cost of the discriminator-side switches do_Dis_only_gray, useRandomGen and useRandomDis (trainer_council.py:499-510, 736-765) at
male2female 256x256, council of 4, batch 8 (the shipped configuration, a2b).

    python scripts/prof_dis_options.py [steps]

1. The three kernels on tensors of the step's shapes: cg_gather_images_gray as dis_update calls it ([fake ; real] for every member),
   cg_gray_fold on gen_update's data gradient and cg_gather_members on the discriminator bank.  CUDA events around 20 launches, best of
   3; us per launch, the HBM bytes each must move (every element read once and written once), the achieved rate and the floor that
   bytes / 3.35 TB/s (H100 SXM data sheet) implies.
2. The training step (dis_update, dis_council_update, gen_update), `steps` (default 5) steps per block, alternating 3x in one process
   after a warm-up step of each: every switch off, each switch on alone, and all three on (one trainer; the switches are read per
   call).
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


def best_of_3(fn, n=20):
    fn()
    torch.cuda.synchronize()
    best = None
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        best = ms if best is None else min(best, ms)
    return best


def with_switches(hp, gray=False, random_gen=False, random_dis=False):
    h = copy.deepcopy(hp)
    h['dis']['do_Dis_only_gray'], h['dis']['useRandomGen'], h['gen']['useRandomDis'] = gray, random_gen, random_dis
    return h


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    from council_gan_b200 import Council_Trainer
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    hp, N, B, size, it = load_hp('male2female_256_n4_b8')
    torch.manual_seed(1)
    np.random.seed(1)
    tr = Council_Trainer(hp, 'cuda:0')
    ops = tr.ops

    # ---- the kernels ----------------------------------------------------------------------------------------------------------
    gen = torch.Generator().manual_seed(0)
    fake = torch.rand(N * B, size, size, 4, generator=gen).cuda() * 2 - 1
    real = torch.rand(B, size, size, 4, generator=gen).cuda() * 2 - 1
    idx = torch.tensor([[g * B + b for b in range(B)] + [N * B + b for b in range(B)] for g in range(N)], dtype=torch.int32).cuda()
    d_x = torch.randn(N, B, size, size, 4, generator=gen).cuda()
    dis = tr._nets['dis_a2b']
    scratch = dis.bank_like()
    segs = dis.bank.member_segments()
    member_floats = sum(n for _, n in segs)
    cases = (('gather_images_gray', lambda: ops.gather_images_gray((fake, real), idx, N, 2 * B), 2 * 4 * N * 2 * B * size * size * 4),
             ('gray_fold', lambda: ops.gray_fold(d_x), 2 * 4 * d_x.numel()),
             ('gather_members', lambda: ops.gather_members(dis.bank.data, scratch.data, segs, [2, 3, 2, 3]), 2 * 4 * N * member_floats))
    print('discriminator bank: %d segments, %.2f M floats per member' % (len(segs), member_floats / 1e6))
    for name, fn, nbytes in cases:
        ms = best_of_3(fn)
        print('%-20s %7.1f us/launch  %6.1f MB  %5.2f TB/s  (floor %.1f us at 3.35 TB/s)'
              % (name, ms * 1e3, nbytes / 1e6, nbytes / ms / 1e9, nbytes / HBM_BYTES_PER_S * 1e6))
    del fake, real, d_x, scratch

    # ---- the training step ------------------------------------------------------------------------------------------------------
    xa, xb = (t.cuda() for t in synth(B, size, 123))

    def block(h, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            tr.dis_update(xa, xb, h)
            tr.dis_council_update(xa, xb, h)
            tr.gen_update(xa, xb, h, it)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    runs = (('all off', with_switches(hp)), ('do_Dis_only_gray', with_switches(hp, gray=True)),
            ('useRandomGen', with_switches(hp, random_gen=True)), ('useRandomDis', with_switches(hp, random_dis=True)),
            ('all three on', with_switches(hp, True, True, True)))
    res = {name: [] for name, _ in runs}
    for _, h in runs:
        block(h, 1)
    for _ in range(3):
        for name, h in runs:
            res[name].append(block(h, steps))
    assert set(tr._dis_pick) == {'a2b'}  # useRandomDis ran
    base = sum(res['all off']) / 3
    for name, _ in runs:
        mean = sum(res[name]) / 3
        print('%-18s %s ms   %.1f images/s   %+.2f ms vs all off' % (name, '  '.join('%.2f' % t for t in res[name]), B * 1e3 / mean,
                                                                   mean - base))


if __name__ == '__main__':
    main()
