"""Cost of the council abs loss council_abs_w (trainer_council.py:224-228, 595-619) at male2female 256x256, council of 4, batch 8,
both directions (the term needs both).

    python scripts/prof_council_abs.py [steps]

1. The two kernels, cg_council_abs_fwd / _bwd, in colour and gray scale on tensors of the step's shapes: CUDA events around 20
   launches, best of 3; us per launch, the HBM bytes each must move (pass 1 reads two x_fake stacks; pass 2 reads two and reads and
   writes d_x), the achieved rate and the floor that bytes / 3.35 TB/s (H100 SXM data sheet) implies.
2. The training step (dis_update, dis_council_update, gen_update), `steps` (default 5) steps per block, alternating 3x in one process
   after a warm-up step of each: council_w 4 with council_abs_w 0 and 1 (one trainer), and council_w 0 with council_abs_w 1 (a
   trainer without council discriminators).  Step time and, per block, the peak device memory above what was allocated when the block
   started (the step's working set; both trainers stay resident).
Prints the card's name, power limit and max SM clock beside the numbers."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    from council_gan_b200 import Council_Trainer
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    hp, N, B, size, it = load_hp('male2female_256_n4_b8')
    hp_dc = dict(hp, do_a2b=True, do_b2a=True, council_w=4, council_abs_w=0)
    hp_both = dict(hp_dc, council_abs_w=1)
    hp_free = dict(hp_dc, council_w=0, council_abs_w=1)
    torch.manual_seed(1)
    tr = Council_Trainer(hp_both, 'cuda:0')
    ops = tr.ops

    # ---- the kernels ----------------------------------------------------------------------------------------------------------
    gen = torch.Generator().manual_seed(0)
    x_fake = torch.rand(N, B, size, size, 4, generator=gen).cuda() * 2 - 1
    d_x, sums, pub, total = torch.zeros_like(x_fake), ops.empty(N), ops.empty(N), ops.zeros(N)
    peers = [1, 2, 3, 0]
    stack = 4 * x_fake.numel()
    for gray in (False, True):
        numel = (1 if gray else 3) * B * size * size
        fwd = best_of_3(lambda: ops.council_abs_fwd(x_fake, peers, gray, sums))
        bwd = best_of_3(lambda: ops.council_abs_bwd(x_fake, peers, gray, sums, numel, 1e-9, total, pub, d_x))
        for name, ms, nbytes in (('pass 1 %s' % ('gray' if gray else 'colour'), fwd, 2 * stack),
                                 ('pass 2 %s' % ('gray' if gray else 'colour'), bwd, 4 * stack)):
            print('%-14s %7.1f us/launch  %6.1f MB  %5.2f TB/s  (floor %.1f us at 3.35 TB/s)'
                  % (name, ms * 1e3, nbytes / 1e6, nbytes / ms / 1e9, nbytes / HBM_BYTES_PER_S * 1e6))
    del x_fake, d_x

    # ---- the training step ------------------------------------------------------------------------------------------------------
    free = Council_Trainer(hp_free, 'cuda:0')
    xa, xb = (t.cuda() for t in synth(B, size, 123))

    def block(t, h, n):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            t.dis_update(xa, xb, h)
            t.dis_council_update(xa, xb, h)
            t.gen_update(xa, xb, h, it)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n, (torch.cuda.max_memory_allocated() - base) / 2 ** 30

    runs = (('council_w 4, council_abs_w 0', tr, hp_dc), ('council_w 4, council_abs_w 1', tr, hp_both),
            ('council_w 0, council_abs_w 1', free, hp_free))
    res = {name: [] for name, _, _ in runs}
    for _, t, h in runs:
        block(t, h, 1)
    for _ in range(3):
        for name, t, h in runs:
            res[name].append(block(t, h, steps))
    assert not free.do_dis_council and all(torch.is_tensor(v) for v in free.council_loss_ab_s)  # the term was live
    mean = {}
    for name, _, _ in runs:
        mean[name] = sum(t for t, _ in res[name]) / 3
        print('%-30s %s ms   working set %s GiB   %.1f images/s' % (name, '  '.join('%.1f' % t for t, _ in res[name]),
                                                                   '  '.join('%.2f' % m for _, m in res[name]), B * 1e3 / mean[name]))
    a, b, c = (mean[name] for name, _, _ in runs)
    print('council_abs_w 1 on top of the council discriminators: %+.1f ms per step' % (b - a))
    print('without council discriminators (council_w 0, abs 1) vs discriminators only (council_w 4, abs 0): %+.1f ms per step' % (c - a))


if __name__ == '__main__':
    main()
