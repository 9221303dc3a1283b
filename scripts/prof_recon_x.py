"""Cost of the image reconstruction term recon_x_w (trainer_council.py:339-345, 455-459) at male2female 256x256, council of 4, batch 8,
both directions (the term needs both).

    python scripts/prof_recon_x.py [steps]

One trainer (built with recon_x_w on, so its style encoder is trainable) runs the whole training step (dis_update, dis_council_update,
gen_update) with the term off and with recon_x_w = 1, alternating 3x in one process, `steps` (default 5) steps per block after a
warm-up step of each.  Reports the step time and peak device memory of each block, then the per-launch time, bytes and TB/s of the
two reconstruction-head kernels in one step with the term on (CUDA events, CudaOps.start_timing), and the card's name, power limit
and max SM clock."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from bench import load_hp, synth


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    from council_gan_b200 import Council_Trainer
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    hp, N, B, size, it = load_hp('male2female_256_n4_b8')
    hp_off = dict(hp, do_a2b=True, do_b2a=True, recon_x_w=0)
    hp_on = dict(hp_off, recon_x_w=1)
    torch.manual_seed(1)
    tr = Council_Trainer(hp_on, 'cuda:0')
    xa, xb = (t.cuda() for t in synth(B, size, 123))

    def block(h, n):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            tr.dis_update(xa, xb, h)
            tr.dis_council_update(xa, xb, h)
            tr.gen_update(xa, xb, h, it)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n, torch.cuda.max_memory_allocated() / 2 ** 30

    res = {'off': [], 'on': []}
    for h in (hp_off, hp_on):
        block(h, 1)
    for _ in range(3):
        for key, h in (('off', hp_off), ('on', hp_on)):
            res[key].append(block(h, steps))
    assert len(tr.loss_gen_recon_x_a_s) == N and len(tr.loss_gen_recon_x_b_s) == N  # the term was live in the 'on' blocks
    for key in ('off', 'on'):
        print('step, term %-3s  %s ms   peak %s GiB' % (key, '  '.join('%.1f' % t for t, _ in res[key]),
                                                       '  '.join('%.2f' % m for _, m in res[key])))
    mean = {k: sum(t for t, _ in v) / len(v) for k, v in res.items()}
    print('difference of the means: %+.1f ms per step (%.1f -> %.1f images/s)'
          % (mean['on'] - mean['off'], B * 1e3 / mean['off'], B * 1e3 / mean['on']))

    tr.ops.start_timing()
    block(hp_on, 1)
    for key, (ms, n, nbytes) in sorted(tr.ops.stop_timing().items()):
        if 'recon_head' in key:
            print('%-44s %3d launches  %8.1f us/launch  %7.1f MB  %5.2f TB/s' % (key, n, ms / n * 1e3, nbytes / 1e6, nbytes / (ms / n) / 1e9))


if __name__ == '__main__':
    main()
