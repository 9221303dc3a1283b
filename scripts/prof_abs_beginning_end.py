"""Cost of the abs_beginning_end term (trainer_council.py:477-495) at the male2female 256x256 configuration (council of 4, batch 8).

    python scripts/prof_abs_beginning_end.py [iters] [steps]

1. The two kernels, cg_abs_beginning_end_fwd / _bwd, under CUDA events over `iters` (default 200) launches after warm-up: ms per
   launch, the HBM bytes each must move (pass 1 reads x_fake and x; pass 2 reads x_fake and x and reads and writes d_x) and the
   share of the 3.35 TB/s data-sheet bandwidth that implies.
2. The whole training step (dis_update, dis_council_update, gen_update) with the term on (abs_beginning_end 1, weight constant) and
   off, alternating 3x in one process, `steps` (default 10) steps per block after 3 warm-up steps of each.
Prints the card's name, power limit and max SM clock beside the numbers."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from bench import load_hp, synth

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def events(fn, n):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    from council_gan_b200 import Council_Trainer
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    hp, N, B, size, it = load_hp('male2female_256_n4_b8')
    hp_on = dict(hp, abs_beginning_end=1, abs_beginning_end_less_by=1, abs_beginning_end_minimume=0)
    torch.manual_seed(1)
    tr = Council_Trainer(hp_on, 'cuda:0')  # the gate starts from the constructor's value; hp (term off) leaves it alone
    ops = tr.ops

    # ---- the kernels on tensors of the step's shapes ------------------------------------------------------------------------
    gen = torch.Generator().manual_seed(0)
    x = torch.rand(1, B, size, size, 4, generator=gen).cuda() * 2 - 1
    x_fake = torch.rand(N, B, size, size, 4, generator=gen).cuda() * 2 - 1
    d_x, sums, pub, total = torch.zeros_like(x_fake), ops.empty(N, 2), ops.empty(N), ops.zeros(N)
    fwd_ms = events(lambda: ops.abs_beginning_end_fwd(x_fake, x, sums), iters)
    bwd_ms = events(lambda: ops.abs_beginning_end_bwd(x_fake, x, sums, 3 * B * size * size, [1e-9] * N, total, pub, d_x), iters)
    for name, ms, nbytes in (('pass 1 (sums)', fwd_ms, 4 * (x_fake.numel() + x.numel())),
                             ('pass 2 (value, gradient)', bwd_ms, 4 * (3 * x_fake.numel() + x.numel()))):
        print('%-26s %8.1f us/launch  %6.1f MB  %5.2f TB/s  (%.0f %% of 3.35 TB/s)'
              % (name, ms * 1e3, nbytes / 1e6, nbytes / ms / 1e9, 100 * nbytes / ms / 1e9 / 3.35))
    del x, x_fake, d_x

    # ---- the training step, term on / off ---------------------------------------------------------------------------------
    xa, xb = (t.cuda() for t in synth(B, size, 123))

    def step(h):
        tr.dis_update(xa, xb, h)
        tr.dis_council_update(xa, xb, h)
        tr.gen_update(xa, xb, h, it)

    res = {'on': [], 'off': []}
    for key, h in (('on', hp_on), ('off', hp)):
        events(lambda: step(h), 1)
    for _ in range(3):
        for key, h in (('on', hp_on), ('off', hp)):
            res[key].append(events(lambda: step(h), steps))
    assert len(tr.loss_gen_beginning_end_a_ab_s) == N  # the term was live in the 'on' blocks
    for key in ('on', 'off'):
        print('step, term %-3s  %s ms' % (key, '  '.join('%.2f' % v for v in res[key])))
    print('difference of the means: %+.2f ms per step' % (sum(res['on']) / 3 - sum(res['off']) / 3))


if __name__ == '__main__':
    main()
