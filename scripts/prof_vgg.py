"""Cost of the perceptual loss vgg_w (trainer_council.py:531-538, 636-641) at male2female 256x256, council of 4, batch 8, both
directions (the term needs both).

    python scripts/prof_vgg.py [steps]

One trainer (built with vgg_w on; the frozen VGG-16 is the seeded synthetic one of the tests, written to a temporary directory: the
cost does not depend on the weight values) runs the whole training step with vgg_w = 0 and vgg_w = 1, alternating 3x in one process,
`steps` (default 3) steps per block after a warm-up step of each.  Reports the step time and peak device memory of each block, then,
for one step with the term on (CUDA events, CudaOps.start_timing): every VGG convolution's forward and data-gradient time and TFLOP/s
(FLOPs from shapes) against the 495 TFLOP/s TF32 dense data-sheet rate of the H100 SXM, the max-pool, preprocessing and loss kernels
with their HBM bytes, and the card's name, power limit and max SM clock."""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import torch

from bench import load_hp, synth
from vgg_oracle import synth_vgg16, write_vgg16

TF32_PEAK = 495e12  # H100 SXM5 dense TF32 data-sheet rate


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    from council_gan_b200 import Council_Trainer
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    hp, N, B, size, it = load_hp('male2female_256_n4_b8')
    tmp = tempfile.mkdtemp()
    write_vgg16(synth_vgg16(16), tmp)
    hp_off = dict(hp, do_a2b=True, do_b2a=True, vgg_w=0, vgg_model_path=tmp)
    hp_on = dict(hp_off, vgg_w=1)
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
    assert len(tr.loss_gen_vgg_a_s) == N and len(tr.loss_gen_vgg_b_s) == N  # the term was live in the 'on' blocks
    for key in ('off', 'on'):
        print('step, vgg_w %-3s  %s ms   peak %s GiB' % (key, '  '.join('%.1f' % t for t, _ in res[key]),
                                                        '  '.join('%.2f' % m for _, m in res[key])))
    mean = {k: sum(t for t, _ in v) / len(v) for k, v in res.items()}
    print('difference of the means: %+.1f ms per step (%.1f -> %.1f images/s)'
          % (mean['on'] - mean['off'], B * 1e3 / mean['off'], B * 1e3 / mean['on']))

    tr.ops.start_timing()
    block(hp_on, 1)
    timing = tr.ops.stop_timing()
    vgg_shape = 'G1 B%d' % (2 * N * B)
    tgt_shape = 'G1 B%d' % (2 * B)
    conv_ms, conv_fl = 0.0, 0.0
    for key, (ms, n, work) in sorted(timing.items()):
        if key.startswith(('conv_fwd', 'conv_dgrad')) and (' %s ' % vgg_shape in key or ' %s ' % tgt_shape in key) and ' k3 ' in key:
            per = ms / n
            conv_ms += ms
            conv_fl += work * n
            print('%-56s %2d x %8.3f ms  %6.1f TFLOP/s (%4.1f %% of %d)' % (key, n, per, work / per / 1e9, 100 * work / per / 1e9 / (TF32_PEAK / 1e12),
                                                                           TF32_PEAK / 1e12))
    print('VGG convolutions: %.1f ms, %.2f TFLOP per step, %.1f TFLOP/s' % (conv_ms, conv_fl / 1e12, conv_fl / conv_ms / 1e9))
    for key, (ms, n, nbytes) in sorted(timing.items()):
        if any(s in key for s in ('maxpool2x2', 'vgg_loss', 'vgg_preprocess', 'in_stats G1 B%d' % (2 * N * B), 'in_stats G1 B%d' % (2 * B))):
            print('%-52s %3d launches  %8.1f us/launch  %8.1f MB  %5.2f TB/s' % (key, n, ms / n * 1e3, nbytes / 1e6, nbytes / (ms / n) / 1e9))


if __name__ == '__main__':
    main()
