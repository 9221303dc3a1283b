"""Per-tile fixed cost of conv_tc_kernel: the time a tile spends outside its main loop (epilogue, tile switch), at the production
shapes of the 256x256 configuration (council of 4, batch 8) with their production epilogues.

    python scripts/prof_conv_epilogue.py [iters] [--modes]

For each shape the launch is timed (CUDA events, `iters` launches after warm-up, best of three) at several lengths of the
reduction dimension K while the output, the N tile and the tile count stay the same: the input channels of a forward, the output
channels (dy channels) of a data gradient.  A persistent CTA runs ceil(tiles / SMs) rounds of one tile each, so

    time / rounds = a + b * (K chunks of 32 channels per tile)

is fitted by least squares.  The intercept `a` is the per-tile cost outside the main loop; `a * rounds / time` at the production
K is the share of the launch it takes.  With --modes every shape is also timed with mode bit 27 (every launch on the register
epilogue), alternating, so the intercepts of the two epilogues are side by side.  Prints the card name and power limit."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from council_gan_b200.ops import CudaOps, ACT_LRELU

# (label, kind, epilogue, G, B, H, W, K channels swept (production first), N, KH, stride, pad, ups)
#   fwd: input H x W, Cin = swept K, Cout = N;   dgrad: forward input H x W, Cin = N, forward Cout = swept K
SHAPES = [
    ('gen residual', 'fwd', 'stats', 4, 8, 64, 64, (256, 32, 64, 128), 256, 3, 1, 1, False),
    ('gen residual', 'dgrad', 'addend', 4, 8, 64, 64, (256, 32, 64, 128), 256, 3, 1, 1, False),
    ('gen decoder ups', 'fwd', 'stats', 4, 8, 64, 64, (256, 32, 64, 128), 128, 3, 1, 1, True),
    ('gen decoder ups', 'fwd', 'stats', 4, 8, 128, 128, (128, 32, 64), 64, 3, 1, 1, True),
    ('gen decoder', 'fwd', 'stats', 4, 8, 128, 128, (256, 32, 64, 128), 128, 3, 1, 1, False),
    ('gen decoder', 'dgrad', 'plain', 4, 8, 128, 128, (128, 32, 64, 256), 256, 3, 1, 1, False),
    ('gen decoder', 'fwd', 'stats', 4, 8, 128, 128, (128, 32, 64, 256), 128, 3, 1, 1, False),
    ('gen decoder', 'dgrad', 'plain', 4, 8, 128, 128, (128, 32, 64, 256), 128, 3, 1, 1, False),
    ('image patch 1x1', 'fwd', 'stats', 4, 8, 256, 256, (160, 32, 64, 96), 64, 1, 1, 0, False),
    ('council D', 'fwd', 'bias+lrelu', 4, 32, 256, 256, (64, 32, 128), 128, 4, 2, 1, False),
    ('council D', 'dgrad', 'mask', 4, 32, 256, 256, (128, 32, 64, 256), 64, 4, 2, 1, False),
    ('council D', 'fwd', 'bias+lrelu', 4, 32, 128, 128, (128, 32, 64, 256), 256, 4, 2, 1, False),
    ('council D', 'dgrad', 'mask', 4, 32, 128, 128, (256, 32, 64, 128), 128, 4, 2, 1, False),
    ('council D', 'fwd', 'bias+lrelu', 4, 32, 64, 64, (256, 32, 64, 128), 512, 4, 2, 1, False),
    ('council D', 'dgrad', 'mask', 4, 32, 64, 64, (512, 64, 128, 256), 256, 4, 2, 1, False),
]
BM = 128


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / iters)
    return best


def geometry(kind, H, W, N, KH, s, pad, ups):
    """(output pixels per image and class, classes, taps per class) of the conv_tc_kernel launch"""
    if kind == 'fwd':
        if ups:
            return H * W, 4, 4
        Ho, Wo = (H + 2 * pad - KH) // s + 1, (W + 2 * pad - KH) // s + 1
        return Ho * Wo, 1, KH * KH
    return (H // s) * (W // s), s * s, (KH // s) ** 2


def main():
    args = [a for a in sys.argv[1:] if not a.startswith('--')]
    iters = int(args[0]) if args else 10
    modes = [('default', 1)] + ([('bit 27', 7 | (1 << 27))] if '--modes' in sys.argv else [])
    ops = CudaOps('cuda:0')
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s | %d SMs' % (torch.cuda.get_device_name(0), q.stdout.strip(), sms))
    for label, kind, epi, G, B, H, W, ks, N, KH, s, pad, ups in SHAPES:
        pix, ncls, taps = geometry(kind, H, W, N, KH, s, pad, ups)
        bn = 256 if N % 256 == 0 else N
        tiles = G * ncls * (B * pix // BM) * (N // bn)
        rounds = -(-tiles // sms)
        gen = torch.Generator().manual_seed(0)
        res = {name: [] for name, _ in modes}
        for k in ks:
            if kind == 'fwd':
                x = torch.randn(G, B, H, W, k, generator=gen).cuda()
                w = (torch.randn(G, N, KH, KH, k, generator=gen) / (KH * KH * k) ** 0.5).cuda()
                b = torch.randn(G, N, generator=gen).cuda()
                if epi == 'stats':
                    fn = lambda: ops.conv_fwd_stats(x, w, s, pad, ups=ups)[0]
                else:
                    fn = lambda: ops.conv_fwd(x, w, b, s, pad, act=ACT_LRELU, slope=0.2)
            else:
                xs = (G, B, H, W, N)
                Ho, Wo = (H + 2 * pad - KH) // s + 1, (W + 2 * pad - KH) // s + 1
                w = (torch.randn(G, k, KH, KH, N, generator=gen) / (KH * KH * k) ** 0.5).cuda()
                dy = torch.randn(G, B, Ho, Wo, k, generator=gen).cuda()
                opnd = torch.randn(*xs, generator=gen).cuda() if epi in ('addend', 'mask') else None
                fn = lambda: ops.conv_dgrad(dy, w, xs, s, pad, addend=opnd if epi == 'addend' else None,
                                            mask_src=opnd if epi == 'mask' else None, mask_slope=0.2)
            times = {name: [] for name, _ in modes}
            for _ in range(2):
                for name, m in modes:
                    ops.set_tensor_core_mode(m)
                    times[name].append(timed(fn, iters))
            ops.set_tensor_core_mode(1)
            for name, _ in modes:
                res[name].append((taps * k // 32, min(times[name])))
            del fn
            torch.cuda.empty_cache()
        for name, _ in modes:
            kc = np.array([c for c, _ in res[name]], dtype=np.float64)
            tr = np.array([t for _, t in res[name]]) * 1e3 / rounds  # us per round
            b_fit, a_fit = np.polyfit(kc, tr, 1)
            t_prod = res[name][0][1]
            print('%-16s %-5s %-10s %dx%d s%d%s K%d->N%d %dx%d BN%d tiles %d rounds %d %-7s: %s ms | a = %.2f us/tile, b = %.3f us/chunk, '
                  'a share %.1f %% (%.3f ms of %.3f)'
                  % (label, kind, epi, KH, KH, s, ' ups' if ups else '', ks[0], N, H, W, bn, tiles, rounds, name,
                     ' '.join('K%d:%.3f' % (k, t) for k, (_, t) in zip(ks, res[name])), a_fit, b_fit,
                     100 * a_fit * rounds / 1e3 / t_prod, a_fit * rounds / 1e3, t_prod), flush=True)


if __name__ == '__main__':
    main()
