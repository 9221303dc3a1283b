"""Forward and data-gradient convolutions of the 256x256 configuration (council of 4, batch 8) on conv_tc_kernel: the largest
launches of the step, at their production shapes.

    python scripts/prof_conv_tc.py [iters]

CUDA events over `iters` (default 20) launches after warm-up.  Every launch runs with the default epilogue and tile walk, with the
register epilogue (mode bit 27) and with the previous epilogue and walk (mode bit 26), alternating three times in one process; the
best of the three is reported for each.  Prints ms per
launch, algorithmic TFLOP/s and its ratio to the TF32 cuBLAS rate measured in the same process (torch.matmul 8192^3, best of 10, as
bench.py measures it), and the card it ran on with its power limit.  Epilogues as in the training step: the forward of the
generator layers with the fused statistics, of the discriminator layers with bias and LeakyReLU; the data gradient of the
discriminator layers masked by the layer input, of the residual layer with the residual addend."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from council_gan_b200.ops import CudaOps, ACT_LRELU

# (label, G, B, H, W, Cin, Cout, K, stride, pad): input map H x W
GEOMS = [('gen residual', 4, 8, 64, 64, 256, 256, 3, 1, 1),
         ('gen decoder', 4, 8, 128, 128, 256, 128, 3, 1, 1),
         ('gen decoder', 4, 8, 128, 128, 128, 128, 3, 1, 1),
         ('council D', 4, 32, 256, 256, 64, 128, 4, 2, 1),
         ('council D', 4, 32, 128, 128, 128, 256, 4, 2, 1),
         ('council D', 4, 32, 64, 64, 256, 512, 4, 2, 1)]


def cublas_tf32_tflops():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    ma, mb = torch.randn(8192, 8192, device='cuda'), torch.randn(8192, 8192, device='cuda')
    for _ in range(3):
        torch.matmul(ma, mb)
    best = 1e9
    for _ in range(10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.matmul(ma, mb)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    torch.backends.cuda.matmul.allow_tf32 = prev
    return 2.0 * 8192 ** 3 / (best * 1e-3) / 1e12


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


MODES = [('default', 1), ('bit 27', 7 | (1 << 27)), ('bit 26', 7 | (1 << 26))]


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    ops = CudaOps('cuda:0')
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    lib = cublas_tf32_tflops()
    print('TF32 cuBLAS (torch.matmul 8192^3): %.0f TFLOP/s' % lib)
    for label, G, B, H, W, Cin, Cout, K, s, pad in GEOMS:
        Ho, Wo = (H + 2 * pad - K) // s + 1, (W + 2 * pad - K) // s + 1
        gen = torch.Generator().manual_seed(0)
        x = torch.randn(G, B, H, W, Cin, generator=gen).cuda()
        w = (torch.randn(G, Cout, K, K, Cin, generator=gen) / (K * K * Cin) ** 0.5).cuda()
        b = torch.randn(G, Cout, generator=gen).cuda()
        dy = torch.randn(G, B, Ho, Wo, Cout, generator=gen).cuda()
        flops = 2.0 * G * B * Ho * Wo * Cout * K * K * Cin
        if s == 1:  # generator layers feed instance norm / AdaIN: statistics in the epilogue
            fwd = lambda: ops.conv_fwd_stats(x, w, s, pad)[0]
            dgrad = lambda: ops.conv_dgrad(dy, w, x.shape, s, pad, addend=x if label == 'gen residual' else None)
        else:  # discriminator layers: bias and LeakyReLU 0.2
            fwd = lambda: ops.conv_fwd(x, w, b, s, pad, act=ACT_LRELU, slope=0.2)
            dgrad = lambda: ops.conv_dgrad(dy, w, x.shape, s, pad, mask_src=x, mask_slope=0.2)
        for kind, fn in (('fwd', fwd), ('dgrad', dgrad)):
            times = {m: [] for _, m in MODES}
            for _ in range(3):
                for _, m in MODES:
                    ops.set_tensor_core_mode(m)
                    times[m].append(timed(fn, iters))
            ops.set_tensor_core_mode(1)
            for name, m in MODES:
                t = min(times[m])
                print('%-12s %-5s %dx%d s%d %d->%d %dx%d G%d B%d (%.1f GFLOP) %-8s: %s ms, %.0f TFLOP/s, %.2f of cuBLAS'
                      % (label, kind, K, K, s, Cin, Cout, H, W, G, B, flops / 1e9, name, ' '.join('%.3f' % v for v in times[m]),
                         flops / t / 1e9, flops / t / 1e9 / lib), flush=True)
        del x, w, b, dy
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
