"""Weight gradients of the stride-1 3x3 generator layers (256x256 configuration: council of 4, batch 8), the TMA-fed kernel
against the previous tensor-core kernel (mode bit 25), alternating 3x in one process.

    python scripts/prof_wgrad.py [iters]

CUDA events over `iters` (default 20) launches after warm-up; the new path's time includes its transpose.  Prints ms per launch,
algorithmic TFLOP/s, the max difference old vs new relative to the result's magnitude, and the card it ran on."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from council_gan_b200.ops import CudaOps

NEW, OLD = 1, 7 | (1 << 25)
# (G, B, H, W, Cin, Cout): output map H x W, 3x3, pad 1
GEOMS = [(4, 8, 64, 64, 256, 256), (4, 8, 128, 128, 256, 128), (4, 8, 128, 128, 128, 128),
         (4, 8, 256, 256, 128, 64), (4, 8, 256, 256, 64, 64)]


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    ops = CudaOps('cuda:0')
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    for G, B, H, W, Cin, Cout in GEOMS:
        gen = torch.Generator().manual_seed(0)
        x = torch.randn(G, B, H, W, Cin, generator=gen).cuda()
        dy = torch.randn(G, B, H, W, Cout, generator=gen).cuda()
        dw = {m: torch.empty(G, Cout, 3, 3, Cin, device='cuda') for m in (NEW, OLD)}
        flops = 2.0 * G * B * H * W * Cout * 9 * Cin
        times = {NEW: [], OLD: []}
        for _ in range(3):
            for m in (NEW, OLD):
                ops.set_tensor_core_mode(m)
                for _ in range(3):
                    ops.conv_wgrad(x, dy, dw[m], None, 1, 1)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    ops.conv_wgrad(x, dy, dw[m], None, 1, 1)
                e1.record()
                torch.cuda.synchronize()
                times[m].append(e0.elapsed_time(e1) / iters)
        ops.set_tensor_core_mode(1)
        rel = ((dw[NEW].double() - dw[OLD].double()).abs().max() / dw[OLD].double().abs().max()).item()
        tn, to = min(times[NEW]), min(times[OLD])
        print('3x3 %d->%d %dx%d G%d B%d (%.1f GFLOP): new %s ms (%.0f TFLOP/s) | old %s ms (%.0f TFLOP/s) | x%.2f | max rel diff %.2e'
              % (Cin, Cout, H, W, G, B, flops / 1e9, ' '.join('%.3f' % t for t in times[NEW]), flops / tn / 1e9,
                 ' '.join('%.3f' % t for t in times[OLD]), flops / to / 1e9, to / tn, rel))
        del x, dy, dw
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
