"""Weight gradients of the generator's stride-1 3x3 layers and of the stride-2 4x4 layers of the discriminators and the encoder
(256x256 configuration: council of 4, batch 8), the TMA-fed kernel against the previous tensor-core kernel (mode bit 25),
alternating 3x in one process.

    python scripts/prof_wgrad.py [iters]

CUDA events over `iters` (default 20) launches after warm-up; the new path's time includes its transpose.  Prints ms per launch,
algorithmic TFLOP/s, the new path's HBM floor (x read once, dy read, its channel-major copy written and read back, at 3.35 TB/s),
the max difference old vs new relative to the result's magnitude, and the card it ran on."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from council_gan_b200.ops import CudaOps

NEW, OLD = 1, 7 | (1 << 25)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
# (G, B, H, W, Cin, Cout, K, stride): input map H x W, pad 1
GEOMS = [(4, 8, 64, 64, 256, 256, 3, 1), (4, 8, 128, 128, 256, 128, 3, 1), (4, 8, 128, 128, 128, 128, 3, 1),
         (4, 8, 256, 256, 128, 64, 3, 1), (4, 8, 256, 256, 64, 64, 3, 1),
         # council discriminator (real, own fake and peers' fakes per call), both scales
         (4, 32, 256, 256, 64, 128, 4, 2), (4, 32, 128, 128, 128, 256, 4, 2), (4, 32, 64, 64, 256, 512, 4, 2),
         (4, 32, 128, 128, 64, 128, 4, 2), (4, 32, 64, 64, 128, 256, 4, 2), (4, 32, 32, 32, 256, 512, 4, 2),
         # discriminator (fake + real), scale 0; encoder E1, E2
         (4, 16, 128, 128, 64, 128, 4, 2), (4, 16, 64, 64, 128, 256, 4, 2), (4, 16, 32, 32, 256, 512, 4, 2),
         (4, 8, 256, 256, 64, 128, 4, 2), (4, 8, 128, 128, 128, 256, 4, 2)]


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    ops = CudaOps('cuda:0')
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), q.stdout.strip()))
    for G, B, H, W, Cin, Cout, K, s in GEOMS:
        Ho, Wo = (H + 2 - K) // s + 1, (W + 2 - K) // s + 1
        gen = torch.Generator().manual_seed(0)
        x = torch.randn(G, B, H, W, Cin, generator=gen).cuda()
        dy = torch.randn(G, B, Ho, Wo, Cout, generator=gen).cuda()
        dw = {m: torch.empty(G, Cout, K, K, Cin, device='cuda') for m in (NEW, OLD)}
        flops = 2.0 * G * B * Ho * Wo * Cout * K * K * Cin
        floor_ms = 4.0 * (x.numel() + 3 * dy.numel()) / HBM_BYTES_PER_S * 1e3
        times = {NEW: [], OLD: []}
        for _ in range(3):
            for m in (NEW, OLD):
                ops.set_tensor_core_mode(m)
                for _ in range(3):
                    ops.conv_wgrad(x, dy, dw[m], None, s, 1)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    ops.conv_wgrad(x, dy, dw[m], None, s, 1)
                e1.record()
                torch.cuda.synchronize()
                times[m].append(e0.elapsed_time(e1) / iters)
        ops.set_tensor_core_mode(1)
        rel = ((dw[NEW].double() - dw[OLD].double()).abs().max() / dw[OLD].double().abs().max()).item()
        tn, to = min(times[NEW]), min(times[OLD])
        print('%dx%d s%d %d->%d %dx%d G%d B%d (%.1f GFLOP): new %s ms (%.0f TFLOP/s, HBM floor %.3f ms) | old %s ms (%.0f TFLOP/s) '
              '| x%.2f | max rel diff %.2e'
              % (K, K, s, Cin, Cout, H, W, G, B, flops / 1e9, ' '.join('%.3f' % t for t in times[NEW]), flops / tn / 1e9, floor_ms,
                 ' '.join('%.3f' % t for t in times[OLD]), flops / to / 1e9, to / tn, rel))
        del x, dy, dw
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
