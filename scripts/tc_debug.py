"""Bring-up harness for the tensor-core convolution: each case runs in its own subprocess with a timeout so a
hang cannot take the whole GPU visit down; prints error statistics instead of asserting."""
import json
import subprocess
import sys
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [
    # name, kind, G, Gx, B, H, W, Cin, Cout, K, stride, pad
    ('1x1_c32_o64_1tile', 'fwd', 1, 1, 1, 8, 16, 32, 64, 1, 1, 0),
    ('1x1_c64_o64', 'fwd', 1, 1, 1, 16, 16, 64, 64, 1, 1, 0),
    ('1x1_c64_o256', 'fwd', 1, 1, 2, 16, 16, 64, 256, 1, 1, 0),
    ('3x3_c32_o64', 'fwd', 1, 1, 1, 16, 16, 32, 64, 3, 1, 1),
    ('3x3_c256_o256_g2', 'fwd', 2, 2, 2, 16, 16, 256, 256, 3, 1, 1),
    ('4x4s2_c64_o128', 'fwd', 2, 2, 2, 32, 32, 64, 128, 4, 2, 1),
    ('4x4s2_c256_o512', 'fwd', 2, 2, 2, 32, 32, 256, 512, 4, 2, 1),
    ('3x3_partial_tile', 'fwd', 2, 2, 3, 12, 12, 64, 64, 3, 1, 1),
    ('3x3_many_tiles', 'fwd', 4, 4, 4, 64, 64, 256, 256, 3, 1, 1),
    ('pair_half_tile', 'fwd', 2, 2, 5, 8, 16, 64, 256, 3, 1, 1),
    ('pair_partial', 'fwd', 2, 2, 3, 12, 20, 32, 512, 3, 1, 1),
    ('dgrad_3x3', 'dgrad', 2, 2, 2, 16, 16, 128, 256, 3, 1, 1),
    ('dgrad_1x1', 'dgrad', 2, 2, 2, 16, 16, 64, 64, 1, 1, 0),
    ('dgrad_4x4s2', 'dgrad', 2, 2, 2, 32, 32, 64, 128, 4, 2, 1),
    ('dgrad_4x4s2_big', 'dgrad', 2, 2, 2, 32, 32, 256, 512, 4, 2, 1),
    ('wgrad_1x1_c32_o128', 'wgrad', 1, 1, 1, 16, 16, 32, 128, 1, 1, 0),
    ('wgrad_1x1_c64_o64', 'wgrad', 2, 2, 2, 16, 16, 64, 64, 1, 1, 0),
    ('wgrad_3x3_c64_o128', 'wgrad', 1, 1, 2, 16, 16, 64, 128, 3, 1, 1),
    ('wgrad_3x3_c256_o256', 'wgrad', 2, 2, 2, 32, 32, 256, 256, 3, 1, 1),
    ('wgrad_4x4s2_c128_o256', 'wgrad', 2, 2, 2, 32, 32, 128, 256, 4, 2, 1),
    ('wgrad_4x4s2_c256_o512', 'wgrad', 2, 2, 4, 32, 32, 256, 512, 4, 2, 1),
    ('wgrad_pair_c64_o256', 'wgrad', 2, 2, 2, 16, 16, 64, 256, 3, 1, 1),
    ('wgrad_pair_c192_o256', 'wgrad', 1, 1, 2, 16, 16, 192, 256, 3, 1, 1),
    ('wgrad_pair_1x1_c512_o512', 'wgrad', 3, 3, 4, 8, 8, 512, 512, 1, 1, 0),
    ('wgrad_xm_3x3_c128_o64', 'wgrad', 2, 2, 2, 16, 16, 128, 64, 3, 1, 1),
    ('wgrad_xm_4x4s2_c32_o64', 'wgrad', 2, 2, 2, 32, 32, 32, 64, 4, 2, 1),
    ('wgrad_xm_1x1_c96_o64', 'wgrad', 2, 1, 2, 16, 16, 96, 64, 1, 1, 0),
    ('wgrad_shared_x', 'wgrad', 2, 1, 2, 16, 16, 64, 128, 3, 1, 1),
]


def run_case(idx):
    import torch
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
    from council_gan_b200.ops import CudaOps
    from ops_torch import TorchOps
    name, kind, G, Gx, B, H, W, Cin, Cout, K, stride, pad = CASES[idx]
    ops = CudaOps('cuda:0')
    ref = TorchOps('cuda:0', torch.float64)
    g = torch.Generator().manual_seed(idx)
    x = torch.randn(Gx, B, H, W, Cin, generator=g).cuda()
    w = (torch.randn(G, Cout, K, K, Cin, generator=g) * 0.1).cuda()
    b = torch.randn(G, Cout, generator=g).cuda()
    out = {'case': name}
    if kind == 'fwd':
        ops.set_tensor_core_mode(1)
        y = ops.conv_fwd(x, w, b, stride, pad)
        torch.cuda.synchronize()
        want = ref.conv_fwd(x.double(), w.double(), b.double(), stride, pad)
        ops.set_tensor_core_mode(0)
        y0 = ops.conv_fwd(x, w, b, stride, pad)
    elif kind == 'wgrad':
        Ho = (H + 2 * pad - K) // stride + 1
        dy = torch.randn(G, B, Ho, Ho * W // H, Cout, generator=g).cuda()
        ops.set_tensor_core_mode(int(os.environ.get('TC_MODE', '1')))
        y = torch.zeros_like(w)
        ops.conv_wgrad(x, dy, y, None, stride, pad)
        torch.cuda.synchronize()
        want = torch.zeros_like(w, dtype=torch.float64)
        ref.conv_wgrad(x.double(), dy.double(), want, None, stride, pad)
        ops.set_tensor_core_mode(0)
        y0 = torch.zeros_like(w)
        ops.conv_wgrad(x, dy, y0, None, stride, pad)
    else:
        Ho = (H + 2 * pad - K) // stride + 1
        dy = torch.randn(G, B, Ho, Ho * W // H, Cout, generator=g).cuda()
        add = torch.randn(G, B, H, W, Cin, generator=g).cuda()
        ops.set_tensor_core_mode(1)
        y = ops.conv_dgrad(dy, w, (G, B, H, W, Cin), stride, pad, addend=add, mask_src=add, mask_slope=0.2)
        torch.cuda.synchronize()
        want = ref.conv_dgrad(dy.double(), w.double(), (G, B, H, W, Cin), stride, pad, addend=add.double(), mask_src=add.double(), mask_slope=0.2)
        ops.set_tensor_core_mode(0)
        y0 = ops.conv_dgrad(dy, w, (G, B, H, W, Cin), stride, pad, addend=add, mask_src=add, mask_slope=0.2)
    err = (y.double() - want).abs()
    mag = want.abs().max().item()
    out.update(max_err=err.max().item(), mean_err=err.mean().item(), mag=mag, rel=err.max().item() / mag,
               simt_rel=(y0.double() - want).abs().max().item() / mag,
               frac_bad=(err > 1e-2 * mag).double().mean().item(), nan=int(torch.isnan(y).sum().item()))
    if out['frac_bad'] > 0:  # where are the bad elements?  (group, image, row, col, channel) histogram heads
        bad = (err > 1e-2 * mag).nonzero()
        out['first_bad'] = bad[:6].tolist()
        out['bad_by_dim'] = [sorted(set(bad[:, d].tolist()))[:12] for d in range(5)]
    print('RESULT ' + json.dumps(out), flush=True)


if __name__ == '__main__':
    if len(sys.argv) > 1:
        run_case(int(sys.argv[1]))
    else:
        only = os.environ.get('TC_ONLY', '')
        for i, c in enumerate(CASES):
            if only and c[1] not in only.split(','):
                continue
            if os.environ.get('TC_NAME') and os.environ['TC_NAME'] not in c[0]:
                continue
            try:
                r = subprocess.run([sys.executable, __file__, str(i)], capture_output=True, text=True, timeout=int(os.environ.get('TC_TIMEOUT', '45')))
                lines = [l for l in r.stdout.splitlines() if l.startswith('RESULT')]
                print(c[0], lines[0] if lines else 'NO RESULT rc=%d %s' % (r.returncode, (r.stderr or '')[-600:]), flush=True)
            except subprocess.TimeoutExpired:
                print(c[0], 'TIMEOUT (hang)', flush=True)
