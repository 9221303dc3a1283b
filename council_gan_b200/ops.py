"""ctypes binding of libcouncil_b200.so (the C ABI declared in include/council_b200.h).

PyTorch is used here for device memory (``torch.empty``), the current CUDA stream and nothing else:
every method hands raw device pointers to a hand-written sm_90a kernel.  There is NO fallback:
if the shared library is missing or no CUDA device is present, constructing :class:`CudaOps` raises.

Tensor conventions (see the header): fp32, channels-last activations stacked over the council
``[G, B, H, W, C]``; weights stacked OHWI ``[G, Cout, KH, KW, Cin]``.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libcouncil_b200.so')

ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH = 0, 1, 2, 3


class ConvGeom(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('G', 'x_groups', 'B', 'H', 'W', 'Cin', 'Ho', 'Wo', 'Cout',
                                         'KH', 'KW', 'stride', 'pad', 'ups')]


LOSS_MAX_MAPS, LOSS_MAX_G, LOSS_MAX_SEG = 4, 8, 8


class LsganDesc(C.Structure):  # cg_lsgan_desc
    _fields_ = [('nmaps', C.c_int32), ('G', C.c_int32), ('nseg', C.c_int32), ('_pad', C.c_int32),
                ('out', C.c_void_p * LOSS_MAX_MAPS), ('dout', C.c_void_p * LOSS_MAX_MAPS),
                ('n_per_seg', C.c_int32 * LOSS_MAX_MAPS), ('target', C.c_float * LOSS_MAX_SEG),
                ('weight', (C.c_float * LOSS_MAX_SEG) * LOSS_MAX_G), ('loss_scale', C.c_float), ('grad_scale', C.c_float)]


class GenLossDesc(C.Structure):  # cg_gen_loss_desc
    _fields_ = [('G', C.c_int32), ('B', C.c_int32), ('H', C.c_int32), ('W', C.c_int32), ('n_adv', C.c_int32), ('n_cl', C.c_int32),
                ('adv_out', C.c_void_p * 2), ('adv_dout', C.c_void_p * 2), ('cl_out', C.c_void_p * 2), ('cl_dout', C.c_void_p * 2),
                ('adv_n', C.c_int32 * 2), ('cl_n', C.c_int32 * 2), ('mask', C.c_void_p),
                ('center', C.c_float), ('eps', C.c_float), ('adv_grad_scale', C.c_float), ('_pad', C.c_float)]


class GenLossHp(C.Structure):  # cg_gen_loss_hp
    _fields_ = [(n, C.c_int32) for n in ('world', 'hist_size', 'head_gan', 'head_council', 'gan_on', 'council_on', 'focus_on',
                                         'matching', 'small_abs', 'small_square')] + \
               [(n, C.c_double) for n in ('gan_w', 'council_w', 'w01', 'wtot', 'wtv', 'numel')] + \
               [(n, C.c_int32) for n in ('focus_matching', 'head_focus', 'head_focus01', '_pad')] + \
               [(n, C.c_void_p) for n in ('hist_focus', 'hist_focus01', 'focus_src', 'focus_w')]


_fp = C.c_void_p
_SIGS = {
    'cg_last_error': (C.c_char_p, []),
    'cg_device_info': (C.c_int, [C.POINTER(C.c_int)] * 3),
    'cg_set_tensor_core_mode': (C.c_int, [C.c_int]),
    'cg_launch_count': (C.c_uint64, []),
    'cg_tensor_map_cache_stats': (None, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    'cg_conv_fwd': (C.c_int, [C.POINTER(ConvGeom), _fp, _fp, _fp, _fp, C.c_int, C.c_float, _fp, C.c_size_t, _fp]),
    'cg_conv_fwd_stats': (C.c_int, [C.POINTER(ConvGeom), _fp, _fp, _fp, _fp, _fp, C.c_float, _fp, C.c_size_t, _fp]),
    'cg_conv_fwd_stats_workspace_bytes': (C.c_size_t, [C.POINTER(ConvGeom)]),
    'cg_conv_dgrad': (C.c_int, [C.POINTER(ConvGeom), _fp, _fp, _fp, _fp, _fp, C.c_float, _fp, C.c_size_t, _fp]),
    'cg_conv_wgrad': (C.c_int, [C.POINTER(ConvGeom), _fp, _fp, _fp, _fp, _fp, C.c_size_t, _fp]),
    'cg_conv_workspace_bytes': (C.c_size_t, [C.POINTER(ConvGeom), C.c_int]),
    'cg_in_stats': (C.c_int, [_fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _fp, C.c_size_t, _fp]),
    'cg_norm_act_fwd': (C.c_int, [_fp, _fp, _fp, _fp, C.c_int, C.c_int, _fp, _fp] + [C.c_int] * 7 + [_fp]),
    'cg_norm_act_bwd': (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, _fp, _fp] + [C.c_int] * 7 + [_fp, C.c_size_t, _fp]),
    'cg_ln_workspace_bytes': (C.c_size_t, [C.c_int] * 4),
    'cg_ln_stats': (C.c_int, [_fp, _fp, _fp] + [C.c_int] * 4 + [_fp, C.c_size_t, _fp]),
    'cg_ln_act_fwd': (C.c_int, [_fp] * 5 + [C.c_float, _fp] + [C.c_int] * 6 + [_fp]),
    'cg_ln_act_bwd': (C.c_int, [_fp] * 6 + [C.c_float] + [_fp] * 3 + [C.c_int] * 6 + [_fp, C.c_size_t, _fp]),
    'cg_upsample2x_bwd': (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_mask_head_fwd': (C.c_int, [_fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_head_fused': (C.c_int, [_fp, _fp, _fp, _fp, C.c_int, C.c_int] + [_fp] * 9 + [C.c_int] * 3 + [_fp]),
    'cg_mask_head_bwd': (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_avgpool_fwd': (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_avgpool_bwd': (C.c_int, [_fp, _fp] + [C.c_int] * 7 + [_fp]),
    'cg_acc_slice': (C.c_int, [_fp, _fp, C.c_long, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_gather_images': (C.c_int, [_fp, C.c_int, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_gather_images_gray': (C.c_int, [_fp, C.c_int, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_gray_fold': (C.c_int, [_fp, C.c_long, _fp]),
    'cg_gather_members': (C.c_int, [_fp, _fp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_int32), C.c_int, _fp]),
    'cg_nchw_to_nhwc': (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_nhwc_to_nchw': (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_lsgan_fwd': (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_lsgan_bwd': (C.c_int, [_fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_focus_fwd': (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, _fp, C.c_size_t, _fp]),
    'cg_focus_bwd': (C.c_int, [_fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, _fp]),
    'cg_lsgan_fused': (C.c_int, [C.POINTER(LsganDesc), _fp, C.c_int, _fp, _fp, C.c_size_t, _fp]),
    'cg_gen_loss_fwd': (C.c_int, [C.POINTER(GenLossDesc), _fp, _fp, C.c_size_t, _fp]),
    'cg_gen_loss_bwd': (C.c_int, [C.POINTER(GenLossDesc), C.POINTER(GenLossHp), _fp, _fp, _fp, _fp, C.c_int, _fp, _fp, _fp, C.c_size_t, _fp]),
    'cg_abs_beginning_end_fwd': (C.c_int, [_fp, _fp, _fp] + [C.c_int] * 4 + [_fp, C.c_size_t, _fp]),
    'cg_abs_beginning_end_bwd': (C.c_int, [_fp, _fp, _fp, C.c_double, C.POINTER(C.c_double), _fp, _fp, _fp] + [C.c_int] * 4 +
                                 [_fp, C.c_size_t, _fp]),
    'cg_council_abs_fwd': (C.c_int, [_fp, C.POINTER(C.c_int32), C.c_int, _fp] + [C.c_int] * 4 + [_fp, C.c_size_t, _fp]),
    'cg_council_abs_bwd': (C.c_int, [_fp, C.POINTER(C.c_int32), C.c_int, _fp, C.c_double, C.c_double, _fp, _fp, _fp] + [C.c_int] * 4 +
                           [_fp, C.c_size_t, _fp]),
    'cg_latent_l1': (C.c_int, [_fp, _fp, C.c_int, _fp, _fp, C.c_float, C.c_int, _fp, C.c_int, C.c_long, _fp, C.c_size_t, _fp]),
    'cg_recon_finalize': (C.c_int, [_fp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int, C.c_int, _fp, _fp, _fp, C.c_size_t,
                                    _fp]),
    'cg_recon_head_fwd': (C.c_int, [_fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp, C.c_size_t, _fp]),
    'cg_recon_head_bwd': (C.c_int, [_fp, _fp, C.c_float, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_vgg_preprocess': (C.c_int, [_fp, _fp, C.c_long, _fp]),
    'cg_vgg_preprocess_bwd': (C.c_int, [_fp, _fp, C.c_long, C.c_int, _fp]),
    'cg_maxpool2x2_fwd': (C.c_int, [_fp, _fp] + [C.c_int] * 4 + [_fp]),
    'cg_maxpool2x2_bwd': (C.c_int, [_fp, _fp, _fp] + [C.c_int] * 4 + [_fp]),
    'cg_vgg_loss': (C.c_int, [_fp] * 6 + [C.c_int] * 5 + [C.c_float, _fp, _fp, _fp, C.c_size_t, _fp]),
    'cg_reflect_pad': (C.c_int, [_fp, _fp] + [C.c_int] * 6 + [_fp]),
    'cg_reflect_pad_bwd': (C.c_int, [_fp, _fp, _fp, _fp, C.c_float] + [C.c_int] * 5 + [_fp]),
    'cg_global_avgpool_fwd': (C.c_int, [_fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_global_avgpool_bwd': (C.c_int, [_fp, _fp, _fp, C.c_int, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_loss_workspace_bytes': (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    'cg_zero': (C.c_int, [_fp, C.c_size_t, _fp]),
    'cg_aug_color': (C.c_int, [_fp, _fp, _fp, _fp, _fp, C.c_int, C.c_int, C.c_int, _fp]),
    'cg_aug_resize_crop': (C.c_int, [_fp] * 5 + [C.c_int] * 7 + [_fp, _fp, C.c_int, _fp, _fp, C.c_int, _fp, _fp, _fp, _fp]),
    'cg_adam_step': (C.c_int, [_fp, _fp, _fp, _fp, C.c_long] + [C.c_float] * 5 + [C.c_int, C.c_float, _fp]),
}
EXPORTS = tuple(_SIGS)


def load_library(path=LIB_PATH):
    """dlopen the library and attach argtypes.  Works without a GPU (symbol check only)."""
    if not os.path.exists(path):
        raise RuntimeError('%s not found: build it with `python -m council_gan_b200.build` '
                           '(there is no CPU or PyTorch fallback for this path)' % path)
    lib = C.CDLL(path)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


def _p(t):
    return None if t is None else t.data_ptr()


def conv_out_size(h, k, stride, pad, ups):
    return ((2 * h if ups else h) + 2 * pad - k) // stride + 1


class CudaOps:
    """The product op-set: every method is one (or a few) launches of our own kernels."""

    name = 'cuda'
    dtype = torch.float32

    def __init__(self, device='cuda:0', workspace_bytes=256 << 20):
        if not torch.cuda.is_available():
            raise RuntimeError('council_gan_b200 needs a CUDA device (sm_90a); no CPU path exists')
        self.lib = load_library()
        self._stream_cached = None
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        sm, maj, mnr = C.c_int(), C.c_int(), C.c_int()
        rc = self.lib.cg_device_info(C.byref(sm), C.byref(maj), C.byref(mnr))
        if rc < 0:
            raise RuntimeError('cg_device_info: ' + self.lib.cg_last_error().decode())
        self.sm_count, self.cc = sm.value, (maj.value, mnr.value)
        if self.cc != (9, 0):
            raise RuntimeError('libcouncil_b200.so is built for sm_90a only; device is sm_%d%d' % self.cc)
        self._ws = torch.empty(workspace_bytes, dtype=torch.uint8, device=self.device)
        # dedicated, zero-initialised scratch of the fused loss kernels (ticket counter + partial sums); grown on demand
        self._loss_ws = self._zero_bytes(1 << 16)
        # small per-step host data (style noise, peer index tables): ONE pinned staging buffer and ONE async H2D copy per
        # update instead of a pageable `torch.tensor(...).to(device)` (a hidden host sync) per table
        self._stage_ring = [None] * 8
        self._ws_sizes = {}
        self._stage_next = 0

    # -- plumbing ---------------------------------------------------------------------------------
    def _stream(self):
        c = self._stream_cached
        return c if c is not None else torch.cuda.current_stream(self.device).cuda_stream

    def pin_stream(self):
        """Resolve torch's current stream ONCE for a run of launches (the trainer pins it for the duration of an update: a per-launch
        lookup is a noticeable share of the host time of a step on the launch-bound small configurations)."""
        self._stream_cached = torch.cuda.current_stream(self.device).cuda_stream

    def unpin_stream(self):
        self._stream_cached = None

    def _ck(self, rc, what):
        if rc != 0:
            raise RuntimeError('%s failed (%d): %s' % (what, rc, self.lib.cg_last_error().decode()))

    def _conv_ws(self, g, which):
        """Workspace of a convolution call; the size query is cached per (geometry, direction, kernel-selection mode)."""
        key = (which, self._tc_mode, g.G, g.x_groups, g.B, g.H, g.W, g.Cin, g.Ho, g.Wo, g.Cout, g.KH, g.KW, g.stride, g.pad, g.ups)
        n = self._ws_sizes.get(key)
        if n is None:
            n = int(self.lib.cg_conv_workspace_bytes(C.byref(g), which))
            self._ws_sizes[key] = n
        return self._ws_for(n)

    def _ws_for(self, nbytes):
        if nbytes > self._ws.numel():
            self._ws = torch.empty(int(nbytes * 1.25) + 1024, dtype=torch.uint8, device=self.device)
        return self._ws

    def empty(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self.device)

    def _zero_bytes(self, n):
        t = torch.empty(n, dtype=torch.uint8, device=self.device)
        self._ck(self.lib.cg_zero(t.data_ptr(), n, self._stream()), 'cg_zero')
        return t

    def zeros(self, *shape):
        t = torch.empty(*shape, dtype=torch.float32, device=self.device)
        self._ck(self.lib.cg_zero(t.data_ptr(), t.numel() * 4, self._stream()), 'cg_zero')
        return t

    def launch_count(self):
        return int(self.lib.cg_launch_count())

    def tensor_map_cache_stats(self):
        h, m = C.c_uint64(), C.c_uint64()
        self.lib.cg_tensor_map_cache_stats(C.byref(h), C.byref(m))
        return {'hits': int(h.value), 'misses': int(m.value)}

    _tc_mode = 1

    pdl = False

    def set_tensor_core_mode(self, mode):
        """mode as cg_set_tensor_core_mode documents it; the programmatic-dependent-launch bit (1 << 22) is added here when set_pdl(True)"""
        self._tc_mode = mode = int(mode)
        eff = 7 if mode == 1 else mode
        if self.pdl and mode:
            eff |= 1 << 22
        return self.lib.cg_set_tensor_core_mode(eff)

    def set_pdl(self, on):
        """Programmatic dependent launch between the library's kernels: pays on launch-bound small maps, costs ~2 % on long kernels."""
        on = bool(on)
        if on != self.pdl:
            self.pdl = on
            self.set_tensor_core_mode(self._tc_mode)

    # -- live per-kernel timing (bench.py roofline): CUDA events on the launching stream ----------
    _timing = None

    def start_timing(self):
        self._timing = {}

    def stop_timing(self):
        """-> {kernel key: (total ms, launches, algorithmic FLOPs (conv_*) or HBM bytes (hbm:*) per launch)}."""
        rec, self._timing = self._timing or {}, None
        torch.cuda.synchronize(self.device)
        return {k: (sum(a.elapsed_time(b) for a, b in evs), len(evs), fl) for k, (evs, fl) in rec.items()}

    def _timed(self, kind, g, fn):
        if self._timing is None:
            return fn()
        key = '%s G%d B%d %dx%d Cin%d Cout%d k%d s%d%s' % (kind, g.G, g.B, g.H, g.W, g.Cin, g.Cout, g.KH, g.stride,
                                                          ' ups' if g.ups else '')
        flops = 2.0 * g.G * g.B * g.Ho * g.Wo * g.Cout * g.KH * g.KW * g.Cin
        return self._timed_raw(key, flops, fn)

    def _timed_raw(self, key, work, fn):
        """work = algorithmic FLOPs (conv_* keys) or algorithmic HBM bytes (hbm:* keys) of one launch."""
        if self._timing is None:
            return fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        self._timing.setdefault(key, ([], work))[0].append((e0, e1))
        return out

    @staticmethod
    def _chk(*ts):
        for t in ts:
            if t is not None:
                assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda, 'need contiguous fp32 CUDA tensors'

    # -- convolution ------------------------------------------------------------------------------
    def _geom(self, xshape, w, stride, pad, ups):
        Gx, B, H, W, Cin = xshape
        G, Cout, KH, KW, Cin2 = w.shape
        assert Cin == Cin2, (xshape, tuple(w.shape))
        Ho, Wo = conv_out_size(H, KH, stride, pad, ups), conv_out_size(W, KW, stride, pad, ups)
        return ConvGeom(G, Gx, B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, int(bool(ups)))

    def conv_fwd(self, x, w, bias, stride, pad, ups=False, act=ACT_NONE, slope=0.2):
        self._chk(x, w, bias)
        g = self._geom(x.shape, w, stride, pad, ups)
        y = self.empty(g.G, g.B, g.Ho, g.Wo, g.Cout)
        ws = self._conv_ws(g, 0)
        self._timed('conv_fwd', g, lambda: self._ck(self.lib.cg_conv_fwd(
            C.byref(g), _p(x), _p(w), _p(bias), _p(y), act, slope, _p(ws), ws.numel(), self._stream()), 'cg_conv_fwd'))
        return y

    def conv_fwd_stats(self, x, w, stride, pad, ups=False, eps=1e-5):
        """conv (no bias / activation) + instance-norm statistics of its output: (y, mean, rstd)."""
        self._chk(x, w)
        g = self._geom(x.shape, w, stride, pad, ups)
        y = self.empty(g.G, g.B, g.Ho, g.Wo, g.Cout)
        mean, rstd = self.empty(g.G, g.B, g.Cout), self.empty(g.G, g.B, g.Cout)
        ws = self._ws_for(self.lib.cg_conv_fwd_stats_workspace_bytes(C.byref(g)))
        self._timed('conv_fwd', g, lambda: self._ck(self.lib.cg_conv_fwd_stats(
            C.byref(g), _p(x), _p(w), _p(y), _p(mean), _p(rstd), eps, _p(ws), ws.numel(), self._stream()), 'cg_conv_fwd_stats'))
        return y, mean, rstd

    def conv_dgrad(self, dy, w, x_shape, stride, pad, ups=False, addend=None, mask_src=None, mask_slope=0.0):
        self._chk(dy, w, addend, mask_src)
        G = w.shape[0]
        g = self._geom((G,) + tuple(x_shape[1:]), w, stride, pad, ups)
        assert tuple(dy.shape) == (g.G, g.B, g.Ho, g.Wo, g.Cout), (tuple(dy.shape), (g.G, g.B, g.Ho, g.Wo, g.Cout))
        dx = self.empty(g.G, g.B, g.H, g.W, g.Cin)
        ws = self._conv_ws(g, 1)
        self._timed('conv_dgrad', g, lambda: self._ck(self.lib.cg_conv_dgrad(
            C.byref(g), _p(dy), _p(w), _p(dx), _p(addend), _p(mask_src), mask_slope, _p(ws), ws.numel(), self._stream()),
            'cg_conv_dgrad'))
        return dx

    def conv_wgrad(self, x, dy, dw, db, stride, pad, ups=False):
        """dw [G,Cout,KH,KW,Cin] and db [G,Cout] (or None) are OUTPUT views (overwritten)."""
        self._chk(x, dy, dw, db)
        g = self._geom(x.shape, dw, stride, pad, ups)
        assert tuple(dy.shape) == (g.G, g.B, g.Ho, g.Wo, g.Cout)
        ws = self._conv_ws(g, 2)
        self._timed('conv_wgrad', g, lambda: self._ck(self.lib.cg_conv_wgrad(
            C.byref(g), _p(x), _p(dy), _p(dw), _p(db), _p(ws), ws.numel(), self._stream()), 'cg_conv_wgrad'))

    # -- instance norm / AdaIN --------------------------------------------------------------------
    def in_stats(self, y, eps=1e-5):
        self._chk(y)
        G, B, H, W, Cc = y.shape
        mean, rstd = self.empty(G, B, Cc), self.empty(G, B, Cc)
        ws = self._ws_for(((H * W + 127) // 128) * G * B * Cc * 8)
        self._timed_raw('hbm:in_stats G%d B%d %dx%d C%d' % (G, B, H, W, Cc), 4.0 * y.numel(),
                        lambda: self._ck(self.lib.cg_in_stats(_p(y), _p(mean), _p(rstd), G, B, H * W, Cc, eps, _p(ws), ws.numel(),
                                                              self._stream()), 'cg_in_stats'))
        return mean, rstd

    def norm_act_fwd(self, y, mean, rstd, adain=None, off=0, res=None, act=ACT_NONE, ups=False):
        self._chk(y, mean, rstd, adain, res)
        G, B, H, W, Cc = y.shape
        z = self.empty(G, B, 2 * H if ups else H, 2 * W if ups else W, Cc)
        P = adain.shape[-1] if adain is not None else 0
        units = 1 + (1 if res is not None else 0) + (4 if ups else 1)  # read y (+ residual), write z (x4 when upsampling)
        self._timed_raw('hbm:norm_act_fwd G%d B%d %dx%d C%d%s%s' % (G, B, H, W, Cc, ' res' if res is not None else '', ' ups' if ups else ''),
                        4.0 * units * y.numel(),
                        lambda: self._ck(self.lib.cg_norm_act_fwd(_p(y), _p(mean), _p(rstd), _p(adain), P, off, _p(res), _p(z), G, B, H, W,
                                                                  Cc, act, int(bool(ups)), self._stream()), 'cg_norm_act_fwd'))
        return z

    def norm_act_bwd(self, dz, y, mean, rstd, adain=None, off=0, act=ACT_NONE, ups=False, d_adain=None):
        self._chk(dz, y, mean, rstd, adain, d_adain)
        G, B, H, W, Cc = y.shape
        dy = self.empty(G, B, H, W, Cc)
        P = adain.shape[-1] if adain is not None else 0
        ws = self._ws_for((((H * W + 127) // 128) + 1) * G * B * Cc * 8)
        units = 2 * (1 + (4 if ups else 1)) + 1  # two passes over (y, dz) -- the reduction, then the apply -- and one write of dy
        self._timed_raw('hbm:norm_act_bwd G%d B%d %dx%d C%d%s' % (G, B, H, W, Cc, ' ups' if ups else ''), 4.0 * units * y.numel(),
                        lambda: self._ck(self.lib.cg_norm_act_bwd(_p(dz), _p(y), _p(mean), _p(rstd), _p(adain), P, off, _p(dy), _p(d_adain),
                                                                  G, B, H, W, Cc, act, int(bool(ups)), _p(ws), ws.numel(), self._stream()),
                                         'cg_norm_act_bwd'))
        return dy

    # -- layer norm (the discriminators' dis.norm ln) -------------------------------------------------
    def ln_stats(self, y):
        """-> (mean, std) [G,B]: each sample's mean and unbiased std over H*W*C"""
        self._chk(y)
        G, B, H, W, Cc = y.shape
        mean, std = self.empty(G, B), self.empty(G, B)
        ws = self._ws_for(self.lib.cg_ln_workspace_bytes(G, B, H * W, Cc))
        self._timed_raw('hbm:ln_stats G%d B%d %dx%d C%d' % (G, B, H, W, Cc), 4.0 * y.numel(),
                        lambda: self._ck(self.lib.cg_ln_stats(_p(y), _p(mean), _p(std), G, B, H * W, Cc, _p(ws), ws.numel(),
                                                              self._stream()), 'cg_ln_stats'))
        return mean, std

    def ln_act_fwd(self, y, mean, std, gamma, beta, act=ACT_LRELU, eps=1e-5):
        """act((y - mean) / (std + eps) * gamma + beta); gamma, beta [G,C]"""
        self._chk(y, mean, std, gamma, beta)
        G, B, H, W, Cc = y.shape
        z = self.empty(G, B, H, W, Cc)
        self._timed_raw('hbm:ln_act_fwd G%d B%d %dx%d C%d' % (G, B, H, W, Cc), 8.0 * y.numel(),
                        lambda: self._ck(self.lib.cg_ln_act_fwd(_p(y), _p(mean), _p(std), _p(gamma), _p(beta), eps, _p(z), G, B, H, W, Cc,
                                                                act, self._stream()), 'cg_ln_act_fwd'))
        return z

    def ln_act_bwd(self, dz, y, mean, std, gamma, beta, dgamma, dbeta, act=ACT_LRELU, eps=1e-5):
        """-> d(y); dgamma, dbeta [G,C] are OUTPUT views (overwritten with the sums over each member's samples)"""
        self._chk(dz, y, mean, std, gamma, beta, dgamma, dbeta)
        G, B, H, W, Cc = y.shape
        dy = self.empty(G, B, H, W, Cc)
        ws = self._ws_for(self.lib.cg_ln_workspace_bytes(G, B, H * W, Cc))
        # two passes over (y, dz) -- the reduction, then the apply -- and one write of dy
        self._timed_raw('hbm:ln_act_bwd G%d B%d %dx%d C%d' % (G, B, H, W, Cc), 20.0 * y.numel(),
                        lambda: self._ck(self.lib.cg_ln_act_bwd(_p(dz), _p(y), _p(mean), _p(std), _p(gamma), _p(beta), eps, _p(dy),
                                                                _p(dgamma), _p(dbeta), G, B, H, W, Cc, act, _p(ws), ws.numel(),
                                                                self._stream()), 'cg_ln_act_bwd'))
        return dy

    def upsample2x_bwd(self, d_up):
        self._chk(d_up)
        G, B, H2, W2, Cc = d_up.shape
        dx = self.empty(G, B, H2 // 2, W2 // 2, Cc)
        self._ck(self.lib.cg_upsample2x_bwd(_p(d_up), _p(dx), G * B, H2 // 2, W2 // 2, Cc, self._stream()),
                 'cg_upsample2x_bwd')
        return dx

    # -- mask head --------------------------------------------------------------------------------
    def mask_head_fwd(self, h, x_in):
        self._chk(h, x_in)
        G, B, H, W, _ = h.shape
        x_fake, mask = self.empty(G, B, H, W, 4), self.empty(G, B, H, W, 4)
        self._ck(self.lib.cg_mask_head_fwd(_p(h), _p(x_in), _p(x_fake), _p(mask), G, B, H * W, self._stream()),
                 'cg_mask_head_fwd')
        return x_fake, mask

    def head_fused(self, y, mean, rstd, adain, off, w1, b1, w2, b2, w3, b3, x_in):
        """AdaIN + ReLU of the last 3x3 block, the three 1x1 head convolutions and the mask compositing in ONE launch
        (no-grad decoder passes): y [G,B,H,W,64] raw conv output -> (x_fake, mask) [G,B,H,W,4]"""
        self._chk(y, mean, rstd, adain, w1, b1, w2, b2, w3, b3, x_in)
        G, B, H, W, Cc = y.shape
        assert Cc == 64 and tuple(w1.shape[1:]) == (64, 1, 1, 64) and tuple(w3.shape[1:]) == (12, 1, 1, 64)
        x_fake, mask = self.empty(G, B, H, W, 4), self.empty(G, B, H, W, 4)
        P = adain.shape[-1] if adain is not None else 0
        self._timed_raw('hbm:head_fused G%d B%d %dx%d' % (G, B, H, W), 4.0 * (y.numel() + 3 * x_fake.numel()),
                        lambda: self._ck(self.lib.cg_head_fused(_p(y), _p(mean), _p(rstd), _p(adain), P, off, _p(w1), _p(b1), _p(w2), _p(b2),
                                                                _p(w3), _p(b3), _p(x_in), _p(x_fake), _p(mask), G, B, H * W, self._stream()),
                                         'cg_head_fused'))
        return x_fake, mask

    def head_fused_supported(self, y_shape):
        # a wgmma (TF32) kernel: not used when the exact-fp32 SIMT mode is selected (cg_set_tensor_core_mode(0))
        return (self._tc_mode & 1) == 1 and y_shape[-1] == 64 and (y_shape[2] * y_shape[3]) % 128 == 0

    def mask_head_bwd(self, h, x_in, d_xfake, d_mask=None):
        self._chk(h, x_in, d_xfake, d_mask)
        G, B, H, W, _ = h.shape
        dh = self.empty(G, B, H, W, 12)
        self._ck(self.lib.cg_mask_head_bwd(_p(h), _p(x_in), _p(d_xfake), _p(d_mask), _p(dh), G, B, H * W,
                                           self._stream()), 'cg_mask_head_bwd')
        return dh

    # -- image-space helpers ----------------------------------------------------------------------
    def avgpool_fwd(self, x):
        self._chk(x)
        G, B, H, W, Cc = x.shape
        y = self.empty(G, B, H // 2, W // 2, Cc)
        self._ck(self.lib.cg_avgpool_fwd(_p(x), _p(y), G * B, H, W, Cc, self._stream()), 'cg_avgpool_fwd')
        return y

    def avgpool_bwd(self, dy, dx, nch, accumulate):
        self._chk(dy, dx)
        G, B, H, W, Cx = dx.shape
        self._ck(self.lib.cg_avgpool_bwd(_p(dy), _p(dx), G * B, H, W, dy.shape[-1], Cx, nch, int(bool(accumulate)),
                                         self._stream()), 'cg_avgpool_bwd')

    def global_avgpool_fwd(self, h):
        """h [G,B,H,W,C] -> [G,B,1,1,C], the mean over H x W (the style encoder's nn.AdaptiveAvgPool2d(1))"""
        self._chk(h)
        G, B, H, W, Cc = h.shape
        y = self.empty(G, B, 1, 1, Cc)
        self._ck(self.lib.cg_global_avgpool_fwd(_p(h), _p(y), G * B, H * W, Cc, self._stream()), 'cg_global_avgpool_fwd')
        return y

    def global_avgpool_bwd(self, dy, h, relu_gate=True):
        """dy [G,B,1,1,C], h [G,B,H,W,C] (the pooled ReLU output) -> dh = dy / HW, gated by h > 0 when relu_gate"""
        self._chk(dy, h)
        G, B, H, W, Cc = h.shape
        assert tuple(dy.shape) == (G, B, 1, 1, Cc)
        dh = self.empty(G, B, H, W, Cc)
        self._timed_raw('hbm:global_avgpool_bwd G%d B%d %dx%d C%d' % (G, B, H, W, Cc), 4.0 * (2 if relu_gate else 1) * h.numel(),
                        lambda: self._ck(self.lib.cg_global_avgpool_bwd(_p(dy), _p(h), _p(dh), G * B, H * W, Cc, int(bool(relu_gate)),
                                                                        self._stream()), 'cg_global_avgpool_bwd'))
        return dh

    def add_(self, dst, src):
        """dst += src elementwise (contiguous tensors of the same size), one launch"""
        self._chk(dst, src)
        assert dst.numel() == src.numel()
        self._ck(self.lib.cg_acc_slice(_p(dst), _p(src), dst.numel(), 1, 1, 1, self._stream()), 'cg_acc_slice')

    def acc_slice(self, dst, src, nch):
        self._chk(dst, src)
        npix = dst.numel() // dst.shape[-1]
        assert npix == src.numel() // src.shape[-1]
        self._ck(self.lib.cg_acc_slice(_p(dst), _p(src), npix, dst.shape[-1], src.shape[-1], nch, self._stream()),
                 'cg_acc_slice')

    def gather_images(self, pools, idx, x_in, G, Bt):
        """pools: one or two tensors [S_k,H,W,4] (slot k < S_0 reads pools[0], else pools[1] -- no torch.cat); idx int32
        [G,Bt] slot table on the device; x_in [1,B,H,W,4] or None -> [G,Bt,H,W,4|8]"""
        if torch.is_tensor(pools):
            pools = (pools,)
        self._chk(x_in, *pools)
        assert idx.dtype == torch.int32 and idx.is_cuda and idx.is_contiguous() and idx.numel() == G * Bt
        S0, H, W, _ = pools[0].shape
        p1 = pools[1] if len(pools) > 1 else None
        B = x_in.shape[1] if x_in is not None else 1
        y = self.empty(G, Bt, H, W, 8 if x_in is not None else 4)
        self._ck(self.lib.cg_gather_images(_p(pools[0]), S0, _p(p1), idx.data_ptr(), _p(x_in), _p(y), G, Bt, B, H * W,
                                           self._stream()), 'cg_gather_images')
        return y

    def gather_images_gray(self, pools, idx, G, Bt):
        """gather_images without x_in, each slot converted to gray scale (do_Dis_only_gray): {m, m, m, 0}, m = (x0 + x1 + x2) / 3
        -> [G,Bt,H,W,4]"""
        if torch.is_tensor(pools):
            pools = (pools,)
        self._chk(*pools)
        assert idx.dtype == torch.int32 and idx.is_cuda and idx.is_contiguous() and idx.numel() == G * Bt
        S0, H, W, _ = pools[0].shape
        p1 = pools[1] if len(pools) > 1 else None
        y = self.empty(G, Bt, H, W, 4)
        self._timed_raw('hbm:gather_images_gray G%d Bt%d %dx%d' % (G, Bt, H, W), 4.0 * 2 * y.numel(),
                        lambda: self._ck(self.lib.cg_gather_images_gray(_p(pools[0]), S0, _p(p1), idx.data_ptr(), None, _p(y), G, Bt, 1,
                                                                        H * W, self._stream()), 'cg_gather_images_gray'))
        return y

    def gray_fold(self, d_x):
        """in place on a data gradient [..., 4] w.r.t. a gray_images input: lanes 0..2 = g0/3 + g1/3 + g2/3, lane 3 kept"""
        self._chk(d_x)
        assert d_x.shape[-1] == 4
        self._timed_raw('hbm:gray_fold n%d' % d_x.numel(), 4.0 * 2 * d_x.numel(),
                        lambda: self._ck(self.lib.cg_gray_fold(_p(d_x), d_x.numel() // 4, self._stream()), 'cg_gray_fold'))

    def gather_members(self, src, dst, segments, member_map):
        """dst[g] = src[member_map[g]] in every member-major segment (offset, floats per member) of two flat buffers laid out
        alike (the data of two ParamBanks with one table).  member_map: G python ints.  ONE launch."""
        self._chk(src, dst)
        G = len(member_map)
        assert src.numel() == dst.numel() and len(segments) >= 1
        nseg = len(segments)
        off = (C.c_int64 * nseg)(*[o for o, _ in segments])
        n = (C.c_int64 * nseg)(*[k for _, k in segments])
        self._timed_raw('hbm:gather_members G%d n%d' % (G, src.numel()), 4.0 * 2 * G * sum(k for _, k in segments),
                        lambda: self._ck(self.lib.cg_gather_members(_p(src), _p(dst), off, n, nseg, (C.c_int32 * G)(*member_map), G,
                                                                    self._stream()), 'cg_gather_members'))

    # -- host -> device staging -------------------------------------------------------------------
    def stage(self, arrays):
        """arrays: list of CPU tensors (float32 / int32).  Packs them into one pinned buffer, issues ONE asynchronous H2D
        copy on the current stream and returns device views with the same shapes / dtypes."""
        sizes = [(a.numel() * 4 + 15) // 16 * 16 for a in arrays]
        total = max(16, sum(sizes))
        k = self._stage_next
        self._stage_next = (k + 1) % len(self._stage_ring)
        slot = self._stage_ring[k]
        if slot is None or slot[0].numel() < total:
            cap = max(total, 1 << 16)
            slot = [torch.empty(cap, dtype=torch.uint8).pin_memory(), torch.empty(cap, dtype=torch.uint8, device=self.device), None]
            self._stage_ring[k] = slot
        host, dev, ev = slot
        if ev is not None:
            ev.synchronize()  # the copy that last used this pinned buffer (8 updates ago) has long finished
        off, views = 0, []
        for a, sz in zip(arrays, sizes):
            assert a.dtype in (torch.float32, torch.int32) and not a.is_cuda, a.dtype
            n = a.numel() * 4
            host[off:off + n].view(a.dtype).copy_(a.reshape(-1))
            views.append(dev[off:off + n].view(a.dtype).view(a.shape))
            off += sz
        dev[:off].copy_(host[:off], non_blocking=True)
        slot[2] = torch.cuda.Event()
        slot[2].record()
        return views

    def nchw_to_nhwc(self, x, Cp):
        self._chk(x)
        N, Cc, H, W = x.shape
        y = self.empty(N, H, W, Cp)
        self._ck(self.lib.cg_nchw_to_nhwc(_p(x), _p(y), N, Cc, H * W, Cp, self._stream()), 'cg_nchw_to_nhwc')
        return y

    def nhwc_to_nchw(self, x, Cc):
        self._chk(x)
        *lead, H, W, Cp = x.shape
        N = 1
        for d in lead:
            N *= d
        y = self.empty(*lead, Cc, H, W)
        self._ck(self.lib.cg_nhwc_to_nchw(_p(x), _p(y), N, Cc, H * W, Cp, self._stream()), 'cg_nhwc_to_nchw')
        return y

    # -- losses -----------------------------------------------------------------------------------
    def lsgan_fwd(self, out, targets, weights, nseg, loss, accumulate):
        """out [G, nseg*B, h, w, 1]; targets device [nseg], weights device [G, nseg]; returns sums [G,nseg] and updates
        loss[G] (+)= sum_seg weights[seg] * mean_seg((out - target[seg])^2)."""
        self._chk(out, targets, weights, loss)
        G = out.shape[0]
        assert weights.numel() == G * nseg
        n_per_seg = out[0].numel() // nseg
        sums = self.empty(G, nseg)
        self._ck(self.lib.cg_lsgan_fwd(_p(out), _p(targets), _p(weights), _p(sums), _p(loss), G, nseg, n_per_seg,
                                       int(bool(accumulate)), self._stream()), 'cg_lsgan_fwd')
        return sums

    def lsgan_bwd(self, out, targets, coef, nseg):
        self._chk(out, targets, coef)
        G = out.shape[0]
        n_per_seg = out[0].numel() // nseg
        dout = torch.empty_like(out)
        self._ck(self.lib.cg_lsgan_bwd(_p(out), _p(targets), _p(coef), _p(dout), G, nseg, n_per_seg, self._stream()),
                 'cg_lsgan_bwd')
        return dout

    def focus_fwd(self, mask, center, eps):
        self._chk(mask)
        G, B, H, W, _ = mask.shape
        sums = self.empty(G, 4)
        ws = self._ws_for(((B * H * W + 2047) // 2048) * G * 16)
        self._ck(self.lib.cg_focus_fwd(_p(mask), _p(sums), G, B, H, W, center, eps, _p(ws), ws.numel(), self._stream()),
                 'cg_focus_fwd')
        return sums

    def focus_bwd(self, mask, coef, center, eps):
        self._chk(mask, coef)
        G, B, H, W, _ = mask.shape
        dmask = torch.empty_like(mask)
        self._ck(self.lib.cg_focus_bwd(_p(mask), _p(coef), _p(dmask), G, B, H, W, center, eps, self._stream()),
                 'cg_focus_bwd')
        return dmask

    # -- fused losses (the training path uses these; the four calls above remain for the per-kernel tests) --------
    def _loss_scratch(self, G, B=0, H=0, W=0):
        need = int(self.lib.cg_loss_workspace_bytes(G, B, H, W))
        if need > self._loss_ws.numel():
            self._loss_ws = self._zero_bytes(need + 4096)
        return self._loss_ws

    def lsgan_fused(self, outs, nseg, targets, weights, loss_scale, grad_scale, loss_total, accumulate, loss_plain=None,
                    want_grad=True):
        """outs: patch maps [G, nseg*B, h, w, 1] of every scale; targets [nseg], weights [G][nseg] python floats.
        loss_total[g] (+)= loss_scale * sum_maps sum_seg weights[g][seg] * mean_seg((out - target[seg])^2); returns the
        gradients d(out) = grad_scale * weights[g][seg] * 2/n_seg * (out - target[seg]), one per map.  ONE launch."""
        self._chk(loss_total, loss_plain, *outs)
        G = outs[0].shape[0]
        d = LsganDesc()
        d.nmaps, d.G, d.nseg = len(outs), G, nseg
        douts = [torch.empty_like(o) for o in outs] if want_grad else [None] * len(outs)
        for m, o in enumerate(outs):
            d.out[m], d.dout[m], d.n_per_seg[m] = _p(o), _p(douts[m]), o[0].numel() // nseg
        for k in range(nseg):
            d.target[k] = targets[k]
        for g in range(G):
            for k in range(nseg):
                d.weight[g][k] = weights[g][k]
        d.loss_scale, d.grad_scale = loss_scale, grad_scale
        ws = self._loss_scratch(G)
        self._ck(self.lib.cg_lsgan_fused(C.byref(d), _p(loss_total), int(bool(accumulate)), _p(loss_plain), _p(ws), ws.numel(),
                                         self._stream()), 'cg_lsgan_fused')
        return douts

    def _gen_desc(self, adv_outs, cl_outs, mask, center, eps, adv_grad_scale, adv_douts=None, cl_douts=None):
        d = GenLossDesc()
        if mask is not None:
            d.G, d.B, d.H, d.W, _ = mask.shape
        elif adv_outs or cl_outs:
            d.G = (adv_outs + cl_outs)[0].shape[0]
        d.n_adv, d.n_cl = len(adv_outs), len(cl_outs)
        for m, o in enumerate(adv_outs):
            d.adv_out[m], d.adv_n[m] = _p(o), o[0].numel()
            d.adv_dout[m] = _p(adv_douts[m]) if adv_douts else None
        for m, o in enumerate(cl_outs):
            d.cl_out[m], d.cl_n[m] = _p(o), o[0].numel()
            d.cl_dout[m] = _p(cl_douts[m]) if cl_douts else None
        d.mask = _p(mask)
        d.center, d.eps, d.adv_grad_scale = center, eps, adv_grad_scale
        return d

    def gen_loss_fwd(self, adv_outs, cl_outs, mask, center, eps, adv_grad_scale, scal):
        """Pass 1 of the generator loss: scal[G,6] = {adv, council, focus sums x4} of this rank in ONE launch; returns the
        gradients of the adversarial patch maps (their coefficient gan_w * 2 / (n * world) does not depend on loss values)."""
        self._chk(scal, mask, *adv_outs, *cl_outs)
        adv_douts = [torch.empty_like(o) for o in adv_outs]
        d = self._gen_desc(adv_outs, cl_outs, mask, center, eps, adv_grad_scale, adv_douts)
        d.G = scal.shape[0]
        ws = self._loss_scratch(d.G, d.B, d.H, d.W)
        self._ck(self.lib.cg_gen_loss_fwd(C.byref(d), _p(scal), _p(ws), ws.numel(), self._stream()), 'cg_gen_loss_fwd')
        return adv_douts

    def gen_loss_bwd(self, cl_outs, mask, center, eps, scal, hp, hist_gan, hist_council, total, accumulate, pub, want_dmask, *,
                     hist_focus=None, hist_focus01=None, focus_src=None, focus_w=None):
        """Pass 2: loss assembly, history matching and publication on the device + council-map / mask gradients, ONE launch.
        hp: dict with the cg_gen_loss_hp scalar fields.  Returns (cl_douts, d_mask or None).
        Focus matching (hp['focus_matching'], heads hp['head_focus'] / hp['head_focus01']): hist_focus / hist_focus01 are the float64
        rings [G, hist+1] of the mask-total and zero-one terms; focus_src the a2b call's pub [G, 8] when this is the b2a call;
        focus_w (optional, [G, 2]) receives the two ratios of every member."""
        self._chk(scal, mask, total, pub, focus_src, focus_w, *cl_outs)
        assert hist_gan.dtype == torch.float64 and hist_council.dtype == torch.float64
        for r in (hist_focus, hist_focus01):
            assert r is None or (r.dtype == torch.float64 and r.is_contiguous() and tuple(r.shape) == tuple(hist_gan.shape))
        cl_douts = [torch.empty_like(o) for o in cl_outs]
        d = self._gen_desc([], cl_outs, mask, center, eps, 0.0, None, cl_douts)
        d.G = total.shape[0]
        assert focus_src is None or focus_src.numel() == d.G * 8
        assert focus_w is None or focus_w.numel() == d.G * 2
        h = GenLossHp()
        for k, v in hp.items():
            setattr(h, k, v)
        h.hist_focus, h.hist_focus01, h.focus_src, h.focus_w = _p(hist_focus), _p(hist_focus01), _p(focus_src), _p(focus_w)
        d_mask = torch.empty_like(mask) if want_dmask else None
        ws = self._loss_scratch(d.G, d.B, d.H, d.W)
        self._ck(self.lib.cg_gen_loss_bwd(C.byref(d), C.byref(h), _p(scal), hist_gan.data_ptr(), hist_council.data_ptr(), _p(total),
                                          int(bool(accumulate)), _p(pub), _p(d_mask), _p(ws), ws.numel(), self._stream()),
                 'cg_gen_loss_bwd')
        return cl_douts, d_mask

    def abs_beginning_end_fwd(self, x_fake, x, sums):
        """Pass 1 of abs_beginning_end: sums[G,2] = {sum |x_fake - x|, sum (x_fake - x)^2} over the 3 live lanes of this rank.
        x_fake [G,B,H,W,4], x [1,B,H,W,4] (shared).  ONE launch."""
        self._chk(x_fake, x, sums)
        G, B, H, W, _ = x_fake.shape
        assert tuple(x.shape) == (1, B, H, W, 4) and sums.numel() == 2 * G
        ws = self._loss_scratch(G, B, H, W)
        self._ck(self.lib.cg_abs_beginning_end_fwd(_p(x_fake), _p(x), _p(sums), G, B, H, W, _p(ws), ws.numel(), self._stream()),
                 'cg_abs_beginning_end_fwd')

    def abs_beginning_end_bwd(self, x_fake, x, sums, numel, weights, total, pub, d_x):
        """Pass 2: picks L1 or L2 per member from the (globally summed) sums, pub[g] = the unweighted loss, total[g] += weights[g] *
        loss, d_x += its gradient.  weights: python floats, 0 = no contribution.  Must follow gen_loss_bwd of the same direction
        (the direction totals share its double accumulator).  ONE launch."""
        self._chk(x_fake, x, sums, total, pub, d_x)
        G, B, H, W, _ = x_fake.shape
        assert tuple(d_x.shape) == tuple(x_fake.shape) and len(weights) == G
        w = (C.c_double * G)(*weights)
        ws = self._loss_scratch(G)  # never grows the scratch: a new buffer would drop the accumulator gen_loss_bwd left in it
        self._ck(self.lib.cg_abs_beginning_end_bwd(_p(x_fake), _p(x), _p(sums), float(numel), w, _p(total), _p(pub), _p(d_x), G, B, H, W,
                                                   _p(ws), ws.numel(), self._stream()), 'cg_abs_beginning_end_bwd')

    def council_abs_fwd(self, x_fake, peers, gray, sums):
        """Pass 1 of council_abs_w: sums[g] = sum |x_fake[g] - x_fake[peers[g]]| over the 3 live lanes (gray: of the channel sums) on
        this rank.  x_fake [G,B,H,W,4]; peers: G python ints, each another member.  ONE launch."""
        self._chk(x_fake, sums)
        G, B, H, W, _ = x_fake.shape
        assert len(peers) == G and sums.numel() == G
        ws = self._loss_scratch(G, B, H, W)
        self._timed_raw('hbm:council_abs_fwd G%d B%d %dx%d' % (G, B, H, W), 4.0 * 2 * x_fake.numel(),
                        lambda: self._ck(self.lib.cg_council_abs_fwd(_p(x_fake), (C.c_int32 * G)(*peers), int(bool(gray)), _p(sums), G, B, H,
                                                                     W, _p(ws), ws.numel(), self._stream()), 'cg_council_abs_fwd'))

    def council_abs_bwd(self, x_fake, peers, gray, sums, numel, w, total, pub, d_x):
        """Pass 2: pub[g] = w * sums[g] / numel (the weighted term), total[g] += pub[g], d_x[g] += w / numel * sign(d) on the 3 live
        lanes; the peers take no gradient.  numel: of the GLOBAL minibatch.  Must follow gen_loss_bwd of the same direction (the
        direction totals share its double accumulator).  ONE launch."""
        self._chk(x_fake, sums, total, pub, d_x)
        G, B, H, W, _ = x_fake.shape
        assert tuple(d_x.shape) == tuple(x_fake.shape) and len(peers) == G
        ws = self._loss_scratch(G)  # never grows the scratch: a new buffer would drop the accumulator gen_loss_bwd left in it
        self._timed_raw('hbm:council_abs_bwd G%d B%d %dx%d' % (G, B, H, W), 4.0 * 4 * x_fake.numel(),
                        lambda: self._ck(self.lib.cg_council_abs_bwd(_p(x_fake), (C.c_int32 * G)(*peers), int(bool(gray)), _p(sums),
                                                                     float(numel), float(w), _p(total), _p(pub), _p(d_x), G, B, H, W,
                                                                     _p(ws), ws.numel(), self._stream()), 'cg_council_abs_bwd'))

    def add_column(self, dst, k, src):
        """dst[:, k] += src for dst [n, C] and src [n] (contiguous), one launch"""
        self._chk(dst, src)
        n, Cd = dst.shape
        assert src.numel() == n and 0 <= k < Cd
        self._ck(self.lib.cg_acc_slice(dst.data_ptr() + 4 * k, _p(src), n, Cd, 1, 1, self._stream()), 'cg_acc_slice')

    def latent_l1(self, a, b, sums, coef, da=None, db=None, accumulate=False):
        """recon_criterion(a, b) = mean |a - b| per member (recon_c / recon_s): sums[g] = sum |a - b| of member g on this rank; in the
        same launch da (+)= coef * sign(a - b) and db (+)= -coef * sign(a - b) (None: not wanted).  a [G, ...]; b [G, ...] of the same
        shape, or [1, ...] shared by all members (then db must be None)."""
        self._chk(a, b, sums, da, db)
        G = a.shape[0]
        n = a.numel() // G
        shared = b.shape[0] == 1 and G > 1
        assert b.numel() == (n if shared else a.numel()) and sums.numel() == G
        for t in (da, db):
            assert t is None or t.numel() == a.numel()
        ws = self._loss_scratch(G)
        self._timed_raw('hbm:latent_l1 G%d n%d' % (G, n), 4.0 * a.numel() * (2 + (da is not None) + (db is not None)),
                        lambda: self._ck(self.lib.cg_latent_l1(_p(a), _p(b), int(shared), _p(da), _p(db), float(coef), int(bool(accumulate)),
                                                               _p(sums), G, n, _p(ws), ws.numel(), self._stream()), 'cg_latent_l1'))

    def recon_finalize(self, sums, numel, weights, total, pub):
        """After the all-reduce: pub[k, g] = sums[k, g] / numel[k]; total[g] += sum_k weights[k] * pub[k, g] through gen_loss_bwd's
        double accumulator (so it follows every gen_loss_bwd call of the update).  sums, pub [K, G]; numel, weights: K python floats."""
        self._chk(sums, total, pub)
        K, G = sums.shape
        assert len(numel) == len(weights) == K and tuple(pub.shape) == (K, G)
        ws = self._loss_scratch(G)  # never grows the scratch: a new buffer would drop the accumulator gen_loss_bwd left in it
        self._ck(self.lib.cg_recon_finalize(_p(sums), (C.c_double * K)(*numel), (C.c_double * K)(*weights), K, G, _p(total), _p(pub),
                                            _p(ws), ws.numel(), self._stream()), 'cg_recon_finalize')

    def recon_head_fwd(self, h, x_in, sums):
        """recon_x pass 1: sums[g] = sum |x_recon - x_in| over the 3 live lanes of member g on this rank, x_recon the mask_head_fwd
        composite of h [G,B,H,W,12] (tanh output of the last head layer) over x_in [1,B,H,W,4].  x_recon is never written.  ONE launch."""
        self._chk(h, x_in, sums)
        G, B, H, W, _ = h.shape
        assert tuple(x_in.shape) == (1, B, H, W, 4) and sums.numel() == G
        ws = self._loss_scratch(G, B, H, W)
        self._timed_raw('hbm:recon_head_fwd G%d B%d %dx%d' % (G, B, H, W), 4.0 * (h.numel() + x_in.numel()),
                        lambda: self._ck(self.lib.cg_recon_head_fwd(_p(h), _p(x_in), _p(sums), G, B, H * W, _p(ws), ws.numel(),
                                                                    self._stream()), 'cg_recon_head_fwd'))

    def recon_head_bwd(self, h, x_in, coef):
        """recon_x backward: the gradient w.r.t. the pre-tanh head output [G,B,H,W,12] for d(x_recon) = coef * sign(x_recon - x_in)
        (sign(0) = 0) and no mask gradient, the composite recomputed.  ONE launch."""
        self._chk(h, x_in)
        G, B, H, W, _ = h.shape
        assert tuple(x_in.shape) == (1, B, H, W, 4)
        dh = self.empty(G, B, H, W, 12)
        self._timed_raw('hbm:recon_head_bwd G%d B%d %dx%d' % (G, B, H, W), 4.0 * (2 * h.numel() + x_in.numel()),
                        lambda: self._ck(self.lib.cg_recon_head_bwd(_p(h), _p(x_in), float(coef), _p(dh), G, B, H * W, self._stream()),
                                         'cg_recon_head_bwd'))
        return dh

    # -- perceptual loss (vgg_w): the frozen VGG-16's preprocessing, max-pools and loss ------------------------------------------------
    def vgg_preprocess(self, x, out=None):
        """vgg_preprocess (utils.py:380-390) of channels-last images [..., 4]: {B', G', R', 0}, c' = (x_c + 1) * 255 * 0.5 - mean_c.
        out: a tensor of the same size to write into (default: a new one).  ONE launch."""
        self._chk(x, out)
        assert x.shape[-1] == 4
        y = self.empty(*x.shape) if out is None else out
        assert y.numel() == x.numel()
        self._timed_raw('hbm:vgg_preprocess n%d' % x.numel(), 4.0 * 2 * x.numel(),
                        lambda: self._ck(self.lib.cg_vgg_preprocess(_p(x), _p(y), x.numel() // 4, self._stream()), 'cg_vgg_preprocess'))
        return y

    def vgg_preprocess_bwd(self, dy, d_x, accumulate):
        """d_x[..., c] (+)= 127.5 * dy[..., 2 - c] for c < 3 (lane 3: written 0, or kept when accumulating).  ONE launch."""
        self._chk(dy, d_x)
        assert dy.numel() == d_x.numel() and d_x.shape[-1] == 4
        self._timed_raw('hbm:vgg_preprocess_bwd n%d' % dy.numel(), 4.0 * (3 if accumulate else 2) * dy.numel(),
                        lambda: self._ck(self.lib.cg_vgg_preprocess_bwd(_p(dy), _p(d_x), dy.numel() // 4, int(bool(accumulate)),
                                                                        self._stream()), 'cg_vgg_preprocess_bwd'))

    def maxpool2x2_fwd(self, x):
        """F.max_pool2d(x, 2, 2) of [G,B,H,W,C] (floor size) -> [G,B,H/2,W/2,C].  ONE launch."""
        self._chk(x)
        G, B, H, W, Cc = x.shape
        y = self.empty(G, B, H // 2, W // 2, Cc)
        self._timed_raw('hbm:maxpool2x2_fwd B%d %dx%d C%d' % (G * B, H, W, Cc), 4.0 * (x.numel() + y.numel()),
                        lambda: self._ck(self.lib.cg_maxpool2x2_fwd(_p(x), _p(y), G * B, H, W, Cc, self._stream()), 'cg_maxpool2x2_fwd'))
        return y

    def maxpool2x2_bwd(self, dy, x):
        """The gradient w.r.t. the pre-activation of x = relu(pre) [G,B,H,W,C] through max_pool2d(x, 2, 2), from dy [G,B,H/2,W/2,C]:
        each window's first maximum takes dy where x > 0, every other position 0.  No index tensor.  ONE launch."""
        self._chk(dy, x)
        G, B, H, W, Cc = x.shape
        assert tuple(dy.shape) == (G, B, H // 2, W // 2, Cc)
        dx = self.empty(G, B, H, W, Cc)
        self._timed_raw('hbm:maxpool2x2_bwd B%d %dx%d C%d' % (G * B, H, W, Cc), 4.0 * (2 * x.numel() + dy.numel()),
                        lambda: self._ck(self.lib.cg_maxpool2x2_bwd(_p(dy), _p(x), _p(dx), G * B, H, W, Cc, self._stream()),
                                         'cg_maxpool2x2_bwd'))
        return dx

    def vgg_loss(self, f_img, f_tgt, B, per_dir, coef, sums):
        """compute_vgg_loss (trainer_council.py:636-641) of stacked relu5_3 rows f_img [1,R,h,w,C] against f_tgt [1,T,h,w,C], image row r
        paired with target row (r // per_dir) * B + r % B: sums[k] = sum (IN(f_img) - IN(f_tgt))^2 over rows [k B, k B + B) on this rank
        (R // B values); returns d(pre-activation of conv5_3) [1,R,h,w,C] of coef * that sum (the targets take no gradient).  The
        statistics come from in_stats; the loss and its gradient are ONE more launch."""
        self._chk(f_img, f_tgt, sums)
        _, R, h, w, Cc = f_img.shape
        assert f_tgt.shape[0] == 1 and tuple(f_tgt.shape[2:]) == (h, w, Cc) and sums.numel() == R // B
        mi, ri = self.in_stats(f_img)
        mt, rt = self.in_stats(f_tgt)
        d_pre = self.empty(*f_img.shape)
        need = 16 + 8 * LOSS_MAX_G + 4 * R * (Cc // 32)
        if need > self._loss_ws.numel():
            self._loss_ws = self._zero_bytes(need + 4096)
        ws = self._loss_ws
        self._timed_raw('hbm:vgg_loss R%d %dx%d C%d' % (R, h, w, Cc), 4.0 * (5 * f_img.numel()),
                        lambda: self._ck(self.lib.cg_vgg_loss(_p(f_img), _p(mi), _p(ri), _p(f_tgt), _p(mt), _p(rt), R, B, per_dir, h * w, Cc,
                                                              float(coef), _p(sums), _p(d_pre), _p(ws), ws.numel(), self._stream()),
                                         'cg_vgg_loss'))
        return d_pre

    # -- reflection padding (pad_type: reflect) --------------------------------------------------------------------------------------
    def reflect_pad(self, x, p, ups=False):
        """nn.ReflectionPad2d(p) of x [G,B,H,W,C] (after a nearest x2 upsample with ups) -> [G,B,Hs+2p,Ws+2p,C], the input of a
        pad-0 convolution.  Raises when p is not smaller than the (upsampled) map.  ONE launch."""
        self._chk(x)
        G, B, H, W, Cc = x.shape
        Hs, Ws = (2 * H, 2 * W) if ups else (H, W)
        xp = self.empty(G, B, Hs + 2 * p, Ws + 2 * p, Cc)
        self._timed_raw('hbm:reflect_pad G%d B%d %dx%d C%d p%d%s' % (G, B, H, W, Cc, p, ' ups' if ups else ''), 4.0 * (x.numel() + xp.numel()),
                        lambda: self._ck(self.lib.cg_reflect_pad(_p(x), _p(xp), G * B, H, W, Cc, p, int(bool(ups)), self._stream()),
                                         'cg_reflect_pad'))
        return xp

    def reflect_pad_bwd(self, dxp, p, addend=None, mask_src=None, mask_slope=0.0):
        """The data gradient through reflect_pad (no upsample): dxp [G,B,H+2p,W+2p,C] -> (fold + addend) * act'(mask_src)
        [G,B,H,W,C], addend / mask_src as in conv_dgrad.  ONE launch."""
        self._chk(dxp, addend, mask_src)
        G, B, Hp, Wp, Cc = dxp.shape
        H, W = Hp - 2 * p, Wp - 2 * p
        dx = self.empty(G, B, H, W, Cc)
        for t in (addend, mask_src):
            assert t is None or tuple(t.shape) == tuple(dx.shape), (tuple(t.shape), tuple(dx.shape))
        units = (dxp.numel() + dx.numel() * (1 + (addend is not None) + (mask_src is not None))) / dx.numel()
        self._timed_raw('hbm:reflect_pad_bwd G%d B%d %dx%d C%d p%d' % (G, B, H, W, Cc, p), 4.0 * units * dx.numel(),
                        lambda: self._ck(self.lib.cg_reflect_pad_bwd(_p(dxp), _p(dx), _p(addend), _p(mask_src), mask_slope, G * B, H, W, Cc,
                                                                     p, self._stream()), 'cg_reflect_pad_bwd'))
        return dx

    # -- input pipeline (council_gan_b200/data.py) ------------------------------------------------------
    def aug_color(self, pix, desc, opcode, param, B, max_pixels, any_contrast):
        """one colour phase of the transform stack, in place on the packed uint8 batch (csrc/augment.cu)"""
        lsum = torch.empty(B, dtype=torch.int64, device=self.device)
        self._ck(self.lib.cg_aug_color(pix.data_ptr(), desc.data_ptr(), opcode.data_ptr(), param.data_ptr(), lsum.data_ptr(), B,
                                       int(max_pixels), int(bool(any_contrast)), self._stream()), 'cg_aug_color')

    def aug_resize_crop(self, pix, src_off, flip, slot, crop, n, H, W, oh, ow, ch, cw, bh, kh, ksh, bv, kv, ksv, out, nchw):
        """flip + Pillow bilinear resize + crop + ToTensor + Normalize of n same-sized images into their batch slots"""
        tmp = torch.empty(n * H * ow * 3, dtype=torch.uint8, device=self.device)
        self._ck(self.lib.cg_aug_resize_crop(pix.data_ptr(), src_off.data_ptr(), flip.data_ptr(), slot.data_ptr(), crop.data_ptr(), n, H, W,
                                             oh, ow, ch, cw, bh.data_ptr(), kh.data_ptr(), ksh, bv.data_ptr(), kv.data_ptr(), ksv,
                                             tmp.data_ptr(), _p(out), _p(nchw), self._stream()), 'cg_aug_resize_crop')

    # -- optimiser --------------------------------------------------------------------------------
    def adam_step(self, p, g, m, v, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0):
        self._chk(p, g, m, v)
        self._ck(self.lib.cg_adam_step(_p(p), _p(g), _p(m), _p(v), p.numel(), lr, beta1, beta2, eps, weight_decay,
                                       step, grad_scale, self._stream()), 'cg_adam_step')
