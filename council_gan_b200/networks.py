"""Council-stacked networks: AdaIN generator, multi-scale PatchGAN discriminator, council discriminator.

GPU-first restructuring of the reference's ``networks.py``: instead of N independent ``nn.Module``
copies executed one after the other (trainer_council.py:101-119, loops at :328,558,747,826,858), the N
council members of one family live in ONE flat fp32 parameter buffer (stacked ``[N, ...]`` per layer) and
every layer is ONE grouped kernel launch over all members.  Forward *and* backward are written out
explicitly (no autograd): each step below is a call into libcouncil_b200.so through ``ops``.

Layer-by-layer correspondence with the reference (paths relative to /root/reference):
  ContentEncoder       networks.py:355-369      -> CouncilGen.encode
  MLP                  networks.py:432-443      -> CouncilGen._mlp
  Decoder_V2_atten     networks.py:374-415      -> CouncilGen.decode
  assign_adain_params  networks.py:303-312      -> column offsets into the MLP output (no copies)
  MsImageDis           networks.py:17-54        -> CouncilDis(council=False)
  MsImageDisCouncil    networks.py:116-156      -> CouncilDis(council=True)
Per-member ``state_dict`` views keep the reference's key names and OIHW shapes (see MemberView).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch

from .ops import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH

IMG_C = 4  # image tensors carry 3 live lanes + 1 zero lane (16-byte pixels)


def _pad_type(pad_type):
    """True for reflect: the pad_type of a network's Conv2dBlocks (networks.py:470-474), 'zero' or 'reflect' on the accelerated path"""
    assert pad_type in ('zero', 'reflect')
    return pad_type == 'reflect'


def _padded(ops, x, s, reflect, ups=False):
    """-> (the input a layer's convolution reads, the pad it applies): under reflect a layer with pad > 0 reads
    nn.ReflectionPad2d(pad) of x (of x nearest-upsampled x2 with ups) with pad 0, since the convolutions pad with zeros only"""
    if reflect and s.pad > 0:
        return ops.reflect_pad(x, s.pad, ups), 0
    return x, s.pad


# ------------------------------------------------------------------------------------------------------
# parameter storage
# ------------------------------------------------------------------------------------------------------
class ParamBank:
    """One flat fp32 buffer (+ grad, Adam moments) holding every parameter of a family for all members.

    ``entries``: list of (name, per-member kernel-layout shape).  Each entry is stored ``[G, *shape]``,
    its offset rounded up to 64 floats (256 B) so any slice is a valid TMA / float4 base address.
    The flat ``grad`` buffer is what data parallelism all-reduces; ``data/grad/exp_avg/exp_avg_sq`` are
    what the fused Adam kernel walks.
    """

    def __init__(self, ops, G, entries, trainable=True):
        self.ops, self.G = ops, G
        self._views = {}
        self.table = OrderedDict()
        off = 0
        for name, shape in entries:
            n = G * int(math.prod(shape))
            self.table[name] = (off, tuple(shape), n)
            off += (n + 63) // 64 * 64
        self.total = off
        self.data = ops.zeros(off)
        self.trainable = trainable
        if trainable:
            self.grad = ops.zeros(off)
            self.exp_avg = ops.zeros(off)
            self.exp_avg_sq = ops.zeros(off)
        self.step = 0

    def _view(self, buf, name, base=0):
        """view of `name` in buf, a flat buffer laid out like grad[base:]"""
        # views are cached per (buffer object, name): ~430 lookups per step, each a slice + view (8 % of the host time of a step on the
        # launch-bound small configuration)
        hit = self._views.get((id(buf), name))
        if hit is not None and hit[0] is buf:
            return hit[1]
        off, shape, n = self.table[name]
        v = buf[off - base:off - base + n].view((self.G,) + shape)
        self._views[(id(buf), name)] = (buf, v)
        return v

    def p(self, name):
        return self._view(self.data, name)

    def member_segments(self):
        """[(offset, floats per member)] of every entry: the member-major segments of ops.gather_members"""
        return [(off, n // self.G) for off, _, n in self.table.values()]

    def g(self, name):
        return self._view(self.grad, name)


class LayerSpec:
    """A convolution (or linear, as 1x1 on a 1x1 map) with its reference key and lane mapping."""

    def __init__(self, key, cout, cin, k, stride, pad, lanes=None, linear=False):
        self.key, self.cout, self.cin, self.k, self.stride, self.pad = key, cout, cin, k, stride, pad
        self.lanes = lanes  # kernel lane index of each reference input channel (None: identity)
        self.cin_p = cin if lanes is None else (max(lanes) // 4 + 1) * 4
        self.linear = linear
        self.wname = key + '.weight'
        self.bname = key + '.bias'
        self.vecs = []  # names of per-channel [cout] parameters stored before the weight (a layer norm's gamma / beta)

    def entries(self):
        return [(n, (self.cout,)) for n in self.vecs] + [(self.wname, (self.cout, self.k, self.k, self.cin_p)), (self.bname, (self.cout,))]

    # reference <-> kernel layout
    def export_weight(self, w):  # w: [Cout,KH,KW,Cin_p] one member
        if self.lanes is not None:
            w = w[..., self.lanes]
        w = w.permute(0, 3, 1, 2)
        return (w.reshape(self.cout, self.cin) if self.linear else w).contiguous().clone()

    def import_weight(self, dst, ref):  # dst: [Cout,KH,KW,Cin_p] view; ref: reference tensor
        """OIHW -> the kernel layout, assembled on the HOST and moved with one plain copy (no permute / fill kernels on the
        device: checkpoint loading stays out of the kernel launch list)."""
        ref = ref.detach().to('cpu', dst.dtype)
        if self.linear:
            ref = ref.reshape(self.cout, self.cin, 1, 1)
        ref = ref.permute(0, 2, 3, 1)
        if self.lanes is not None:
            full = torch.zeros(dst.shape, dtype=dst.dtype)
            full[..., self.lanes] = ref
            ref = full
        dst.copy_(ref.contiguous())


class MemberView:
    """Reference-shaped view of council member ``i`` of a stacked network (``gen_a2b_s[i]`` etc.).

    Provides what the reference's callers use on those objects (train.py / test_on_folder.py /
    trainer_council.py:898-992): ``state_dict`` / ``load_state_dict`` with the reference's keys and OIHW
    shapes, ``cuda_device``, ``eval`` / ``train``, and for generators ``encode`` / ``decode`` /
    ``dec.mask_s``.
    """

    def __init__(self, net, i):
        self.net, self.i = net, i
        self.cuda_device = str(net.ops.device)
        self.training = True

    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        self.training = mode
        return self

    def state_dict(self):
        return self.net.member_state_dict(self.i)

    def load_state_dict(self, sd, strict=True):
        self.net.load_member_state_dict(self.i, sd, strict)

    def parameters(self):
        return [v for k, v in self.state_dict().items() if not k.endswith(('running_mean', 'running_var'))]


class _StackedNet:
    """Shared state_dict plumbing for the three stacked network types."""

    def _specs(self):
        raise NotImplementedError

    def _banks(self):
        raise NotImplementedError

    def _bank_of(self, name):
        for b in self._banks():
            if name in b.table:
                return b
        raise KeyError(name)

    def extra_state(self):
        return OrderedDict()

    _before_access = None  # set by the trainer: joins a pending (data-parallel, deferred) optimiser step of this family

    def _sync(self):
        if self._before_access is not None:
            self._before_access()

    def member_state_dict(self, i):
        self._sync()
        sd = OrderedDict()
        for spec in self._specs():
            b = self._bank_of(spec.wname)
            sd[spec.wname] = spec.export_weight(b.p(spec.wname)[i])
            sd[spec.bname] = b.p(spec.bname)[i].clone()
            for n in spec.vecs:
                sd[n] = b.p(n)[i].clone()
        for k, v in self.extra_state().items():
            sd[k] = v.clone()
        # reference key order (state_dict of the nn.Module tree)
        order = self.reference_key_order()
        return OrderedDict((k, sd[k]) for k in order)

    def load_member_state_dict(self, i, sd, strict=True):
        self._sync()
        keys = set(self.reference_key_order())
        if strict:
            missing, unexpected = keys - set(sd), set(sd) - keys
            if missing or unexpected:
                raise RuntimeError('state_dict mismatch: missing %s unexpected %s' % (sorted(missing), sorted(unexpected)))
        for spec in self._specs():
            b = self._bank_of(spec.wname)
            if spec.wname in sd:
                spec.import_weight(b.p(spec.wname)[i], sd[spec.wname])
            if spec.bname in sd:
                b.p(spec.bname)[i].copy_(sd[spec.bname].detach().to('cpu', b.data.dtype).reshape(-1))
            for n in spec.vecs:
                if n in sd:
                    b.p(n)[i].copy_(sd[n].detach().to('cpu', b.data.dtype).reshape(-1))
        self.params_changed()

    def params_changed(self):
        self._load_epoch = getattr(self, '_load_epoch', 0) + 1

    def member(self, i):
        return MemberView(self, i)


# ------------------------------------------------------------------------------------------------------
# generator
# ------------------------------------------------------------------------------------------------------
class _DecView:
    def __init__(self):
        self.mask_s = []


class GenMemberView(MemberView):
    """``gen_a2b_s[i]``: encode/decode of a single member through the stacked kernels (G sliced to 1)."""

    def __init__(self, net, i):
        super().__init__(net, i)
        self.dec = _DecView()

    def encode(self, images):
        """AdaINGen.encode networks.py:278-283 -> (content NCHW, style_fake [B,style_dim,1,1])."""
        return self.net.member_encode(self.i, images)

    def decode(self, content, style, images, return_mask=False):
        """AdaINGen.decode networks.py:285-301; sets ``self.dec.mask_s`` like networks.py:400."""
        out, mask = self.net.member_decode(self.i, content, style, images)
        self.dec.mask_s = mask
        if return_mask:
            return out, mask
        return out


class CouncilGen(_StackedNet):
    def __init__(self, ops, hp, G, input_dim=3):
        g = hp['gen']
        assert not g['do_my_style'], 'do_my_style generators are outside the accelerated path'
        assert g['activ'] == 'relu'
        self.reflect = _pad_type(g['pad_type'])
        assert input_dim == 3 and g['num_of_mask_dim_to_add'] == 3, 'mask head kernel is specialised for RGB + 3 masks'
        self.ops, self.hp, self.G = ops, hp, G
        self.dim, self.style_dim, self.nd, self.nr, self.mlp_dim = g['dim'], g['style_dim'], g['n_downsample'], g['n_res'], g['mlp_dim']
        dim, nd, nr = self.dim, self.nd, self.nr
        img_lanes = [0, 1, 2]
        # --- content encoder (networks.py:355-366)
        self.enc = [LayerSpec('enc_content.model.0.conv', dim, input_dim, 7, 1, 3, lanes=img_lanes)]
        d = dim
        for i in range(nd):
            self.enc.append(LayerSpec('enc_content.model.%d.conv' % (1 + i), 2 * d, d, 4, 2, 1))
            d *= 2
        self.enc_res = [[LayerSpec('enc_content.model.%d.model.%d.model.%d.conv' % (1 + nd, r, j), d, d, 3, 1, 1)
                         for j in range(2)] for r in range(nr)]
        self.cdim = d
        # --- decoder (networks.py:374-396)
        self.dec_res = [[LayerSpec('dec.model.0.model.%d.model.%d.conv' % (r, j), d, d, 3, 1, 1) for j in range(2)]
                        for r in range(nr)]
        self.dec_up = []
        idx = 1
        for i in range(nd):
            idx += 1
            self.dec_up.append((LayerSpec('dec.model.%d.conv' % idx, d // 2, d, 3, 1, 1),
                                LayerSpec('dec.model.%d.conv' % (idx + 1), d // 2, d // 2, 3, 1, 1)))
            idx += 2
            d //= 2
        self.head = [LayerSpec('dec.model.%d.conv' % idx, d, d, 1, 1, 0),
                     LayerSpec('dec.model.%d.conv' % (idx + 1), d, d, 1, 1, 0),
                     LayerSpec('dec.model.%d.conv' % (idx + 2), 12, d, 1, 1, 0)]
        # AdaIN column offsets in modules() order (networks.py:303-312)
        self.adain_off = {}
        off = 0
        for blk in self.dec_res:
            for s in blk:
                self.adain_off[s.key] = off
                off += 2 * s.cout
        for a, b in self.dec_up:
            for s in (a, b):
                self.adain_off[s.key] = off
                off += 2 * s.cout
        self.n_adain = off
        # --- MLP (networks.py:432-440)
        self.mlp = [LayerSpec('mlp.model.0.fc', self.mlp_dim, self.style_dim, 1, 1, 0, linear=True),
                    LayerSpec('mlp.model.1.fc', self.mlp_dim, self.mlp_dim, 1, 1, 0, linear=True),
                    LayerSpec('mlp.model.2.fc', self.n_adain, self.mlp_dim, 1, 1, 0, linear=True)]
        # --- style encoder (networks.py:337-350): run by encode() / sample(), and in training only by the style and image
        # reconstructions (recon_s_w, recon_x_w != 0), the terms that give it a gradient; otherwise its parameters are kept for the API /
        # checkpoints
        d = dim
        self.sty = [LayerSpec('enc_style.model.0.conv', d, input_dim, 7, 1, 3, lanes=img_lanes)]
        for i in range(2):
            self.sty.append(LayerSpec('enc_style.model.%d.conv' % (1 + i), 2 * d, d, 4, 2, 1))
            d *= 2
        for i in range(2):
            self.sty.append(LayerSpec('enc_style.model.%d.conv' % (3 + i), d, d, 4, 2, 1))
        self.sty_out = LayerSpec('enc_style.model.6', self.style_dim, d, 1, 1, 0)

        live = self.enc + [s for b in self.enc_res for s in b] + [s for b in self.dec_res for s in b] + \
            [s for ab in self.dec_up for s in ab] + self.head + self.mlp
        self.live_specs = live
        self.bank = ParamBank(ops, G, [e for s in live for e in s.entries()])
        # flat-buffer offset where the content encoder's parameters end: the decoder / head / MLP gradients [enc_end:] are
        # complete before the encoder backward starts, so data parallelism all-reduces them while it runs
        self.enc_end = self.bank.table[self.dec_res[0][0].wname][0] if self.dec_res else self.bank.table[self.head[0].wname][0]
        # its own bank: gradients, Adam moments and step count only when recon_s_w or recon_x_w trains it (torch's Adam starts a
        # parameter's state at its first gradient, so this bank's step count can lag the generator's, e.g. after resuming with the
        # terms off)
        self.sty_bank = ParamBank(ops, G, [e for s in self.sty + [self.sty_out] for e in s.entries()],
                                  trainable=hp.get('recon_s_w', 0) != 0 or hp.get('recon_x_w', 0) != 0)
        # biases feeding IN / AdaIN are mathematically dead (SURVEY.md 7.3-5): their gradient is exactly 0 here
        self.dead_bias = set(s.bname for s in live if s not in self.head and s not in self.mlp)
        self._enc_grad2 = self._dec_grad2 = self._sty_grad2 = None

    @property
    def frozen(self):  # the style-encoder bank's earlier name
        return self.sty_bank

    def reencode_grad(self):
        """Zero-initialised flat buffer laid out like bank.grad[:enc_end]: the content encoder's weight gradients of its second pass
        in gen_update (the re-encode of the other direction's translation), added to bank.grad after the first pass's backward.
        The dead biases are never written, so they stay 0."""
        if self._enc_grad2 is None:
            self._enc_grad2 = self.ops.zeros(self.enc_end)
        return self._enc_grad2

    def decode_grad(self):
        """Zero-initialised flat buffer laid out like bank.grad[enc_end:]: the decoder, head and MLP weight gradients of this
        generator's second decoder pass in gen_update (recon_x: the other direction's image reconstruction), added to bank.grad after
        the first pass's decoder backward.  The dead biases are never written, so they stay 0."""
        if self._dec_grad2 is None:
            self._dec_grad2 = self.ops.zeros(self.bank.total - self.enc_end)
        return self._dec_grad2

    def style_grad(self):
        """Zero-initialised flat buffer laid out like sty_bank.grad: the style encoder's weight gradients of its second pass in
        gen_update when it runs twice (recon_s on the other direction's translation, recon_x on the source image)."""
        if self._sty_grad2 is None:
            self._sty_grad2 = self.ops.zeros(self.sty_bank.total)
        return self._sty_grad2

    def _gv(self, grad, name):
        """weight-gradient view of `name`: in bank.grad (grad None), decode_grad() or reencode_grad()"""
        if grad is None:
            return self.bank.g(name)
        return self.bank._view(grad, name, self.enc_end if grad is self._dec_grad2 else 0)

    # -- state_dict plumbing -------------------------------------------------------------------------
    def _specs(self):
        return self.sty + [self.sty_out] + self.live_specs

    def _banks(self):
        return (self.bank, self.sty_bank)

    def extra_state(self):
        out = OrderedDict()
        for blk in self.dec_res:
            for s in blk:
                p = s.key[:-5]
                out[p + '.norm.running_mean'] = torch.zeros(s.cout)
                out[p + '.norm.running_var'] = torch.ones(s.cout)
        for ab in self.dec_up:
            for s in ab:
                p = s.key[:-5]
                out[p + '.norm.running_mean'] = torch.zeros(s.cout)
                out[p + '.norm.running_var'] = torch.ones(s.cout)
        return out

    def reference_key_order(self):
        keys = []
        for s in self.sty + [self.sty_out] + self.enc + [s for b in self.enc_res for s in b]:
            keys += [s.wname, s.bname]
        for s in [s for b in self.dec_res for s in b] + [s for ab in self.dec_up for s in ab]:
            p = s.key[:-5]
            keys += [p + '.norm.running_mean', p + '.norm.running_var', s.wname, s.bname]
        for s in self.head + self.mlp:
            keys += [s.wname, s.bname]
        return keys

    def member(self, i):
        return GenMemberView(self, i)

    # -- building blocks -------------------------------------------------------------------------------
    def _w(self, s, sl=None):
        w, b = self.bank.p(s.wname), self.bank.p(s.bname)
        if sl is not None:
            w, b = w[sl:sl + 1], b[sl:sl + 1]
        return w, b

    def _conv_norm(self, x, s, sl, adain, act, res, ups_out, saved, ups_in=False):
        """conv(+bias) -> IN/AdaIN statistics -> normalise(+gamma/beta) -> activation (+residual).
        ups_out: the normalise pass writes its result nearest-upsampled x2 (nn.Upsample, networks.py:385), so
        the following convolution is a plain 3x3 on the materialised tensor (TMA im2col cannot halve indices)."""
        ops = self.ops
        w, b = self._w(s, sl)
        # the bias of a convolution that feeds IN / AdaIN is removed again by the mean subtraction: skip the add
        # ups_in (no-grad passes): the x2 nearest upsample is folded into this convolution (four 2x2 parity classes)
        off = self.adain_off.get(s.key, 0)
        # statistics in the convolution epilogue (cg_conv_fwd_stats) on the wide layers (>= 128 output channels, K >= 1024), whose main
        # loop is an order of magnitude longer than the epilogue and hides the reduction; a separate pass on the narrow
        # full-resolution layers, which are epilogue-bound
        wide = s.cout >= 128 and s.k * s.k * s.cin >= 1024
        if self.reflect and s.pad > 0:  # the upsample goes into the padding pass, whose output the weight gradient reads
            x, pad, ups_in = ops.reflect_pad(x, s.pad, ups_in), 0, False
        else:
            pad = s.pad
        if wide:
            y, mean, rstd = ops.conv_fwd_stats(x, w, s.stride, pad, ups=ups_in)
        else:
            y = ops.conv_fwd(x, w, None, s.stride, pad, ups=ups_in)
            mean, rstd = ops.in_stats(y)
        z = ops.norm_act_fwd(y, mean, rstd, adain, off, res, act, ups_out)
        if saved is not None:
            saved.append((x, y, mean, rstd))
        return z

    def _conv_norm_bwd(self, dz, s, rec, adain, d_adain, act, ups_out, addend, need_dx=True, grad=None):
        """Backward of _conv_norm: fills the weight gradient (in bank.grad, or in the flat buffer grad laid out like it), returns
        d(input).  With ups_out, dz has the upsampled shape and the 2x2 fan-in is summed while it is read."""
        ops = self.ops
        x, y, mean, rstd = rec  # x: the padded input under reflect
        off = self.adain_off.get(s.key, 0)
        dy = ops.norm_act_bwd(dz, y, mean, rstd, adain, off, act, ups_out, d_adain)
        reflect = self.reflect and s.pad > 0
        pad = 0 if reflect else s.pad
        ops.conv_wgrad(x, dy, self._gv(grad, s.wname), None, s.stride, pad)
        if not need_dx:
            return None
        if reflect:
            return ops.reflect_pad_bwd(ops.conv_dgrad(dy, self.bank.p(s.wname), x.shape, s.stride, 0), s.pad, addend=addend)
        return ops.conv_dgrad(dy, self.bank.p(s.wname), x.shape, s.stride, s.pad, addend=addend)

    # -- forward ---------------------------------------------------------------------------------------
    def encode(self, x_img, saved=None, sl=None):
        """x_img [1,B,H,W,4] (shared by all members) -> content [G,B,H/2^nd,W/2^nd,C]."""
        x = x_img
        for s in self.enc:
            x = self._conv_norm(x, s, sl, None, ACT_RELU, None, False, saved)
        for blk in self.enc_res:
            res = x
            x = self._conv_norm(x, blk[0], sl, None, ACT_RELU, None, False, saved)
            x = self._conv_norm(x, blk[1], sl, None, ACT_NONE, res, False, saved)
        return x

    def _mlp(self, style, saved=None, sl=None):
        """style [1,B,1,1,style_dim] -> AdaIN parameters [G,B,n_adain]."""
        ops = self.ops
        h = style
        acts = []
        for li, s in enumerate(self.mlp):
            w, b = self._w(s, sl)
            h_in = h
            h = ops.conv_fwd(h, w, b, 1, 0, act=ACT_RELU if li < 2 else ACT_NONE)
            acts.append((h_in, h))
        if saved is not None:
            saved.append(acts)
        return h.view(h.shape[0], h.shape[1], self.n_adain)

    def decode(self, content, style, x_img, saved=None, sl=None, recon_sums=None):
        """content [G,B,h,w,C], style [1|G,B,1,1,S] (shared, or one code per member), x_img [1,B,H,W,4] -> (x_fake, mask) [G,B,H,W,4].
        recon_sums [G]: end in the image reconstruction head instead (recon_x_w): recon_sums[g] = sum |x_recon - x_img| of member g,
        the image and its mask are never written, and the result is None.  Needs saved."""
        ops = self.ops
        assert recon_sums is None or saved is not None
        adain = self._mlp(style, saved, sl)
        x = content
        nres, nup = len(self.dec_res), len(self.dec_up)
        # passes that keep activations for backward materialise the upsampled tensor (the weight / data gradient
        # kernels read it); no-grad passes fold the upsample into the consumer convolution instead
        fold = saved is None
        for r, blk in enumerate(self.dec_res):
            res = x
            x = self._conv_norm(x, blk[0], sl, adain, ACT_RELU, None, False, saved)
            x = self._conv_norm(x, blk[1], sl, adain, ACT_NONE, res, r == nres - 1 and nup > 0 and not fold, saved)
        for u, (a, b) in enumerate(self.dec_up):
            x = self._conv_norm(x, a, sl, adain, ACT_RELU, None, False, saved, ups_in=fold)
            if fold and u + 1 == nup and b.cout == 64 and ops.head_fused_supported((1, 1, x.shape[2], x.shape[3], 64)):
                # no-grad pass: the rest of the decoder (AdaIN + ReLU of this block, the three 1x1 head layers, mask compositing)
                # is one kernel; the 64-channel full-resolution map is read once instead of making four HBM round trips
                w, _ = self._w(b, sl)
                xb, pad = _padded(ops, x, b, self.reflect)
                y = ops.conv_fwd(xb, w, None, b.stride, pad)
                mean, rstd = ops.in_stats(y)
                (w1, b1), (w2, b2), (w3, b3) = (self._w(s, sl) for s in self.head)
                return ops.head_fused(y, mean, rstd, adain, self.adain_off[b.key], w1, b1, w2, b2, w3, b3, x_img)
            x = self._conv_norm(x, b, sl, adain, ACT_RELU, None, u + 1 < nup and not fold, saved)
        acts = [x]
        for li, s in enumerate(self.head):
            w, b = self._w(s, sl)
            x = ops.conv_fwd(x, w, b, 1, 0, act=ACT_RELU if li < 2 else ACT_TANH)
            acts.append(x)
        if recon_sums is not None:
            ops.recon_head_fwd(x, x_img, recon_sums)
            saved.append((adain, acts, x_img))
            return None
        x_fake, mask = ops.mask_head_fwd(x, x_img)
        if saved is not None:
            saved.append((adain, acts, x_img))
        return x_fake, mask

    # -- backward (gen_update only) -------------------------------------------------------------------
    def backward(self, d_xfake, d_mask, enc_saved, dec_saved, on_decoder_done=None, d_content=None):
        """Fills ``self.bank.grad`` for every live parameter given d(loss)/d(x_fake), d(loss)/d(mask).
        on_decoder_done: called when grad[enc_end:] (decoder, head, MLP) is final, before the encoder backward.
        d_content: a further gradient of the content code (the recon_c target), added to what the decoder sends back."""
        d, _ = self.decoder_backward(dec_saved, d_xfake, d_mask)
        if on_decoder_done is not None:
            on_decoder_done()
        if d_content is not None:
            self.ops.add_(d, d_content)
        self.encode_backward(d, enc_saved)

    def decoder_backward(self, dec_saved, d_xfake=None, d_mask=None, recon_coef=None, grad=None, want_dstyle=False):
        """Backward of decode(..., saved=dec_saved) from d(loss)/d(x_fake), d(loss)/d(mask) -- or, for a pass that ended in the
        reconstruction head, from recon_coef (d(x_recon) = recon_coef * sign(x_recon - x_img)).  Decoder, head and MLP weight gradients
        go into bank.grad[enc_end:] (grad None) or decode_grad().  -> (d(content), d(style) [G,B,1,1,S] when want_dstyle else None)."""
        ops = self.ops
        dec_saved = list(dec_saved)
        adain, acts, x_img = dec_saved.pop()
        mlp_acts = dec_saved.pop(0)
        d_adain = ops.empty(*adain.shape)  # every column is written by exactly one AdaIN layer's backward
        # head: 1x1 convs with fused activations; grad w.r.t. pre-tanh output of head[2]
        if recon_coef is not None:
            d = ops.recon_head_bwd(acts[3], x_img, recon_coef)
        else:
            d = ops.mask_head_bwd(acts[3], x_img, d_xfake, d_mask)
        for li in (2, 1, 0):
            s = self.head[li]
            ops.conv_wgrad(acts[li], d, self._gv(grad, s.wname), self._gv(grad, s.bname), 1, 0)
            d = ops.conv_dgrad(d, self.bank.p(s.wname), acts[li].shape, 1, 0,
                               mask_src=acts[li] if li > 0 else None, mask_slope=0.0)
        # upsampling blocks, last to first
        recs = dec_saved  # one record per conv in forward order: dec_res (2*nr) then dec_up (2*nd)
        k = len(recs) - 1
        nup = len(self.dec_up)
        for u in range(nup - 1, -1, -1):
            a, b = self.dec_up[u]
            d = self._conv_norm_bwd(d, b, recs[k], adain, d_adain, ACT_RELU, u + 1 < nup, None, grad=grad)
            d = self._conv_norm_bwd(d, a, recs[k - 1], adain, d_adain, ACT_RELU, False, None, grad=grad)
            k -= 2
        if nup > 0:
            d = ops.upsample2x_bwd(d)  # the last residual block's output was written upsampled
        for blk in reversed(self.dec_res):
            d_out = d
            d = self._conv_norm_bwd(d_out, blk[1], recs[k], adain, d_adain, ACT_NONE, False, None, grad=grad)
            d = self._conv_norm_bwd(d, blk[0], recs[k - 1], adain, d_adain, ACT_RELU, False, d_out, grad=grad)
            k -= 2
        assert k == -1
        # MLP (gradients reach it through every AdaIN gamma/beta); layer 0's data gradient is d(style)
        dm = d_adain.view(d_adain.shape[0], d_adain.shape[1], 1, 1, self.n_adain)
        d_style = None
        for li in (2, 1, 0):
            s = self.mlp[li]
            h_in, _ = mlp_acts[li]
            ops.conv_wgrad(h_in, dm, self._gv(grad, s.wname), self._gv(grad, s.bname), 1, 0)
            if li > 0:
                dm = ops.conv_dgrad(dm, self.bank.p(s.wname), h_in.shape, 1, 0, mask_src=h_in, mask_slope=0.0)
            elif want_dstyle:
                d_style = ops.conv_dgrad(dm, self.bank.p(s.wname), h_in.shape, 1, 0)
        return d, d_style

    def encode_backward(self, d, enc_saved, grad=None, want_dx=False, addend=None):
        """Backward of encode(x, enc_saved) from d(content): weight gradients into bank.grad (or the flat buffer grad laid out like
        it); returns d(x) + addend when want_dx (x: a per-member image [G,B,H,W,4]), else None."""
        recs = list(enc_saved)
        k = len(recs) - 1
        for blk in reversed(self.enc_res):
            d_out = d
            d = self._conv_norm_bwd(d_out, blk[1], recs[k], None, None, ACT_NONE, False, None, grad=grad)
            d = self._conv_norm_bwd(d, blk[0], recs[k - 1], None, None, ACT_RELU, False, d_out, grad=grad)
            k -= 2
        for li in range(len(self.enc) - 1, -1, -1):
            d = self._conv_norm_bwd(d, self.enc[li], recs[k], None, None, ACT_RELU, False, addend if li == 0 else None,
                                    need_dx=li > 0 or want_dx, grad=grad)
            k -= 1
        assert k == -1
        return d

    # -- single-member API (reference's gen.encode / gen.decode on NCHW tensors) -----------------------
    def member_encode(self, i, images):
        self._sync()
        ops = self.ops
        x = ops.nchw_to_nhwc(images.to(ops.device, ops.dtype).contiguous(), IMG_C)[None]
        c = self.encode(x, None, sl=i)
        content = ops.nhwc_to_nchw(c[0], self.cdim)
        return content, self.member_style_encode(i, x)

    def style_encode(self, x, sl=None, saved=None):
        """StyleEncoder networks.py:337-353 (norm none, relu), all members (or member sl) at once:
        x [1|G,B,H,W,4] -> style codes [G,B,1,1,style_dim].  In training only the style reconstruction (recon_s_w) runs it, on the
        other direction's translations, and the image reconstruction (recon_x_w), on the source images; saved (a list) keeps what
        style_backward needs."""
        ops, sb = self.ops, self.sty_bank

        def wb(s):
            w, b = sb.p(s.wname), sb.p(s.bname)
            return (w, b) if sl is None else (w[sl:sl + 1], b[sl:sl + 1])
        acts = []  # the input of each layer (padded under reflect), then the last layer's output
        h = x
        for s in self.sty:
            h, pad = _padded(ops, h, s, self.reflect)
            acts.append(h)
            h = ops.conv_fwd(h, *wb(s), s.stride, pad, act=ACT_RELU)
        acts.append(h)
        # global average pool, then the 1x1 conv as a linear layer.  Training (saved) pools with the library's kernel, which
        # style_backward differentiates; the no-grad API path (encode(), sample()) keeps the tensor mean it has always used, so its
        # results are unchanged and op sets without the pool op can still serve it.
        if saved is not None:
            pooled = ops.global_avgpool_fwd(h)
            saved.extend([acts, pooled])
        else:
            pooled = h.mean(dim=(2, 3), keepdim=True).contiguous()
        return ops.conv_fwd(pooled, *wb(self.sty_out), 1, 0)

    def style_backward(self, d_s, saved, addend=None, want_dx=True, grad=None):
        """Backward of style_encode(x, saved=saved) from d(style code) [G,B,1,1,S]: weight and bias gradients into sty_bank.grad (or
        style_grad()); returns d(x) [G,B,H,W,4] (+ addend), or None without want_dx (x a real image: the 7x7 data gradient is skipped)."""
        ops, sb = self.ops, self.sty_bank

        def gv(name):
            return sb.g(name) if grad is None else sb._view(grad, name)
        acts, pooled = saved
        s = self.sty_out
        ops.conv_wgrad(pooled, d_s, gv(s.wname), gv(s.bname), 1, 0)
        d = ops.conv_dgrad(d_s, sb.p(s.wname), pooled.shape, 1, 0)
        d = ops.global_avgpool_bwd(d, acts[-1])  # gated by the last layer's ReLU
        for li in range(len(self.sty) - 1, -1, -1):
            s = self.sty[li]
            reflect = self.reflect and s.pad > 0
            pad = 0 if reflect else s.pad
            ops.conv_wgrad(acts[li], d, gv(s.wname), gv(s.bname), s.stride, pad)
            if li == 0 and not want_dx:
                return None
            add = addend if li == 0 else None
            # the ReLU gate read from the padded input gates every copy of a pixel alike, so it stays in the data gradient
            d = ops.conv_dgrad(d, sb.p(s.wname), acts[li].shape, s.stride, pad, addend=None if reflect else add,
                               mask_src=acts[li] if li > 0 else None, mask_slope=0.0)
            if reflect:
                d = ops.reflect_pad_bwd(d, s.pad, addend=add)
        return d

    def member_style_encode(self, i, x):
        """-> [B, style_dim, 1, 1] of member i (AdaINGen.encode's second result, networks.py:278-283)."""
        return self.style_encode(x, sl=i)[0].permute(0, 3, 1, 2).contiguous()

    def member_decode(self, i, content, style, images):
        self._sync()
        ops = self.ops
        x = ops.nchw_to_nhwc(images.to(ops.device, ops.dtype).contiguous(), IMG_C)[None]
        c = ops.nchw_to_nhwc(content.to(ops.device, ops.dtype).contiguous(), self.cdim)[None]
        st = style.to(ops.device, ops.dtype).reshape(1, style.shape[0], 1, 1, self.style_dim).contiguous()
        x_fake, mask = self.decode(c, st, x, None, sl=i)
        return ops.nhwc_to_nchw(x_fake[0], 3), ops.nhwc_to_nchw(mask[0], 3)


# ------------------------------------------------------------------------------------------------------
# discriminators
# ------------------------------------------------------------------------------------------------------
class CouncilDis(_StackedNet):
    """MsImageDis (council=False) / MsImageDisCouncil (council=True), all members stacked.

    dis.norm (networks.py:40-44, 137-143): layers 1 .. n_layer-1 of every scale normalise between the convolution and the LeakyReLU.
      * 'in'  -- nn.InstanceNorm2d (no parameters): the convolution's epilogue gives the statistics (cg_conv_fwd_stats), then one
                 normalise + LeakyReLU pass.  The conv bias is removed again by the mean subtraction: it is never added and its
                 gradient is exactly 0 (as the generators' dead biases).
      * 'ln'  -- LayerNorm (networks.py:659-686): the convolution with its (live) bias, the per-sample statistics over C*H*W with the
                 unbiased std (cg_ln_stats), then (y - mean) / (std + eps) * gamma + beta and the LeakyReLU (cg_ln_act_fwd).  gamma /
                 beta are bank entries 'cnns.<s>.<i>.norm.{gamma,beta}', stored before the block's conv weight and bias as the
                 reference's parameters() lists them.
    """

    NORMS = ('none', 'in', 'ln')

    def __init__(self, ops, hp, G, input_dim=3, council=False):
        dp = hp['dis']
        assert dp['gan_type'] == 'lsgan', 'only the LSGAN objective is on the accelerated path'
        assert dp['norm'] in self.NORMS and dp['activ'] == 'lrelu'
        self.norm = dp['norm']
        self.reflect = _pad_type(dp['pad_type'])
        assert input_dim == 3
        self.ops, self.hp, self.G, self.council = ops, hp, G, council
        self.num_scales, self.n_layer = dp['num_scales'], dp['n_layer']
        self.scales = []
        for sc in range(self.num_scales):
            d = dp['dim']
            if council:  # networks.py:138: 3x3 stride 1 on cat(x, x_input)
                layers = [LayerSpec('cnns.%d.0.conv' % sc, d, 2 * input_dim, 3, 1, 1, lanes=[0, 1, 2, 4, 5, 6])]
            else:        # networks.py:40: 4x4 stride 2
                layers = [LayerSpec('cnns.%d.0.conv' % sc, d, input_dim, 4, 2, 1, lanes=[0, 1, 2])]
            for i in range(self.n_layer - 1):
                s = LayerSpec('cnns.%d.%d.conv' % (sc, i + 1), 2 * d, d, 4, 2, 1)
                if self.norm == 'ln':
                    s.vecs = ['cnns.%d.%d.norm.gamma' % (sc, i + 1), 'cnns.%d.%d.norm.beta' % (sc, i + 1)]
                layers.append(s)
                d *= 2
            n = self.n_layer
            tail = []
            if council:  # networks.py:142-143: two 1x1 convs, no activation between them
                tail.append(LayerSpec('cnns.%d.%d' % (sc, n), d, d, 1, 1, 0))
                n += 1
            tail.append(LayerSpec('cnns.%d.%d' % (sc, n), 1, d, 1, 1, 0))
            self.scales.append((layers, tail))
        self.specs = [s for layers, tail in self.scales for s in layers + tail]
        self.bank = ParamBank(ops, G, [e for s in self.specs for e in s.entries()])
        # the normalised layers, and under 'in' their dead conv biases (their gradient stays exactly 0)
        self.normed = set(s.key for layers, _ in self.scales for s in layers[1:]) if self.norm != 'none' else set()
        self.dead_bias = set(s.bname for s in self.specs if s.key in self.normed) if self.norm == 'in' else set()

    def _specs(self):
        return self.specs

    def _banks(self):
        return (self.bank,)

    def bank_like(self):
        """a parameter bank with self.bank's layout, data only (zero-initialised)"""
        return ParamBank(self.ops, self.G, [e for s in self.specs for e in s.entries()], trainable=False)

    def reference_key_order(self):
        return [k for s in self.specs for k in s.vecs + [s.wname, s.bname]]

    def _conv_norm(self, h, s, bank, pad):
        """Conv2dBlock.forward of a normalised layer: -> (LeakyReLU output, what _conv_norm_bwd needs)"""
        ops = self.ops
        w = bank.p(s.wname)
        G, B = w.shape[0], h.shape[1]
        ho = (h.shape[2] + 2 * pad - s.k) // s.stride + 1
        wo = (h.shape[3] + 2 * pad - s.k) // s.stride + 1
        if self.norm == 'in':
            if ho * wo == 1:  # nn.InstanceNorm2d in training mode (F.instance_norm's check)
                raise ValueError('Expected more than 1 spatial element when training, got input size torch.Size([%d, %d, 1, 1])'
                                 % (B, s.cout))
            y, mean, rstd = ops.conv_fwd_stats(h, w, s.stride, pad)
            return ops.norm_act_fwd(y, mean, rstd, act=ACT_LRELU), (y, mean, rstd)
        y = ops.conv_fwd(h, w, bank.p(s.bname), s.stride, pad)
        mean, std = ops.ln_stats(y)
        gamma, beta = bank.p(s.vecs[0]), bank.p(s.vecs[1])
        return ops.ln_act_fwd(y, mean, std, gamma, beta, act=ACT_LRELU), (y, mean, std)

    def _conv_norm_bwd(self, d, s, rec, bank, want_wgrad):
        """d(LeakyReLU output) of a normalised layer -> d(conv output); under 'ln' with want_wgrad also d gamma / d beta"""
        ops = self.ops
        y, mean, st = rec
        if self.norm == 'in':
            return ops.norm_act_bwd(d, y, mean, st, act=ACT_LRELU)
        gamma, beta = bank.p(s.vecs[0]), bank.p(s.vecs[1])
        if want_wgrad:
            dgamma, dbeta = bank.g(s.vecs[0]), bank.g(s.vecs[1])
        else:  # the data gradient alone (gen_update): the parameter gradients go to scratch
            dgamma, dbeta = ops.empty(*gamma.shape), ops.empty(*beta.shape)
        return ops.ln_act_bwd(d, y, mean, st, gamma, beta, dgamma, dbeta, act=ACT_LRELU)

    def forward(self, x, saved=None, bank=None):
        """x [G,Bt,H,W,4|8] -> list over scales of patch outputs [G,Bt,h,w,1].  bank: parameters laid out like self.bank (None:
        self.bank), e.g. members drawn from it by ops.gather_members."""
        ops, bank = self.ops, self.bank if bank is None else bank
        outs = []
        for sc, (layers, tail) in enumerate(self.scales):
            h = x
            acts = []  # the input of each layer (padded under reflect), then the output
            norms = {}  # layer index -> the record of its normalisation
            for li, s in enumerate(layers):
                h, pad = _padded(ops, h, s, self.reflect)
                acts.append(h)
                if s.key in self.normed:
                    h, norms[li] = self._conv_norm(h, s, bank, pad)
                else:
                    h = ops.conv_fwd(h, bank.p(s.wname), bank.p(s.bname), s.stride, pad, act=ACT_LRELU, slope=0.2)
            for s in tail:
                acts.append(h)
                h = ops.conv_fwd(h, bank.p(s.wname), bank.p(s.bname), 1, 0)
            acts.append(h)
            outs.append(h)
            if saved is not None:
                saved.append((acts, norms))
            if sc + 1 < self.num_scales:
                x = ops.avgpool_fwd(x)
        return outs

    def backward(self, d_outs, saved, want_wgrad, want_dx, bank=None):
        """d_outs: per-scale d(loss)/d(out).  want_wgrad: fill bank.grad (dis/dis_council update).
        want_dx: return d(loss)/d(x) [G,Bt,H,W,lanes of x] accumulated over scales (gen_update).  bank: the parameters forward ran
        with (None: self.bank)."""
        ops, bank = self.ops, self.bank if bank is None else bank
        dx_scales = []
        for sc, (layers, tail) in enumerate(self.scales):
            acts, norms = saved[sc]
            d = d_outs[sc]
            allspecs = layers + tail
            nl = len(layers)
            for li in range(len(allspecs) - 1, -1, -1):
                s = allspecs[li]
                a_in = acts[li]
                reflect = self.reflect and s.pad > 0
                pad = 0 if reflect else s.pad
                if li in norms:  # d arrives as d(LeakyReLU output), ungated: through the LeakyReLU and the norm to d(conv output)
                    d = self._conv_norm_bwd(d, s, norms[li], bank, want_wgrad)
                if want_wgrad:
                    ops.conv_wgrad(a_in, d, bank.g(s.wname), None if s.bname in self.dead_bias else bank.g(s.bname), s.stride, pad)
                if li == 0 and not want_dx:
                    break
                # a_in is the lrelu OUTPUT of layer li-1 when that layer is one of `layers` (padded under reflect: the gate read from
                # it gates every copy of a pixel alike); a normalised layer li-1 applies its LeakyReLU gate in its own backward
                masked = 1 <= li <= nl and (li - 1) not in norms
                d = ops.conv_dgrad(d, bank.p(s.wname), a_in.shape, s.stride, pad,
                                   mask_src=a_in if masked else None, mask_slope=0.2)
                if reflect:
                    d = ops.reflect_pad_bwd(d, s.pad)
            if want_dx:
                dx_scales.append(d)
        if not want_dx:
            return None
        # fold the image pyramid back: x_{s+1} = avgpool(x_s)
        dx = dx_scales[-1]
        for sc in range(self.num_scales - 2, -1, -1):
            up = dx_scales[sc]
            ops.avgpool_bwd(dx, up, min(4, up.shape[-1]), True)
            if up.shape[-1] == 8:  # second image of the pair (x_input) is data: its lanes 4..7 are ignored
                pass
            dx = up
        return dx


# ------------------------------------------------------------------------------------------------------
# the frozen feature network of the perceptual loss (vgg_w)
# ------------------------------------------------------------------------------------------------------
class Vgg16:
    """Vgg16 networks.py:573-622 up to relu5_3, frozen, for compute_vgg_loss (trainer_council.py:636-641).  One weight group (G = 1): the
    trainer stacks every translation of every member and both directions into the batch of one pass.  The parameters are loaded from
    the reference's ``vgg16.weight`` (a torch.save'd state_dict with keys conv{1_1..5_3}.{weight,bias}, utils.py:350-366); conv1_1's
    3 input channels sit on lanes 0..2 of 4.  No gradient, optimiser state or checkpoint of its own: it is not one of the trainer's
    networks."""

    STAGES = ((('conv1_1', 3, 64), ('conv1_2', 64, 64)),
              (('conv2_1', 64, 128), ('conv2_2', 128, 128)),
              (('conv3_1', 128, 256), ('conv3_2', 256, 256), ('conv3_3', 256, 256)),
              (('conv4_1', 256, 512), ('conv4_2', 512, 512), ('conv4_3', 512, 512)),
              (('conv5_1', 512, 512), ('conv5_2', 512, 512), ('conv5_3', 512, 512)))
    POOL_AFTER = ('conv1_2', 'conv2_2', 'conv3_3')  # F.max_pool2d(h, 2, 2) follows these (none after conv4_3)

    def __init__(self, ops):
        self.ops = ops
        self.specs = [LayerSpec(k, cout, cin, 3, 1, 1, lanes=[0, 1, 2] if cin == 3 else None)
                      for stage in self.STAGES for k, cin, cout in stage]
        self.bank = ParamBank(ops, 1, [e for s in self.specs for e in s.entries()], trainable=False)

    @staticmethod
    def weight_path(vgg_model_path):
        """where load_vgg16 (utils.py:350-366) reads the weights for hp['vgg_model_path'] (trainer_council.py:202)"""
        import os
        return os.path.join(vgg_model_path + '/models', 'vgg16.weight')

    def load_state_dict(self, sd):
        for s in self.specs:
            s.import_weight(self.bank.p(s.wname)[0], sd[s.wname])
            self.bank.p(s.bname)[0].copy_(sd[s.bname].detach().to('cpu', self.bank.data.dtype))

    def load(self, vgg_model_path):
        """Load <vgg_model_path>/models/vgg16.weight.  Never downloads or converts (the reference would fetch vgg16.t7 with wget)."""
        import os
        path = self.weight_path(vgg_model_path)
        if not os.path.isfile(path):
            raise FileNotFoundError('vgg_w needs the VGG-16 weights at %s (a torch.save\'d Vgg16 state_dict, as the reference\'s '
                                    'load_vgg16 writes it); they are not downloaded' % path)
        self.load_state_dict(torch.load(path, map_location='cpu'))
        return self

    def forward(self, x, saved=None):
        """x [1,Bt,H,W,4]: preprocessed images (ops.vgg_preprocess) -> relu5_3 [1,Bt,H/8,W/8,512].  saved (a list): every ReLU output,
        in layer order -- the masks of the data gradient and what the max-pool backward recomputes its windows from."""
        ops, bank = self.ops, self.bank
        h = x
        for s in self.specs:
            h = ops.conv_fwd(h, bank.p(s.wname), bank.p(s.bname), 1, 1, act=ACT_RELU)
            if saved is not None:
                saved.append(h)
            if s.key in self.POOL_AFTER:
                h = ops.maxpool2x2_fwd(h)
        return h

    def backward(self, d_pre, x_shape, saved):
        """Data gradient only: d_pre = d(loss)/d(conv5_3's pre-activation) -> d(loss)/d(x) [1,Bt,H,W,4]."""
        ops, bank = self.ops, self.bank
        d = d_pre
        for li in range(len(self.specs) - 1, -1, -1):
            s = self.specs[li]
            if li == 0:
                return ops.conv_dgrad(d, bank.p(s.wname), x_shape, 1, 1)
            prev = self.specs[li - 1]
            if prev.key in self.POOL_AFTER:  # d(pool output), then through the pool and the previous layer's ReLU
                pooled = saved[li - 1]
                d = ops.conv_dgrad(d, bank.p(s.wname), (1,) + tuple(pooled.shape[1:2]) + (pooled.shape[2] // 2, pooled.shape[3] // 2,
                                                                                          pooled.shape[4]), 1, 1)
                d = ops.maxpool2x2_bwd(d, pooled)
            else:
                d = ops.conv_dgrad(d, bank.p(s.wname), saved[li - 1].shape, 1, 1, mask_src=saved[li - 1], mask_slope=0.0)
        return d
