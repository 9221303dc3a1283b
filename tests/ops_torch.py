"""Plain-PyTorch fp32 reference of every op in the C ABI (include/council_b200.h)  --  TEST DOUBLE.

Lives under tests/ and is never imported by the product package.  Two uses:
  * ``-m gpu`` tests: the per-kernel numerics reference each CUDA op is compared against;
  * ``-m "not gpu"`` tests: injected into the trainer (``Council_Trainer(..., _ops=TorchOps())``) so the
    HOST logic (gating, RNG order, manual backward wiring, loss weighting, Adam bookkeeping) can be
    checked against the oracle without a GPU.
Same method signatures and tensor conventions as ``council_gan_b200.ops.CudaOps``.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH = 0, 1, 2, 3


def _act(v, act, slope):
    if act == ACT_RELU:
        return F.relu(v)
    if act == ACT_LRELU:
        return F.leaky_relu(v, slope)
    if act == ACT_TANH:
        return torch.tanh(v)
    return v


class TorchOps:
    name = 'torch-reference'

    def __init__(self, device='cpu', dtype=torch.float32):
        self.device = torch.device(device)
        self.dtype = dtype
        self.sm_count = 0
        self._launches = 0
        self._tot64 = {}

    def empty(self, *shape):
        return torch.empty(*shape, dtype=self.dtype, device=self.device)

    def zeros(self, *shape):
        return torch.zeros(*shape, dtype=self.dtype, device=self.device)

    def launch_count(self):
        return self._launches

    def set_tensor_core_mode(self, mode):
        return 0

    # -- convolution ------------------------------------------------------------------------------
    @staticmethod
    def _conv_pre(x, w, bias, stride, pad, ups):
        """x [Gx,B,H,W,Ci], w [G,Co,KH,KW,Ci] -> pre-activation [G,B,Ho,Wo,Co] (autograd-capable)."""
        G = w.shape[0]
        outs = []
        for g in range(G):
            xg = x[g if x.shape[0] > 1 else 0].permute(0, 3, 1, 2)
            if ups:
                xg = F.interpolate(xg, scale_factor=2)
            y = F.conv2d(xg, w[g].permute(0, 3, 1, 2), None if bias is None else bias[g], stride, pad)
            outs.append(y.permute(0, 2, 3, 1))
        return torch.stack(outs).contiguous()

    def conv_fwd(self, x, w, bias, stride, pad, ups=False, act=ACT_NONE, slope=0.2):
        return _act(self._conv_pre(x, w, bias, stride, pad, ups), act, slope)

    def conv_fwd_stats(self, x, w, stride, pad, ups=False, eps=1e-5):
        y = self.conv_fwd(x, w, None, stride, pad, ups=ups)
        mean, rstd = self.in_stats(y, eps)
        return y, mean, rstd

    def conv_dgrad(self, dy, w, x_shape, stride, pad, ups=False, addend=None, mask_src=None, mask_slope=0.0):
        G = w.shape[0]
        x = torch.zeros((G,) + tuple(x_shape[1:]), dtype=dy.dtype, device=dy.device, requires_grad=True)
        with torch.enable_grad():
            y = self._conv_pre(x, w, None, stride, pad, ups)
        dx, = torch.autograd.grad(y, x, dy)
        if addend is not None:
            dx = dx + addend
        if mask_src is not None:
            dx = dx * torch.where(mask_src > 0, torch.ones_like(dx), torch.full_like(dx, mask_slope))
        return dx.contiguous()

    def conv_wgrad(self, x, dy, dw, db, stride, pad, ups=False):
        w = torch.zeros_like(dw, requires_grad=True)
        with torch.enable_grad():
            y = self._conv_pre(x, w, None, stride, pad, ups)
        g, = torch.autograd.grad(y, w, dy)
        dw.copy_(g)
        if db is not None:
            db.copy_(dy.sum(dim=(1, 2, 3)))

    # -- instance norm / AdaIN --------------------------------------------------------------------
    def in_stats(self, y, eps=1e-5):
        mean = y.mean(dim=(2, 3))
        var = y.var(dim=(2, 3), unbiased=False)
        return mean.contiguous(), (1.0 / torch.sqrt(var + eps)).contiguous()

    @staticmethod
    def _gb(adain, off, Cc, like):
        if adain is None:
            return torch.ones(1, 1, 1, 1, Cc, device=like.device, dtype=like.dtype), torch.zeros(1, 1, 1, 1, Cc, device=like.device, dtype=like.dtype)
        beta = adain[:, :, off:off + Cc][:, :, None, None, :]
        gamma = adain[:, :, off + Cc:off + 2 * Cc][:, :, None, None, :]
        return gamma, beta

    def _norm_fwd(self, y, mean, rstd, adain, off, res, act, ups):
        Cc = y.shape[-1]
        gamma, beta = self._gb(adain, off, Cc, y)
        z = (y - mean[:, :, None, None, :]) * rstd[:, :, None, None, :] * gamma + beta
        z = _act(z, act, 0.0)
        if res is not None:
            z = z + res
        if ups:
            z = z.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        return z

    def norm_act_fwd(self, y, mean, rstd, adain=None, off=0, res=None, act=ACT_NONE, ups=False):
        return self._norm_fwd(y, mean, rstd, adain, off, res, act, ups).contiguous()

    def norm_act_bwd(self, dz, y, mean, rstd, adain=None, off=0, act=ACT_NONE, ups=False, d_adain=None):
        # differentiate the *whole* normalisation (statistics included) with autograd
        Cc = y.shape[-1]
        yy = y.detach().clone().requires_grad_(True)
        ad = adain.detach().clone().requires_grad_(True) if adain is not None else None
        with torch.enable_grad():
            m = yy.mean(dim=(2, 3))
            v = yy.var(dim=(2, 3), unbiased=False)
            z = self._norm_fwd(yy, m, 1.0 / torch.sqrt(v + 1e-5), ad, off, None, act, ups)
        if ad is not None:
            dy, dad = torch.autograd.grad(z, [yy, ad], dz)
            d_adain[:, :, off:off + 2 * Cc] = dad[:, :, off:off + 2 * Cc]
        else:
            dy, = torch.autograd.grad(z, [yy], dz)
        return dy.contiguous()

    def upsample2x_bwd(self, d_up):
        G, B, H2, W2, Cc = d_up.shape
        return d_up.reshape(G, B, H2 // 2, 2, W2 // 2, 2, Cc).sum(dim=(3, 5)).contiguous()

    # -- mask head --------------------------------------------------------------------------------
    @staticmethod
    def _mask_head(h, x_in):
        mask = (torch.tanh(10 * h[..., 9:12]) + 1) / 2
        im = x_in[..., :3]
        for k in range(3):
            m = mask[..., k:k + 1]
            im = (1 - m) * im + m * h[..., 3 * k:3 * k + 3]
        return im, mask

    def mask_head_fwd(self, h, x_in):
        im, mask = self._mask_head(h, x_in)
        pad = torch.zeros_like(im[..., :1])
        return torch.cat((im, pad), -1).contiguous(), torch.cat((mask, pad), -1).contiguous()

    def head_fused(self, y, mean, rstd, adain, off, w1, b1, w2, b2, w3, b3, x_in):
        z = self.norm_act_fwd(y, mean, rstd, adain, off, None, ACT_RELU, False)
        z = self.conv_fwd(z, w1, b1, 1, 0, act=ACT_RELU)
        z = self.conv_fwd(z, w2, b2, 1, 0, act=ACT_RELU)
        return self.mask_head_fwd(self.conv_fwd(z, w3, b3, 1, 0, act=ACT_TANH), x_in)

    def head_fused_supported(self, y_shape):
        return y_shape[-1] == 64

    def mask_head_bwd(self, h, x_in, d_xfake, d_mask=None):
        # h is the tanh OUTPUT of the last conv; return the gradient w.r.t. its pre-activation
        pre = torch.atanh(h.detach().double().clamp(-1 + 1e-15, 1 - 1e-15)).requires_grad_(True)
        with torch.enable_grad():
            hh = torch.tanh(pre)
            im, mask = self._mask_head(hh, x_in.double())
            outs, grads = [im], [d_xfake[..., :3].double()]
            if d_mask is not None:
                outs.append(mask)
                grads.append(d_mask[..., :3].double())
        g, = torch.autograd.grad(outs, pre, grads)
        return g.to(h.dtype).contiguous()

    # -- image-space helpers ----------------------------------------------------------------------
    def avgpool_fwd(self, x):
        G, B, H, W, Cc = x.shape
        y = F.avg_pool2d(x.reshape(G * B, H, W, Cc).permute(0, 3, 1, 2), 3, 2, 1, count_include_pad=False)
        return y.permute(0, 2, 3, 1).reshape(G, B, H // 2, W // 2, Cc).contiguous()

    def avgpool_bwd(self, dy, dx, nch, accumulate):
        G, B, H, W, Cx = dx.shape
        x = torch.zeros(G * B, nch, H, W, device=dy.device, dtype=dy.dtype, requires_grad=True)
        with torch.enable_grad():
            y = F.avg_pool2d(x, 3, 2, 1, count_include_pad=False)
        g, = torch.autograd.grad(y, x, dy[..., :nch].reshape(G * B, H // 2, W // 2, nch).permute(0, 3, 1, 2))
        g = g.permute(0, 2, 3, 1).reshape(G, B, H, W, nch)
        if accumulate:
            dx[..., :nch] += g
        else:
            dx[..., :nch] = g

    def acc_slice(self, dst, src, nch):
        dst[..., :nch] += src.reshape(dst.shape[:-1] + (src.shape[-1],))[..., :nch]

    def gather_images(self, pools, idx, x_in, G, Bt):
        pool = pools if torch.is_tensor(pools) else torch.cat(tuple(pools), 0)
        y = pool[idx.reshape(-1).long()].reshape(G, Bt, *pool.shape[1:])
        if x_in is not None:
            B = x_in.shape[1]
            reps = Bt // B
            xi = x_in[0].repeat(reps, 1, 1, 1)[None].expand(G, -1, -1, -1, -1)
            y = torch.cat((y, xi), -1)
        return y.contiguous()

    def stage(self, arrays):
        return [a.to(self.device) if a.dtype == torch.int32 else a.to(self.device, self.dtype) for a in arrays]

    def nchw_to_nhwc(self, x, Cp):
        N, Cc, H, W = x.shape
        y = torch.zeros(N, H, W, Cp, dtype=x.dtype, device=x.device)
        y[..., :Cc] = x.permute(0, 2, 3, 1)
        return y

    def nhwc_to_nchw(self, x, Cc):
        nd = x.dim()
        perm = list(range(nd - 3)) + [nd - 1, nd - 3, nd - 2]
        return x[..., :Cc].permute(*perm).contiguous()

    # -- losses -----------------------------------------------------------------------------------
    def lsgan_fwd(self, out, targets, weights, nseg, loss, accumulate):
        G = out.shape[0]
        o = out.reshape(G, nseg, -1)
        sq = (o - targets[None, :, None]) ** 2
        sums = sq.sum(-1)
        tot = (sq.mean(-1) * weights.reshape(G, nseg)).sum(-1)
        if accumulate:
            loss += tot
        else:
            loss.copy_(tot)
        return sums

    def lsgan_bwd(self, out, targets, coef, nseg):
        G = out.shape[0]
        o = out.reshape(G, nseg, -1)
        return (coef[:, :, None] * (o - targets[None, :, None])).reshape(out.shape).contiguous()

    def focus_fwd(self, mask, center, eps):
        m = mask[..., :3]
        s0 = (1 / ((m - center).abs() + eps)).sum(dim=(1, 2, 3, 4))
        s1 = m.sum(dim=(1, 2, 3, 4))
        s2 = (m[:, :, 1:] - m[:, :, :-1]).abs().sum(dim=(1, 2, 3, 4))
        s3 = (m[:, :, :, 1:] - m[:, :, :, :-1]).abs().sum(dim=(1, 2, 3, 4))
        return torch.stack((s0, s1, s2, s3), -1).contiguous()

    def focus_bwd(self, mask, coef, center, eps):
        m = mask[..., :3].detach().clone().requires_grad_(True)
        with torch.enable_grad():
            s0 = (1 / ((m - center).abs() + eps)).sum(dim=(1, 2, 3, 4))
            s1 = m.sum(dim=(1, 2, 3, 4))
            s2 = (m[:, :, 1:] - m[:, :, :-1]).abs().sum(dim=(1, 2, 3, 4)) + \
                (m[:, :, :, 1:] - m[:, :, :, :-1]).abs().sum(dim=(1, 2, 3, 4))
            tot = (coef[:, 0] * s0 + coef[:, 1] * s1 + coef[:, 2] * s2).sum()
        g, = torch.autograd.grad(tot, m)
        return torch.cat((g, torch.zeros_like(g[..., :1])), -1).contiguous()

    # -- fused losses (same contracts as CudaOps.lsgan_fused / gen_loss_fwd / gen_loss_bwd) -------------------
    def lsgan_fused(self, outs, nseg, targets, weights, loss_scale, grad_scale, loss_total, accumulate, loss_plain=None,
                    want_grad=True):
        G = outs[0].shape[0]
        t = torch.tensor(targets, dtype=self.dtype, device=self.device)
        w = torch.tensor(weights, dtype=self.dtype, device=self.device).reshape(G, nseg)
        tot, plain, douts = 0, 0, []
        for out in outs:
            o = out.reshape(G, nseg, -1)
            n = o.shape[-1]
            df = o - t[None, :, None]
            mean = (df ** 2).sum(-1) / n
            tot = tot + (mean * w).sum(-1)
            plain = plain + mean.sum(-1)
            douts.append((grad_scale * w[:, :, None] * 2.0 / n * df).reshape(out.shape).contiguous() if want_grad else None)
        tot = tot * loss_scale
        if accumulate:
            loss_total += tot
        else:
            loss_total.copy_(tot)
        if loss_plain is not None:
            loss_plain.copy_(plain * loss_scale)
        return douts

    def gen_loss_fwd(self, adv_outs, cl_outs, mask, center, eps, adv_grad_scale, scal):
        G = scal.shape[0]
        scal.zero_()
        douts = []
        for out in adv_outs:
            o = out.reshape(G, -1)
            scal[:, 0] += ((o - 1) ** 2).sum(-1) / o.shape[-1]
            douts.append((adv_grad_scale * 2.0 / o.shape[-1] * (o - 1)).reshape(out.shape).contiguous())
        for out in cl_outs:
            o = out.reshape(G, -1)
            scal[:, 1] += ((o - 1) ** 2).sum(-1) / o.shape[-1]
        if mask is not None:
            scal[:, 2:] = self.focus_fwd(mask, center, eps)
        return douts

    def gen_loss_bwd(self, cl_outs, mask, center, eps, scal, hp, hist_gan, hist_council, total, accumulate, pub, want_dmask):
        """Plain restatement of the device finalisation (csrc/losses.cu gen_loss_bwd_kernel) in float64."""
        import numpy as np
        G = total.shape[0]
        R = hp['hist_size'] + 1
        sc = scal.detach().double().cpu().numpy()
        coef = np.zeros((G, 3))
        cdis = np.zeros(G)
        for g in range(G):
            adv, cl = sc[g, 0] / hp['world'], sc[g, 1] / hp['world']
            l01, msum, ltv = sc[g, 2] / hp['numel'], sc[g, 3] / hp['numel'], (sc[g, 4] + sc[g, 5]) / hp['numel']
            tot, ltot = 0.0, 0.0
            if hp['focus_on']:
                if hp['w01'] != 0:
                    tot += hp['w01'] * l01
                    coef[g, 0] = hp['w01'] / hp['numel']
                if hp['wtv'] != 0:
                    tot += hp['wtv'] * ltv
                    coef[g, 2] = hp['wtv'] / hp['numel']
                if hp['wtot'] != 0:
                    if hp['small_abs']:
                        ltot += abs(msum)
                        coef[g, 1] += hp['wtot'] * np.sign(msum) / hp['numel']
                    if hp['small_square']:
                        ltot += msum ** 2
                        coef[g, 1] += hp['wtot'] * 2.0 * msum / hp['numel']
                    tot += hp['wtot'] * ltot

            def window(ring, head, drop_first):
                return [float(ring[g, (head + k) % R]) for k in range(1 if drop_first else 0, hp['hist_size'])]
            adv32 = float(np.float32(adv)) if self.dtype == torch.float32 else adv
            if hp['gan_on'] and hp['matching']:
                mean_gan = (sum(window(hist_gan, hp['head_gan'], True)) + adv32) / hp['hist_size']
                hist_gan[g, (hp['head_gan'] + hp['hist_size']) % R] = adv32
            else:
                mean_gan = sum(window(hist_gan, hp['head_gan'], False)) / hp['hist_size']
            if hp['gan_on']:
                tot += hp['gan_w'] * adv
            w, closs = 1.0, 0.0
            if hp['council_on']:
                if hp['matching']:
                    cl32 = float(np.float32(cl)) if self.dtype == torch.float32 else cl
                    mean_c = (sum(window(hist_council, hp['head_council'], True)) + cl32) / hp['hist_size']
                    hist_council[g, (hp['head_council'] + hp['hist_size']) % R] = cl32
                    w = mean_gan / mean_c
                w_used = float(np.float32(w)) if self.dtype == torch.float32 else w
                closs = cl * w_used * hp['council_w']
                tot += closs
                cdis[g] = w * hp['council_w']
            prev = self._tot64[g] if accumulate else 0.0
            self._tot64[g] = prev + tot
            total[g] = self._tot64[g]
            pub[g] = torch.tensor([tot, adv, l01, ltot, ltv, closs, w, cl], dtype=pub.dtype)
        cl_douts = []
        for out in cl_outs:
            o = out.reshape(G, -1)
            cf = torch.tensor(cdis * 2.0 / (o.shape[-1] * hp['world']), dtype=self.dtype, device=self.device)
            cl_douts.append((cf[:, None] * (o - 1)).reshape(out.shape).contiguous())
        d_mask = None
        if want_dmask:
            d_mask = self.focus_bwd(mask, torch.tensor(coef, dtype=self.dtype, device=self.device), center, eps)
        return cl_douts, d_mask

    # -- input pipeline: the numpy oracle stands in for csrc/augment.cu --------------------------------------
    def aug_color(self, pix, desc, opcode, param, B, max_pixels, any_contrast):
        import augment_oracle as ao
        buf = pix.numpy()
        for b in range(B):
            off, h, w, _ = [int(v) for v in desc[b]]
            img = buf[off:off + h * w * 3].reshape(h, w, 3)
            op, f = int(opcode[b]), float(param[b])
            if op == 1:
                img[:] = ao.grayscale3(img)
            elif op == 2:
                img[:] = ao.adjust_brightness(img, f)
            elif op == 3:
                img[:] = ao.adjust_contrast(img, f)
            elif op == 4:
                img[:] = ao.adjust_saturation(img, f)
            elif op == 5:
                hsv = ao.rgb_to_hsv(img)
                hsv[..., 0] = (hsv[..., 0].astype('int64') + int(f)) % 256
                img[:] = ao.hsv_to_rgb(hsv)

    def aug_resize_crop(self, pix, src_off, flip, slot, crop, n, H, W, oh, ow, ch, cw, bh, kh, ksh, bv, kv, ksv, out, nchw):
        import numpy as np
        import augment_oracle as ao
        buf = pix.numpy()
        for i in range(n):
            off = int(src_off[i])
            img = buf[off:off + H * W * 3].reshape(H, W, 3)
            if int(flip[i]):
                img = img[:, ::-1, :]
            r = ao.resize_bilinear(np.ascontiguousarray(img), oh, ow)
            ci, cj = int(crop[i][0]), int(crop[i][1])
            x = r[ci:ci + ch, cj:cj + cw, :].astype(np.float32) / np.float32(255.0)
            x = (x - np.float32(0.5)) / np.float32(0.5)
            s_ = int(slot[i])
            out[0, s_, :, :, :3] = torch.from_numpy(x).to(out.dtype)
            out[0, s_, :, :, 3] = 0
            if nchw is not None:
                nchw[s_] = torch.from_numpy(x.transpose(2, 0, 1).copy()).to(nchw.dtype)

    # -- optimiser --------------------------------------------------------------------------------
    def adam_step(self, p, g, m, v, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0):
        import math
        gg = g * grad_scale + weight_decay * p
        m.mul_(beta1).add_(gg, alpha=1 - beta1)
        v.mul_(beta2).addcmul_(gg, gg, value=1 - beta2)
        bc1, bc2 = 1 - beta1 ** step, 1 - beta2 ** step
        denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
        p.addcdiv_(m, denom, value=-lr / bc1)
