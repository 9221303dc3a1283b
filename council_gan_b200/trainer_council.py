"""``Council_Trainer`` -- drop-in for the reference's training step, driven through libcouncil_b200.so.

Same constructor, method names, argument meaning, attribute names and error behaviour as
``/root/reference/trainer_council.py`` for the path train.py:241-250 exercises::

    trainer = Council_Trainer(config, cuda_device)
    trainer.dis_update(images_a, images_b, config)
    trainer.dis_council_update(images_a, images_b, config)
    trainer.gen_update(images_a, images_b, config, iterations)
    trainer.update_learning_rate()

What is different underneath (GPU-first, see DESIGN.md):
  * the N council members are stacked: one grouped kernel launch per layer serves all of them
    (the reference loops ``for i in range(self.council_size)`` in Python, :328,558,747,826,858);
  * forward and backward are explicit sequences of our own CUDA kernels; no autograd graph, no
    cuDNN/cuBLAS; the dead work the reference performs is skipped (style encoder :754/829/331, D/DC
    weight gradients inside gen_update, the second/third evaluation of the same content encoding);
  * NO host<->device synchronisation inside an iteration: the losses of all scales, the focus terms, the
    loss-history matching (:518-524,576-586: float64 ring buffers on the device) and every loss gradient are
    three fused kernels (csrc/losses.cu); the published loss attributes are 0-d device tensors exactly like the
    reference's, so the only sync is the one the caller makes when it reads them (write_loss, utils.py:277-305);
  * data parallel: when ``torch.distributed`` is initialised every rank holds all members, takes its
    slice of the global minibatch and the flat gradient buffer of each family is all-reduced (NCCL)
    once per optimiser step -- asynchronously: the discriminators' all-reduce + Adam are joined only when that
    family's parameters are next needed (dis: during dis_council_update; dis_council: during gen_update's
    generator forward; gen: decoder bucket during the encoder backward).
  * abs_beginning_end (:477-495, the input-to-output pixel loss whose weight decays with ``iterations``): its gate and
    weight are host arithmetic on Python floats (``abs_beginning_end_w_conf``, with the reference's member-0 quirk); its value,
    branch (L1 or L2) and gradient are two more launches per direction (csrc/losses.cu) whose sums join the scalar all-reduce.
    With ``abs_beginning_end: 0`` (the shipped configs) nothing of it runs.
  * recon_c_w / recon_s_w (:359-369, 460-469, the latent reconstructions; both directions required): after both forwards each
    translation is re-encoded by the other direction's generator (content encoder for recon_c, style encoder for recon_s).
    One launch per term computes mean |recon - target| and its gradient; the sums join the scalar all-reduce and one launch
    after pass 2 publishes ``loss_gen_recon_{s,c}_{a,b}_s`` and adds the weighted values to the totals.  The re-encode
    backward runs before either generator's own backward: its d(x_fake) joins d_x, the recon_c target gradient joins the
    content gradient, and the content encoder's weight gradients of its two passes are summed.  recon_s_w is the only term
    that trains the style encoder; its bank then has its own Adam state.  With both weights 0 (the shipped configs) nothing
    of it runs.
  * recon_x_w (:339-345, 455-459, the within-domain image reconstruction; both directions required): each source image is
    style-encoded by its own generator, and the other direction's generator decodes (own content code, own style code, source
    image) through a reconstruction head that composites like the mask head but writes only the per-member sums of |x_recon - x|
    (one more pair of rows in the scalar all-reduce).  Its backward runs with the re-encode backward: the other generator's
    decoder, head and MLP gradients go into a scratch added after that generator's own decoder backward, d(content) joins the
    content gradient, and d(style) trains this generator's style encoder on the source image (summed with recon_s's pass when both
    are on).  The reconstruction's mask takes no loss.  With recon_x_w 0 (the shipped configs) nothing of it runs.
  * council_abs_w (:224-228, 595-619, the council loss without a discriminator; both directions required): while the council gate is
    open, one peer per member is drawn on the host with ``random.choice`` in member order (the reference's draw; it serves both
    directions), and two launches per direction compute mean |x_i - x_peer| (or of the channel sums with council_abs_gray_scale) and
    its gradient, the peer detached; the sums join the scalar all-reduce.  Each direction's term is published in the OTHER
    direction's council list (``council_loss_ab_s`` holds the b2a term, as :616-619 do).  With council_w 0 there are no council
    discriminators and dis_council_update returns at once.  With council_abs_w 0 (the shipped configs) nothing of it runs and
    gen_update draws nothing from ``random``.
  * do_Dis_only_gray / useRandomGen / useRandomDis (:499-510, 736-765, the discriminator-side switches): with gray scale D sees
    sum_c x / 3 on every live lane -- dis_update gathers its minibatch through a converting gather, gen_update converts the
    translations and folds D's data gradient back to colour before the council discriminator's colour gradient joins it.  With
    useRandomGen dis_update draws one generator per member from numpy (np.random.randint, member order, both directions) and D_g
    trains on that generator's slot of the stacked translations; the table goes up with the style noise.  With useRandomDis (and
    gan_w != 0) gen_update draws one discriminator per member and runs D on a scratch bank whose member g holds discriminator
    dis_map[g]'s parameters (one gather launch per direction).  Under data parallelism every rank must seed numpy identically.  With
    all three off (the shipped configs) nothing of it runs and neither update draws from numpy.
  * vgg_w (:199-205, 531-538, 636-641, the perceptual loss; both directions required): the frozen VGG-16 is loaded from
    <vgg_model_path>/models/vgg16.weight at construction (never downloaded).  After both forwards every translation of every member
    and both directions is preprocessed into the batch of ONE VGG pass ([x_ab ; x_ba], one weight group), the targets [x_a ; x_b]
    once per update, forward only.  One launch computes the sums of the instance-normalised squared error of relu5_3 (they join the
    scalar all-reduce) and its gradient; the VGG data gradient runs before the per-direction backward, and its d(x_fake) joins d_x.
    ``loss_gen_vgg_{a,b}_s`` are published through the reconstruction terms' finalize launch.  The network is not one of the
    trainer's networks: no optimiser state, checkpoint or all-reduce.  With vgg_w 0 (the shipped configs) nothing of it runs.
  * do_w_loss_matching_focus (:398-410, 433-445, ``focus_loss.do_w_loss_matching_focus``): while the focus gate is open, gen_update's
    pass 2 scales the zero-one term (mask_zero_or_one_w != 0) and the mask-total term of each member by mean(its GAN history before
    this update's append) / mean(its own focus history after appending the unscaled term), the ratio rounded to float32.  The
    b2a mask-total history appends a2b's SCALED term (:441), read from a2b's published values on the device.  The two float64 rings
    per direction live on the device like the GAN / council ones; ``los_hist_focus{,_zero_one}_{a2b,b2a}_s`` read them back and
    ``w_match_focus{,_zero_one}_{a2b,b2a}_conf`` keep the last member's ratios.  No launch is added.  A focus weight with
    mask_total_w 0 or without do_a2b raises NotImplementedError (the reference fails there).  Off (the shipped configs), or with
    both focus weights 0, nothing of it runs.
  * pad_type: reflect (networks.py:463-520, ``gen.pad_type`` / ``dis.pad_type``; every shipped config documents zero/reflect): each
    Conv2dBlock with a pad reads a reflect-padded copy of its input (cg_reflect_pad) through a convolution with pad 0, and the weight
    gradient reads that copy, kept instead of the input.  The data gradient runs at the padded shape, and cg_reflect_pad_bwd folds the
    reflected positions back and adds the residual gradient.  The no-grad decoder (encode / sample) pads the nearest-upsampled map in
    the same pass instead of folding the upsample into the convolution.  The AvgPool pyramid, the MLP, the 1x1 layers and the VGG keep
    zero padding; parameter names and checkpoints do not change.  Other pad types fail the networks' assertion.  With zero (the
    shipped configs) nothing of it runs.
  * dis.norm: in / ln (networks.py:40-44, 137-143, 659-686): both discriminator families normalise layers 1 .. n_layer-1 between
    the convolution and the LeakyReLU (CouncilDis).  'ln' adds each block's LayerNorm gamma / beta to the discriminator banks, the
    checkpoints and optimizer_<i>.pt in the reference's parameter order; gamma starts U(0,1), beta 0.  'bn' and 'sn' raise
    NotImplementedError; other values fail the networks' assertion.  With none (the shipped configs) nothing of it runs.
Paths outside the live configuration space of the reference's three configs (recon_x_cyc loss, nsgan/RaHinge, do_my_style)
raise NotImplementedError.
"""
from __future__ import annotations

import math
import functools
import os
import random
from collections import deque

import numpy as np
import torch
import torch.nn as nn

from .networks import IMG_C, CouncilDis, CouncilGen, Vgg16
from .utils import get_model_list

_DIRS = ('a2b', 'b2a')


class _VecEntry:
    """A per-channel parameter that is not a layer's bias (a layer norm's gamma / beta) in the optimiser's parameter list"""

    def __init__(self, name):
        self.key = self.bname = name
        self.wname = None


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist
    return None


_PDL_MAX_PIXELS = 128 * 128 * 4             # batch x height x width up to which programmatic dependent launch is switched on


def _pinned(fn):
    """Run an update with the launch stream resolved once (ops.pin_stream) instead of once per kernel."""
    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        ops = self.ops
        if not hasattr(ops, 'pin_stream') or ops._stream_cached is not None:
            return fn(self, *args, **kwargs)
        ops.pin_stream()
        # programmatic dependent launch on launch-bound small maps only: early-scheduled dependents cost more than the launch gaps
        # they hide once kernels are long
        for x in args:
            if torch.is_tensor(x):
                pix = x.numel() // (IMG_C if x.dim() == 5 else max(int(x.shape[1]), 1)) if x.dim() >= 4 else 0
                ops.set_pdl(0 < pix <= _PDL_MAX_PIXELS)
                break
        try:
            return fn(self, *args, **kwargs)
        finally:
            ops.unpin_stream()
    return wrapper


class Council_Trainer(nn.Module):
    def __init__(self, hyperparameters, cuda_device='cuda:0', _ops=None):
        super(Council_Trainer, self).__init__()
        hp = hyperparameters
        # ---- the same bookkeeping attributes as trainer_council.py:23-68 --------------------------------
        self.council_size = hp['council']['council_size']
        self.council_size_conf = self.council_size
        self.do_dis_council = hp['council_w'] != 0
        self.do_ads_council_loss = hp['council_abs_w'] != 0
        self.numberOfCouncil_dis_relative_iteration_conf = hp['council']['numberOfCouncil_dis_relative_iteration']
        self.discriminetro_less_style_by_conf = hp['council']['discriminetro_less_style_by']
        self.cuda_device = cuda_device
        self.recon_x_w_conf = hp['recon_x_w']
        self.recon_c_w_conf = hp['recon_c_w']
        self.recon_s_w_conf = hp['recon_s_w']
        self.recon_x_cyc_w_conf = hp['recon_x_cyc_w']
        self.gan_w_conf = hp['gan_w']
        self.vgg_w_conf = hp['vgg_w']
        self.abs_beginning_end_w_conf = hp['abs_beginning_end']
        self.flipOnOff_On_iteration_conf = hp['council']['flipOnOff_On_iteration']
        self.flipOnOff_Off_iteration_conf = hp['council']['flipOnOff_start_with']  # sic, :46-47
        self.council_abs_w_conf = hp['council_abs_w']
        self.council_w_conf = hp['council_w']
        self.council_start_at_iter_conf = hp['council']['council_start_at_iter']
        self.focus_loss_start_at_iter_conf = hp['focus_loss']['focus_loss_start_at_iter']
        self.mask_zero_or_one_w_conf = hp['mask_zero_or_one_w']
        self.mask_zero_or_one_center_conf = hp['focus_loss']['mask_zero_or_one_center']
        self.mask_zero_or_one_epsilon_conf = hp['focus_loss']['mask_zero_or_one_epsilon']
        self.mask_total_w_conf = hp['mask_total_w']
        self.mask_tv_w_conf = hp['mask_tv_w']
        self.batch_size_conf = hp['batch_size']
        self.do_w_loss_matching = hp['do_w_loss_matching']
        self.do_w_loss_matching_focus = hp['focus_loss']['do_w_loss_matching_focus']
        self.los_matching_hist_size_conf = hp['loss_matching_hist_size']
        self.do_a2b_conf = hp['do_a2b']
        self.do_b2a_conf = hp['do_b2a']
        self.w_match_b2a_conf = 1
        self.w_match_a2b_conf = 1
        self.w_match_focus_a2b_conf = 1
        self.w_match_focus_b2a_conf = 1
        self.w_match_focus_zero_one_a2b_conf = 1
        self.w_match_focus_zero_one_b2a_conf = 1
        self._check_supported(hp)
        self._dirs = [d for d in _DIRS if hp['do_' + d]]
        N, hist = self.council_size, self.los_matching_hist_size_conf
        focus_match = bool(self.do_w_loss_matching_focus)
        for d in self._dirs if not focus_match else ():  # :70-92; the gan / council histories live on the device (see _rings);
            # without focus matching these two are never updated
            setattr(self, 'los_hist_focus_%s_s' % d, [deque(np.ones(hist)) for _ in range(N)])
            setattr(self, 'los_hist_focus_zero_one_%s_s' % d, [deque(np.ones(hist)) for _ in range(N)])
        self.do_council_loss = None

        # ---- device op-set: our CUDA library.  No fallback: without it construction fails loudly. -------
        if _ops is None:
            from .ops import CudaOps
            _ops = CudaOps(cuda_device)
        object.__setattr__(self, 'ops', _ops)
        # loss histories of the matching (:81-92, deque(np.ones(hist))): float64 rings [N][hist+1] on the device, window start
        # kept on the host; exported as deques by the los_hist_{gan,council}_{a2b,b2a}_s attributes
        rings = {d: {'gan': torch.ones(N, hist + 1, dtype=torch.float64).to(_ops.device),
                     'council': torch.ones(N, hist + 1, dtype=torch.float64).to(_ops.device),
                     'head_gan': 0, 'head_council': 0} for d in self._dirs}
        if focus_match:  # the focus histories (:398-445) likewise, exported by los_hist_focus{,_zero_one}_{a2b,b2a}_s
            for d in self._dirs:
                for kind in ('focus', 'focus_zero_one'):
                    rings[d][kind] = torch.ones(N, hist + 1, dtype=torch.float64).to(_ops.device)
                    rings[d]['head_' + kind] = 0
        object.__setattr__(self, '_rings', rings)
        dist = _dist()
        self.world = dist.get_world_size() if dist else 1
        self.rank = dist.get_rank() if dist else 0

        # ---- networks (:101-133), stacked over the council ---------------------------------------------
        nets = {}
        for d in self._dirs:
            cin = hp['input_dim_a'] if d == 'a2b' else hp['input_dim_b']
            nets['gen_' + d] = CouncilGen(_ops, hp, N, cin)
            nets['dis_' + d] = CouncilDis(_ops, hp, N, cin, council=False)
            if self.do_dis_council:
                nets['dis_council_' + d] = CouncilDis(_ops, hp, N, cin, council=True)
        object.__setattr__(self, '_nets', nets)
        self.gen_a2b_s, self.gen_b2a_s, self.dis_a2b_s, self.dis_b2a_s = [], [], [], []
        if self.do_dis_council:
            self.dis_council_a2b_s, self.dis_council_b2a_s = [], []
        for name, net in nets.items():
            net._before_access = self._flush
            object.__setattr__(self, name + '_s', [net.member(i) for i in range(N)])
        self.style_dim = hp['gen']['style_dim']
        # the frozen VGG-16 of the perceptual loss (:199-205): loaded once, on every rank, from the same file
        self.vgg = Vgg16(_ops).load(hp['vgg_model_path']) if hp.get('vgg_w', 0) > 0 else None

        display_size = int(hp['display_size'])  # :136-138
        self.s_a = torch.randn(display_size, self.style_dim, 1, 1).to(_ops.device)
        self.s_b = torch.randn(display_size, self.style_dim, 1, 1).to(_ops.device)

        # ---- optimiser state (:140-183): flat fused Adam per family + StepLR bookkeeping -----------------
        self._lr0 = hp['lr']
        self._betas = (hp['beta1'], hp['beta2'])
        self._wd = hp['weight_decay']
        self._lr_policy = hp.get('lr_policy', 'constant')
        if self._lr_policy not in ('constant', 'step'):
            raise NotImplementedError('learning rate policy [%s] is not implemented' % self._lr_policy)
        self._step_size, self._gamma = hp.get('step_size', 1), hp.get('gamma', 1.0)
        self._sched_epoch = {'gen': 0, 'dis': 0, 'dis_council': 0}

        self._init_weights(hp['init'])  # :186-197
        self._img_cache = {}
        self._enc_cache = {}
        self._idx_cache = {}
        self._dis_pick = {}  # direction -> scratch bank of the discriminators gen_update draws with useRandomDis
        self.img_cache_misses = 0  # image batches uploaded / converted (bench.py checks its e2e leg really copies)
        object.__setattr__(self, '_pending', {})  # family -> [(net, bucket, async work)] awaiting all-reduce completion + Adam
        self.hyperparameters = hp
        self.sync_parameters()

    def __getattr__(self, name):
        # los_hist_gan_a2b_s etc. (trainer_council.py:81-92): lists of deques, read back from the device rings on demand
        kind = next((k for k in ('gan', 'council', 'focus_zero_one', 'focus') if name.startswith('los_hist_%s_' % k)), None)
        if kind is not None:
            d = name[len('los_hist_%s_' % kind):][:3]
            rings = self.__dict__.get('_rings', {})
            if d in rings and kind in rings[d] and name == 'los_hist_%s_%s_s' % (kind, d):
                r = rings[d]
                R = r[kind].shape[1]
                host = r[kind].detach().cpu().numpy()
                head = r['head_' + kind]
                return [deque(host[i, [(head + k) % R for k in range(R - 1)]]) for i in range(host.shape[0])]
        return super().__getattr__(name)

    def sync_parameters(self):
        """Data parallel: every rank must hold the same parameters and optimiser state.  Only gradients are all-reduced
        during training, so rank 0's banks are broadcast after construction / resume() (ranks seeded differently, e.g.
        seed + rank, would otherwise train replicas that never re-synchronise).  No-op without a process group."""
        dist = _dist()
        if dist is None or self.world <= 1:
            return
        self._flush()
        for net in self._nets.values():
            for bank in net._banks():
                dist.broadcast(bank.data, 0)
                if bank.trainable:
                    dist.broadcast(bank.exp_avg, 0)
                    dist.broadcast(bank.exp_avg_sq, 0)
            net.params_changed()

    # ------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_supported(hp):
        bad = [k for k in ('recon_x_cyc_w',) if hp.get(k, 0) != 0]
        if bad:
            raise NotImplementedError('loss terms %s are not on the accelerated training path' % bad)
        if hp.get('vgg_w', 0) != 0 and not (hp['do_a2b'] and hp['do_b2a']):
            raise NotImplementedError('vgg_w compares both directions\' translations with their sources, so it needs do_a2b and do_b2a '
                                      '(with one direction the reference fails with an IndexError)')
        if hp.get('vgg_w', 0) < 0:
            raise NotImplementedError('vgg_w must not be negative (the reference fails with an AttributeError on int.cuda)')
        if any(hp.get(k, 0) != 0 for k in ('recon_x_w', 'recon_c_w', 'recon_s_w')) and not (hp['do_a2b'] and hp['do_b2a']):
            raise NotImplementedError('recon_x_w / recon_c_w / recon_s_w decode or re-encode with the other direction\'s generator, so '
                                      'they need do_a2b and do_b2a (with one direction the reference fails with an IndexError)')
        if hp.get('council_abs_w', 0) != 0 and not (hp['do_a2b'] and hp['do_b2a']):
            raise NotImplementedError('council_abs_w publishes each direction\'s term with the other direction\'s council loss, so it '
                                      'needs do_a2b and do_b2a (with one direction the reference fails with an AttributeError)')
        if hp['dis']['gan_type'] != 'lsgan':
            assert 0, "Unsupported GAN type: {}".format(hp['dis']['gan_type'])
        if hp['focus_loss'].get('do_w_loss_matching_focus') and (hp['mask_zero_or_one_w'] != 0 or hp['mask_total_w'] != 0):
            if hp['mask_total_w'] == 0:
                raise NotImplementedError('do_w_loss_matching_focus matches the mask-total term whenever the focus gate is open, so it '
                                          'needs mask_total_w != 0 (with mask_total_w 0 the reference fails with an AttributeError)')
            if not hp['do_a2b']:
                raise NotImplementedError('do_w_loss_matching_focus fills the b2a mask-total history from the a2b term, so it needs '
                                          'do_a2b (with b2a alone the reference fails with an IndexError)')
        if hp['dis']['norm'] in ('bn', 'sn'):
            raise NotImplementedError('dis.norm %s is not on the accelerated training path (in, ln and none are): batch norm takes '
                                      'statistics across the batch of each forward and would need them synchronised across ranks; '
                                      'spectral norm is not a documented option' % hp['dis']['norm'])
        if not (hp['do_a2b'] or hp['do_b2a']):
            raise ValueError('at least one of do_a2b / do_b2a must be set')

    def _init_weights(self, init_type):
        """weights_init (utils.py:402-422): kaiming fan_in normal (or N(0,0.02)) for generators, N(0,0.02) for
        discriminators, zero biases.  A layer norm's gamma is U(0,1) and its beta 0, as LayerNorm.__init__ draws them
        (networks.py:666-667; weights_init touches Conv and Linear modules only).  Drawn from the torch CPU generator; the
        stream is not the reference's (module construction order differs) -- parity tests load explicit state_dicts instead."""
        for name, net in self._nets.items():
            kind = init_type if name.startswith('gen_') else 'gaussian'
            if kind not in ('gaussian', 'kaiming', 'default'):
                raise NotImplementedError('init [%s] is not implemented' % kind)
            for spec in net._specs():
                b = net._bank_of(spec.wname)
                w = b.p(spec.wname)
                fan_in = spec.cin * spec.k * spec.k
                std = math.sqrt(2.0 / fan_in) if kind == 'kaiming' else 0.02
                ref = torch.randn(net.G, spec.cout, spec.cin, spec.k, spec.k) * std
                for i in range(net.G):
                    spec.import_weight(w[i], ref[i])
                for n in spec.vecs:  # gamma, beta
                    b.p(n).copy_(torch.rand(net.G, spec.cout) if n.endswith('.gamma') else torch.zeros(net.G, spec.cout))

    # nn.Module surface the reference's callers touch
    def cuda(self, device=None):
        return self

    def _gate(self, hp, for_gen):
        """flip on/off + start gating, trainer_council.py:541-555 (gen) / :787-801 (dis_council)."""
        c = hp['council']
        cyc = hp['iteration'] % (c['flipOnOff_On_iteration'] + c['flipOnOff_Off_iteration'])
        start = c['flipOnOff_On_iteration'] if c['flipOnOff_start_with'] else c['flipOnOff_Off_iteration']
        do = c['flipOnOff_start_with'] if cyc < start else (not c['flipOnOff_start_with'])
        if not c['flipOnOff']:
            do = True if for_gen else c['flipOnOff_start_with']
        if for_gen and hp['iteration'] < c['council_start_at_iter']:
            do = False
        return do

    def _abs_beginning_end_weights(self, hp, iterations):
        """Gate and weight of the abs_beginning_end term, trainer_council.py:477-495, on host floats.  Member i gets the term while
        abs_beginning_end != 0 and abs_beginning_end_w_conf > 0.005; the weight is recomputed inside the member loop, so member 0 is
        gated by the previous call's weight and the others by this call's.  Once the weight is at or below 0.005 the block is never
        entered again and the weight stops updating.  -> None when the term is off, else the weights of the members whose gate
        is open (a prefix of the council, possibly empty)."""
        if hp['abs_beginning_end'] == 0:
            return None
        weights = []
        for _ in range(self.council_size):
            if not self.abs_beginning_end_w_conf > 0.005:
                break
            self.abs_beginning_end_w_conf = max(hp['abs_beginning_end'] * hp['abs_beginning_end_less_by'] ** iterations,
                                                hp['abs_beginning_end_minimume'])
            weights.append(self.abs_beginning_end_w_conf)
        return weights

    # ---- small host/device helpers ---------------------------------------------------------------------
    def _img(self, x):
        """NCHW image batch (any device) -> shared channels-last [1,B,H,W,4] on the device.  Cached per tensor OBJECT (the
        three updates of one iteration receive the same tensors, train.py:241-250); a new tensor is always uploaded."""
        if x.dim() == 5:  # already the step's layout: a DeviceAugment / DeviceFolderLoader batch (data.py)
            if x.shape[0] != 1 or x.shape[-1] != IMG_C or x.device.type != torch.device(self.ops.device).type or x.dtype != self.ops.dtype:
                raise ValueError('channels-last image batches must be [1, B, H, W, %d] %s tensors on %s' % (IMG_C, self.ops.dtype, self.ops.device))
            return x
        key = (x.data_ptr(), x._version, tuple(x.shape), str(x.device))
        for slot in ('k', 'k2'):
            hit = self._img_cache.get(slot)
            if hit is not None and hit[0] == key and hit[2] is x:
                return hit[1]
        xd = x.detach().to(self.ops.device, self.ops.dtype, non_blocking=True).contiguous()
        img = self.ops.nchw_to_nhwc(xd, IMG_C)[None]
        self.img_cache_misses += 1
        self._img_cache['k2'] = self._img_cache.get('k')
        self._img_cache['k'] = (key, img, x)
        return img

    @staticmethod
    def _bsz(x):
        return x.shape[1] if x.dim() == 5 else x.size(0)

    def _noise(self, batch):
        """torch.randn(B, style_dim, 1, 1) on the CPU generator (:284-285,741,744,807,809) as a HOST tensor [1,B,1,1,S];
        ops.stage() moves it.  Under data parallelism the GLOBAL batch is drawn on every rank (all ranks must be seeded
        identically: same torch / python `random` seeds) and sliced."""
        s = torch.randn(batch * self.world, self.style_dim, 1, 1)
        s = s[self.rank * batch:(self.rank + 1) * batch]
        return s.reshape(1, batch, 1, 1, self.style_dim)

    def _idx(self, key, build):
        t = self._idx_cache.get(key)
        if t is None:
            t = torch.tensor(build(), dtype=torch.int32).to(self.ops.device)
            self._idx_cache[key] = t
        return t

    def _encode(self, d, src_img, save):
        """Content encoding shared by the three updates of one iteration: same generator parameters and same
        images give the same result (the reference recomputes it 3x, :754-756, :829-832, :331-335)."""
        gen = self._nets['gen_' + d]
        key = (id(src_img), gen.bank.step, getattr(gen, '_load_epoch', 0))
        hit = self._enc_cache.get(d)
        if hit is not None and hit[0] == key and (hit[3] or not save):
            return hit[1], hit[2]
        saved = []
        c = gen.encode(src_img, saved)
        self._enc_cache[d] = (key, c, saved, True, src_img)
        return c, saved

    def _lr(self, fam):
        if self._lr_policy == 'constant':
            return self._lr0
        return self._lr0 * self._gamma ** (self._sched_epoch[fam] // self._step_size)

    # ---- optimiser step, data-parallel gradient exchange ---------------------------------------------------
    def _reduce_async(self, fam, net, lo=0, hi=None, bank=None):
        """Queue the all-reduce of grad[lo:hi] of one bank of a network (default: its main bank; NCCL stream, ordered after
        everything issued so far)."""
        dist = _dist()
        work = None
        bank = net.bank if bank is None else bank
        if dist is not None and self.world > 1:
            g = bank.grad if (lo == 0 and hi is None) else bank.grad[lo:hi]
            work = dist.all_reduce(g, async_op=True)  # SUM; local coefficients already carry 1/world
        self._pending.setdefault(fam, []).append((net, bank, work))

    def _finish(self, fam):
        """Join the family's queued all-reduces (stream-side wait, no host block on NCCL) and run its fused Adam."""
        items = self._pending.pop(fam, None)
        if not items:
            return
        for _, _, work in items:
            if work is not None:
                work.wait()  # every bucket of the family first
        done = []
        for net, bank, _ in items:
            if any(bank is b for b in done):
                continue  # a bank with several buckets steps once
            done.append(bank)
            bank.step += 1
            self.ops.adam_step(bank.data, bank.grad, bank.exp_avg, bank.exp_avg_sq, self._lr(fam), self._betas[0],
                               self._betas[1], 1e-8, self._wd, bank.step)
            net.params_changed()

    def _flush(self):
        for fam in list(self._pending):
            self._finish(fam)

    def synchronize(self):
        """Join every deferred optimiser step (data parallel: the gradient all-reduce of the last update is still in flight
        when gen_update returns).  Called implicitly by the next update, save(), sample() and every state_dict access."""
        self._flush()

    def _adam(self, fam, defer=False):
        """All-reduce the flat gradient of a family (data parallel) and run the fused Adam kernel on it.  defer: leave both
        queued until the family's parameters are next needed (_finish), so that the all-reduce overlaps the next update."""
        for d in self._dirs:
            net = self._nets.get('%s_%s' % (fam, d))
            if net is None:
                continue
            if not any(net.bank is b for _, b, _ in self._pending.get(fam, [])):
                self._reduce_async(fam, net)
        if not (defer and self.world > 1):
            self._finish(fam)

    def _src(self, d, a, b):
        return a if d == 'a2b' else b

    def _global_sum(self, t):
        """Reported loss values are means over the GLOBAL minibatch (equal shards); the local values already carry 1/world."""
        dist = _dist()
        if dist is not None and self.world > 1:
            dist.all_reduce(t)
        return t

    # ==================================================================================================
    # dis_update   (trainer_council.py:735-780)
    # ==================================================================================================
    @_pinned
    def dis_update(self, x_a=None, x_b=None, hyperparameters=None):
        hp = hyperparameters
        self._check_supported(hp)
        self._flush()
        ops, N = self.ops, self.council_size
        gray = bool(hp['dis'].get('do_Dis_only_gray'))
        # useRandomGen (:748-750): D_g trains on the translation of generator gen_map[g], one draw per member serving both directions
        gen_map = [int(np.random.randint(N)) for _ in range(N)] if hp['dis'].get('useRandomGen') else None
        img_a, img_b = self._img(x_a), self._img(x_b)
        noise = []
        if self.do_a2b_conf:  # :740-745
            noise.append(('a2b', self._noise(self._bsz(x_b))))
        if self.do_b2a_conf:
            noise.append(('b2a', self._noise(self._bsz(x_a))))
        tables = []
        if gen_map is not None:  # slot tables [translation of gen_map[g] ; real], in the same pinned copy as the noise
            for d in self._dirs:
                B = self._bsz(self._src(d, x_a, x_b))
                tables.append(torch.tensor([[gen_map[g] * B + b for b in range(B)] + [N * B + b for b in range(B)] for g in range(N)],
                                           dtype=torch.int32))
        dev = ops.stage([v for _, v in noise] + tables)
        s = dict(zip((k for k, _ in noise), dev[:len(noise)]))
        random_idx = dict(zip(self._dirs, dev[len(noise):]))
        total = ops.empty(N)
        inv_world = 1.0 / self.world
        for di, d in enumerate(self._dirs):
            gen, dis = self._nets['gen_' + d], self._nets['dis_' + d]
            src, real = self._src(d, img_a, img_b), self._src(d, img_b, img_a)
            B, H, W = src.shape[1:4]
            c, _ = self._encode(d, src, save=True)
            x_fake, _ = gen.decode(c, s[d], src)
            # D minibatch per member: [own fake ; real]   (calc_dis_loss networks.py:56-64); slots >= N*B read the real batch
            idx = random_idx.get(d)
            if idx is None:
                idx = self._idx(('dis', N, B), lambda: [[g * B + b for b in range(B)] + [N * B + b for b in range(B)]
                                                        for g in range(N)])
            pools = (x_fake.view(N * B, H, W, IMG_C), real[0])
            # do_Dis_only_gray (:736-737, 761, 765): D sees the translation and the real batch in gray scale
            xin = ops.gather_images_gray(pools, idx, N, 2 * B) if gray else ops.gather_images(pools, idx, None, N, 2 * B)
            saved = []
            outs = dis.forward(xin, saved)
            wdir = float(hp['gan_w']) if d == 'a2b' else 1.0  # :775 vs :777 (no gan_w on the b2a branch)
            plain = ops.empty(N)
            # loss of both scales + d(loss)/d(out) = wdir * 2 / (n * world) * (out - target): one launch
            d_outs = ops.lsgan_fused(outs, 2, [0.0, 1.0], [[wdir, wdir]] * N, inv_world, inv_world, total, di > 0, plain)
            plain = self._global_sum(plain)
            setattr(self, 'loss_dis_%s_s' % d, [plain[i] for i in range(N)])  # :765-768, only for active directions
            dis.backward(d_outs, saved, want_wgrad=True, want_dx=False)
        total = self._global_sum(total)
        self.loss_dis_total_s = [total[i] for i in range(N)]
        self._adam('dis', defer=True)  # joined when the D parameters are next needed (gen_update / the next dis_update)

    # ==================================================================================================
    # dis_council_update   (trainer_council.py:782-883)
    # ==================================================================================================
    @_pinned
    def dis_council_update(self, x_a=None, x_b=None, hyperparameters=None):
        hp = hyperparameters
        cc = hp['council']
        if self.council_size <= 1 or cc['numberOfCouncil_dis_relative_iteration'] == 0:
            print('no council discriminetor is needed (council size <= 1 or numberOfCouncil_dis_relative_iteration == 0)')
            return
        self.do_council_loss = self._gate(hp, for_gen=False)
        if not self.do_council_loss or hp['council_w'] == 0 or hp['iteration'] < cc['council_start_at_iter']:
            return
        self._check_supported(hp)
        self._finish('dis_council')
        self._finish('gen')
        ops, N = self.ops, self.council_size
        img_a, img_b = self._img(x_a), self._img(x_b)
        noise = []
        if self.do_b2a_conf:  # :806-809: s_a first, then s_b
            noise.append(('b2a', self._noise(self._bsz(x_a))))
        if self.do_a2b_conf:
            noise.append(('a2b', self._noise(self._bsz(x_b))))
        less = cc['discriminetro_less_style_by']
        # peers: python `random`, without replacement, pool refilled when exhausted (:861-868)
        Kcfg = cc['numberOfCouncil_dis_relative_iteration']
        peers = []
        for i in range(N):
            pool_i = list(range(0, i)) + list(range(i + 1, N))
            js = []
            for k in range(Kcfg):
                if k == N:
                    break
                if len(pool_i) == 0:
                    pool_i = list(range(0, i)) + list(range(i + 1, N))
                j = random.choice(pool_i)
                pool_i.remove(j)
                js.append(j)
            peers.append(js)
        # a peer drawn twice (K_cfg >= N refills the pool, :865-866) gives an identical term: evaluate each distinct peer
        # once and weight it by its multiplicity (x + x == 2x exactly)
        uniq = [sorted(set(js)) for js in peers]
        mult = [[js.count(j) for j in u] for js, u in zip(peers, uniq)]
        Krun = len(peers[0])
        U = len(uniq[0])
        assert all(len(u) == U for u in uniq)
        # every small host table of this update (style noise, less-style noise, slot tables) goes up in ONE pinned copy
        Bs = {d: self._src(d, img_a, img_b).shape[1] for d in self._dirs}
        comp0 = {d: (N * Bs[d] if less != 0 else 0) for d in self._dirs}
        tables = [torch.tensor([[g * Bs[d] + b for b in range(Bs[d])] +
                                [comp0[d] + j * Bs[d] + b for j in uniq[g] for b in range(Bs[d])] for g in range(N)], dtype=torch.int32)
                  for d in self._dirs]
        host = [v for _, v in noise] + ([v * less for _, v in noise] if less != 0 else []) + tables
        dev = ops.stage(host)
        s = dict(zip((k for k, _ in noise), dev[:len(noise)]))
        s_less = dict(zip((k for k, _ in noise), dev[len(noise):2 * len(noise)])) if less != 0 else {}
        idx = dict(zip(self._dirs, dev[-len(self._dirs):]))
        total = ops.empty(N)
        inv_world = 1.0 / self.world
        for di, d in enumerate(self._dirs):
            gen, disc = self._nets['gen_' + d], self._nets['dis_council_' + d]
            src = self._src(d, img_a, img_b)
            B, H, W = src.shape[1:4]
            c, _ = self._encode(d, src, save=True)
            x_fake, _ = gen.decode(c, s[d], src)
            pools = [x_fake.view(N * B, H, W, IMG_C)]
            if less != 0:
                x_less, _ = gen.decode(c, s_less[d], src)
                pools.append(x_less.view(N * B, H, W, IMG_C))
            if di == 0:
                self._finish('dis')  # dis_update's all-reduce had the generator decodes above to complete behind
            xin = ops.gather_images(pools, idx[d], src, N, (1 + U) * B)
            saved = []
            outs = disc.forward(xin, saved)
            # sum_k [ mean(D(fake_i)^2) + mean((D(less_jk)-1)^2) ] * council_w / Kcfg   (:872, :878)
            wk = float(hp['council_w']) / Kcfg
            wrows = [[wk * Krun] + [wk * m for m in mult[g]] for g in range(N)]
            d_outs = ops.lsgan_fused(outs, 1 + U, [0.0] + [1.0] * U, wrows, inv_world, inv_world, total, di > 0)
            disc.backward(d_outs, saved, want_wgrad=True, want_dx=False)
        total = self._global_sum(total)
        self.loss_dis_council_total_s = [total[i] for i in range(N)]
        self._adam('dis_council', defer=True)  # joined before gen_update evaluates the council discriminators

    # ==================================================================================================
    # gen_update   (trainer_council.py:280-634)
    # ==================================================================================================
    @_pinned
    def gen_update(self, x_a, x_b, hyperparameters, iterations=0):
        hp = hyperparameters
        self.hyperparameters = hp
        self._check_supported(hp)
        self._finish('gen')
        ops, N = self.ops, self.council_size
        fl = hp['focus_loss']
        img_a, img_b = self._img(x_a), self._img(x_b)
        s_a = self._noise(self._bsz(x_a))  # :284-285 both are always drawn, a first
        s_b = self._noise(self._bsz(x_b))
        s_a, s_b = ops.stage([s_a, s_b])
        s = {'a2b': s_b, 'b2a': s_a}
        it = hp['iteration']
        focus_gate = it > fl['focus_loss_start_at_iter']
        self.council_w_conf = hp['council_w'] if it > hp['council']['council_start_at_iter'] else 0  # :323-326
        self.mask_zero_or_one_w_conf = hp['mask_zero_or_one_w'] if focus_gate else 0
        self.mask_total_w_conf = hp['mask_total_w'] if focus_gate else 0
        self.mask_tv_w_conf = hp['mask_tv_w'] if focus_gate else 0
        focus_on = focus_gate and (hp['mask_zero_or_one_w'] != 0 or hp['mask_total_w'] != 0)  # :390
        if focus_on and hp['mask_total_w'] != 0:
            assert fl['mask_small_use_abs'] or fl['mask_small_use_square'], \
                'at leas one small mask loss should be true, mask_small_use_abs or mask_small_use_square'
        self.do_council_loss = self._gate(hp, for_gen=True)
        council_on = (hp['council_w'] != 0) and self.do_council_loss and N > 1 and self.do_dis_council  # :559,567
        ca_w = hp['council_abs_w']
        ca_on = ca_w != 0 and self.do_council_loss and N > 1  # :559,595
        if ca_on:  # :596-597: one peer per member, in member order, serving both directions
            peers = [random.choice(list(range(0, i)) + list(range(i + 1, N))) for i in range(N)]
            ca_gray = bool(hp['council_abs_gray_scale'])
        gan_on = hp['gan_w'] != 0
        # useRandomDis (:499-501, only with gan_w != 0): member g's adversarial loss comes from discriminator dis_map[g], drawn in member
        # order from numpy; its loss history and w_match stay member g's
        dis_map = [int(np.random.randint(N)) for _ in range(N)] if gan_on and hp['gen'].get('useRandomDis') else None
        dis_gray = bool(hp['dis'].get('do_Dis_only_gray'))
        center, eps = float(fl['mask_zero_or_one_center']), float(fl['mask_zero_or_one_epsilon'])
        be_w = self._abs_beginning_end_weights(hp, iterations)
        be_on = bool(be_w)
        # image and latent reconstruction (:339-345, 359-369, 455-469): the terms in the reference's order, as (kind, domain, weight);
        # x: the source of domain dom decoded by the other direction's generator, s / c: the translation of direction d re-encoded
        recon = [(kind, dom, hp['recon_%s_w' % kind]) for kind in ('x', 's', 'c') if hp['recon_%s_w' % kind] != 0 for dom in ('a', 'b')]
        if (hp['recon_s_w'] != 0 or hp['recon_x_w'] != 0) and not all(self._nets['gen_' + d].sty_bank.trainable for d in self._dirs):
            raise NotImplementedError('recon_s_w / recon_x_w train the style encoder: they must be non-zero when the trainer is built')
        vgg_w = hp['vgg_w']
        if vgg_w != 0 and self.vgg is None:
            raise NotImplementedError('vgg_w loads the VGG-16 when the trainer is built: it must be positive then')
        # the terms of the finalize launch: the reconstructions, then the perceptual loss of x_ab (vgg_b) and of x_ba (vgg_a)
        fin = recon + ([('vgg', 'b', vgg_w), ('vgg', 'a', vgg_w)] if vgg_w != 0 else [])

        # ---- forward of every direction; pass 1 of the loss (all reductions, one launch per direction) -----------
        fw = {}
        nd = len(self._dirs)
        extra = (nd * N * 2 if be_on else 0) + (nd * N if ca_on else 0) + len(fin) * N
        if extra:  # the abs_beginning_end sums [|d|, d^2], the council abs sums and the recon sums ride behind the other scalars:
            red = ops.empty(nd * N * 6 + extra)  # still one all-reduce
            scal, off = red[:nd * N * 6].view(nd, N, 6), nd * N * 6
            if be_on:
                be_sums, off = red[off:off + nd * N * 2].view(nd, N, 2), off + nd * N * 2
            if ca_on:
                ca_sums, off = red[off:off + nd * N].view(nd, N), off + nd * N
            if fin:
                rc_sums = red[off:].view(len(fin), N)
        else:
            red = scal = ops.empty(nd, N, 6)  # per direction and member: [adv, council, focus sums x4] of THIS rank
        for di, d in enumerate(self._dirs):
            gen = self._nets['gen_' + d]
            src = self._src(d, img_a, img_b)
            B, H, W = src.shape[1:4]
            c, enc_saved = self._encode(d, src, save=True)
            dec_saved = []
            x_fake, mask = gen.decode(c, s[d], src, dec_saved)
            rec = {'enc': enc_saved, 'dec': dec_saved, 'x_fake': x_fake, 'mask': mask, 'B': B, 'H': H, 'W': W,
                   'dis_outs': [], 'disc_outs': []}
            if gan_on:  # calc_gen_loss networks.py:84-90
                if di == 0:
                    self._finish('dis')
                rec['dis_bank'] = self._dis_members(d, dis_map) if dis_map is not None else None
                x_dis = x_fake
                if dis_gray:  # :504, 510: D sees the gray translation; the gradient flows back through the conversion
                    idx = self._idx(('id', N, B), lambda: [[g * B + b for b in range(B)] for g in range(N)])
                    x_dis = ops.gather_images_gray(x_fake.view(N * B, H, W, IMG_C), idx, N, B)
                rec['dis_saved'] = []
                rec['dis_outs'] = self._nets['dis_' + d].forward(x_dis, rec['dis_saved'], bank=rec['dis_bank'])
            if council_on:  # MsImageDisCouncil.calc_gen_loss networks.py:188-194
                if di == 0:
                    self._finish('dis_council')
                idx = self._idx(('id', N, B), lambda: [[g * B + b for b in range(B)] for g in range(N)])
                xin = ops.gather_images(x_fake.view(N * B, H, W, IMG_C), idx, src, N, B)
                rec['disc_saved'] = []
                rec['disc_outs'] = self._nets['dis_council_' + d].forward(xin, rec['disc_saved'])
            rec['d_adv'] = ops.gen_loss_fwd(rec['dis_outs'], rec['disc_outs'], mask if focus_on else None, center, eps,
                                            float(hp['gan_w']) / self.world, scal[di])
            if be_on:
                ops.abs_beginning_end_fwd(x_fake, src, be_sums[di])
            if ca_on:
                ops.council_abs_fwd(x_fake, peers, ca_gray, ca_sums[di])
            if recon:
                rec['c'], rec['src'] = c, src
            fw[d] = rec
        fin_numel = self._recon_forward(fw, s, recon, rc_sums) if recon else []
        if vgg_w != 0:
            vgg_numel, vgg_rec = self._vgg_forward(fw, img_a, img_b, rc_sums[len(recon):], vgg_w)
            fin_numel += [vgg_numel] * 2
        self._flush()  # (a family gated off above still steps here)
        dist = _dist()
        if dist is not None and self.world > 1:
            dist.all_reduce(red)  # sums over ranks; pass 2 divides the means by world and uses the GLOBAL (sum m / numel)^2
        d_x_re = self._recon_backward(fw, recon) if recon else {}
        if vgg_w != 0:  # d(VGG input) of both directions, [1, 2NB, H, W, 4]
            d_vgg = self.vgg.backward(*vgg_rec)
            del vgg_rec

        # ---- pass 2 (loss assembly + history matching on the device, remaining loss gradients) and the backward ------
        total = ops.empty(N)
        pub = ops.empty(len(self._dirs), N, 8)
        if be_on:
            be_pub = ops.empty(nd, N)
            be_weights = [float(w) for w in be_w] + [0.0] * (N - len(be_w))  # 0: this member's gate is closed
        if ca_on:
            ca_pub = ops.empty(nd, N)
        matching = bool(self.do_w_loss_matching)
        focus_match = focus_on and bool(self.do_w_loss_matching_focus)
        if focus_match:
            focus_w = ops.empty(nd, N, 2)  # per direction and member: the zero-one and mask-total ratios
        data_parallel = self.world > 1
        recon_x_on = hp['recon_x_w'] != 0

        def decoder_done(g):  # grad[enc_end:] of g is final once recon_x's pass through its decoder is added
            if recon_x_on:
                ops.add_(g.bank.grad[g.enc_end:], g.decode_grad())
            if data_parallel:
                self._reduce_async('gen', g, g.enc_end, None)
        for di, d in enumerate(self._dirs):
            rec = fw[d]
            gen = self._nets['gen_' + d]
            ring = self._rings[d]
            hpd = {'world': self.world, 'hist_size': self.los_matching_hist_size_conf, 'head_gan': ring['head_gan'],
                   'head_council': ring['head_council'], 'gan_on': int(gan_on), 'council_on': int(council_on),
                   'focus_on': int(focus_on), 'matching': int(matching), 'small_abs': int(bool(fl['mask_small_use_abs'])),
                   'small_square': int(bool(fl['mask_small_use_square'])), 'gan_w': float(hp['gan_w']),
                   'council_w': float(hp['council_w']), 'w01': float(hp['mask_zero_or_one_w']), 'wtot': float(hp['mask_total_w']),
                   'wtv': float(hp['mask_tv_w']), 'numel': float(rec['B'] * self.world * 3 * rec['H'] * rec['W'])}
            focus_kw = {}
            if focus_match:  # :398-410, 433-445; b2a's mask-total history appends a2b's scaled term (:441), pub[0][:, 3]
                hpd.update(focus_matching=1, head_focus=ring['head_focus'], head_focus01=ring['head_focus_zero_one'])
                focus_kw = dict(hist_focus=ring['focus'], hist_focus01=ring['focus_zero_one'], focus_w=focus_w[di],
                                focus_src=pub[self._dirs.index('a2b')] if d == 'b2a' else None)
            d_cl, d_mask = ops.gen_loss_bwd(rec['disc_outs'], rec['mask'] if focus_on else None, center, eps, scal[di], hpd,
                                            ring['gan'], ring['council'], total, di > 0, pub[di], focus_on, **focus_kw)
            R = self.los_matching_hist_size_conf + 1
            if focus_match and hp['mask_zero_or_one_w'] != 0:
                ring['head_focus_zero_one'] = (ring['head_focus_zero_one'] + 1) % R
            if focus_match:  # the mask-total term is matched whenever the gate is open (mask_total_w != 0, _check_supported)
                ring['head_focus'] = (ring['head_focus'] + 1) % R
            if gan_on and matching:  # :518-524 append + popleft
                ring['head_gan'] = (ring['head_gan'] + 1) % R
            if council_on and matching:  # :576-586
                ring['head_council'] = (ring['head_council'] + 1) % R
            d_x = None
            if gan_on:
                d_x = self._nets['dis_' + d].backward(rec['d_adv'], rec['dis_saved'], want_wgrad=False, want_dx=True, bank=rec['dis_bank'])
                if dis_gray:  # before the council discriminator's colour gradient joins d_x
                    ops.gray_fold(d_x)
            if council_on:
                d_x8 = self._nets['dis_council_' + d].backward(d_cl, rec['disc_saved'], want_wgrad=False, want_dx=True)
                if d_x is None:
                    d_x = ops.zeros(*rec['x_fake'].shape)
                ops.acc_slice(d_x, d_x8, 4)
            if d in d_x_re:  # d(recon) / d(x_fake) through the other generator's re-encode
                if d_x is None:
                    d_x = d_x_re[d]
                else:
                    ops.add_(d_x, d_x_re[d])
            if vgg_w != 0:  # through vgg_preprocess: d_x += 127.5 * the lane-swapped gradient of this direction's half of the batch
                d_vd = d_vgg[0, di * N * rec['B']:(di + 1) * N * rec['B']]
                fresh = d_x is None
                if fresh:
                    d_x = ops.empty(*rec['x_fake'].shape)
                ops.vgg_preprocess_bwd(d_vd, d_x, accumulate=not fresh)
            if d_x is None:
                d_x = ops.zeros(*rec['x_fake'].shape)
            if be_on:  # after gen_loss_bwd of this direction: the totals share its accumulator
                ops.abs_beginning_end_bwd(rec['x_fake'], self._src(d, img_a, img_b), be_sums[di], hpd['numel'], be_weights, total,
                                          be_pub[di], d_x)
            if ca_on:  # likewise after gen_loss_bwd of this direction
                numel = rec['B'] * self.world * rec['H'] * rec['W'] * (1 if ca_gray else 3)
                ops.council_abs_bwd(rec['x_fake'], peers, ca_gray, ca_sums[di], numel, float(ca_w), total, ca_pub[di], d_x)
            gen.backward(d_x, d_mask, rec['enc'], rec['dec'],
                         on_decoder_done=(lambda g=gen: decoder_done(g)) if recon_x_on or data_parallel else None,
                         d_content=rec.get('d_c'))
            if hp['recon_c_w'] != 0:  # the content encoder ran twice: add the re-encode pass's weight gradients
                ops.add_(gen.bank.grad[:gen.enc_end], gen.reencode_grad())
            if data_parallel:
                self._reduce_async('gen', gen, 0, gen.enc_end)  # encoder bucket; the decoder bucket went out during the encoder backward
        if fin:  # after every gen_loss_bwd / abs_beginning_end_bwd of this update: the member totals share their accumulator
            rc_pub = ops.empty(len(fin), N)
            ops.recon_finalize(rc_sums, fin_numel, [float(w) for _, _, w in fin], total, rc_pub)
        if ca_on:  # :616-619: each direction's published council loss takes the OTHER direction's abs term (both directions are on)
            for di in range(nd):
                ops.add_column(pub[di], 5, ca_pub[nd - 1 - di])
        self._adam('gen', defer=True)  # joined at the start of the next update (or by save / state_dict / sample)
        self._enc_cache.clear()

        # ---- publish the reference's loss attributes (:302-322, :556-557): 0-d DEVICE tensors, no sync here -------------
        self.loss_gen_total_s = [total[i] for i in range(N)]
        for d in _DIRS:
            ab = 'ab' if d == 'a2b' else 'ba'
            if d in fw:
                di = self._dirs.index(d)

                def col(k, on=True):
                    return [pub[di, i, k] for i in range(N)] if on else []
                setattr(self, 'loss_gen_adv_%s_s' % d, col(1, gan_on))
                setattr(self, 'loss_gen_mask_zero_one_%s_s' % ab, col(2, focus_on and hp['mask_zero_or_one_w'] != 0))
                setattr(self, 'loss_gen_mask_total_%s_s' % ab, col(3) if focus_on and hp['mask_total_w'] != 0 else [0] * N)
                setattr(self, 'loss_gen_mask_TV_%s_s' % ab, col(4) if focus_on and hp['mask_tv_w'] != 0 else [0] * N)
                setattr(self, 'council_loss_%s_s' % ab, col(5) if council_on or ca_on else [0] * N)
                if council_on and matching:
                    setattr(self, 'w_match_%s_conf' % d, pub[di, N - 1, 6])  # the reference keeps the last member's ratio (:583)
                if focus_match:  # likewise for the focus ratios (:402, 408, 437, 443)
                    if hp['mask_zero_or_one_w'] != 0:
                        setattr(self, 'w_match_focus_zero_one_%s_conf' % d, focus_w[di, N - 1, 0])
                    setattr(self, 'w_match_focus_%s_conf' % d, focus_w[di, N - 1, 1])
            else:
                setattr(self, 'loss_gen_adv_%s_s' % d, [0] * N if gan_on else [])
                setattr(self, 'loss_gen_mask_zero_one_%s_s' % ab, [])
                setattr(self, 'loss_gen_mask_total_%s_s' % ab, [])
                setattr(self, 'loss_gen_mask_TV_%s_s' % ab, [])
                setattr(self, 'council_loss_%s_s' % ab, [])
        if be_w is not None:  # :477-484: one entry per member whose gate was open, the int 0 for an inactive direction
            for d, name in (('a2b', 'loss_gen_beginning_end_a_ab_s'), ('b2a', 'loss_gen_beginning_end_b_ba_s')):
                setattr(self, name, [be_pub[self._dirs.index(d), i] for i in range(len(be_w))] if d in fw else [0] * len(be_w))
        if recon:  # :308-313, :455-469: one entry per member, [] for a term whose weight is 0
            for kind in ('x', 's', 'c'):
                for dom in ('a', 'b'):
                    setattr(self, 'loss_gen_recon_%s_%s_s' % (kind, dom), [])
            for k, (kind, dom, _) in enumerate(recon):
                setattr(self, 'loss_gen_recon_%s_%s_s' % (kind, dom), [rc_pub[k, i] for i in range(N)])
        if vgg_w != 0:  # :531-536: one entry per member, vgg_a the b2a translation's term
            self.loss_gen_vgg_b_s = [rc_pub[len(recon), i] for i in range(N)]
            self.loss_gen_vgg_a_s = [rc_pub[len(recon) + 1, i] for i in range(N)]
        self._last_fw = {d: {'x_fake': fw[d]['x_fake'], 'mask': fw[d]['mask']} for d in self._dirs}

    def _dis_members(self, d, dis_map):
        """The discriminators of direction d with member g's parameters copied from member dis_map[g] (useRandomDis), in a scratch bank
        allocated once per direction: its address stays the same for the tensor-map cache, which is keyed by pointer."""
        dis = self._nets['dis_' + d]
        bank = self._dis_pick.get(d)
        if bank is None:
            bank = self._dis_pick[d] = dis.bank_like()
        self.ops.gather_members(dis.bank.data, bank.data, dis.bank.member_segments(), dis_map)
        return bank

    def _recon_forward(self, fw, s, recon, sums):
        """The reconstruction passes, keeping activations for the backward, and their terms: sums[k] = this rank's sum |recon - target|
        of term k.  recon_x (:339-345): the source of direction d, style-encoded by its own generator, decoded by the other one through
        the reconstruction head.  recon_s / recon_c (:359-369): each translation re-encoded by the other direction's generator; their
        gradients are written together with the sums (they do not depend on the loss value).  -> numel of each term over the GLOBAL
        minibatch."""
        ops = self.ops
        other = {'a2b': 'b2a', 'b2a': 'a2b'}
        numel = []
        for k, (kind, dom, w) in enumerate(recon):
            if kind == 'x':  # x_a_recon = gen_b2a.decode(c_a, s_a', x_a): mean |x_recon - x| over B x 3 x H x W
                d = 'a2b' if dom == 'a' else 'b2a'
                rec = fw[d]
                rec['sx_saved'], rec['x_dec_saved'] = [], []
                s_prime = self._nets['gen_' + d].style_encode(rec['src'], saved=rec['sx_saved'])
                self._nets['gen_' + other[d]].decode(rec['c'], s_prime, rec['src'], rec['x_dec_saved'], recon_sums=sums[k])
                n = rec['B'] * 3 * rec['H'] * rec['W'] * self.world
                rec['x_coef'] = float(w) / n
                numel.append(float(n))
                continue
            # recon_c_a / recon_s_b come from re-encoding x_ab (direction a2b), recon_c_b / recon_s_a from x_ba
            d = ('a2b' if dom == 'a' else 'b2a') if kind == 'c' else ('a2b' if dom == 'b' else 'b2a')
            rec = fw[d]
            gen_o = self._nets['gen_' + other[d]]
            if kind == 'c':  # mean |c_recon - c|; the target c is not detached (:466-467): it takes the opposite gradient
                rec['c_saved'] = []
                c_rec = gen_o.encode(rec['x_fake'], rec['c_saved'])
                n = rec['c'][0].numel() * self.world
                rec['d_c_rec'], rec['d_c'] = ops.empty(*c_rec.shape), ops.empty(*c_rec.shape)
                ops.latent_l1(c_rec, rec['c'], sums[k], float(w) / n, da=rec['d_c_rec'], db=rec['d_c'])
            else:  # mean |s_recon - s|, s the style noise this direction decoded with
                rec['s_saved'] = []
                s_rec = gen_o.style_encode(rec['x_fake'], saved=rec['s_saved'])
                n = s[d][0].numel() * self.world
                rec['d_s_rec'] = ops.empty(*s_rec.shape)
                ops.latent_l1(s_rec, s[d], sums[k], float(w) / n, da=rec['d_s_rec'])
            numel.append(float(n))
        return numel

    def _vgg_forward(self, fw, img_a, img_b, sums, w):
        """The perceptual loss, compute_vgg_loss (:636-641) for every member and both directions in ONE VGG pass: the batch
        [x_ab (N B) ; x_ba (N B)] keeps its ReLU outputs, the targets [x_a ; x_b] run once, forward only.  sums [2, N] = this rank's
        sums of the squared error of x_ab against x_a (vgg_b) and of x_ba against x_b (vgg_a); their gradient w.r.t. conv5_3's
        pre-activation is written in the same launch.  -> (numel of each term over the GLOBAL minibatch, arguments of Vgg16.backward)"""
        ops, N = self.ops, self.council_size
        xa, xb = fw['a2b']['x_fake'], fw['b2a']['x_fake']
        assert xa.shape == xb.shape and img_a.shape == img_b.shape, 'vgg_w stacks both directions: their batches must have one shape'
        _, B, H, W, _ = xa.shape
        x = ops.empty(1, 2 * N * B, H, W, IMG_C)
        ops.vgg_preprocess(xa, out=x[0, :N * B])
        ops.vgg_preprocess(xb, out=x[0, N * B:])
        tgt = ops.empty(1, 2 * B, H, W, IMG_C)
        ops.vgg_preprocess(img_a, out=tgt[0, :B])
        ops.vgg_preprocess(img_b, out=tgt[0, B:])
        saved = []
        f = self.vgg.forward(x, saved)
        f_tgt = self.vgg.forward(tgt)
        _, _, h, wd, Cf = f.shape
        numel = float(B * self.world * Cf * h * wd)
        d_pre = ops.vgg_loss(f, f_tgt, B, N * B, w / numel, sums)
        return numel, (d_pre, x.shape, saved)

    def _recon_backward(self, fw, recon):
        """Backward of the reconstruction passes, before either generator's own backward.  recon_x: the other generator's decoder
        (weight gradients into its decode_grad() buffer), its d(content) joining the content gradient of the direction and its d(style)
        training this generator's style encoder without a data gradient to the image.  recon_s / recon_c: the other generator's
        style-encoder and content-encoder gradients (the latter into its reencode_grad() buffer).  A style encoder that ran twice sums
        its two passes, and each style bank's all-reduce is queued once, after all of its contributions.  -> d(recon) / d(x_fake) of
        every direction that has a re-encode term."""
        ops = self.ops
        other = {'a2b': 'b2a', 'b2a': 'a2b'}
        kinds = set(kind for kind, _, _ in recon)
        both_styles = 'x' in kinds and 's' in kinds
        d_x = {}
        for d in self._dirs:
            rec = fw[d]
            gen_d, gen_o = self._nets['gen_' + d], self._nets['gen_' + other[d]]
            if 'x_dec_saved' in rec:
                d_c, d_s = gen_o.decoder_backward(rec['x_dec_saved'], recon_coef=rec['x_coef'], grad=gen_o.decode_grad(), want_dstyle=True)
                if 'd_c' in rec:
                    ops.add_(rec['d_c'], d_c)
                else:
                    rec['d_c'] = d_c
                gen_d.style_backward(d_s, rec['sx_saved'], want_dx=False, grad=gen_d.style_grad() if both_styles else None)
            dx = None
            if 's_saved' in rec:
                dx = gen_o.style_backward(rec['d_s_rec'], rec['s_saved'])
            if 'c_saved' in rec:
                dx = gen_o.encode_backward(rec['d_c_rec'], rec['c_saved'], grad=gen_o.reencode_grad(), want_dx=True, addend=dx)
            if dx is not None:
                d_x[d] = dx
        if kinds & {'x', 's'}:
            for d in self._dirs:
                gen = self._nets['gen_' + d]
                if both_styles:
                    ops.add_(gen.sty_bank.grad, gen.style_grad())
                self._reduce_async('gen', gen, bank=gen.sty_bank)
        return d_x

    # ==================================================================================================
    # the rest of the reference surface
    # ==================================================================================================
    def update_learning_rate(self):
        """StepLR.step() on every optimiser (:885-896; get_scheduler utils.py:392-400)."""
        for fam in self._sched_epoch:
            if fam == 'dis_council' and not self.do_dis_council:
                continue
            self._sched_epoch[fam] += 1

    @_pinned
    def sample(self, x_a=None, x_b=None, s_a=None, s_b=None, council_member_to_sample_vec=None, return_mask=True):
        """Translation of every image by every member (:643-733): returns the same 8-tuple, rows ordered image-major /
        member-minor like the reference's double loop.  All members and all images run as ONE stacked pass per network
        (the reference runs batch-1 passes in a Python double loop); instance norm / AdaIN are per-sample, so the result
        per image is the same.  (eval() == train() for this network: no dropout, no running statistics.)"""
        self._flush()
        ops, N = self.ops, self.council_size
        members = list(range(N)) if council_member_to_sample_vec is None else list(council_member_to_sample_vec)
        res = {}
        for d in _DIRS:
            if not getattr(self, 'do_%s_conf' % d):
                res[d] = (None, None, None, None)
                continue
            x = x_a if d == 'a2b' else x_b
            if x.dim() == 5:
                raise ValueError('sample() takes NCHW images like the reference (trainer_council.py:643)')
            B = x.size(0)
            fixed = (self.s_b if s_b is None else s_b) if d == 'a2b' else (self.s_a if s_a is None else s_a)
            s2 = torch.randn(B, self.style_dim, 1, 1)  # :649 / :655
            gen = self._nets['gen_' + d]
            img = ops.nchw_to_nhwc(x.detach().to(ops.device, ops.dtype).contiguous(), IMG_C)[None]

            def st(t):  # [B, S, 1, 1] -> shared style [1, B, 1, 1, S]
                return t[:B].to(ops.device, ops.dtype).reshape(1, B, 1, 1, self.style_dim).contiguous()
            c = gen.encode(img)
            first, mask1 = gen.decode(c, st(fixed), img)
            third, _ = gen.decode(c, st(s2), img)
            if return_mask:
                second = mask1
            else:
                second, _ = gen.decode(c, gen.style_encode(img), img)  # recon with each member's own style code

            def rows(t):  # [N, B, H, W, 4] -> [B * len(members), 3, H, W], image-major
                t = ops.nhwc_to_nchw(t, 3)[members]
                return t.permute(1, 0, 2, 3, 4).reshape(B * len(members), 3, t.shape[-2], t.shape[-1])
            xs = x.detach().to(ops.device, ops.dtype).repeat_interleave(len(members), dim=0)
            res[d] = (xs, rows(second), rows(first), rows(third))
        return res['a2b'] + res['b2a']

    def forward(self, *args, **kwargs):
        raise NotImplementedError('Council_Trainer.forward is broken in the reference (trainer_council.py:267 '
                                  'references a nonexistent self.gen_a2b); use sample()')

    def save(self, snapshot_dir, iterations):
        """Per-member checkpoint files with the reference's names, keys and optimiser layout (:969-992): the reference's
        resume() loads them, and ours loads the reference's."""
        self._flush()
        for i in range(self.council_size):
            for fam in ('gen', 'dis', 'dis_council'):
                if fam == 'dis_council' and not self.do_dis_council:
                    continue
                for d in self._dirs:
                    name = os.path.join(snapshot_dir, '%s_%s_%d_%08d.pt' % (d, fam, i, iterations + 1))
                    torch.save({d: getattr(self, '%s_%s_s' % (fam, d))[i].state_dict()}, name)
            opt = {fam: self._opt_state_dict(fam, i) for fam in ('gen', 'dis', 'dis_council')
                   if fam != 'dis_council' or self.do_dis_council}
            torch.save(opt, os.path.join(snapshot_dir, 'optimizer_%d.pt' % i))

    def _opt_params(self, fam):
        """The parameter list of the reference's per-member optimiser (:152-179): a2b network then b2a network, each in
        nn.Module.parameters() order (= state_dict order without buffers).  -> [(net, spec, is_weight)]"""
        out = []
        for d in self._dirs:
            net = self._nets['%s_%s' % (fam, d)]
            by_key = {}
            for spec in net._specs():
                by_key[spec.wname] = (net, spec, True)
                by_key[spec.bname] = (net, spec, False)
                for n in spec.vecs:  # a layer norm's gamma / beta: per-channel like a bias
                    by_key[n] = (net, _VecEntry(n), False)
            out += [by_key[k] for k in net.reference_key_order() if k in by_key]
        return out

    def _opt_state_dict(self, fam, i):
        """torch.optim.Adam.state_dict() of member i's optimiser for one family, from the flat moment buffers.
        Parameters that never receive a gradient (the style encoder) have no state entry, as in the reference."""
        state = {}
        plist = self._opt_params(fam)
        for idx, (net, spec, is_w) in enumerate(plist):
            name = spec.wname if is_w else spec.bname
            bank = net._bank_of(name)
            if not bank.trainable or bank.step == 0:
                continue
            m, v = bank._view(bank.exp_avg, name)[i], bank._view(bank.exp_avg_sq, name)[i]
            if is_w:
                m, v = spec.export_weight(m), spec.export_weight(v)
            state[idx] = {'step': torch.tensor(float(bank.step)), 'exp_avg': m.detach().clone().cpu(),
                          'exp_avg_sq': v.detach().clone().cpu()}
        group = {'lr': self._lr(fam), 'betas': tuple(self._betas), 'eps': 1e-8, 'weight_decay': self._wd, 'amsgrad': False,
                 'maximize': False, 'foreach': None, 'capturable': False, 'differentiable': False, 'fused': None,
                 'decoupled_weight_decay': False, 'initial_lr': self._lr0, 'params': list(range(len(plist)))}
        return {'state': state, 'param_groups': [group]}

    def _load_opt_state_dict(self, fam, i, sd):
        """Inverse of _opt_state_dict; accepts what torch.optim.Adam.state_dict() of the reference wrote (:988-992)."""
        plist = self._opt_params(fam)
        steps = {}  # bank -> largest step of its entries
        for idx, ent in sd.get('state', {}).items():
            net, spec, is_w = plist[int(idx)]
            name = spec.wname if is_w else spec.bname
            bank = net._bank_of(name)
            if not bank.trainable:
                continue
            for key, buf in (('exp_avg', bank.exp_avg), ('exp_avg_sq', bank.exp_avg_sq)):
                dst = bank._view(buf, name)[i]
                if is_w:
                    spec.import_weight(dst, ent[key])
                else:
                    dst.copy_(ent[key].detach().to('cpu', dst.dtype).reshape(-1))
            steps[bank] = max(steps.get(bank, 0), int(float(ent['step'])))
        return steps

    def resume(self, checkpoint_dir, hyperparameters):
        """Load the latest per-member checkpoints (:898-967); returns the iteration parsed from the file name."""
        self._flush()
        iterations = 0
        # the flat Adam keeps ONE step count per family for the main banks (the reference: one per parameter, all equal in practice)
        # and one per style-encoder bank, whose parameters have state only once recon_s_w has given them a gradient
        steps = {}
        sty_steps = {}
        for d in self._dirs:
            sb = self._nets['gen_' + d].sty_bank
            if sb.trainable:  # a checkpoint without style-encoder entries (written with the term off) starts its moments at zero
                sb.exp_avg, sb.exp_avg_sq, sb.step = self.ops.zeros(sb.total), self.ops.zeros(sb.total), 0
                sty_steps[sb] = 0
        for i in range(self.council_size):
            for fam in ('gen', 'dis', 'dis_council'):
                if fam == 'dis_council' and not self.do_dis_council:
                    continue
                last = get_model_list(checkpoint_dir, '%s_%d' % (fam, i))
                if last is None:
                    import warnings
                    warnings.warn('Failed to find %s checkpoint, did not load model' % fam)
                    continue
                base = os.path.basename(last)
                for d in self._dirs:
                    path = os.path.join(checkpoint_dir, d + base[3:])
                    state = torch.load(path, map_location='cpu')
                    getattr(self, '%s_%s_s' % (fam, d))[i].load_state_dict(state[d])
                if fam == 'gen':
                    iterations = int(last[-11:-3])
            opt_path = os.path.join(checkpoint_dir, 'optimizer_%d.pt' % i)
            try:
                opt = torch.load(opt_path, map_location='cpu')
                for fam in ('dis', 'gen') + (('dis_council',) if self.do_dis_council else ()):
                    for bank, st in self._load_opt_state_dict(fam, i, opt[fam]).items():
                        if bank in sty_steps:
                            sty_steps[bank] = max(sty_steps[bank], st)
                        else:
                            steps[fam] = max(steps.get(fam, 0), st)
            except Exception as e:  # the reference warns and carries on as well (:958-959)
                import warnings
                warnings.warn('some optimizer FAILED to load (%s: %s): Adam moments restart from zero' % (type(e).__name__, e))
        for fam, st in steps.items():
            for d in self._dirs:
                self._nets['%s_%s' % (fam, d)].bank.step = st
        for bank, st in sty_steps.items():
            bank.step = st
        if iterations > 0:
            print('Resume from iteration %d' % iterations)
            for fam in self._sched_epoch:  # get_scheduler(..., last_epoch=iterations) :953-957
                self._sched_epoch[fam] = iterations
        else:
            import warnings
            warnings.warn('FAILED TO RESUME STARTED FROM 0')
        self.sync_parameters()
        return iterations
