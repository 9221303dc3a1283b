"""CPU oracle of the discriminators' normalisation dis.norm ('in', 'ln')  --  TEST INFRASTRUCTURE ONLY.

MsImageDis (networks.py:40-44) and MsImageDisCouncil (networks.py:137-143) build layers 1 .. n_layer-1 of every scale as
``Conv2dBlock(..., norm=params['norm'], activation='lrelu')``: conv(pad(x)) + bias, then the norm, then LeakyReLU(0.2)
(networks.py:515-520).  Layer 0 and the final 1x1 convolutions have no norm.
  * 'in': nn.InstanceNorm2d(C) -- affine=False, no running statistics, biased variance, eps 1e-5 (F.instance_norm, which raises
    ValueError on a 1x1 map in training);
  * 'ln': the reference's LayerNorm (networks.py:659-686) -- per sample, mean and UNBIASED std over C*H*W, (x - mean) / (std + eps)
    with eps 1e-5, then * gamma[c] + beta[c].  Its parameters are 'cnns.<s>.<i>.norm.gamma' / '.norm.beta', listed before the
    block's conv weight and bias (Conv2dBlock registers norm before conv).

``normalising(hp)`` runs council_oracle's ms_dis / ms_dis_council that way while it is entered; every oracle trainer built on
council_oracle (dis_options_oracle's included) reads them through those names, and the blocks go through ``co.conv_block``, so
``pad_oracle.padding`` composes with it.  ``synth_all_states`` adds gamma ~ U(0,1) (LayerNorm.__init__'s draw) and a small non-zero
beta to the synthetic states.  Pinned against the unmodified reference by ``oracle/make_golden_dis_norm.py``
(tests/golden/*_dis_in*.json, *_dis_ln*.json).  Like the base oracle it is the checker, never the product.
"""
from __future__ import annotations

import contextlib
from collections import OrderedDict

import torch
import torch.nn.functional as F

import council_oracle as co

EPS = 1e-5
_synth_base = co.synth_all_states  # synth_all_states below may stand in for it (oracle/make_golden_dis_norm.py)


def layer_norm(x, gamma, beta, eps=EPS):
    """LayerNorm.forward networks.py:673-686 (the batch-1 branch computes the same statistics over the one sample)"""
    shape = [-1] + [1] * (x.dim() - 1)
    if x.size(0) == 1:
        mean = x.view(-1).mean().view(*shape)
        std = x.view(-1).std().view(*shape)
    else:
        mean = x.view(x.size(0), -1).mean(1).view(*shape)
        std = x.view(x.size(0), -1).std(1).view(*shape)
    x = (x - mean) / (std + eps)
    shape = [1, -1] + [1] * (x.dim() - 2)
    return x * gamma.view(*shape) + beta.view(*shape)


def norm_block(p, prefix, x, stride, pad, norm):
    """Conv2dBlock(..., norm, 'lrelu').forward of layer `prefix` ('cnns.<s>.<i>')"""
    x = co.conv_block(p, prefix + '.conv', x, stride, pad, 'none', 'none')
    if norm == 'in':
        x = F.instance_norm(x, eps=EPS)
    elif norm == 'ln':
        x = layer_norm(x, p[prefix + '.norm.gamma'], p[prefix + '.norm.beta'])
    else:
        assert norm == 'none', norm
    return F.leaky_relu(x, 0.2)


def ms_dis(p, hp, x):
    """MsImageDis.forward networks.py:48-54 with dis.norm"""
    dp = hp['dis']
    outs = []
    for s in range(dp['num_scales']):
        h = co.conv_block(p, 'cnns.%d.0.conv' % s, x, 2, 1, 'none', 'lrelu')
        for i in range(1, dp['n_layer']):
            h = norm_block(p, 'cnns.%d.%d' % (s, i), h, 2, 1, dp['norm'])
        n = dp['n_layer']
        outs.append(F.conv2d(h, p['cnns.%d.%d.weight' % (s, n)], p['cnns.%d.%d.bias' % (s, n)]))
        x = co._avgpool(x)
    return outs


def ms_dis_council(p, hp, x, x_input):
    """MsImageDisCouncil.forward networks.py:147-156 with dis.norm"""
    dp = hp['dis']
    outs = []
    for s in range(dp['num_scales']):
        h = co.conv_block(p, 'cnns.%d.0.conv' % s, torch.cat((x, x_input), 1), 1, 1, 'none', 'lrelu')
        for i in range(1, dp['n_layer']):
            h = norm_block(p, 'cnns.%d.%d' % (s, i), h, 2, 1, dp['norm'])
        n = dp['n_layer']
        h = F.conv2d(h, p['cnns.%d.%d.weight' % (s, n)], p['cnns.%d.%d.bias' % (s, n)])
        outs.append(F.conv2d(h, p['cnns.%d.%d.weight' % (s, n + 1)], p['cnns.%d.%d.bias' % (s, n + 1)]))
        x = co._avgpool(x)
        x_input = co._avgpool(x_input)
    return outs


@contextlib.contextmanager
def normalising(hp):
    """council_oracle.ms_dis / ms_dis_council with hp's dis.norm while the context is entered"""
    assert hp['dis']['norm'] in ('none', 'in', 'ln'), hp['dis']['norm']
    base = co.ms_dis, co.ms_dis_council
    co.ms_dis, co.ms_dis_council = ms_dis, ms_dis_council
    try:
        yield
    finally:
        co.ms_dis, co.ms_dis_council = base


def dis_param_shapes(hp, council=False):
    """council_oracle.dis_param_shapes with the LayerNorm parameters of the normalised blocks, in the reference's key order"""
    out = []
    for key, shape in co.dis_param_shapes(hp, council):
        parts = key.split('.')
        if hp['dis']['norm'] == 'ln' and key.endswith('.conv.weight') and parts[2] != '0':
            prefix = key[:-len('.conv.weight')]
            out += [(prefix + '.norm.gamma', (shape[0],)), (prefix + '.norm.beta', (shape[0],))]
        out.append((key, shape))
    return out


def synth_all_states(hp, seed=7):
    """council_oracle.synth_all_states; under 'ln' every normalised block also gets gamma ~ U(0,1) (LayerNorm.__init__,
    networks.py:666) and beta ~ 0.01 N(0,1) (non-zero, to exercise it), one generator per tensor, in the reference's key order"""
    states = _synth_base(hp, seed)
    if hp['dis']['norm'] != 'ln':
        return states
    for ni, name in enumerate(sorted(states)):
        if not name.startswith('dis'):
            continue
        lst = states[name]
        shapes = dis_param_shapes(hp, name.startswith('dis_council'))
        for i, sd in enumerate(lst):
            full = OrderedDict()
            for n, (k, shape) in enumerate(shapes):
                if k in sd:
                    full[k] = sd[k]
                    continue
                gen = torch.Generator().manual_seed(seed * 100003 + 1000 * ni + 50 * i + n)
                full[k] = torch.rand(shape, generator=gen) if k.endswith('.gamma') else torch.randn(shape, generator=gen) * 0.01
            lst[i] = full
    return states
