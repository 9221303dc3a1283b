"""CPU oracle of pad_type: reflect  --  TEST INFRASTRUCTURE ONLY.

The reference's Conv2dBlock (networks.py:463-520) pads with ``nn.ReflectionPad2d(padding)`` when its ``pad_type`` is 'reflect' and
runs its convolution with padding 0.  ``padding(hp)`` runs ``council_oracle``'s blocks that way: while it is entered,
``council_oracle.conv_block`` pads the discriminators' layers (keys ``cnns.*``, MsImageDis / MsImageDisCouncil) as
``hp['dis']['pad_type']`` says and every generator layer (content and style encoders, decoder) as ``hp['gen']['pad_type']`` says;
'zero' keeps ``council_oracle``'s ``F.pad`` with zeros.  Every oracle trainer built on ``council_oracle`` (the recon, recon_x and
abs_beginning_end extensions included) reads its blocks through that name, so any of them runs under it.  Pinned against the
unmodified reference by ``oracle/make_golden_pad.py`` (tests/golden/*_reflect*.json).  Like the base oracle it is the checker, never
the product.
"""
from __future__ import annotations

import contextlib

import torch.nn.functional as F

import council_oracle as co


@contextlib.contextmanager
def padding(hp):
    """council_oracle.conv_block with the pad types of hp while the context is entered"""
    base = co.conv_block
    modes = {'gen': hp['gen']['pad_type'], 'dis': hp['dis']['pad_type']}
    assert set(modes.values()) <= {'zero', 'reflect'}, modes

    def conv_block(p, prefix, x, stride, pad, norm='none', act='relu', adain=None):
        if pad > 0 and modes['dis' if prefix.startswith('cnns.') else 'gen'] == 'reflect':
            x, pad = F.pad(x, (pad, pad, pad, pad), mode='reflect'), 0  # nn.ReflectionPad2d, networks.py:470
        return base(p, prefix, x, stride, pad, norm, act, adain)
    co.conv_block = conv_block
    try:
        yield
    finally:
        co.conv_block = base
