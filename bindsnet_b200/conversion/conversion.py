"""ANN-to-SNN conversion (reference: ``bindsnet/conversion/conversion.py``): a trained ``torch.nn`` model becomes a
``Network`` of ``SubtractiveResetIFNodes`` (one per ``nn.Linear`` / ``nn.Conv2d``) and ``PassThroughNodes`` (one per
``nn.MaxPool2d``), optionally after rescaling its weights on sample data so that the chosen percentile of every ReLU's
activations is 1.  The result runs on the generic window kernel like any other ``Network``; its pooling connections
need learning off (``network.train(False)``), as in the reference.

The reference's behaviour is kept where it is peculiar: layer names count the ANN's children (ReLU and Flatten
included), so they skip numbers and a connection key's source may name no layer; ``nn.Linear`` weights are handed over
as ``weight.t()``; an ``nn.Conv2d`` without bias gets a zero bias of the output *height*, which fails (RuntimeError) when
the network's plan is built unless height and channel count agree; and a ``Permute`` or ``nn.ConstantPad2d`` raises
``TypeError`` because its connection cannot be constructed.
"""
from __future__ import annotations

import warnings
from copy import deepcopy
from typing import Dict, Optional, Sequence, Union

import numpy as np
import torch
import torch.nn as nn
from torch.nn.modules.utils import _pair

from ..network import Network
from ..network import nodes as _nodes
from ..network import topology as _topology
from .nodes import PassThroughNodes, SubtractiveResetIFNodes
from .topology import ConstantPad2dConnection, PermuteConnection


class Permute(nn.Module):
    """``x.permute(*dims).contiguous()`` as a module (reference: conversion.py:15-42)."""

    def __init__(self, dims):
        super().__init__()
        self.dims = dims

    def forward(self, x):
        return x.permute(*self.dims).contiguous()


class FeatureExtractor(nn.Module):
    """The output of every direct child of ``submodule`` on one input, keyed by the child's name, plus ``"input"``
    (reference: conversion.py:45-79).  An ``nn.Linear`` child gets its input flattened to ``[-1, in_features]``."""

    def __init__(self, submodule):
        super().__init__()
        self.submodule = submodule

    def forward(self, x: torch.Tensor) -> Dict[str, torch.Tensor]:
        out = {"input": x}
        for name, module in self.submodule._modules.items():
            if isinstance(module, nn.Linear):
                x = x.view(-1, module.in_features)
            x = module(x)
            out[name] = x
        return out


def data_based_normalization(ann: Union[nn.Module, str], data: torch.Tensor, percentile: float = 99.9):
    """Rescale ``ann`` in place so that the ``percentile`` of every ReLU's activations on ``data`` is 1 (reference:
    conversion.py:82-155): at each ReLU that follows an ``nn.Linear`` / ``nn.Conv2d``, with ``p`` the percentile of that
    ReLU's output and ``f`` the previous such factor (1 at first), the weight is multiplied by ``f / p`` and the bias
    divided by ``p``.  The children of a top-level ``nn.Sequential`` are visited one level down, on activations computed
    from ``data`` by that Sequential alone; after it, the checks of the top level see its LAST child, and a top-level
    ``nn.Linear`` rescales with the activations of the module visited before it — both as in the reference."""
    if isinstance(ann, str):
        ann = torch.load(ann)
    assert isinstance(ann, nn.Module)
    for p in ann.parameters():
        p.requires_grad = False

    prev_module, prev_factor = None, 1
    activations = None

    def rescale(acts):
        nonlocal prev_factor
        scale = np.percentile(acts.cpu(), percentile)
        prev_module.weight *= prev_factor / scale
        prev_module.bias /= scale
        prev_factor = scale

    top = FeatureExtractor(ann).forward(data)
    for name, module in ann._modules.items():
        if isinstance(module, nn.Sequential):
            inner = FeatureExtractor(module).forward(data)
            for name2, child in module.named_children():
                activations = inner[name2]
                if isinstance(child, nn.ReLU):
                    if prev_module is not None:
                        rescale(activations)
                elif isinstance(child, (nn.Linear, nn.Conv2d)):
                    prev_module = child
                module = child
        if isinstance(module, nn.Linear):
            if prev_module is not None:
                rescale(activations)
        else:
            activations = top[name]
            if isinstance(module, nn.ReLU):
                if prev_module is not None:
                    rescale(activations)
            elif isinstance(module, (nn.Linear, nn.Conv2d)):
                prev_module = module
    return ann


def _out_hw(prev, module):
    """The reference's output size of a convolution or pooling: ``int((size - kernel + 2 * padding) / stride + 1)``
    (no dilation) on the previous layer's [C, H, W]."""
    (kh, kw), (ph, pw), (sh, sw) = module.kernel_size, module.padding, module.stride
    return int((prev.shape[1] - kh + 2 * ph) / sh + 1), int((prev.shape[2] - kw + 2 * pw) / sw + 1)


def _convert(prev, module, node_type, last: bool = False, **kwargs):
    """The (layer, connection) one ANN child becomes, or (None, None) for a child without a counterpart (ReLU,
    Flatten, ...).  Reference: conversion.py:158-264."""
    if isinstance(module, nn.Linear):
        layer = node_type(n=module.out_features, reset=0, thresh=1, refrac=0, sum_input=last, **kwargs)
        bias = module.bias if module.bias is not None else torch.zeros(layer.n)
        return layer, _topology.Connection(source=prev, target=layer, w=module.weight.t(), b=bias)
    if isinstance(module, nn.Conv2d):
        layer = node_type(shape=(module.out_channels, *_out_hw(prev, module)), reset=0, thresh=1, refrac=0, sum_input=last,
                          **kwargs)
        bias = module.bias if module.bias is not None else torch.zeros(layer.shape[1])
        conn = _topology.Conv2dConnection(source=prev, target=layer, kernel_size=module.kernel_size, stride=module.stride,
                                          padding=module.padding, dilation=module.dilation, w=module.weight, b=bias)
        return layer, conn
    if isinstance(module, nn.MaxPool2d):
        module.kernel_size, module.padding, module.stride = _pair(module.kernel_size), _pair(module.padding), _pair(module.stride)
        layer = PassThroughNodes(shape=(prev.shape[0], *_out_hw(prev, module)))
        conn = _topology.MaxPool2dConnection(source=prev, target=layer, kernel_size=module.kernel_size, stride=module.stride,
                                             padding=module.padding, dilation=module.dilation, decay=1)
        return layer, conn
    if isinstance(module, Permute):
        layer = PassThroughNodes(shape=[prev.shape[d] for d in module.dims[:3]])
        return layer, PermuteConnection(source=prev, target=layer, dims=module.dims)
    if isinstance(module, nn.ConstantPad2d):
        p = module.padding
        layer = PassThroughNodes(shape=[prev.shape[0], p[0] + p[1] + prev.shape[1], p[2] + p[3] + prev.shape[2]])
        return layer, ConstantPad2dConnection(source=prev, target=layer, padding=module.padding)
    return None, None


def ann_to_snn(
    ann: Union[nn.Module, str],
    input_shape: Sequence[int],
    data: Optional[torch.Tensor] = None,
    percentile: float = 99.9,
    node_type: Optional[type] = SubtractiveResetIFNodes,
    **kwargs,
) -> Network:
    """Convert ``ann`` (a copy of it: the argument is left as it is) into a spiking ``Network`` (reference:
    conversion.py:267-345).  ``data`` (``[n_examples, ...]``): rescale the copy first with
    ``data_based_normalization``; without it a ``RuntimeWarning`` says that nothing is scaled.  The children of the
    model (those of a top-level ``nn.Sequential`` spliced in) are converted in order behind an ``Input`` layer named
    ``"Input"``; the layer made from child ``i`` (counting from 1) is named ``str(i)`` and fed by connection
    ``(str(i - 1), str(i))``.  The last child's layer sums its input (``sum_input=True``).  ``kwargs`` go to every
    ``node_type`` layer."""
    ann = torch.load(ann) if isinstance(ann, str) else deepcopy(ann)
    assert isinstance(ann, nn.Module)
    if data is None:
        warnings.warn("Data is None. Weights will not be scaled.", RuntimeWarning)
    else:
        ann = data_based_normalization(ann=ann, data=data.detach(), percentile=percentile)

    snn = Network()
    prev = _nodes.Input(shape=input_shape)
    snn.add_layer(prev, name="Input")
    children = []
    for c in ann.children():
        children += list(c.children()) if isinstance(c, nn.Sequential) else [c]
    for i, module in enumerate(children, start=1):
        layer, conn = _convert(prev, module, node_type, last=i == len(children), **kwargs)
        if layer is None and conn is None:
            continue
        snn.add_layer(layer, name=str(i))
        snn.add_connection(conn, source=str(i - 1), target=str(i))
        prev = layer
    return snn
