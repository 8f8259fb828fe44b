"""The two populations ``ann_to_snn`` builds besides ``Input`` (reference: ``bindsnet/conversion/nodes.py``).  Like
every population of this package they hold state only; their step runs in the generic window kernel
(``SNN_NODE_SUBIF`` / ``SNN_NODE_PASSTHROUGH`` in include/snn_b200.h)."""
from __future__ import annotations

from typing import Iterable, Optional, Union

import torch

from .. import _abi
from ..network.nodes import Nodes, Scalar, _scalar


class SubtractiveResetIFNodes(Nodes):
    """Integrate-and-fire neurons with reset by subtraction (reference: conversion/nodes.py:8-121; forward :73-99).
    The input is integrated only while the refractory counter is exactly 0, the counter decreases only while it is
    positive, and a spike subtracts ``thresh`` from the voltage instead of resetting it."""

    kind = _abi.SNN_NODE_SUBIF

    def __init__(
        self,
        n: Optional[int] = None,
        shape: Optional[Iterable[int]] = None,
        traces: bool = False,
        traces_additive: bool = False,
        tc_trace: Scalar = 20.0,
        trace_scale: Scalar = 1.0,
        sum_input: bool = False,
        thresh: Scalar = -52.0,
        reset: Scalar = -65.0,
        refrac: Union[int, torch.Tensor] = 5,
        lbound: float = None,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )
        self.register_buffer("reset", torch.tensor(reset, dtype=torch.float))
        self.register_buffer("thresh", torch.tensor(thresh, dtype=torch.float))
        self.register_buffer("refrac", torch.tensor(refrac))
        self.register_buffer("v", torch.zeros(0))
        self.register_buffer("refrac_count", torch.zeros(0))
        self.lbound = lbound

    def reset_state_variables(self) -> None:
        """conversion/nodes.py:101-108."""
        super().reset_state_variables()
        self.v.fill_(self.reset)
        self.refrac_count.zero_()

    def set_batch_size(self, batch_size) -> None:
        """conversion/nodes.py:110-121."""
        super().set_batch_size(batch_size=batch_size)
        dev = self.v.device
        self.v = self.reset * torch.ones(batch_size, *self.shape, device=dev)
        self.refrac_count = torch.zeros_like(self.v)

    def _fill_desc(self, d) -> None:
        super()._fill_desc(d)
        d.reset = _scalar(self.reset, "reset")
        d.thresh = _scalar(self.thresh, "thresh")
        d.refrac = _scalar(self.refrac, "refrac")
        d.has_lbound = int(self.lbound is not None)
        d.lbound = _scalar(self.lbound, "lbound") if self.lbound is not None else 0.0


class PassThroughNodes(Nodes):
    """A population whose spikes are its input (reference: conversion/nodes.py:124-150; forward :137-144: ``s = x``).
    Its ``s`` is float32, as the reference's is after a step; the window kernel carries it as spikes and refuses inputs
    outside {0, 1}.  Its traces and summed input never change (the reference's forward never reaches Nodes.forward)."""

    kind = _abi.SNN_NODE_PASSTHROUGH

    def __init__(
        self,
        n: Optional[int] = None,
        shape: Optional[Iterable[int]] = None,
        traces: bool = False,
        traces_additive: bool = False,
        tc_trace: Scalar = 20.0,
        trace_scale: Scalar = 1.0,
        sum_input: bool = False,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )
        self.register_buffer("v", torch.zeros(self.shape))

    def reset_state_variables(self) -> None:
        """conversion/nodes.py:146-150: the spikes only."""
        self.s.zero_()

    def set_batch_size(self, batch_size) -> None:
        super().set_batch_size(batch_size=batch_size)
        self.s = self.s.float()

    def _fill_desc(self, d) -> None:
        super()._fill_desc(d)
        d.traces = d.sum_input = 0
