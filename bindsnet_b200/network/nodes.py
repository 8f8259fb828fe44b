"""Neuron populations — host-side mirror of ``bindsnet/network/nodes.py``.

These classes carry the same constructor signatures, attribute names and state tensors as
the reference (``Nodes`` nodes.py:9-162, ``Input`` :172-228, ``LIFNodes`` :418-559,
``DiehlAndCookNodes`` :981-1144) so that models written against BindsNET construct
unchanged.  They hold state only: the arithmetic of ``forward`` runs inside the CUDA
window kernels (``bindsnet_b200/csrc``), reached through ``Network.run`` or, for a single
population, through ``Nodes.forward`` which submits a one-layer, one-step window.
"""
from __future__ import annotations

from functools import reduce
from operator import mul
from typing import Iterable, Optional, Union

import torch

from .. import _abi

Scalar = Union[float, int, torch.Tensor]


def _exp_decay(dt: torch.Tensor, tc: torch.Tensor) -> torch.Tensor:
    """``exp(-dt / tc)`` evaluated on CPU fp32 tensors exactly as the reference does
    (nodes.py:129-131,546-548,1128-1133) so that the constants handed to the kernels are
    bit-identical to the reference's whatever device the layer lives on."""
    return torch.exp(-dt.detach().cpu().float() / tc.detach().cpu().float()).to(tc.device)


_SCALAR_CACHE: dict = {}


def _scalar(value: Scalar, name: str) -> float:
    """Host float of a (possibly device-resident) scalar parameter.  Reading a CUDA tensor costs a
    device synchronisation, so the value is cached per tensor object and version: building the
    plan of a window must not stall the stream the previous window is still running on."""
    if isinstance(value, torch.Tensor):
        if value.numel() != 1:
            raise NotImplementedError(
                f"per-neuron tensor for '{name}' is not supported by the CUDA core yet (scalar only)"
            )
        key = id(value)
        hit = _SCALAR_CACHE.get(key)
        if hit is not None and hit[0] is value and hit[1] == value._version:
            return hit[2]
        out = float(value.detach().cpu().reshape(()).item())
        if len(_SCALAR_CACHE) > 4096:
            _SCALAR_CACHE.clear()
        _SCALAR_CACHE[key] = (value, value._version, out)
        return out
    return float(value)


def _per_neuron(value) -> bool:
    """A parameter given as a tensor of more than one element (one element stays a scalar, whatever its shape)."""
    return isinstance(value, torch.Tensor) and value.numel() != 1


def _no_tensor_fill(value, name: str, op: str = "masked_fill_") -> None:
    """The reference writes ``refrac`` / ``reset`` / ``lbound`` / a non-additive ``trace_scale`` with ``masked_fill_`` and
    ``rest`` with ``fill_``, which take a 0-dim value only: its first step (or reset) raises this ``RuntimeError``."""
    if _per_neuron(value):
        if op == "fill_":
            raise RuntimeError(f"fill_ only supports 0-dimension value tensor but got tensor with {value.dim()} dimensions. "
                               f"('{name}' is a per-neuron tensor)")
        raise RuntimeError(f"masked_fill_ only supports a 0-dimensional value tensor, but got tensor with {value.dim()} "
                           f"dimension(s). ('{name}' is a per-neuron tensor)")


_ROW_CACHE: dict = {}


def _neuron_row(value: torch.Tensor, name: str, shape, device) -> torch.Tensor:
    """A per-neuron parameter as ``[n]`` fp32 on ``device``, cached per tensor object and version like ``_scalar``.  It
    must broadcast to the layer's shape without growing it (``[n]``, the full shape, or e.g. ``[C, 1, 1]`` of a
    ``[C, H, W]`` layer): the reference broadcasts it elementwise against ``[B, *shape]``."""
    shape = tuple(shape)
    try:
        out_shape = torch.broadcast_shapes(tuple(value.shape), shape)
    except RuntimeError as e:
        raise RuntimeError(f"per-neuron '{name}' of shape {tuple(value.shape)} does not broadcast to the layer's shape "
                           f"{shape}: {e}") from None
    if tuple(out_shape) != shape:
        raise NotImplementedError(f"per-neuron '{name}' of shape {tuple(value.shape)} broadcasts the layer's state {shape} "
                                  f"to {tuple(out_shape)}; the CUDA core keeps one value per neuron")
    key = (id(value), str(device))
    hit = _ROW_CACHE.get(key)
    if hit is not None and hit[0] is value and hit[1] == value._version:
        return hit[2]
    with torch.no_grad():
        row = value.detach().to(device, torch.float32).expand(shape).reshape(-1).contiguous()
    if len(_ROW_CACHE) > 4096:
        _ROW_CACHE.clear()
    _ROW_CACHE[key] = (value, value._version, row)
    return row


class Nodes(torch.nn.Module):
    """Base class of all populations (reference: nodes.py:9-162)."""

    kind: Optional[int] = None  # SNN_NODE_*; None = not executable by the CUDA core

    def __init__(
        self,
        n: Optional[int] = None,
        shape: Optional[Iterable[int]] = None,
        traces: bool = False,
        traces_additive: bool = False,
        tc_trace: Scalar = 20.0,
        trace_scale: Scalar = 1.0,
        sum_input: bool = False,
        learning: bool = True,
        **kwargs,
    ) -> None:
        super().__init__()
        assert n is not None or shape is not None, "Must provide either no. of neurons or shape of layer"
        self.n = int(reduce(mul, shape)) if n is None else int(n)
        self.shape = [self.n] if shape is None else list(shape)
        assert self.n == reduce(mul, self.shape), "No. of neurons and shape do not match"

        self.traces = traces
        self.traces_additive = traces_additive
        self.sum_input = sum_input
        self.register_buffer("s", torch.zeros(0, dtype=torch.bool))
        if self.traces:
            self.register_buffer("x", torch.zeros(0))
            self.register_buffer("tc_trace", torch.as_tensor(tc_trace, dtype=torch.float))
            self.register_buffer("trace_scale", torch.as_tensor(trace_scale, dtype=torch.float))
            self.register_buffer("trace_decay", torch.empty_like(self.tc_trace))
        if self.sum_input:
            self.register_buffer("summed", torch.zeros(0))
        self.dt = None
        self.batch_size = None
        self.learning = learning

    # -- reference API -------------------------------------------------------------------
    def forward(self, x: torch.Tensor) -> None:
        """One simulation step of this population alone (reference: ``Nodes.forward`` and
        its overrides).  ``x`` is the input of the step, shape ``[B, *shape]``.

        For the populations the CUDA core implements (``kind`` set) this submits a one-layer, one-step window.  For a
        USER-DEFINED population (a subclass that computes ``v`` / ``s`` itself with torch ops and then calls
        ``super().forward(x)``, the extension contract of docs/source/guide/guide_part_ii.rst:69-73) it is the
        reference's base behaviour — spike traces and summed input (nodes.py:96-107) — in torch ops on the layer's
        own device; ``Network.run`` drives such layers step by step (the scripted tier)."""
        if self.kind is not None:
            from . import _plan

            _plan.step_single_layer(self, x)
            return
        if self.traces:
            self.x *= self.trace_decay
            if self.traces_additive:
                self.x += self.trace_scale * self.s.float()
            else:
                self.x.masked_fill_(self.s.bool(), float(self.trace_scale))
        if self.sum_input:
            self.summed += x.float()

    def reset_state_variables(self) -> None:
        """nodes.py:109-120."""
        self.s.zero_()
        if self.traces:
            self.x.zero_()
        if self.sum_input:
            self.summed.zero_()

    def _reset_plan(self):
        """(tensors to zero, [(tensor, fill value)]) of ``reset_state_variables`` — lets
        ``Network.reset_state_variables`` clear a whole network with one multi-tensor launch."""
        zeros = [self.s]
        if self.traces:
            zeros.append(self.x)
        if self.sum_input:
            zeros.append(self.summed)
        return zeros, []

    def compute_decays(self, dt) -> None:
        """nodes.py:122-131."""
        self.dt = torch.tensor(dt)
        if self.traces:
            self.trace_decay = _exp_decay(self.dt, self.tc_trace)

    def set_batch_size(self, batch_size) -> None:
        """nodes.py:133-151 — (re)allocates, i.e. resets, the per-sample state."""
        self.batch_size = batch_size
        dev = self.s.device
        self.s = torch.zeros(batch_size, *self.shape, device=dev, dtype=torch.bool)
        if self.traces:
            self.x = torch.zeros(batch_size, *self.shape, device=dev)
        if self.sum_input:
            self.summed = torch.zeros(batch_size, *self.shape, device=dev)

    def train(self, mode: bool = True) -> "Nodes":
        """nodes.py:153-162."""
        self.learning = mode
        return super().train(mode)

    # -- plan export -----------------------------------------------------------------------
    def _fill_desc(self, d: "_abi.SnnLayer", rows: Optional[dict] = None) -> None:
        """``rows``: collects the per-neuron parameters (``{SNN_PN_*: (name, tensor)}``) of a population that runs them
        (``LIFNodes``, ``AdaptiveLIFNodes``, ``DiehlAndCookNodes``); without it a tensor parameter is refused."""
        if self.kind is None:
            raise NotImplementedError(
                f"{type(self).__name__} has no CUDA implementation in bindsnet_b200 "
                "(built in: Input, McCullochPitts, IFNodes, LIFNodes, BoostedLIFNodes, CurrentLIFNodes, AdaptiveLIFNodes, "
                "DiehlAndCookNodes; a subclass with its own forward() runs on the scripted tier)"
            )
        d.kind = self.kind
        d.n = self.n
        d.traces = int(bool(self.traces))
        d.traces_additive = int(bool(self.traces_additive))
        d.sum_input = int(bool(self.sum_input))
        d.learning = int(bool(self.learning))
        d.dt = float(self.dt) if self.dt is not None else 1.0
        if self.traces:
            d.trace_decay = self._param(self.trace_decay, "tc_trace", _abi.SNN_PN_TRACE_DECAY, rows)
            if rows is not None and not self.traces_additive:
                _no_tensor_fill(self.trace_scale, "trace_scale")
            d.trace_scale = self._param(self.trace_scale, "trace_scale", _abi.SNN_PN_TRACE_SCALE, rows)

    @staticmethod
    def _param(value, name: str, row: int, rows: Optional[dict]) -> float:
        """The scalar field of a parameter; a per-neuron tensor goes to ``rows`` (its scalar field is then unused)."""
        if rows is not None and _per_neuron(value):
            rows[row] = (name, value)
            return 0.0
        return _scalar(value, name)

    def _fill_rows(self, d: "_abi.SnnLayer", rows: dict) -> None:
        """The per-neuron block of ``rows`` (include/snn_b200.h SNN_NODE_PN): ``[SNN_PN_ROWS, n]`` fp32 on the layer's
        device, rebuilt only when one of its tensors changed."""
        if not rows:
            return
        device = self.s.device
        key = (tuple(sorted((r, id(t), t._version) for r, (_, t) in rows.items())), str(device), self.n)
        cached = getattr(self, "_b200_pn", None)
        if cached is None or cached[0] != key:
            block = torch.zeros(_abi.SNN_PN_ROWS, self.n, dtype=torch.float32, device=device)
            for r, (name, t) in rows.items():
                block[r].copy_(_neuron_row(t, name, self.shape, device))
            mask = sum(1 << r for r in rows)
            cached = (key, block, mask, [t for _, t in rows.values()])
            self._b200_pn = cached
        d.kind = d.kind | _abi.SNN_NODE_PN
        d.pn, d.pn_mask = cached[1].data_ptr(), cached[2]


class AbstractInput:
    """Marker base of externally driven populations (reference: nodes.py:165-169)."""


class Input(Nodes, AbstractInput):
    """Population whose spikes are the user's input (reference: nodes.py:172-228)."""

    kind = _abi.SNN_NODE_INPUT

    def __init__(
        self,
        n: Optional[int] = None,
        shape: Optional[Iterable[int]] = None,
        traces: bool = False,
        traces_additive: bool = False,
        tc_trace: Scalar = 20.0,
        trace_scale: Scalar = 1.0,
        sum_input: bool = False,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )


class LIFNodes(Nodes):
    """Leaky integrate-and-fire population (reference: nodes.py:418-559)."""

    kind = _abi.SNN_NODE_LIF

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
        rest: Scalar = -65.0,
        reset: Scalar = -65.0,
        refrac: Scalar = 5,
        tc_decay: Scalar = 100.0,
        lbound: float = None,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )
        self.register_buffer("rest", torch.as_tensor(rest, dtype=torch.float))
        self.register_buffer("reset", torch.as_tensor(reset, dtype=torch.float))
        self.register_buffer("thresh", torch.as_tensor(thresh, dtype=torch.float))
        self.register_buffer("refrac", torch.as_tensor(refrac))
        self.register_buffer("tc_decay", torch.as_tensor(tc_decay, dtype=torch.float))
        self.register_buffer("decay", torch.zeros(()))
        self.register_buffer("v", torch.zeros(0))
        self.register_buffer("refrac_count", torch.zeros(0))
        self.lbound = None if lbound is None else torch.tensor(lbound, dtype=torch.float)

    def reset_state_variables(self) -> None:
        """nodes.py:531-538."""
        _no_tensor_fill(self.rest, "rest", "fill_")   # (raised before any state changes)
        super().reset_state_variables()
        self.v.fill_(self.rest)
        self.refrac_count.zero_()

    def _reset_plan(self):
        _no_tensor_fill(self.rest, "rest", "fill_")
        zeros, fills = super()._reset_plan()
        return zeros + [self.refrac_count], fills + [(self.v, self.rest)]

    def compute_decays(self, dt) -> None:
        """nodes.py:540-548."""
        super().compute_decays(dt=dt)
        self.decay = _exp_decay(self.dt, self.tc_decay)

    def set_batch_size(self, batch_size) -> None:
        """nodes.py:550-559."""
        super().set_batch_size(batch_size=batch_size)
        dev = self.v.device
        self.v = self.rest * torch.ones(batch_size, *self.shape, device=dev)
        self.refrac_count = torch.zeros_like(self.v)

    def _fill_desc(self, d) -> None:
        # per-neuron thresh / rest / tc_decay / traces on LIFNodes itself (not on CurrentLIFNodes)
        rows = {} if self.kind == _abi.SNN_NODE_LIF else None
        if rows is not None:
            for name in ("refrac", "reset", "lbound"):
                _no_tensor_fill(getattr(self, name), name)
        super()._fill_desc(d, rows)
        d.decay = self._param(self.decay, "tc_decay", _abi.SNN_PN_DECAY, rows)
        d.rest = self._param(self.rest, "rest", _abi.SNN_PN_REST, rows)
        d.reset = _scalar(self.reset, "reset")
        d.thresh = self._param(self.thresh, "thresh", _abi.SNN_PN_THRESH, rows)
        d.refrac = _scalar(self.refrac, "refrac")
        d.has_lbound = int(self.lbound is not None)
        d.lbound = _scalar(self.lbound, "lbound") if self.lbound is not None else 0.0
        if rows is not None:
            self._fill_rows(d, rows)


class DiehlAndCookNodes(Nodes):
    """LIF with adaptive threshold and optional one-spike-per-step arbitration
    (reference: nodes.py:981-1144)."""

    kind = _abi.SNN_NODE_DC

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
        rest: Scalar = -65.0,
        reset: Scalar = -65.0,
        refrac: Scalar = 5,
        tc_decay: Scalar = 100.0,
        theta_plus: Scalar = 0.05,
        tc_theta_decay: Scalar = 1e7,
        lbound: float = None,
        one_spike: bool = True,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )
        self.register_buffer("rest", torch.as_tensor(rest, dtype=torch.float))
        self.register_buffer("reset", torch.as_tensor(reset, dtype=torch.float))
        self.register_buffer("thresh", torch.as_tensor(thresh, dtype=torch.float))
        self.register_buffer("refrac", torch.as_tensor(refrac))
        self.register_buffer("tc_decay", torch.as_tensor(tc_decay, dtype=torch.float))
        self.register_buffer("decay", torch.zeros(()))
        self.register_buffer("theta_plus", torch.as_tensor(theta_plus, dtype=torch.float))
        self.register_buffer("tc_theta_decay", torch.as_tensor(tc_theta_decay, dtype=torch.float))
        self.register_buffer("theta_decay", torch.zeros(()))
        self.register_buffer("v", torch.zeros(0))
        self.register_buffer("theta", torch.zeros(*self.shape))
        self.register_buffer("refrac_count", torch.zeros(0))
        self.lbound = lbound
        self.one_spike = one_spike

    def reset_state_variables(self) -> None:
        """nodes.py:1113-1120 (AdaptiveLIFNodes :948-955) — ``theta`` is deliberately NOT reset."""
        _no_tensor_fill(self.rest, "rest", "fill_")   # (raised before any state changes)
        super().reset_state_variables()
        self.v.fill_(self.rest)
        self.refrac_count.zero_()

    def _reset_plan(self):
        _no_tensor_fill(self.rest, "rest", "fill_")
        zeros, fills = super()._reset_plan()
        return zeros + [self.refrac_count], fills + [(self.v, self.rest)]

    def compute_decays(self, dt) -> None:
        """nodes.py:1122-1133."""
        super().compute_decays(dt=dt)
        self.decay = _exp_decay(self.dt, self.tc_decay)
        self.theta_decay = _exp_decay(self.dt, self.tc_theta_decay)

    def set_batch_size(self, batch_size) -> None:
        """nodes.py:1135-1144."""
        super().set_batch_size(batch_size=batch_size)
        dev = self.v.device
        self.v = self.rest * torch.ones(batch_size, *self.shape, device=dev)
        self.refrac_count = torch.zeros_like(self.v)

    def _fill_desc(self, d) -> None:
        rows = {}
        for name in ("refrac", "reset", "lbound"):
            _no_tensor_fill(getattr(self, name), name)
        super()._fill_desc(d, rows)
        d.decay = self._param(self.decay, "tc_decay", _abi.SNN_PN_DECAY, rows)
        d.rest = self._param(self.rest, "rest", _abi.SNN_PN_REST, rows)
        d.reset = _scalar(self.reset, "reset")
        d.thresh = self._param(self.thresh, "thresh", _abi.SNN_PN_THRESH, rows)
        d.refrac = _scalar(self.refrac, "refrac")
        d.theta_plus = self._param(self.theta_plus, "theta_plus", _abi.SNN_PN_THETA_PLUS, rows)
        d.theta_decay = self._param(self.theta_decay, "tc_theta_decay", _abi.SNN_PN_THETA_DECAY, rows)
        self._fill_rows(d, rows)
        d.one_spike = int(bool(self.one_spike))
        d.has_lbound = int(self.lbound is not None)
        d.lbound = _scalar(self.lbound, "lbound") if self.lbound is not None else 0.0


def _unsupported(name: str, where: str):
    class _Unsupported(Nodes):
        __doc__ = f"``{name}`` (reference: {where}) — not on the accelerated path (SURVEY.md §8f)."

        def __init__(self, *args, **kwargs):
            raise NotImplementedError(
                f"{name} is outside the hot path bindsnet_b200 implements "
                "(Input, LIFNodes, DiehlAndCookNodes); see DESIGN.md 'Out of scope'"
            )

    _Unsupported.__name__ = name
    return _Unsupported


class IFNodes(Nodes):
    """Integrate-and-fire without leak (reference: nodes.py:308-415; forward :377-394)."""

    kind = _abi.SNN_NODE_IF

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
        refrac: Scalar = 5,
        lbound: float = None,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )
        self.register_buffer("reset", torch.as_tensor(reset, dtype=torch.float))
        self.register_buffer("thresh", torch.as_tensor(thresh, dtype=torch.float))
        self.register_buffer("refrac", torch.as_tensor(refrac))
        self.register_buffer("v", torch.zeros(0))
        self.register_buffer("refrac_count", torch.zeros(0))
        self.lbound = None if lbound is None else torch.tensor(lbound, dtype=torch.float)

    def reset_state_variables(self) -> None:
        """nodes.py:396-403."""
        super().reset_state_variables()
        self.v.fill_(self.reset)
        self.refrac_count.zero_()

    def set_batch_size(self, batch_size) -> None:
        """nodes.py:405-415."""
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


class CurrentLIFNodes(LIFNodes):
    """Current-based LIF: the input feeds a decaying synaptic current (reference: nodes.py:681-826; forward
    :770-791)."""

    kind = _abi.SNN_NODE_CURRENT_LIF

    def __init__(self, *args, tc_i_decay: Scalar = 2.0, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        self.register_buffer("tc_i_decay", torch.as_tensor(tc_i_decay, dtype=torch.float))
        self.register_buffer("i_decay", torch.zeros(()))
        self.register_buffer("i", torch.zeros(0))

    def reset_state_variables(self) -> None:
        """nodes.py:793-801."""
        super().reset_state_variables()
        self.i.zero_()

    def _reset_plan(self):
        zeros, fills = super()._reset_plan()
        return zeros + [self.i], fills

    def compute_decays(self, dt) -> None:
        """nodes.py:803-820."""
        super().compute_decays(dt=dt)
        self.i_decay = _exp_decay(self.dt, self.tc_i_decay)

    def set_batch_size(self, batch_size) -> None:
        """nodes.py:822-826."""
        super().set_batch_size(batch_size=batch_size)
        self.i = torch.zeros_like(self.v)

    def _fill_desc(self, d) -> None:
        super()._fill_desc(d)
        d.i_decay = _scalar(self.i_decay, "tc_i_decay")


class AdaptiveLIFNodes(DiehlAndCookNodes):
    """LIF with an adaptive threshold shared across the batch (reference: nodes.py:829-978).  Its ``forward``
    (:921-946) is ``DiehlAndCookNodes.forward`` without the one-spike arbitration, so it runs on the same kernels
    with ``one_spike`` off; only the constructor defaults differ (none, in fact)."""

    def __init__(
        self,
        n: Optional[int] = None,
        shape: Optional[Iterable[int]] = None,
        traces: bool = False,
        traces_additive: bool = False,
        tc_trace: Scalar = 20.0,
        trace_scale: Scalar = 1.0,
        sum_input: bool = False,
        rest: Scalar = -65.0,
        reset: Scalar = -65.0,
        thresh: Scalar = -52.0,
        refrac: Scalar = 5,
        tc_decay: Scalar = 100.0,
        theta_plus: Scalar = 0.05,
        tc_theta_decay: Scalar = 1e7,
        lbound: float = None,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive, tc_trace=tc_trace, trace_scale=trace_scale,
            sum_input=sum_input, thresh=thresh, rest=rest, reset=reset, refrac=refrac, tc_decay=tc_decay, theta_plus=theta_plus,
            tc_theta_decay=tc_theta_decay, lbound=lbound, one_spike=False,
        )


class BoostedLIFNodes(Nodes):
    """LIF without rest / reset / lower bound: voltages decay towards 0 and reset to 0 (reference: nodes.py:562-678;
    forward :620-647)."""

    kind = _abi.SNN_NODE_BOOSTED_LIF

    def __init__(
        self,
        n: Optional[int] = None,
        shape: Optional[Iterable[int]] = None,
        traces: bool = False,
        traces_additive: bool = False,
        tc_trace: Scalar = 20.0,
        trace_scale: Scalar = 1.0,
        sum_input: bool = False,
        thresh: Scalar = 13.0,
        refrac: Scalar = 5,
        tc_decay: Scalar = 100.0,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )
        self.register_buffer("thresh", torch.as_tensor(thresh, dtype=torch.float))
        self.register_buffer("refrac", torch.as_tensor(refrac))
        self.register_buffer("tc_decay", torch.as_tensor(tc_decay, dtype=torch.float))
        self.register_buffer("decay", torch.zeros(()))
        self.register_buffer("v", torch.zeros(0))
        self.register_buffer("refrac_count", torch.zeros(0))

    def reset_state_variables(self) -> None:
        """nodes.py:649-656."""
        super().reset_state_variables()
        self.v.fill_(0)
        self.refrac_count.zero_()

    def _reset_plan(self):
        zeros, fills = super()._reset_plan()
        return zeros + [self.v, self.refrac_count], fills

    def compute_decays(self, dt) -> None:
        """nodes.py:658-666."""
        super().compute_decays(dt=dt)
        self.decay = _exp_decay(self.dt, self.tc_decay)

    def set_batch_size(self, batch_size) -> None:
        """nodes.py:668-678."""
        super().set_batch_size(batch_size=batch_size)
        dev = self.v.device
        self.v = torch.zeros(batch_size, *self.shape, device=dev)
        self.refrac_count = torch.zeros_like(self.v)

    def _fill_desc(self, d) -> None:
        super()._fill_desc(d)
        d.decay = _scalar(self.decay, "tc_decay")
        d.thresh = _scalar(self.thresh, "thresh")
        d.refrac = _scalar(self.refrac, "refrac")


class McCullochPitts(Nodes):
    """McCulloch-Pitts neurons: the voltage IS the input of the step, a spike wherever it reaches the threshold; no
    memory, no refractory period (reference: nodes.py:231-305; forward :278-288)."""

    kind = _abi.SNN_NODE_MCP

    def __init__(
        self,
        n: Optional[int] = None,
        shape: Optional[Iterable[int]] = None,
        traces: bool = False,
        traces_additive: bool = False,
        tc_trace: Scalar = 20.0,
        trace_scale: Scalar = 1.0,
        sum_input: bool = False,
        thresh: Scalar = 1.0,
        **kwargs,
    ) -> None:
        super().__init__(
            n=n, shape=shape, traces=traces, traces_additive=traces_additive,
            tc_trace=tc_trace, trace_scale=trace_scale, sum_input=sum_input,
        )
        self.register_buffer("thresh", torch.as_tensor(thresh, dtype=torch.float))
        self.register_buffer("v", torch.zeros(0))

    def set_batch_size(self, batch_size) -> None:
        """nodes.py:297-305."""
        super().set_batch_size(batch_size=batch_size)
        self.v = torch.zeros(batch_size, *self.shape, device=self.v.device)

    def _fill_desc(self, d) -> None:
        super()._fill_desc(d)
        d.thresh = _scalar(self.thresh, "thresh")




class IzhikevichNodes(Nodes):
    """Izhikevich neurons with their built-in lateral matrix ``S`` (reference: nodes.py:1147-1316; forward :1262-1289).
    A fraction ``excitatory`` of the population (the first ``int(n * excitatory)`` neurons) is regular-spiking with
    positive outgoing ``S`` columns, the rest fast-spiking with negative ones; the per-neuron parameters are drawn at
    construction in the reference's order (excitatory ``r``, its ``S`` columns, inhibitory ``r``, its ``S`` columns), so a
    seeded construction gives the reference's population.  Per-neuron parameter tensors and a population-internal matrix
    are outside what the window kernels describe, so the class has no ``kind``: host torch code on the layer's device,
    scripted tier, everything built-in around it on its kernels."""

    def __init__(self, n: Optional[int] = None, shape: Optional[Iterable[int]] = None, traces: bool = False,
                 traces_additive: bool = False, tc_trace: Scalar = 20.0, trace_scale: Scalar = 1.0, sum_input: bool = False,
                 excitatory: float = 1, thresh: Scalar = 45.0, rest: Scalar = -65.0, lbound: float = None, **kwargs) -> None:
        super().__init__(n=n, shape=shape, traces=traces, traces_additive=traces_additive, tc_trace=tc_trace,
                         trace_scale=trace_scale, sum_input=sum_input)
        n = self.n
        self.register_buffer("rest", torch.tensor(rest))
        self.register_buffer("thresh", torch.tensor(thresh))
        self.lbound = lbound
        ex = int(n * min(max(excitatory, 0), 1))
        r_ex, S_ex = torch.rand(ex), 0.5 * torch.rand(n, ex)            # regular spiking (nodes.py:1203-1210, 1233-1239)
        r_in, S_in = torch.rand(n - ex), -torch.rand(n, n - ex)         # fast spiking (:1211-1218, 1241-1247)
        self.register_buffer("r", torch.cat((r_ex, r_in)))
        self.register_buffer("a", torch.cat((0.02 * torch.ones(ex), 0.02 + 0.08 * r_in)))
        self.register_buffer("b", torch.cat((0.2 * torch.ones(ex), 0.25 - 0.05 * r_in)))
        self.register_buffer("c", torch.cat((-65.0 + 15 * r_ex ** 2, -65.0 * torch.ones(n - ex))))
        self.register_buffer("d", torch.cat((8 - 6 * r_ex ** 2, 2 * torch.ones(n - ex))))
        self.register_buffer("S", torch.cat((S_ex, S_in), dim=1))
        self.register_buffer("excitatory", (torch.arange(n) < ex).byte())
        self.register_buffer("v", self.rest * torch.ones(n))
        self.register_buffer("u", self.b * self.v)

    def forward(self, x: torch.Tensor) -> None:
        self.v = torch.where(self.s, self.c, self.v)                    # last step's spikes: reset v, bump the recovery
        self.u = torch.where(self.s, self.u + self.d, self.u)
        if self.s.any():                                                # lateral input from the neurons that just fired
            x += torch.stack([self.S[:, fired].sum(dim=1) for fired in self.s])
        for _ in range(2):                                              # two half steps (:1276-1277)
            self.v += self.dt * 0.5 * (0.04 * self.v ** 2 + 5 * self.v + 140 - self.u + x)
        self.u += self.dt * self.a * (self.b * self.v - self.u)
        if self.lbound is not None:
            self.v.masked_fill_(self.v < self.lbound, self.lbound)
        self.s = self.v >= self.thresh
        super().forward(x)

    def reset_state_variables(self) -> None:
        super().reset_state_variables()
        self.v.fill_(self.rest)
        self.u = self.b * self.v

    def set_batch_size(self, batch_size) -> None:
        super().set_batch_size(batch_size=batch_size)
        self.v = self.rest * torch.ones(batch_size, *self.shape, device=self.v.device)
        self.u = self.b * self.v
CSRMNodes = _unsupported("CSRMNodes", "nodes.py:1319-1552")


class SRM0Nodes(Nodes):
    """Simplified spike-response neurons with escape noise (reference: nodes.py:1555-1701; forward :1642-1673):
    leaky voltage, input scaled by ``eps_0`` outside the refractory period, a spike with probability
    ``1 - exp(-rho_0 * exp((v - thresh) / d_thresh) * dt)`` per step.

    The spike draw is ``torch.rand_like`` — torch's generator on the layer's device, as in the reference — so there is
    no bit-reproducible kernel form to pin against an oracle: the class has no ``kind``, and a network that contains
    it runs on the scripted tier (``Network._run_scripted``), this ``forward`` as device-resident torch operations in
    the reference's order (so that one seed gives the reference's spikes on the CPU), everything built-in still on
    its kernels."""

    def __init__(self, n: Optional[int] = None, shape: Optional[Iterable[int]] = None, traces: bool = False,
                 traces_additive: bool = False, tc_trace: Scalar = 20.0, trace_scale: Scalar = 1.0, sum_input: bool = False,
                 thresh: Scalar = -50.0, rest: Scalar = -70.0, reset: Scalar = -70.0, refrac: Scalar = 5, tc_decay: Scalar = 10.0,
                 lbound: float = None, eps_0: Scalar = 1.0, rho_0: Scalar = 1.0, d_thresh: Scalar = 5.0, **kwargs) -> None:
        super().__init__(n=n, shape=shape, traces=traces, traces_additive=traces_additive, tc_trace=tc_trace,
                         trace_scale=trace_scale, sum_input=sum_input)
        for name, value in (("rest", rest), ("reset", reset), ("thresh", thresh), ("refrac", refrac), ("tc_decay", tc_decay),
                            ("decay", tc_decay), ("eps_0", eps_0), ("rho_0", rho_0), ("d_thresh", d_thresh)):
            self.register_buffer(name, torch.tensor(value))
        self.register_buffer("v", torch.FloatTensor())
        self.register_buffer("refrac_count", torch.FloatTensor())
        self.lbound = lbound

    def forward(self, x: torch.Tensor) -> None:
        self.v = self.decay * (self.v - self.rest) + self.rest
        self.v += (self.refrac_count <= 0).float() * self.eps_0 * x
        self.rho = self.rho_0 * torch.exp((self.v - self.thresh) / self.d_thresh)      # stochastic intensity
        self.s_prob = 1.0 - torch.exp(-self.rho * self.dt)
        self.refrac_count -= self.dt
        self.s = torch.rand_like(self.s_prob) < self.s_prob
        self.refrac_count.masked_fill_(self.s, self.refrac)
        self.v.masked_fill_(self.s, self.reset)
        if self.lbound is not None:
            self.v.masked_fill_(self.v < self.lbound, self.lbound)
        super().forward(x)

    def reset_state_variables(self) -> None:
        super().reset_state_variables()
        self.v.fill_(self.rest)
        self.refrac_count.zero_()

    def compute_decays(self, dt) -> None:
        super().compute_decays(dt=dt)
        self.decay = torch.exp(-self.dt / self.tc_decay)

    def set_batch_size(self, batch_size) -> None:
        super().set_batch_size(batch_size=batch_size)
        self.v = self.rest * torch.ones(batch_size, *self.shape, device=self.v.device)
        self.refrac_count = torch.zeros_like(self.v)
