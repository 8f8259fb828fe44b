"""Synapse matrices — host-side mirror of ``bindsnet/network/topology.py``.

``Connection`` (reference: topology.py:265-399) and ``MulticompartmentConnection`` with a
``Weight`` feature (topology.py:402-537) keep the reference's constructor signatures and
attributes (``w``, ``b``, ``wmin``, ``wmax``, ``norm``, ``source``, ``target``,
``update_rule`` / ``pipeline``).  ``compute``/``update``/``normalize`` of a whole network run
inside the CUDA window kernels; the standalone methods below submit single-connection
work to the same kernels.
"""
from __future__ import annotations

import warnings
from abc import ABC
from typing import Optional, Sequence, Union

import numpy as np
import torch
from torch.nn import Module, Parameter

from .. import _abi
from .nodes import Nodes, _scalar


_TENSOR_FLAGS: dict = {}


def _tensor_flag(t: torch.Tensor, tag: str, fn) -> bool:
    """``fn(t)`` as a host bool, evaluated once per tensor object and version: reading a device tensor synchronises the
    stream, and building the plan of a window must not stall the window still running on it."""
    key = (tag, id(t))
    hit = _TENSOR_FLAGS.get(key)
    if hit is not None and hit[0] is t and hit[1] == t._version:
        return hit[2]
    with torch.no_grad():
        out = bool(fn(t))
    if len(_TENSOR_FLAGS) > 4096:
        _TENSOR_FLAGS.clear()
    _TENSOR_FLAGS[key] = (t, t._version, out)
    return out


def bounds_clamp(wmin: torch.Tensor, wmax: torch.Tensor) -> bool:
    """learning.py:97-104: the base update clamps when some element of ``wmin`` is not -inf or some element of ``wmax``
    is not +inf (scalars or tensors)."""
    return _tensor_flag(wmin, "lo", lambda t: (t != -np.inf).any()) or _tensor_flag(wmax, "hi", lambda t: (t != np.inf).any())


def nu_any(nu: torch.Tensor, k: int) -> bool:
    """``nu[k].any()`` (the gate of PostPre's and WeightDependentPostPre's terms, learning.py:403, 410, 640, 645)."""
    return _tensor_flag(nu, f"any{k}", lambda t: t[k].any())


def synapse_tensor(t: torch.Tensor, ns: int, nt: int, device: torch.device, name: str, owner=None):
    """``(tensor, form)``: what the kernels read for a bound or rate tensor that broadcasts to ``w``'s ``[ns, nt]``
    (include/snn_b200.h SNN_SYN_*).  A per-target ``[nt]`` / ``[1, nt]``, a per-source ``[ns, 1]``, a one-element or a
    contiguous ``[ns, nt]`` tensor is read in place; any other layout is copied once to a contiguous ``[ns, nt]`` and the
    copy kept on ``owner`` until the tensor changes."""
    if t.device != device:
        raise RuntimeError(f"Expected all tensors to be on the same device, but found at least two devices, {device} and "
                           f"{t.device}! ({name} is on {t.device}, the weights on {device})")
    try:
        ok = tuple(torch.broadcast_shapes(tuple(t.shape), (ns, nt))) == (ns, nt)
    except RuntimeError:
        ok = False
    if not ok:
        raise RuntimeError(f"The size of {name} {list(t.shape)} does not broadcast to the weights' size [{ns}, {nt}]")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    e = t.detach().expand(ns, nt)
    s0 = 0 if ns == 1 else e.stride(0)
    s1 = 0 if nt == 1 else e.stride(1)
    form = {(0, 0): _abi.SNN_SYN_ONE, (0, 1): _abi.SNN_SYN_TGT, (1, 0): _abi.SNN_SYN_SRC, (nt, 1): _abi.SNN_SYN_FULL}.get((s0, s1))
    if form is not None:
        return e, form
    key = (t.data_ptr(), t._version, tuple(t.shape), tuple(t.stride()))
    cache = owner.__dict__.setdefault("_b200_syn_copies", {}) if owner is not None else {}
    hit = cache.get(name)
    if hit is None or hit[0] != key:
        hit = (key, e.contiguous(), t)
        cache[name] = hit
    return hit[1], _abi.SNN_SYN_FULL


def fill_synapse_tensors(d: "_abi.SnnConn", ns: int, nt: int, device: torch.device, wmin: torch.Tensor, wmax: torch.Tensor,
                         nu: Optional[torch.Tensor], owner=None) -> None:
    """The per-synapse fields of a dense connection's plan entry (include/snn_b200.h): each bound that is a tensor of
    more than one element, and ``nu`` (``torch.stack`` of the rule's two rates) when its rates are tensors; ``d.rule``
    is set already.  The scalar fields of a tensor are left as the kernels ignore them, except the rates' gates."""
    for name, t in (("wmin", wmin), ("wmax", wmax), ("nu", nu)):
        if t is not None and t.numel() != 1 and t.device != device:   # the reference's first update fails on it
            raise RuntimeError(f"Expected all tensors to be on the same device, but found at least two devices, {device} and "
                               f"{t.device}! ({name} is on {t.device}, the weights on {device})")
    if d.rule == _abi.SNN_RULE_WDEP_POSTPRE:
        # WeightDependentPostPre multiplies every synapse's term by (w - wmin) / (wmax - w), including the zero terms of
        # silent synapses (learning.py:640-649): an infinite bound turns them into NaN.  With scalar bounds the rule's
        # constructor asserts finite ones; an infinite element of a bound tensor is refused here
        gates = (d.nu0 != 0.0, d.nu1 != 0.0) if nu is None else (nu_any(nu, 0), nu_any(nu, 1))
        for gate, t, name in ((gates[0], wmin, "wmin"), (gates[1], wmax, "wmax")):
            if gate and _tensor_flag(t, "inf", lambda v: torch.isinf(v).any()):
                raise NotImplementedError(f"WeightDependentPostPre with an infinite element of {name}: the reference's update turns "
                                          "every weight of such a synapse into NaN (learning.py:640-649); use finite bounds")
    for name, t, ptr, form in (("wmin", wmin, "wmin_t", "wmin_form"), ("wmax", wmax, "wmax_t", "wmax_form")):
        if t.numel() != 1:
            v, f = synapse_tensor(t, ns, nt, device, name, owner)
            setattr(d, ptr, v.data_ptr())
            setattr(d, form, f)
    if nu is None:
        return
    pair = (nu[0], nu[1])
    gates = [nu_any(nu, 0), nu_any(nu, 1)]
    if d.rule == _abi.SNN_RULE_POSTPRE:
        # PostPre scales the target traces / spikes by nu before torch.bmm (learning.py:403-417): a rate that does not
        # broadcast to [1, n_tgt] makes the bmm fail once its term runs
        for k, r in enumerate(pair):
            if gates[k] and (r.dim() > 2 or (r.dim() == 2 and r.shape[0] != 1) or (r.dim() >= 1 and r.shape[-1] not in (1, nt))):
                raise RuntimeError(f"PostPre: nu[{k}] of shape {list(r.shape)} does not broadcast to [1, {nt}]: torch.bmm fails on "
                                   f"it (Expected size for first two dimensions of batch2 tensor to be: [B, 1] but got: [B, {ns}])")
    if d.rule == _abi.SNN_RULE_HEBBIAN:
        gates = [True, True]   # learning.py:1124-1134 applies both rates without a gate
    if d.rule in (_abi.SNN_RULE_POSTPRE, _abi.SNN_RULE_WDEP_POSTPRE) and not any(gates):
        d.nu0 = d.nu1 = 0.0    # neither term runs: nothing to read
        return
    v0, f0 = synapse_tensor(pair[0], ns, nt, device, "nu[0]", owner)
    v1, f1 = synapse_tensor(pair[1], ns, nt, device, "nu[1]", owner)
    d.nu0_t, d.nu0_form, d.nu1_t, d.nu1_form = v0.data_ptr(), f0, v1.data_ptr(), f1
    d.nu0, d.nu1 = float(gates[0]), float(gates[1])


class AbstractConnection(ABC, Module):
    """Reference: topology.py:17-156."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        **kwargs,
    ) -> None:
        super().__init__()
        assert isinstance(source, Nodes), "Source is not a Nodes object"
        assert isinstance(target, Nodes), "Target is not a Nodes object"
        self.source = source
        self.target = target
        self.weight_decay = weight_decay
        self.reduction = reduction

        from ..learning import NoOp

        self.wmin = Parameter(torch.as_tensor(kwargs.get("wmin", -np.inf), dtype=torch.float32), requires_grad=False)
        self.wmax = Parameter(torch.as_tensor(kwargs.get("wmax", np.inf), dtype=torch.float32), requires_grad=False)
        self.norm = kwargs.get("norm", None)
        self.decay = kwargs.get("decay", None)
        if kwargs.get("Dales_rule", None) is not None:
            raise NotImplementedError("Dales_rule is not implemented by the CUDA core (DESIGN.md 'Out of scope')")
        self.Dales_rule = None

        rule_cls = kwargs.get("update_rule", None) or NoOp
        self.update_rule = rule_cls(connection=self, nu=nu, reduction=reduction, weight_decay=weight_decay, **kwargs)

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        raise NotImplementedError

    def update(self, **kwargs) -> None:
        """topology.py:112-139: apply the learning rule to the current layer state."""
        if kwargs.get("learning", True):
            self.update_rule.update(**kwargs)
        mask = kwargs.get("mask", None)
        if mask is not None:                                              # topology.py:127-131
            self.w.masked_fill_(mask.to(self.w.device).bool(), 0)

    def reset_state_variables(self) -> None:
        pass

    @staticmethod
    def cast_dtype_if_needed(w, w_dtype):
        if w.dtype != w_dtype:
            warnings.warn(f"Provided w has data type {w.dtype} but parameter w_dtype is {w_dtype}")
            return w.to(dtype=w_dtype)
        return w


class Connection(AbstractConnection):
    """Dense all-to-all synapses (reference: topology.py:265-399)."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        w_dtype: torch.dtype = torch.float32,
        **kwargs,
    ) -> None:
        if w_dtype != torch.float32:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
        super().__init__(source, target, nu, reduction, weight_decay, **kwargs)
        w = kwargs.get("w", None)
        if w is None:
            # topology.py:308-313
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(torch.rand(source.n, target.n), self.wmin, self.wmax)
            else:
                w = self.wmin + torch.rand(source.n, target.n) * (self.wmax - self.wmin)
            w = w.to(dtype=w_dtype)
        else:
            # topology.py:314-317
            if (self.wmin != -np.inf).any() or (self.wmax != np.inf).any():
                w = torch.clamp(torch.as_tensor(w), self.wmin, self.wmax)
            w = self.cast_dtype_if_needed(torch.as_tensor(w), w_dtype)
        self.w = Parameter(w.detach().clone().contiguous(), requires_grad=False)
        b = kwargs.get("b", None)
        self.b = Parameter(torch.as_tensor(b, dtype=torch.float32), requires_grad=False) if b is not None else None

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """``s.float() @ w (+ b)`` through the CUDA spike-gather (reference: topology.py:332-346)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def normalize(self) -> None:
        """topology.py:383-392."""
        if self.norm is not None:
            from . import _plan

            _plan.normalize_single_connection(self)

    # per-synapse wmin / wmax and learning-rate tensors run on the generic kernel (LocalConnection and SparseConnection
    # keep scalars)
    _synapse_tensors = True
    # a norm tensor with one value per target neuron runs on the generic kernel (LocalConnection and SparseConnection
    # keep scalars)
    _tensor_norms = True

    def _norm_tensor(self) -> Optional[torch.Tensor]:
        """A tensor ``norm`` as float32 ``[target.n]`` (``w *= norm / |w|.sum(0)``, topology.py:383-392, a true division),
        or None for a number.  A 0-d or one-element norm divides like the scalar path and is read as a number."""
        if not isinstance(self.norm, torch.Tensor) or not self._tensor_norms:
            return None
        if self.norm.dtype == torch.float32 and tuple(self.norm.shape) in ((), (1,)):
            return None
        from . import _plan

        return _plan.norm_tensor(self, self.target.n, self.w.device)

    # -- plan export -----------------------------------------------------------------------
    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        d.kind = _abi.SNN_CONN_DENSE
        tensors = self.wmin.numel() != 1 or self.wmax.numel() != 1
        if tensors and not self._synapse_tensors:
            raise NotImplementedError(f"per-synapse wmin/wmax tensors are not supported by the CUDA core on a {type(self).__name__}")
        d.wmin = _scalar(self.wmin, "wmin") if self.wmin.numel() == 1 else -np.inf
        d.wmax = _scalar(self.wmax, "wmax") if self.wmax.numel() == 1 else np.inf
        d.has_norm = int(self.norm is not None)
        d.norm_abs = 1
        d.norm = float(self.norm) if self.norm is not None and self._norm_tensor() is None else 0.0
        d.dt_scale = 1.0
        if rule:
            self.update_rule._fill_desc(d)
            nu = self.update_rule.nu if getattr(self.update_rule, "_nu_tensors", False) else None
            if tensors or nu is not None:
                fill_synapse_tensors(d, self.source.n, self.target.n, self.w.device, self.wmin, self.wmax, nu, owner=self)
                if nu is not None and d.rule == _abi.SNN_RULE_MSTDPET:
                    d.dt_scale = float(getattr(self, "dt", dt))   # the kernel scales each rate: ((nu * dt) * reward) * e_trace


def _pair(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x, x)


class Conv2dConnection(AbstractConnection):
    """2-D convolutional synapses (reference: topology.py:686-844).  ``w`` is
    ``[out_channels, in_channels, kh, kw]``, ``b`` ``[out_channels]`` (zeros by default, :795-797);
    source / target populations are ``[C, H, W]`` shaped.  Inside ``Network.run`` the convolution is a
    spike-gather over each target neuron's receptive field; ``MSTDP`` is the learning rule the CUDA
    core fuses for it (learning.py:1942-2015)."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        kernel_size,
        stride=1,
        padding=0,
        dilation=1,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        w_dtype: torch.dtype = torch.float32,
        **kwargs,
    ) -> None:
        if w_dtype != torch.float32:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
        # geometry first: the learning rule built by the base constructor looks at it
        self_kernel, self_stride = _pair(kernel_size), _pair(stride)
        self_padding, self_dilation = _pair(padding), _pair(dilation)
        assert len(source.shape) == 3 and len(target.shape) == 3, "Conv2dConnection needs [C, H, W] populations"
        in_channels, input_height, input_width = source.shape
        out_channels = target.shape[0]
        # topology.py:752-772 (the reference swaps the names width / height; the values are these)
        out_h = int((input_height - self_kernel[0] + 2 * self_padding[0]) / self_stride[0] + 1)
        out_w = int((input_width - self_kernel[1] + 2 * self_padding[1]) / self_stride[1] + 1)
        assert target.shape[1] == out_h and target.shape[2] == out_w, (
            "Target dimensionality must be (out_channels, ?,"
            "(input_height - filter_height + 2 * padding_height) / stride_height + 1,"
            "(input_width - filter_width + 2 * padding_width) / stride_width + 1"
        )
        object.__setattr__(self, "_geometry", (self_kernel, self_stride, self_padding, self_dilation))
        super().__init__(source, target, nu, reduction, weight_decay, **kwargs)
        self.kernel_size, self.stride, self.padding, self.dilation = self_kernel, self_stride, self_padding, self_dilation
        self.in_channels, self.out_channels = int(in_channels), int(out_channels)
        w = kwargs.get("w", None)
        shape = (self.out_channels, self.in_channels, *self.kernel_size)
        if w is None:
            # topology.py:775-786
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(torch.rand(*shape), self.wmin, self.wmax)
            else:
                w = (self.wmax - self.wmin) * torch.rand(*shape)
                w = w + self.wmin
        else:
            # topology.py:787-790
            w = torch.as_tensor(w)
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(w, self.wmin, self.wmax)
            w = self.cast_dtype_if_needed(w, w_dtype)
        assert tuple(w.shape) == shape, f"w must have shape {shape}"
        self.w = Parameter(w.detach().clone().float().contiguous(), requires_grad=False)
        self.b = Parameter(torch.as_tensor(kwargs.get("b", torch.zeros(self.out_channels)), dtype=torch.float32).clone(),
                           requires_grad=False)

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """``F.conv2d(s.float(), w, b, stride, padding, dilation)`` for {0,1} spikes (topology.py:799-815), as the
        spike-gather the window kernels use (``snn_b200_conn_compute``)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def normalize(self) -> None:
        """Every (out, in) filter scaled to sum ``norm`` (topology.py:824-837); also runs at the end of every
        ``Network.run`` window."""
        if self.norm is not None:
            from . import _plan

            _plan.normalize_single_connection(self)

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        d.kind = _abi.SNN_CONN_CONV2D
        if self.wmin.numel() != 1 or self.wmax.numel() != 1:
            raise NotImplementedError("per-synapse wmin/wmax tensors are not supported by the CUDA core yet")
        d.wmin = _scalar(self.wmin, "wmin")
        d.wmax = _scalar(self.wmax, "wmax")
        d.has_norm = int(self.norm is not None)
        d.norm_abs = 0
        d.norm = float(self.norm) if self.norm is not None else 0.0
        d.dt_scale = 1.0
        d.cin, d.hin, d.win = (int(v) for v in self.source.shape)
        d.cout, d.hout, d.wout = (int(v) for v in self.target.shape)
        d.kh, d.kw = self.kernel_size
        d.sh, d.sw = self.stride
        d.ph, d.pw = self.padding
        d.dh, d.dw = self.dilation
        if rule:
            self.update_rule._fill_desc(d)


class Conv1dConnection(AbstractConnection):
    """1-D convolutional synapses (reference: topology.py:540-683) between ``[C, L]`` populations.  ``w`` is
    ``[out_channels, in_channels, kernel_size]``, ``b`` ``[out_channels]`` (zeros by default).  Inside ``Network.run`` the
    convolution is a spike-gather over each target neuron's receptive field, and ``PostPre``, ``WeightDependentPostPre``,
    ``Hebbian`` or ``NoOp`` update ``w`` on the generic window kernel; ``normalize`` scales every ``(out, in)`` filter to
    sum ``norm``.

    As in the reference: a dilation other than 1 raises ``NotImplementedError``; a target whose shape is not
    ``[out_channels, int((L - k + 2p) / s + 1)]`` raises ``AssertionError``; ``w`` is drawn with ``torch.rand`` and clamped
    or scaled like ``Conv2dConnection``'s.  The rules' update follows the reference's reshape of the unfolded source,
    which for ``in_channels > 1`` pairs a weight with another source neuron than ``compute`` does (include/snn_b200.h,
    SNN_CONN_CONV1D).  Only ``[C, L]`` source and target populations are built: any other shape raises
    ``NotImplementedError`` before anything else (the reference's ``F.conv1d`` cannot take the batch such a source gives;
    DESIGN.md section 8).  ``MSTDP`` / ``MSTDPET`` on it raise ``NotImplementedError``."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        kernel_size: int,
        stride: int = 1,
        padding: int = 0,
        dilation: int = 1,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        w_dtype: torch.dtype = torch.float32,
        **kwargs,
    ) -> None:
        for name, layer in (("source", source), ("target", target)):
            if not isinstance(layer, Nodes) or len(layer.shape) != 2:
                shape = list(layer.shape) if isinstance(layer, Nodes) else type(layer).__name__
                raise NotImplementedError(f"Conv1dConnection is built between [C, L] populations only; the {name} is {shape}")
        if w_dtype != torch.float32:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
        super().__init__(source, target, nu, reduction, weight_decay, **kwargs)
        if dilation != 1:                                                                   # topology.py:592-595
            raise NotImplementedError("Dilation is not currently supported for 1-D spiking convolution.")
        self.kernel_size, self.stride, self.padding, self.dilation = kernel_size, stride, padding, dilation
        self.in_channels, input_size = source.shape[0], source.shape[1]
        self.out_channels, output_size = target.shape[0], target.shape[1]
        conv_size = (input_size - self.kernel_size + 2 * self.padding) / self.stride + 1       # topology.py:605-613
        assert target.shape[0] == self.out_channels and target.shape[1] == int(conv_size), (
            "Target dimensionality must be (out_channels, ?,(input_size - filter_size + 2 * padding) / stride + 1,"
        )
        w = kwargs.get("w", None)
        shape = (self.out_channels, self.in_channels, self.kernel_size)
        if w is None:
            # topology.py:615-629
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(torch.rand(*shape), self.wmin, self.wmax)
            else:
                w = (self.wmax - self.wmin) * torch.rand(*shape)
                w = w + self.wmin
        else:
            # topology.py:630-633
            w = torch.as_tensor(w)
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(w, self.wmin, self.wmax)
            w = self.cast_dtype_if_needed(w, w_dtype)
        self.w = Parameter(w.detach().clone().float().contiguous(), requires_grad=False)
        self.b = Parameter(torch.as_tensor(kwargs.get("b", torch.zeros(self.out_channels)), dtype=torch.float32).clone(),
                           requires_grad=False)

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """``F.conv1d(s.float(), w, b, stride, padding)`` for {0,1} spikes (topology.py:640-656), as the spike-gather the
        window kernel uses (``snn_b200_conn_compute``)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def normalize(self) -> None:
        """Every (out, in) filter scaled to sum ``norm`` (topology.py:665-676; a filter that sums to zero becomes
        inf / NaN, as in the reference); also runs at the end of every ``Network.run`` window."""
        if self.norm is not None:
            from . import _plan

            _plan.normalize_single_connection(self)

    def _check(self) -> None:
        """The errors of the reference's first ``compute`` (F.conv1d), raised before anything runs."""
        if int(self.target.shape[1]) == 0 or int(self.target.shape[0]) == 0:
            raise RuntimeError(f"Conv1dConnection: calculated output size {list(self.target.shape)} is too small (kernel "
                               f"{self.kernel_size}, padded input {int(self.source.shape[1]) + 2 * self.padding})")
        shape = (int(self.out_channels), int(self.in_channels), int(self.kernel_size))
        if tuple(self.w.shape) != shape:
            raise RuntimeError(f"Conv1dConnection.w has shape {tuple(self.w.shape)}, expected {shape}")
        if tuple(self.b.shape) != (shape[0],):
            raise RuntimeError(f"Given weight of size {list(self.w.shape)}, expected bias to be 1-dimensional with {shape[0]} "
                               f"elements, but got bias of size {list(self.b.shape)} instead")

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        self._check()
        d.kind = _abi.SNN_CONN_CONV1D
        if self.wmin.numel() != 1 or self.wmax.numel() != 1:
            raise NotImplementedError("per-synapse wmin/wmax tensors are not supported by the CUDA core yet")
        d.wmin = _scalar(self.wmin, "wmin")
        d.wmax = _scalar(self.wmax, "wmax")
        d.has_norm = int(self.norm is not None)
        d.norm_abs = 0
        d.norm = float(self.norm) if self.norm is not None else 0.0
        d.dt_scale = 1.0
        d.cin, d.win = (int(v) for v in self.source.shape)
        d.cout, d.wout = (int(v) for v in self.target.shape)
        d.kw, d.sw, d.pw = int(self.kernel_size), int(self.stride), int(self.padding)
        d.hin = d.hout = d.kh = d.sh = 1
        d.ph = 0
        d.dh = d.dw = 1
        if rule:
            self.update_rule._fill_desc(d)


def _triple(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x, x, x)


_MISSING = object()   # a required argument of the reference that was not passed (LocalConnection3D)


class Conv3dConnection(AbstractConnection):
    """3-D convolutional synapses (reference: topology.py:847-1025).  Source and target populations are
    ``[C, D, H, W]`` shaped; ``w`` is ``[out_channels, in_channels, kd, kh, kw]``, ``b`` ``[out_channels]`` (zeros by
    default).  Inside ``Network.run`` the convolution is a spike-gather over each target neuron's receptive field;
    ``normalize`` scales every ``(out, in)`` filter to sum ``norm``.

    As in the reference: a dilation other than 1 raises ``NotImplementedError``; a target whose shape is not
    ``[out_channels, D', H', W']`` with each size ``int((in - k + 2p) / s + 1)`` raises ``AssertionError``; ``w`` is drawn
    with ``torch.rand`` and clamped or scaled like ``Conv2dConnection``'s.  The reference's learning rules on this class
    multiply the bool source spikes by a float trace, which fails; so a learning window whose rule evaluates that
    pre-synaptic term (``PostPre`` / ``WeightDependentPostPre`` with ``nu[0] != 0``, ``Hebbian``, ``MSTDP``, ``MSTDPET``)
    raises the reference's ``RuntimeError`` before it starts.  ``NoOp`` decays ``w``; ``PostPre`` /
    ``WeightDependentPostPre`` with both rates zero decay and clamp it.  Their post-synaptic-only form pairs the kernel
    axes transposed against ``w`` (learning.py:517-530) and is refused when the rule is built (DESIGN.md section 8)."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        kernel_size,
        stride=1,
        padding=0,
        dilation=1,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        w_dtype: torch.dtype = torch.float32,
        **kwargs,
    ) -> None:
        if w_dtype != torch.float32:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
        super().__init__(source, target, nu, reduction, weight_decay, **kwargs)
        if dilation != 1 and dilation != (1, 1, 1):                                       # topology.py:899-903
            raise NotImplementedError("Dilation is not currently supported for 3-D spiking convolution.")
        self.kernel_size, self.stride = _triple(kernel_size), _triple(stride)
        self.padding, self.dilation = _triple(padding), _triple(dilation)
        self.in_channels, input_depth, input_height, input_width = (source.shape[0], source.shape[1], source.shape[2], source.shape[3])
        self.out_channels = target.shape[0]
        # topology.py:922-952 (the reference swaps the names width / height; the values are these)
        out = [int((i - k + 2 * p) / s + 1) for i, k, p, s in
               zip((input_depth, input_height, input_width), self.kernel_size, self.padding, self.stride)]
        assert target.shape[1] == out[0] and target.shape[2] == out[1] and target.shape[3] == out[2], (
            "Target dimensionality must be (out_channels, ?,"
            "(input_depth - filter_depth + 2 * padding_depth) / stride_depth + 1,"
            "(input_height - filter_height + 2 * padding_height) / stride_height + 1,"
            "(input_width - filter_width + 2 * padding_width) / stride_width + 1"
        )
        w = kwargs.get("w", None)
        shape = (self.out_channels, self.in_channels, *self.kernel_size)
        if w is None:
            # topology.py:954-968
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(torch.rand(*shape), self.wmin, self.wmax)
            else:
                w = (self.wmax - self.wmin) * torch.rand(*shape)
                w = w + self.wmin
        else:
            # topology.py:969-972
            w = torch.as_tensor(w)
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(w, self.wmin, self.wmax)
            w = self.cast_dtype_if_needed(w, w_dtype)
        self.w = Parameter(w.detach().clone().float().contiguous(), requires_grad=False)
        self.b = Parameter(torch.as_tensor(kwargs.get("b", torch.zeros(self.out_channels)), dtype=torch.float32).clone(),
                           requires_grad=False)

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """``F.conv3d(s.float(), w, b, stride, padding)`` for {0,1} spikes (topology.py:979-995), as the spike-gather the
        window kernel uses (``snn_b200_conn_compute``)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def normalize(self) -> None:
        """Every (out, in) filter scaled to sum ``norm`` (topology.py:1004-1018; a filter that sums to zero becomes
        inf / NaN, as in the reference); also runs at the end of every ``Network.run`` window."""
        if self.norm is not None:
            from . import _plan

            _plan.normalize_single_connection(self)

    def _check(self) -> None:
        """The errors of the reference's first ``compute`` (F.conv3d), raised before anything runs."""
        if any(int(v) == 0 for v in self.target.shape):
            k = "x".join(str(v) for v in self.kernel_size)
            raise RuntimeError(f"Conv3dConnection: calculated output size {list(self.target.shape)} is too small (kernel {k}, "
                               f"padded input {[int(v) + 2 * p for v, p in zip(self.source.shape[1:], self.padding)]})")
        shape = (int(self.out_channels), int(self.in_channels), *self.kernel_size)
        if tuple(self.w.shape) != shape:
            raise RuntimeError(f"Conv3dConnection.w has shape {tuple(self.w.shape)}, expected {shape}")
        if tuple(self.b.shape) != (shape[0],):
            raise RuntimeError(f"Given weight of size {list(self.w.shape)}, expected bias to be 1-dimensional with {shape[0]} "
                               f"elements, but got bias of size {list(self.b.shape)} instead")

    def _check_learning(self) -> None:
        """The reference's update on this class (learning.py:499-559, 978-1050, 1382-1438, 2017-2121, 2739-2855) fails
        in ``torch.bmm`` whenever it evaluates the pre-synaptic term: the unfolded source spikes stay bool.  Raised when
        a learning window or a standalone update would run it, before any state changes."""
        from ..learning import learning as L

        rule = self.update_rule
        pre = isinstance(rule, (L.Hebbian, L.MSTDP)) or (
            isinstance(rule, (L.PostPre, L.WeightDependentPostPre)) and bool(rule.nu[0] != 0))
        if pre:
            raise RuntimeError("expected m1 and m2 to have the same dtype, but got: float != bool (the reference's "
                               f"{type(rule).__name__} on a Conv3dConnection multiplies the bool source spikes)")
        if isinstance(rule, (L.PostPre, L.WeightDependentPostPre)):
            # the unfolds it runs even at zero rates pair depth with kw, height with kh, width with kd (learning.py:517-545)
            (D, H, W), (p0, p1, p2) = (int(v) for v in self.source.shape[1:]), self.padding
            kd, kh, kw = self.kernel_size
            if D + 2 * p2 < kw or H + 2 * p1 < kh or W + 2 * p0 < kd:
                raise RuntimeError(f"maximum size for tensor at an unfolded dimension is smaller than the kernel: the "
                                   f"reference's {type(rule).__name__} update on this Conv3dConnection fails")

    def _check_window(self, learning: bool) -> None:
        self._check()
        if learning:
            self._check_learning()

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        from ..learning import learning as L

        self._check()
        d.kind = _abi.SNN_CONN_CONV3D
        if self.wmin.numel() != 1 or self.wmax.numel() != 1:
            raise NotImplementedError("per-synapse wmin/wmax tensors are not supported by the CUDA core yet")
        d.wmin = _scalar(self.wmin, "wmin")
        d.wmax = _scalar(self.wmax, "wmax")
        d.has_norm = int(self.norm is not None)
        d.norm_abs = 0
        d.norm = float(self.norm) if self.norm is not None else 0.0
        d.dt_scale = 1.0
        d.cin, d.din, d.hin, d.win = (int(v) for v in self.source.shape)
        d.cout, d.dout, d.hout, d.wout = (int(v) for v in self.target.shape)
        d.kd, d.kh, d.kw = self.kernel_size
        d.sd, d.sh, d.sw = self.stride
        d.pd, d.ph, d.pw = self.padding
        d.dh = d.dw = 1
        # a rule that evaluates the pre-synaptic term never runs (_check_learning refuses its learning windows): the plan
        # of a window without learning carries no rule for it
        if rule and type(self.update_rule) in (L.NoOp, L.PostPre, L.WeightDependentPostPre):
            self.update_rule._fill_desc(d)


class AbstractMulticompartmentConnection(ABC, Module):
    """Reference: topology.py:159-262."""

    def __init__(self, source: Nodes, target: Nodes, device, pipeline: list = None, **kwargs) -> None:
        super().__init__()
        assert isinstance(source, Nodes), "Source is not a Nodes object"
        assert isinstance(target, Nodes), "Target is not a Nodes object"
        self.source = source
        self.target = target
        self.device = device
        self.pipeline = [] if pipeline is None else pipeline
        self.feature_index = {}
        for feature in self.pipeline:
            self.feature_index[feature.name] = feature
            feature.prime_feature(connection=self, device=self.device, **kwargs)

    def append_pipeline(self, feature) -> None:
        self.pipeline.append(feature)
        feature.prime_feature(connection=self, device=self.device)
        self.feature_index[feature.name] = feature


class MulticompartmentConnection(AbstractMulticompartmentConnection):
    """Feature-pipeline connection (reference: topology.py:402-537).  The CUDA core executes pipelines of exactly one
    dense ``Weight`` feature — what every model in ``bindsnet.models`` builds (models.py:185-236) — plus at most one
    ``Probability``, ``Mask`` and ``Intensity`` feature each, in any order.  A spiking source then adds ``w * I`` to a
    target where the mask holds and the synapse's draw transmits (topology.py:437-479); the order of the pipeline
    does not change that single rounding."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        device="cpu",
        pipeline: list = None,
        manual_update: bool = False,
        traces: bool = False,
        **kwargs,
    ) -> None:
        super().__init__(source, target, device, pipeline if pipeline is not None else [], **kwargs)
        self.traces = traces
        self.manual_update = manual_update
        if self.traces:
            raise NotImplementedError("MulticompartmentConnection(traces=True) is not implemented by the CUDA core")

    def _features(self) -> dict:
        """The pipeline by kind: exactly one Weight and at most one Probability, Mask and Intensity feature."""
        from .topology_features import Intensity, Mask, Probability, Weight

        kinds = {}
        for f in self.pipeline:
            k = next((c for c in (Weight, Probability, Mask, Intensity) if isinstance(f, c)), None)
            if k is None:
                raise NotImplementedError(
                    "the CUDA core executes MulticompartmentConnection pipelines of one Weight feature and at most one "
                    f"Probability, Mask and Intensity feature each, not {type(f).__name__}"
                )
            if k.__name__ in kinds:
                raise NotImplementedError(f"a MulticompartmentConnection pipeline with two {k.__name__} features is not implemented by the CUDA core")
            kinds[k.__name__] = f
        if "Weight" not in kinds:
            raise NotImplementedError("the CUDA core executes MulticompartmentConnection pipelines with exactly one Weight feature")
        return kinds

    def _weight(self):
        return self._features()["Weight"]

    @property
    def w(self) -> torch.Tensor:
        return self._weight().value

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """Reference: topology.py:437-479 + Weight.compute topology_features.py:633-645.  With a Probability feature
        every call is a new step of its own: it draws a fresh seed from torch's CPU generator, as a window without
        ``one_spike_seed`` does.  A 'time step' Weight normalises after the product (:641-643)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def update(self, **kwargs) -> None:
        """topology.py:509-518."""
        if kwargs.get("learning", False) and not self.manual_update:
            for f in self.pipeline:
                f.update(**kwargs)

    def normalize(self) -> None:
        """topology.py:520-527."""
        for f in self.pipeline:
            f.normalize()

    def reset_state_variables(self) -> None:
        for f in self.pipeline:
            f.reset_state_variables()

    def _apply(self, fn, *args, **kwargs):
        # Features are not nn.Modules in the reference (they take an explicit device,
        # topology.py:169,192); here Network.to(device) carries their value along.
        out = super()._apply(fn, *args, **kwargs)
        for f in self.pipeline:
            f._apply(fn)
        return out

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        d.kind = _abi.SNN_CONN_MCC
        self._weight()._fill_desc(d, dt, self.manual_update)


class LocalConnection(Connection):
    """Locally connected synapses (reference: topology.py:1304-1484): a dense ``[source.n, target.n]`` matrix that is
    non-zero only inside each target neuron's receptive field.  The reference keeps it dense too — ``compute`` is the
    plain matrix product (:1441-1455) — and holds the structure with a mask of the initially-zero weights that
    ``update`` passes on when the caller gives none (:1457-1469), so here it IS a dense ``Connection`` whose plan always
    carries that mask; ``normalize`` divides by the plain column sum (:1471-1479) and ``norm`` is scaled by the kernel
    size (:1437-1438).  Target neuron ``f * conv_prod + c`` is filter ``f`` at receptive field ``c``."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        kernel_size,
        stride,
        n_filters: int,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        w_dtype: torch.dtype = torch.float32,
        **kwargs,
    ) -> None:
        kernel_size, stride = _pair(kernel_size), _pair(stride)
        shape = kwargs.get("input_shape", None)
        if shape is None:
            shape = _pair(int(np.sqrt(source.n)))                                  # topology.py:1370-1373
        if tuple(kernel_size) == tuple(shape):
            conv_size = (1, 1)
        else:
            conv_size = (int((shape[0] - kernel_size[0]) / stride[0]) + 1, int((shape[1] - kernel_size[1]) / stride[1]) + 1)
        conv_prod, kernel_prod = int(np.prod(conv_size)), int(np.prod(kernel_size))
        assert target.n == n_filters * conv_prod, f"Total neurons in target layer must be {n_filters * conv_prod}. Got {target.n}."
        # topology.py:1393-1407 — the index arithmetic is the reference's (including `k1 * shape[0]`)
        c1, c2, k1, k2 = np.meshgrid(np.arange(conv_size[0]), np.arange(conv_size[1]), np.arange(kernel_size[0]),
                                     np.arange(kernel_size[1]), indexing="ij")
        loc = c1 * stride[0] * shape[1] + c2 * stride[1] + k1 * shape[0] + k2      # [c1, c2, k1, k2]
        locations = torch.from_numpy(loc.transpose(2, 3, 0, 1).reshape(kernel_prod, conv_prod).astype(np.int64))
        w = kwargs.get("w", None)
        if w is None:
            # topology.py:1410-1423: random weights inside the receptive fields only
            lo, hi = kwargs.get("wmin", -np.inf), kwargs.get("wmax", np.inf)
            w = torch.zeros(source.n, target.n)
            cols = (torch.arange(n_filters).view(-1, 1, 1) * conv_prod + torch.arange(conv_prod).view(1, 1, -1)).expand(n_filters, kernel_prod, conv_prod)
            rows = locations.view(1, kernel_prod, conv_prod).expand(n_filters, kernel_prod, conv_prod)
            w[rows.reshape(-1), cols.reshape(-1)] = torch.rand(n_filters * kernel_prod * conv_prod)
            if np.isinf(lo) or np.isinf(hi):
                w = torch.clamp(w, lo, hi)
            else:
                w = lo + w * (hi - lo)
            kwargs = dict(kwargs, w=w)
        kwargs.setdefault("b", torch.zeros(target.n))                              # topology.py:1433
        super().__init__(source, target, nu=nu, reduction=reduction, weight_decay=weight_decay, w_dtype=w_dtype, **kwargs)
        self.kernel_size, self.stride, self.n_filters, self.conv_size = kernel_size, stride, n_filters, conv_size
        self.register_buffer("locations", locations)
        self.register_buffer("mask", self.w == 0)                                  # topology.py:1431
        if self.norm is not None:
            self.norm = self.norm * kernel_prod                                    # topology.py:1437-1438

    _synapse_tensors = False
    _tensor_norms = False

    def update(self, **kwargs) -> None:
        """topology.py:1457-1469."""
        if kwargs.get("mask", None) is None:
            kwargs["mask"] = self.mask
        super().update(**kwargs)

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        super()._fill_desc(d, dt, rule)
        d.norm_abs = 0   # w *= norm / w.sum(0)  (topology.py:1476-1479)


class SparseConnection(Connection):
    """Sparse synapses (reference: topology.py:2009-2017): a ``Connection`` whose ``w`` is a ``torch.sparse_coo``
    ``Parameter``.  A dense ``w`` (or none: dense random, as ``Connection`` draws it) is converted with ``to_sparse()``;
    a sparse ``w`` is taken as given, so a large network never needs its dense matrix.  Inside ``Network.run`` the
    generic window kernel gathers the stored entries only (in ascending source order, bit-identical to a dense
    ``Connection`` holding the same values), and ``learning.NoOp(weight_decay=...)`` decays the stored values in place.

    The pattern is fixed.  Any other learning rule is refused at construction: the reference's rules add an entry
    wherever ``s_pre (x) x_post`` is non-zero (learning.py:403-417), which turns the pattern dense, and fail outright with
    finite ``wmin`` / ``wmax`` (learning.py:101-102).  ``norm`` is refused at construction too; the reference accepts it
    and fails in ``normalize()`` at the end of the first run.  ``masks=`` for it raise, as in the reference
    (topology.py:129-131)."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        w_dtype: torch.dtype = torch.float32,
        **kwargs,
    ) -> None:
        from ..learning import NoOp

        rule = kwargs.get("update_rule", None)
        if rule is not None and rule is not NoOp:
            raise NotImplementedError(
                f"SparseConnection keeps a fixed synapse pattern: learning rule {getattr(rule, '__name__', rule)} is not "
                "supported (the reference's rules grow the pattern into a dense one; only learning.NoOp, i.e. static or "
                "decaying weights, is)"
            )
        if kwargs.get("norm", None) is not None:
            raise NotImplementedError(
                "SparseConnection does not support norm: the reference's normalize() fails on a sparse w "
                "(it would raise at the end of the first run; this raises at construction)"
            )
        w = kwargs.get("w", None)
        if isinstance(w, torch.Tensor) and w.is_sparse:
            if w_dtype != torch.float32:
                raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
            AbstractConnection.__init__(self, source, target, nu, reduction, weight_decay, **kwargs)
            if w.sparse_dim() != 2 or w.dense_dim() != 0 or tuple(w.shape) != (source.n, target.n):
                raise ValueError(f"sparse w must be a 2-D sparse_coo tensor of shape ({source.n}, {target.n})")
            w = self.cast_dtype_if_needed(w, w_dtype)
            if (self.wmin != -np.inf).any() or (self.wmax != np.inf).any():      # topology.py:314-317
                w = torch.sparse_coo_tensor(w._indices(), torch.clamp(w._values(), self.wmin, self.wmax), w.shape,
                                            is_coalesced=w.is_coalesced())
            self.w = Parameter(w.detach(), requires_grad=False)
            b = kwargs.get("b", None)
            self.b = Parameter(torch.as_tensor(b, dtype=torch.float32), requires_grad=False) if b is not None else None
        else:
            super().__init__(source, target, nu, reduction, weight_decay, w_dtype, **kwargs)
            self.w = Parameter(self.w.to_sparse(), requires_grad=False)          # topology.py:2017

    _synapse_tensors = False
    _tensor_norms = False

    def update(self, **kwargs) -> None:
        """topology.py:112-139 with the reference's refusal of masks on a sparse w (:129-131)."""
        if kwargs.get("mask", None) is not None:
            raise NotImplementedError("Mask isn't supported for SparseConnection")
        super().update(**kwargs)

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        super()._fill_desc(d, dt, rule)
        d.kind = _abi.SNN_CONN_SPARSE
        d.norm_abs = 0


class _MaxPoolConnection(AbstractConnection):
    """What MaxPool2dConnection and MaxPoo3dConnection share: no weights, the ``firing_rates`` buffer, the single
    operator, and the reference's failures of ``NoOp.update`` and of ``masks=`` on a connection without ``w``."""

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """topology.py:1163-1185 / :1255-1277: ``firing_rates`` advance in place; returns the pooled spikes ``[B, C,
        *pooled]`` (``snn_b200_conn_compute``)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def update(self, **kwargs) -> None:
        """topology.py:1187-1192 / :1279-1284 -> :112-139: with learning on, learning.NoOp.update reads ``self.w``; so
        does a mask."""
        if kwargs.get("learning", True) or kwargs.get("mask", None) is not None:
            raise AttributeError(self._no_w_message())

    def normalize(self) -> None:
        """No weights, no normalization (topology.py:1194-1199)."""

    def reset_state_variables(self) -> None:
        """topology.py:1201-1211 / :1293-1301 (the reference allocates on the CPU; here the buffer stays on its device)."""
        self.firing_rates = torch.zeros(self.source.batch_size, *self.source.s.shape[1:], device=self.firing_rates.device)

    def _no_w_message(self) -> str:
        name = _pool_dims(self)[1]
        return (f"'{name}' object has no attribute 'w' (the reference's learning.NoOp.update and the masks= of "
                f"Network.run read connection.w, learning.py:87-94 / topology.py:127-131; run {name} networks with "
                "learning off and without masks for it)")

    def _out_shape(self):
        return pool_out_shape(self)

    def _check(self, s_shape) -> None:
        check_pool(self, s_shape)


class MaxPool2dConnection(_MaxPoolConnection):
    """Max pooling by online firing-rate estimates (reference: topology.py:1124-1211).  Each ``compute(s)`` decays the
    ``firing_rates`` buffer (``r -= decay * r``), adds the spikes, and passes on, per channel and window, the spike of
    the source neuron with the highest rate (the first one in row-major window order on a tie; padding never wins).
    Source and target are ``[C, H, W]`` populations with the target ``[C, Hout, Wout]`` as ``F.max_pool2d`` computes it.
    There are no weights and nothing to learn: the rule is ``learning.NoOp``, ``normalize`` does nothing.

    As in the reference, ``decay`` is a keyword argument without default (a ``None`` decay fails in the first
    ``compute``), ``firing_rates`` is ``source.s.shape`` at construction (``[1, C, H, W]`` once the source was added to a
    network, empty before) and ``reset_state_variables`` reallocates it at the source's batch size (here on the buffer's
    device).  Inside ``Network.run`` the generic window kernel keeps the rates in step with the reference's call order;
    shapes the reference's ``fr += s.float().squeeze()`` cannot add (a size-1 channel or spatial dimension at batch size
    > 1, a buffer of another batch size) raise ``RuntimeError`` before anything runs, as do a source that is not
    ``[C, H, W]``, a target that is not ``[C, Hout, Wout]`` and a window that lies entirely in the padding.  A window with learning on raises ``AttributeError``: the reference's ``NoOp.update`` scales
    ``connection.w`` (learning.py:87-94), which this connection does not have; so do ``masks=`` for it."""

    def __init__(self, source: Nodes, target: Nodes, kernel_size, stride=1, padding=0, dilation=1, **kwargs) -> None:
        super().__init__(source, target, None, None, 0.0, **kwargs)
        self.kernel_size = _pair(kernel_size)
        self.stride = _pair(stride)
        self.padding = _pair(padding)
        self.dilation = _pair(dilation)
        self.register_buffer("firing_rates", torch.zeros(source.s.shape))

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        d.kind = _abi.SNN_CONN_MAXPOOL2D
        d.rule = _abi.SNN_RULE_NOOP
        d.weight_decay = 1.0
        d.cin, d.hin, d.win = (int(v) for v in self.source.shape)
        d.cout, d.hout, d.wout = self._out_shape()
        d.kh, d.kw = self.kernel_size
        d.sh, d.sw = self.stride
        d.ph, d.pw = self.padding
        d.dh, d.dw = self.dilation
        d.pool_decay = float(np.float32(float(self.decay))) if self.decay is not None else 0.0
        d.pool_rates = self.firing_rates.data_ptr()


class MaxPoo3dConnection(_MaxPoolConnection):
    """Three-dimensional max pooling by online firing-rate estimates (reference: topology.py:1214-1301; the reference's
    class name, typo included).  Each ``compute(s)`` decays the ``firing_rates`` buffer (``r -= decay * r``), adds the
    spikes, and passes on, per channel and window, the spike of the source neuron with the highest rate (the first one
    in ``(d, h, w)`` row-major window order on a tie; padding never wins).  Source and target are ``[C, D, H, W]``
    populations with the target ``[C, Dout, Hout, Wout]`` as ``F.max_pool3d`` computes it; ``kernel_size``, ``stride``,
    ``padding`` and ``dilation`` are ``(D, H, W)`` triples.  There are no weights and nothing to learn: the rule is
    ``learning.NoOp``, ``normalize`` does nothing.

    As in the reference, ``decay`` is a keyword argument without default, ``firing_rates`` is ``source.s.shape`` at
    construction and ``reset_state_variables`` reallocates it at the source's batch size (here on the buffer's device).
    Inside ``Network.run`` the generic window kernel keeps the rates in step with the reference's call order; the
    reference's failures are raised before anything runs, with its exception types: ``RuntimeError`` for shapes its
    ``fr += s.float().squeeze()`` cannot add (a size-1 dimension at batch size > 1, a buffer of another batch size), a
    target that is not ``[C, Dout, Hout, Wout]``, padding above half the kernel and a window that lies entirely in the
    padding; ``AttributeError`` for a learning window or ``masks=`` for it.  Unlike the reference, a source that is not a
    population of shape ``[C, D, H, W]`` raises ``NotImplementedError`` at construction."""

    def __init__(self, source: Nodes, target: Nodes, kernel_size, stride=1, padding=0, dilation=1, **kwargs) -> None:
        if not isinstance(source, Nodes) or len(source.shape) != 4:
            shape = list(source.shape) if isinstance(source, Nodes) else type(source).__name__
            raise NotImplementedError(f"MaxPoo3dConnection is built from a [C, D, H, W] source population only; the source "
                                      f"is {shape}")
        super().__init__(source, target, None, None, 0.0, **kwargs)
        self.kernel_size = _triple(kernel_size)
        self.stride = _triple(stride)
        self.padding = _triple(padding)
        self.dilation = _triple(dilation)
        self.register_buffer("firing_rates", torch.zeros(source.s.shape))

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        d.kind = _abi.SNN_CONN_MAXPOOL3D
        d.rule = _abi.SNN_RULE_NOOP
        d.weight_decay = 1.0
        fill_pool3d_geometry(d, self)
        d.pool_decay = float(np.float32(float(self.decay))) if self.decay is not None else 0.0
        d.pool_rates = self.firing_rates.data_ptr()


def fill_pool3d_geometry(d: "_abi.SnnConn", conn) -> None:
    """The SNN_CONN_MAXPOOL3D geometry of a MaxPoo3dConnection (this package's or the reference's: the same attributes):
    the depth axis in the depth fields, H and W in the conv fields, ``cin = cout = C``."""
    d.cin, d.din, d.hin, d.win = (int(v) for v in conn.source.shape)
    d.cout, d.dout, d.hout, d.wout = pool_out_shape(conn)
    d.kd, d.kh, d.kw = (int(v) for v in conn.kernel_size)
    d.sd, d.sh, d.sw = (int(v) for v in conn.stride)
    d.pd, d.ph, d.pw = (int(v) for v in conn.padding)
    d.dd, d.dh, d.dw = (int(v) for v in conn.dilation)


class LocalConnection2D(AbstractConnection):
    """Two-dimensional locally connected synapses (reference: topology.py:1623-1767): every target neuron has weights of
    its own over one ``kernel_size`` window of a ``[C, H, W]`` source, ``n_filters`` neurons per window.  ``w`` is
    ``[in_channels, n_filters * conv_prod, kernel_prod]``; target neuron ``f * conv_prod + p`` sees window ``p``.  Inside
    ``Network.run`` the generic window kernel gathers each target's receptive field from the source spikes and applies
    ``PostPre``, ``WeightDependentPostPre``, ``Hebbian`` or ``NoOp``; ``normalize`` scales every ``kernel_prod`` row of
    ``w`` to sum ``norm``.

    As in the reference: ``w`` is drawn with ``torch.rand`` and clamped when a bound is finite; passing ``w=`` raises
    ``AttributeError`` (the reference's shape check reads ``self.out_channels``, which it never sets); ``b`` is stored and
    never used; a target with other than ``n_filters * conv_prod`` neurons raises ``RuntimeError`` when the network runs
    (the reference's ``view`` fails); ``reset_state_variables`` also resets the target layer.  The rules' update follows
    the reference's reshape of the unfolded source, which for ``in_channels > 1`` pairs a weight with another source
    neuron than ``compute`` does (include/snn_b200.h, SNN_CONN_LOCAL2D)."""

    def __init__(self, source: Nodes, target: Nodes, kernel_size, stride, n_filters: int,
                 nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None, reduction: Optional[callable] = None,
                 weight_decay: float = 0.0, w_dtype: torch.dtype = torch.float32, **kwargs) -> None:
        if w_dtype != torch.float32:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
        super().__init__(source, target, nu, reduction, weight_decay, **kwargs)
        self.kernel_size, self.stride, self.n_filters = _pair(kernel_size), _pair(stride), n_filters
        self.in_channels, input_height, input_width = source.shape[0], source.shape[1], source.shape[2]
        height = int((input_height - self.kernel_size[0]) / self.stride[0]) + 1      # topology.py:1677-1682
        width = int((input_width - self.kernel_size[1]) / self.stride[1]) + 1
        self.conv_size = (height, width)
        self.conv_prod = int(np.prod(self.conv_size))
        self.kernel_prod = int(np.prod(self.kernel_size))
        if kwargs.get("w", None) is not None:
            raise AttributeError(f"'{type(self).__name__}' object has no attribute 'out_channels' (the reference's w= shape "
                                 "check, topology.py:1697-1701, reads an attribute it never sets)")
        w = torch.rand(self.in_channels, self.n_filters * self.conv_prod, self.kernel_prod)
        if (self.wmin != -np.inf).any() or (self.wmax != np.inf).any():
            w = torch.clamp(w, self.wmin, self.wmax)
        self.w = Parameter(w.contiguous(), requires_grad=False)
        b = kwargs.get("b", None)
        self.b = Parameter(torch.as_tensor(b, dtype=torch.float32) if b is not None else torch.empty(0), requires_grad=False)

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """topology.py:1717-1740 as the window kernel's receptive-field gather (``snn_b200_conn_compute``)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def normalize(self) -> None:
        """topology.py:1748-1759: every row of ``w`` viewed as ``[in_channels * n, kernel_prod]`` scaled to sum ``norm``
        (a row that sums to zero becomes inf / NaN, as in the reference)."""
        if self.norm is not None:
            from . import _plan

            _plan.normalize_single_connection(self)

    def reset_state_variables(self) -> None:
        """topology.py:1761-1767."""
        super().reset_state_variables()
        self.target.reset_state_variables()

    def _check(self) -> None:
        """The reference's errors at the first ``compute``, raised before anything runs."""
        if len(self.source.shape) != 3:
            raise RuntimeError(f"LocalConnection2D needs a [C, H, W] source population, got {list(self.source.shape)}")
        C_, H, W = (int(v) for v in self.source.shape)
        if self.kernel_size[0] > H or self.kernel_size[1] > W or min(self.kernel_size) < 1 or min(self.stride) < 1:
            raise RuntimeError(f"LocalConnection2D: kernel_size {self.kernel_size} / stride {self.stride} do not fit a "
                               f"{H} x {W} source (unfold fails)")
        n = self.n_filters * self.conv_prod
        if self.target.n != n:
            raise RuntimeError(f"shape '[B, {', '.join(str(int(v)) for v in self.target.shape)}]' is invalid for the "
                               f"LocalConnection2D output of {n} neurons per sample (n_filters * conv_prod)")
        if tuple(self.w.shape) != (C_, n, self.kernel_prod):
            raise RuntimeError(f"LocalConnection2D.w has shape {tuple(self.w.shape)}, expected {(C_, n, self.kernel_prod)}")

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        self._check()
        d.kind = _abi.SNN_CONN_LOCAL2D
        if self.wmin.numel() != 1 or self.wmax.numel() != 1:
            raise NotImplementedError("per-synapse wmin/wmax tensors are not supported by the CUDA core yet")
        d.wmin = _scalar(self.wmin, "wmin")
        d.wmax = _scalar(self.wmax, "wmax")
        d.has_norm = int(self.norm is not None)
        d.norm_abs = 0
        d.norm = float(self.norm) if self.norm is not None else 0.0
        d.dt_scale = 1.0
        d.cin, d.hin, d.win = (int(v) for v in self.source.shape)
        d.cout, (d.hout, d.wout) = int(self.n_filters), self.conv_size
        d.kh, d.kw = self.kernel_size
        d.sh, d.sw = self.stride
        d.ph = d.pw = 0
        d.dh = d.dw = 1
        if rule:
            self.update_rule._fill_desc(d)


class LocalConnection3D(AbstractConnection):
    """Three-dimensional locally connected synapses (reference: topology.py:1770-1917): every target neuron has weights of
    its own over one ``kernel_size`` window of a ``[C, H, W, D]`` source, ``n_filters`` neurons per window.  ``w`` is
    ``[in_channels, n_filters * conv_prod, kernel_prod]``; target neuron ``f * conv_prod + p`` sees window ``p``.  Inside
    ``Network.run`` the generic window kernel gathers each target's receptive field from the source spikes and applies
    ``PostPre``, ``WeightDependentPostPre``, ``Hebbian`` or ``NoOp``; ``normalize`` scales every ``kernel_prod`` row of
    ``w`` to sum ``norm``.

    As in the reference: ``w`` is drawn with ``torch.rand`` and clamped when a bound is finite; passing ``w=`` raises
    ``AttributeError`` (the reference's shape check reads ``self.out_channels``, which it never sets); ``b`` is stored and
    never used; a target with other than ``n_filters * conv_prod`` neurons, or a kernel larger than the source, raises
    ``RuntimeError`` when the network runs (the reference fails in its first ``compute``); ``reset_state_variables`` also
    resets the target layer.  The rules' update follows the reference's reshape of the unfolded source, which for
    ``in_channels > 1`` pairs a weight with another source neuron than ``compute`` does (include/snn_b200.h,
    SNN_CONN_LOCAL3D).  A source or target that is not a population with a ``[C, H, W, D]`` source shape raises
    ``NotImplementedError`` before the other arguments are looked at, so such a call without ``stride`` / ``n_filters``
    raises it where the reference raises ``TypeError`` (DESIGN.md section 8)."""

    def __init__(self, source: Nodes, target: Nodes, kernel_size=_MISSING, stride=_MISSING, n_filters=_MISSING,
                 nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None, reduction: Optional[callable] = None,
                 weight_decay: float = 0.0, w_dtype: torch.dtype = torch.float32, **kwargs) -> None:
        for name, layer in (("source", source), ("target", target)):
            if not isinstance(layer, Nodes) or (name == "source" and len(layer.shape) != 4):
                shape = list(layer.shape) if isinstance(layer, Nodes) else type(layer).__name__
                raise NotImplementedError(f"LocalConnection3D is built from a [C, H, W, D] source population into a population "
                                          f"only; the {name} is {shape}")
        missing = [n for n, v in (("kernel_size", kernel_size), ("stride", stride), ("n_filters", n_filters)) if v is _MISSING]
        if missing:
            names = " and ".join(f"'{n}'" for n in missing) if len(missing) < 3 else "'kernel_size', 'stride', and 'n_filters'"
            raise TypeError(f"LocalConnection3D.__init__() missing {len(missing)} required positional argument"
                            f"{'s' if len(missing) > 1 else ''}: {names}")
        if w_dtype != torch.float32:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
        super().__init__(source, target, nu, reduction, weight_decay, **kwargs)
        self.kernel_size, self.stride, self.n_filters = _triple(kernel_size), _triple(stride), n_filters
        self.in_channels, input_height, input_width, input_depth = (source.shape[0], source.shape[1], source.shape[2],
                                                                    source.shape[3])
        height = int((input_height - self.kernel_size[0]) / self.stride[0]) + 1      # topology.py:1831-1833
        width = int((input_width - self.kernel_size[1]) / self.stride[1]) + 1
        depth = int((input_depth - self.kernel_size[2]) / self.stride[2]) + 1
        self.conv_size = (height, width, depth)
        self.conv_prod = int(np.prod(self.conv_size))
        self.kernel_prod = int(np.prod(self.kernel_size))
        if kwargs.get("w", None) is not None:
            raise AttributeError(f"'{type(self).__name__}' object has no attribute 'out_channels' (the reference's w= shape "
                                 "check, topology.py:1852-1857, reads an attribute it never sets)")
        w = torch.rand(self.in_channels, self.n_filters * self.conv_prod, self.kernel_prod)
        if (self.wmin != -np.inf).any() or (self.wmax != np.inf).any():
            w = torch.clamp(w, self.wmin, self.wmax)
        self.w = Parameter(w.contiguous(), requires_grad=False)
        b = kwargs.get("b", None)
        self.b = Parameter(torch.as_tensor(b, dtype=torch.float32) if b is not None else torch.empty(0), requires_grad=False)

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """topology.py:1866-1896 as the window kernel's receptive-field gather (``snn_b200_conn_compute``)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def normalize(self) -> None:
        """topology.py:1898-1909: every row of ``w`` viewed as ``[in_channels * n, kernel_prod]`` scaled to sum ``norm``
        (a row that sums to zero becomes inf / NaN, as in the reference)."""
        if self.norm is not None:
            from . import _plan

            _plan.normalize_single_connection(self)

    def reset_state_variables(self) -> None:
        """topology.py:1911-1917."""
        super().reset_state_variables()
        self.target.reset_state_variables()

    def _check(self) -> None:
        """The reference's errors at the first ``compute``, raised before anything runs.  ``int((in - k) / s) + 1``
        truncates towards zero, so a kernel larger than the source can still give a conv size of 1 or more; unfold fails."""
        C_, H, W, D = (int(v) for v in self.source.shape)
        if any(k > n for k, n in zip(self.kernel_size, (H, W, D))) or min(self.kernel_size) < 1 or min(self.stride) < 1:
            raise RuntimeError(f"LocalConnection3D: kernel_size {self.kernel_size} / stride {self.stride} do not fit a "
                               f"{H} x {W} x {D} source (unfold fails)")
        n = self.n_filters * self.conv_prod
        if self.target.n != n:
            raise RuntimeError(f"shape '[B, {', '.join(str(int(v)) for v in self.target.shape)}]' is invalid for the "
                               f"LocalConnection3D output of {n} neurons per sample (n_filters * conv_prod)")
        if tuple(self.w.shape) != (C_, n, self.kernel_prod):
            raise RuntimeError(f"LocalConnection3D.w has shape {tuple(self.w.shape)}, expected {(C_, n, self.kernel_prod)}")

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        self._check()
        d.kind = _abi.SNN_CONN_LOCAL3D
        if self.wmin.numel() != 1 or self.wmax.numel() != 1:
            raise NotImplementedError("per-synapse wmin/wmax tensors are not supported by the CUDA core yet")
        d.wmin = _scalar(self.wmin, "wmin")
        d.wmax = _scalar(self.wmax, "wmax")
        d.has_norm = int(self.norm is not None)
        d.norm_abs = 0
        d.norm = float(self.norm) if self.norm is not None else 0.0
        d.dt_scale = 1.0
        fill_local3d_geometry(d, self)
        if rule:
            self.update_rule._fill_desc(d)


def fill_local3d_geometry(d: "_abi.SnnConn", conn) -> None:
    """The SNN_CONN_LOCAL3D geometry of a LocalConnection3D (this package's or the reference's: the same attributes).  The
    reference's axes H, W, D go to the depth, height and width fields, so that D stays the contiguous one."""
    d.cin, d.din, d.hin, d.win = (int(v) for v in conn.source.shape)
    d.cout, (d.dout, d.hout, d.wout) = int(conn.n_filters), (int(v) for v in conn.conv_size)
    d.kd, d.kh, d.kw = (int(v) for v in conn.kernel_size)
    d.sd, d.sh, d.sw = (int(v) for v in conn.stride)
    d.pd = d.ph = d.pw = 0
    d.dh = d.dw = 1


def _pool_dims(conn):
    """The number of spatial axes of a pooling connection (2 or 3: its kernel_size is a pair or a triple), the class
    name and the pooling function its messages name."""
    nd = len(conn.kernel_size)
    return nd, ("MaxPool2dConnection" if nd == 2 else "MaxPoo3dConnection"), f"max_pool{nd}d"


def pool_out_shape(conn):
    """``[C, Hout, Wout]`` of a MaxPool2dConnection, ``[C, Dout, Hout, Wout]`` of a MaxPoo3dConnection (this package's or
    the reference's: the same attributes), or the ``RuntimeError`` the reference's ``compute`` raises for its geometry.
    ``F.max_pool2d`` / ``F.max_pool3d`` without ceil mode; every window must hold an element of the input on every axis (a
    dilated window can lie entirely in the padding, where the reference's gather indexes past the row)."""
    nd, name, fn = _pool_dims(conn)
    shape = tuple(int(v) for v in conn.source.shape)
    if len(shape) != nd + 1:
        axes = "[C, H, W]" if nd == 2 else "[C, D, H, W]"
        raise RuntimeError(f"{name} needs a {axes} source population, got {list(shape)} (the reference's "
                           "gather over s.flatten(2) indexes the wrong dimension)")
    out = []
    for n, k, st, p, d in zip(shape[1:], conn.kernel_size, conn.stride, conn.padding, conn.dilation):
        if k < 1 or st < 1 or d < 1 or p < 0:
            raise RuntimeError(f"{fn}: kernel_size {conn.kernel_size}, stride {conn.stride} and dilation {conn.dilation} must be "
                               f"positive and padding {conn.padding} non-negative")
        if p > k // 2:
            raise RuntimeError(f"pad should be at most half of effective kernel size, but got pad={p}, kernel_size={k} and dilation={d}")
        e = n + 2 * p - d * (k - 1) - 1
        if e < 0:
            raise RuntimeError(f"{fn}: output size is too small for input {list(shape)}")
        m = e // st + 1
        for o in range(m):
            if not any(0 <= o * st - p + j * d < n for j in range(k)):
                raise RuntimeError(f"{fn}: window {o} of kernel_size {k}, stride {st}, padding {p} and dilation {d} lies "
                                   f"entirely in the padding of a dimension of size {n}")
        out.append(m)
    return (shape[0], *out)


def check_pool(conn, s_shape) -> None:
    """The conditions under which the reference's ``MaxPool2dConnection.compute`` / ``MaxPoo3dConnection.compute`` on
    spikes of shape ``s_shape`` succeeds, raised as it raises: ``decay`` set, a buffer that ``fr += s.float().squeeze()``
    adds to element by element (the same shape as ``s``), a geometry ``pool_out_shape`` accepts, a target of the pooled
    shape."""
    nd, name, _ = _pool_dims(conn)
    line = 1175 if nd == 2 else 1265
    if conn.decay is None:
        raise TypeError(f"unsupported operand type(s) for *: 'NoneType' and 'Tensor' ({name} needs the decay= "
                        f"keyword argument, topology.py:{line})")
    fr = tuple(conn.firing_rates.shape)
    sq = tuple(d for d in s_shape if d != 1)
    try:
        ok = tuple(torch.broadcast_shapes(fr, sq)) == fr
    except RuntimeError:
        ok = False
    if not ok or fr != tuple(s_shape):
        raise RuntimeError(
            f"{name}: firing_rates of shape {list(fr)} cannot take the spikes of shape {list(s_shape)} the way "
            f"the reference adds them (firing_rates += s.float().squeeze(), topology.py:{line + 1}); call reset_state_variables() "
            "after the batch size changes, and note that a size-1 channel or spatial dimension at batch size > 1 fails "
            "in the reference too")
    out = pool_out_shape(conn)
    if tuple(int(v) for v in conn.target.shape) != out:
        pooled = "[B, C, Hout, Wout]" if nd == 2 else "[B, C, Dout, Hout, Wout]"
        raise RuntimeError(f"{name}: target shape {list(conn.target.shape)} is not the pooled shape {list(out)} "
                           f"(network.py:248 adds {pooled} into it)")
    if conn.firing_rates.dtype != torch.float32 or not conn.firing_rates.is_contiguous():
        raise TypeError(f"{name}.firing_rates must be a contiguous float32 tensor (it is updated in place)")


class MeanFieldConnection(AbstractConnection):
    """A summary of the whole source population as input to every target neuron (reference: topology.py:1920-2006):
    ``compute(s)`` is ``s.float().mean() * w``.  The mean runs over all of ``[B, *source.shape]``, the batch included, so
    every sample receives the same batch-wide mean (a sample without spikes too), scaled by ``w``.  ``w`` may have any
    shape that broadcasts into ``[B, *target.shape]`` without growing it (0-d, ``[n]`` of the last axis, ``[1, W]``,
    ``[C, 1]``, ``[B, *target.shape]`` per sample...); ``Network.run`` adds the result into the target's input at the
    connection's place in the insertion order.  Inside ``Network.run`` the generic window kernel counts each source's
    spikes with one integer per step and forms the mean from that count, bit-identical to the reference's.

    As in the reference, the constructor passes ``weight_decay`` on in the ``reduction`` slot (topology.py:1957):
    ``reduction`` holds it, ``weight_decay`` is 0.0, and a ``reduction=`` keyword raises ``TypeError``.  Without ``w`` one
    ``torch.randn(1)[0]`` is drawn after the rule is built; a given ``w`` is clamped only when some bound is infinite.
    Only ``learning.NoOp`` constructs (it scales ``w`` by 1.0 and never clamps, so ``w`` does not change); the STDP rules
    and ``MSTDP`` / ``MSTDPET`` raise.  Unlike the reference, ``norm`` raises ``NotImplementedError`` at construction (the
    reference's ``normalize()`` fails at the end of the first run), and so does a run whose ``B * source.n`` reaches
    2**24 (where the float32 mean is no longer the exact count over ``N``).  ``masks=`` for it raise, as for every
    connection but the dense one."""

    def __init__(
        self,
        source: Nodes,
        target: Nodes,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        weight_decay: float = 0.0,
        w_dtype: torch.dtype = torch.float32,
        **kwargs,
    ) -> None:
        if w_dtype != torch.float32:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")
        if kwargs.get("norm", None) is not None:
            raise NotImplementedError(
                "MeanFieldConnection does not support norm: the reference's normalize() assigns a view to the w Parameter "
                "(TypeError), or fails to view w as [1, target.n] (RuntimeError), at the end of the first run; this raises "
                "at construction"
            )
        super().__init__(source, target, nu, weight_decay, **kwargs)   # weight_decay in the reduction slot, topology.py:1957
        w = kwargs.get("w", None)
        if w is None:                                                    # topology.py:1959-1965
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp((torch.randn(1)[0] + 1) / 10, self.wmin, self.wmax)
            else:
                w = self.wmin + ((torch.randn(1)[0] + 1) / 10) * (self.wmax - self.wmin)
            w = w.to(dtype=w_dtype)
        else:                                                            # topology.py:1966-1969
            if (self.wmin == -np.inf).any() or (self.wmax == np.inf).any():
                w = torch.clamp(w, self.wmin, self.wmax)
            w = self.cast_dtype_if_needed(w, w_dtype)
        self.w = Parameter(w.detach().clone().contiguous(), requires_grad=False)
        self._mf_offsets = None   # (key, offsets, stride) of the last plan (meanfield_offsets)

    def compute(self, s: torch.Tensor) -> torch.Tensor:
        """``s.float().mean() * w`` (topology.py:1972-1981), shaped like ``w`` (``snn_b200_conn_compute``)."""
        from . import _plan

        return _plan.compute_single_connection(self, s)

    def update(self, **kwargs) -> None:
        """topology.py:1983-1988 -> :112-139: learning.NoOp scales ``w`` by 1.0 and does not clamp (learning.py:93-104), so
        nothing changes; a user-defined rule runs as it does on any connection.  ``masks=`` are refused by Network.run."""
        if kwargs.get("learning", True) and self.update_rule.rule_code is None:
            self.update_rule.update(**kwargs)

    def normalize(self) -> None:
        """``norm`` is refused at construction, so there is nothing to normalize (topology.py:1990-1999)."""

    def reset_state_variables(self) -> None:
        """No state of its own (topology.py:2001-2006)."""

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, rule: bool = True) -> None:
        d.kind = _abi.SNN_CONN_MEANFIELD
        d.rule = _abi.SNN_RULE_NOOP
        d.weight_decay = 1.0


def meanfield_offsets(conn, B: int, cache: bool = True):
    """The SNN_CONN_MEANFIELD view of ``conn.w`` (this package's or the reference's MeanFieldConnection) at batch size
    ``B``: an int32 ``[target.n]`` tensor on ``w``'s device holding the element of ``w`` each target neuron of sample 0
    reads, and the step between samples (0 unless ``w`` has the batch axis).  Raises what the reference raises before
    anything runs: the ``RuntimeError`` of ``inputs += mean * w`` for a ``w`` that does not broadcast into ``[B,
    *target.shape]`` or would grow it, and ``NotImplementedError`` where ``B * source.n`` reaches 2**24.  Cached on the
    connection per (``w`` shape, target shape, ``B``, device) unless ``cache`` is false (the reference's objects)."""
    w = conn.w
    full = (int(B), *(int(v) for v in conn.target.shape))
    key = (tuple(w.shape), full, w.device)
    cached = getattr(conn, "_mf_offsets", None) if cache else None
    if cached is not None and cached[0] == key:
        return cached[1], cached[2]
    if int(B) * int(conn.source.n) >= 1 << 24:
        raise NotImplementedError(f"MeanFieldConnection with B * source.n = {int(B) * int(conn.source.n)} spikes per step: the "
                                  "float32 mean is exact below 2**24 only")
    # network.py:248: inputs[target] += s.float().mean() * w, with the reference's own error for a shape that fails
    torch.empty(full, device="meta").add_(torch.empty(tuple(w.shape), device="meta"))
    idx = torch.arange(w.numel(), dtype=torch.int64).view(tuple(w.shape)).broadcast_to(full).reshape(full[0], -1)
    stride = int(idx[1, 0] - idx[0, 0]) if full[0] > 1 else 0
    off = idx[0].to(torch.int32).contiguous().to(w.device)
    if cache:
        conn._mf_offsets = (key, off, stride)
    return off, stride


def _unsupported(name: str, where: str):
    class _Unsupported:
        __doc__ = f"``{name}`` (reference: {where}) — not on the accelerated path (SURVEY.md §8f)."

        def __init__(self, *args, **kwargs):
            raise NotImplementedError(
                f"{name} is outside the hot path bindsnet_b200 implements (Connection, "
                "MulticompartmentConnection[Weight]); see DESIGN.md 'Out of scope'"
            )

    _Unsupported.__name__ = name
    return _Unsupported


MaxPool1dConnection = _unsupported("MaxPool1dConnection", "topology.py:1028-1121")
LocalConnection1D = _unsupported("LocalConnection1D", "topology.py:1487-1620")
