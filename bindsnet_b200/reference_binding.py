"""The binding a BindsNET maintainer would add to the REFERENCE: fill the C ABI of ``include/snn_b200.h`` straight
from live ``bindsnet`` objects (no ``bindsnet_b200`` host classes involved) and run one ``Network.run`` window through
a library that implements it — ``libsnn_b200.so`` on CUDA tensors, or the oracle library on CPU tensors (which is how
``tests/test_reference_binding.py`` proves, without a GPU, that the ABI can be driven from the reference's own
``DiehlAndCook2015`` and reproduces the reference's own ``run``).

    from bindsnet_b200 import reference_binding as rb
    rb.run_window(reference_network, {"X": spikes}, time=250)        # drop-in for network.run(...)

Covered: what ``bindsnet.models`` builds for the hot path — ``Input`` / ``LIFNodes`` / ``DiehlAndCookNodes`` layers,
``MulticompartmentConnection`` with one ``Weight`` feature (``MCC_learning.NoOp`` / ``PostPre``) and the classic
``Connection``, ``LocalConnection2D`` and ``LocalConnection3D`` with ``learning.NoOp`` / ``PostPre`` / ``WeightDependentPostPre`` / ``Hebbian``,
``Conv3dConnection`` with the updates the reference can run on it, ``Conv1dConnection`` with ``learning.NoOp`` /
``PostPre`` / ``WeightDependentPostPre`` / ``Hebbian``, ``MaxPool2dConnection`` and ``MaxPoo3dConnection`` with learning off.
Every attribute is read where the
reference keeps it (file:line in the comments); state tensors are handed over by pointer and updated in place.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional

import torch

from . import _abi

_KIND = {"Input": _abi.SNN_NODE_INPUT, "LIFNodes": _abi.SNN_NODE_LIF, "DiehlAndCookNodes": _abi.SNN_NODE_DC,
         "AdaptiveLIFNodes": _abi.SNN_NODE_DC,            # DiehlAndCookNodes.forward without the one-spike arbitration (nodes.py:921-946)
         "IFNodes": _abi.SNN_NODE_IF, "CurrentLIFNodes": _abi.SNN_NODE_CURRENT_LIF, "BoostedLIFNodes": _abi.SNN_NODE_BOOSTED_LIF,
         "McCullochPitts": _abi.SNN_NODE_MCP,
         "SubtractiveResetIFNodes": _abi.SNN_NODE_SUBIF, "PassThroughNodes": _abi.SNN_NODE_PASSTHROUGH}   # conversion/nodes.py


def _f(x) -> float:
    return float(x.item() if isinstance(x, torch.Tensor) else x)


def _u8(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8) if t.dtype == torch.bool else t


def _reduction_code(fn) -> int:
    if fn in (torch.sum, torch.squeeze):       # learning.py:76-80 / MCC_learning.py:68-74
        return _abi.SNN_REDUCE_SUM
    if fn is torch.mean:
        return _abi.SNN_REDUCE_MEAN
    raise NotImplementedError(f"reduction {fn} is not one the core implements (sum, mean)")


def fill_layer(d: "_abi.SnnLayer", layer, B: int, keep: List[torch.Tensor]) -> None:
    """bindsnet.network.nodes: Nodes.__init__ nodes.py:15-86, LIFNodes :425-498, DiehlAndCookNodes :988-1066."""
    kind = _KIND.get(type(layer).__name__)
    if kind is None:
        raise NotImplementedError(f"{type(layer).__name__} is outside the accelerated path")
    d.kind, d.n = kind, int(layer.n)
    d.traces, d.traces_additive = int(layer.traces), int(layer.traces_additive)
    d.sum_input, d.learning = int(layer.sum_input), int(layer.learning)
    d.dt = _f(layer.dt)
    rows = _neuron_rows(layer, kind)
    _g = lambda name: 0.0 if name in rows else _f(getattr(layer, name))                # a per-neuron row replaces the scalar
    if layer.traces:
        d.trace_decay, d.trace_scale = _g("trace_decay"), _g("trace_scale")               # nodes.py:129-131
        d.x = layer.x.data_ptr()
    if layer.sum_input:
        d.summed = layer.summed.data_ptr()
    if kind == _abi.SNN_NODE_PASSTHROUGH:
        # PassThroughNodes.forward stores its float input as s (conversion/nodes.py:137-144); before its first step s is
        # still the bool tensor of Nodes.set_batch_size: hand the core a float32 one with the same values
        if tuple(layer.s.shape) != (B, *layer.shape):
            layer.s = torch.zeros(B, *layer.shape, dtype=torch.float32, device=layer.s.device)
        elif layer.s.dtype != torch.float32 or not layer.s.is_contiguous():
            layer.s = layer.s.float().contiguous()
        d.traces = d.sum_input = 0                                                        # its forward never reaches Nodes.forward
        d.s = layer.s.data_ptr()
        return
    # Input.forward aliases the caller's input into s (nodes.py:219): give the core a private bool tensor
    if layer.s.dtype not in (torch.bool, torch.uint8) or tuple(layer.s.shape) != (B, *layer.shape) or not layer.s.is_contiguous():
        layer.s = torch.zeros(B, *layer.shape, dtype=torch.bool, device=layer.s.device)
    d.s = _u8(layer.s).data_ptr()
    if kind != _abi.SNN_NODE_INPUT:
        d.v = layer.v.data_ptr()
        d.thresh = _g("thresh")
        if kind != _abi.SNN_NODE_MCP:                                                     # McCullochPitts: v = x, no other state
            d.refrac_count, d.refrac = layer.refrac_count.data_ptr(), _f(layer.refrac)
        if hasattr(layer, "decay") and kind not in (_abi.SNN_NODE_IF, _abi.SNN_NODE_MCP):
            d.decay = _g("decay")                                                         # nodes.py:546-548, 1128-1130
        if hasattr(layer, "rest"):
            d.rest = _g("rest")
        if hasattr(layer, "reset"):
            d.reset = _f(layer.reset)
        lb = getattr(layer, "lbound", None)
        d.has_lbound, d.lbound = int(lb is not None), (_f(lb) if lb is not None else 0.0)
    if kind == _abi.SNN_NODE_CURRENT_LIF:
        d.i, d.i_decay = layer.i.data_ptr(), _f(layer.i_decay)                            # nodes.py:771, 818-820
    if kind == _abi.SNN_NODE_DC:
        d.theta = layer.theta.data_ptr()
        d.theta_plus, d.theta_decay = _g("theta_plus"), _g("theta_decay")                 # nodes.py:1131-1133
        d.one_spike = int(getattr(layer, "one_spike", False))
    if rows:   # the per-neuron block (include/snn_b200.h SNN_NODE_PN), [SNN_PN_ROWS, n] fp32 beside v
        block = torch.zeros(_abi.SNN_PN_ROWS, d.n, dtype=torch.float32, device=layer.v.device)
        for name, (r, t) in rows.items():
            block[r].copy_(t.detach().float().expand(tuple(layer.shape)).reshape(-1))
        keep.append(block)
        d.kind |= _abi.SNN_NODE_PN
        d.pn, d.pn_mask = block.data_ptr(), sum(1 << r for r, _ in rows.values())


def _neuron_rows(layer, kind: int) -> Dict[str, tuple]:
    """The parameters of a LIFNodes / AdaptiveLIFNodes / DiehlAndCookNodes population that are tensors of more than one
    element, by buffer name: {name: (SNN_PN_* row, tensor)}.  refrac / reset / lbound and a non-additive trace_scale
    reach masked_fill_, which takes a 0-dim value only: the reference's first step raises that RuntimeError."""
    if kind not in (_abi.SNN_NODE_LIF, _abi.SNN_NODE_DC):
        return {}
    many = lambda t: isinstance(t, torch.Tensor) and t.numel() != 1
    for name in ("refrac", "reset", "lbound") + (() if layer.traces_additive else ("trace_scale",)):
        t = getattr(layer, name, None)
        if layer.traces or name != "trace_scale":
            if many(t):
                raise RuntimeError(f"masked_fill_ only supports a 0-dimensional value tensor, but got tensor with {t.dim()} "
                                   f"dimension(s). ('{name}' is a per-neuron tensor)")
    names = [("thresh", _abi.SNN_PN_THRESH), ("rest", _abi.SNN_PN_REST), ("decay", _abi.SNN_PN_DECAY)]
    if kind == _abi.SNN_NODE_DC:
        names += [("theta_plus", _abi.SNN_PN_THETA_PLUS), ("theta_decay", _abi.SNN_PN_THETA_DECAY)]
    if layer.traces:
        names += [("trace_decay", _abi.SNN_PN_TRACE_DECAY)] + ([("trace_scale", _abi.SNN_PN_TRACE_SCALE)] if layer.traces_additive else [])
    rows = {name: (r, getattr(layer, name)) for name, r in names if many(getattr(layer, name))}
    for name, (_, t) in rows.items():
        if torch.broadcast_shapes(tuple(t.shape), tuple(layer.shape)) != tuple(layer.shape):
            raise NotImplementedError(f"per-neuron '{name}' of shape {tuple(t.shape)} grows the layer's state {tuple(layer.shape)}")
    return rows


def fill_connection(d: "_abi.SnnConn", conn, src: int, tgt: int, dt: float, keep: Optional[List[torch.Tensor]] = None,
                    B: Optional[int] = None, device: Optional[torch.device] = None) -> None:
    """``B`` / ``device``: the run's batch size and the layers' device (default: the source layer's), against which a
    MaxPool2dConnection's or MaxPoo3dConnection's rates buffer is checked."""
    keep = keep if keep is not None else []
    d.src, d.tgt = src, tgt
    d.weight_decay, d.dt_scale = 1.0, 1.0
    if type(conn).__name__ in ("MaxPool2dConnection", "MaxPoo3dConnection"):
        # topology.py:1124-1301: no weights; the firing_rates buffer is updated in place, so it must be [B, *source.shape]
        # for this run (the window reads and writes B * n_src floats) and on the run's device.  The reference allocates it
        # on the CPU at reset_state_variables (:1209-1211) and never resizes it when the batch size changes: move it to the
        # layers' device and reset it after a batch change before binding a run.
        from .network.topology import check_pool, fill_pool3d_geometry, pool_out_shape

        B = int(conn.source.s.shape[0]) if B is None else int(B)
        device = conn.source.s.device if device is None else torch.device(device)
        check_pool(conn, (B, *conn.source.shape))   # the reference's RuntimeError / TypeError, raised before anything runs
        fr = conn.firing_rates
        if fr.device != device:
            raise RuntimeError(f"{type(conn).__name__}.firing_rates is on {fr.device}, the run on {device}: move it to the "
                               "layers' device first")
        d.rule = _abi.SNN_RULE_NOOP
        if type(conn).__name__ == "MaxPoo3dConnection":
            d.kind = _abi.SNN_CONN_MAXPOOL3D
            fill_pool3d_geometry(d, conn)
        else:
            d.kind = _abi.SNN_CONN_MAXPOOL2D
            d.cin, d.hin, d.win = (int(v) for v in conn.source.shape)
            d.cout, d.hout, d.wout = pool_out_shape(conn)
            (d.kh, d.kw), (d.sh, d.sw) = conn.kernel_size, conn.stride
            (d.ph, d.pw), (d.dh, d.dw) = conn.padding, conn.dilation
        d.pool_decay = _f(conn.decay)
        d.pool_rates = fr.data_ptr()
        return
    if type(conn).__name__ == "MeanFieldConnection":
        # topology.py:1920-2006: s.float().mean() * w, w in its own shape and read through a per-target offset map;
        # learning.NoOp leaves it as it is (learning.py:93-104)
        from .network.topology import meanfield_offsets

        if conn.norm is not None:
            raise NotImplementedError("MeanFieldConnection with norm: the reference's normalize() fails at the end of the run")
        if type(conn.update_rule).__name__ != "NoOp":
            raise NotImplementedError(f"{type(conn.update_rule).__name__} on a MeanFieldConnection")
        w = conn.w
        if w.dtype != torch.float32 or not w.is_contiguous():
            raise TypeError("MeanFieldConnection.w must be contiguous float32")
        off, d.mf_stride = meanfield_offsets(conn, int(conn.source.s.shape[0]) if B is None else int(B), cache=False)
        keep.append(off)
        d.kind, d.rule, d.w, d.mf_off = _abi.SNN_CONN_MEANFIELD, _abi.SNN_RULE_NOOP, w.data_ptr(), off.data_ptr()
        return
    if type(conn).__name__ == "LocalConnection2D":
        # topology.py:1623-1767: w [in_channels, n_filters * conv_prod, kernel_prod], b never read; the geometry of the
        # reference's unfold (no padding, no dilation) and its view of the output as the target's shape
        (d.kh, d.kw), (d.sh, d.sw) = conn.kernel_size, conn.stride
        d.kind, d.cin, d.hin, d.win = _abi.SNN_CONN_LOCAL2D, *(int(v) for v in conn.source.shape)
        d.cout, (d.hout, d.wout) = int(conn.n_filters), conn.conv_size
        d.dh = d.dw = 1
        if int(conn.target.n) != d.cout * d.hout * d.wout:
            raise RuntimeError(f"shape '{[B, *conn.target.shape]}' is invalid for the LocalConnection2D output of "
                               f"{d.cout * d.hout * d.wout} neurons per sample")
        w = conn.w
        d.has_norm = int(conn.norm is not None)                                           # topology.py:1748-1759
        d.norm, d.norm_abs = (_f(conn.norm) if conn.norm is not None else 0.0), 0
        rule = conn.update_rule
        name = type(rule).__name__
        d.rule = {"NoOp": _abi.SNN_RULE_NOOP, "PostPre": _abi.SNN_RULE_POSTPRE, "Hebbian": _abi.SNN_RULE_HEBBIAN,
                  "WeightDependentPostPre": _abi.SNN_RULE_WDEP_POSTPRE}.get(name, -1)
        if d.rule < 0:
            raise NotImplementedError(f"learning rule {name} on a LocalConnection2D")
        d.nu0, d.nu1 = _f(rule.nu[0]), _f(rule.nu[1])
        d.reduction = _reduction_code(rule.reduction)
        d.weight_decay = _f(rule.weight_decay)                                            # learning.py:85
        d.wmin, d.wmax = _f(conn.wmin), _f(conn.wmax)
        d.has_clamp = int((math.isfinite(d.wmin) or math.isfinite(d.wmax)) and name != "NoOp")   # learning.py:97-104
        if w.dtype != torch.float32 or not w.is_contiguous():
            raise TypeError("weights must be contiguous float32")
        d.w = w.data_ptr()
        return
    if type(conn).__name__ == "LocalConnection3D":
        # topology.py:1770-1917: w [in_channels, n_filters * conv_prod, kernel_prod], b never read; the reference's axes
        # H, W, D on the depth, height and width fields (include/snn_b200.h SNN_CONN_LOCAL3D), no padding, no dilation
        from .network.topology import fill_local3d_geometry

        if len(conn.source.shape) != 4:
            raise NotImplementedError("LocalConnection3D from a source population other than [C, H, W, D]")
        fill_local3d_geometry(d, conn)
        d.kind = _abi.SNN_CONN_LOCAL3D
        if (d.kd > d.din or d.kh > d.hin or d.kw > d.win) or int(conn.target.n) != d.cout * d.dout * d.hout * d.wout:
            raise RuntimeError(f"LocalConnection3D: kernel_size {tuple(conn.kernel_size)} / stride {tuple(conn.stride)} on a "
                               f"{list(conn.source.shape)} source do not give the target's {int(conn.target.n)} neurons")
        d.has_norm = int(conn.norm is not None)                                           # topology.py:1898-1909
        d.norm, d.norm_abs = (_f(conn.norm) if conn.norm is not None else 0.0), 0
        rule = conn.update_rule
        name = type(rule).__name__
        d.rule = {"NoOp": _abi.SNN_RULE_NOOP, "PostPre": _abi.SNN_RULE_POSTPRE, "Hebbian": _abi.SNN_RULE_HEBBIAN,
                  "WeightDependentPostPre": _abi.SNN_RULE_WDEP_POSTPRE}.get(name, -1)
        if d.rule < 0:
            raise NotImplementedError(f"learning rule {name} on a LocalConnection3D")
        d.nu0, d.nu1 = _f(rule.nu[0]), _f(rule.nu[1])
        d.reduction = _reduction_code(rule.reduction)
        d.weight_decay = _f(rule.weight_decay)                                            # learning.py:85
        d.wmin, d.wmax = _f(conn.wmin), _f(conn.wmax)
        d.has_clamp = int((math.isfinite(d.wmin) or math.isfinite(d.wmax)) and name != "NoOp")   # learning.py:97-104
        if conn.w.dtype != torch.float32 or not conn.w.is_contiguous():
            raise TypeError("weights must be contiguous float32")
        d.w = conn.w.data_ptr()
        return
    if type(conn).__name__ == "Conv3dConnection":
        # topology.py:847-1025: w [out, in, kd, kh, kw], b [out]; the geometry of F.conv3d (dilation 1: the constructor refuses
        # any other).  Its rules: learning.NoOp's decay, or PostPre / WeightDependentPostPre with both rates zero (decay and
        # clamp); the others never run in a learning window (build_net raises the reference's error)
        d.kind = _abi.SNN_CONN_CONV3D
        d.cin, d.din, d.hin, d.win = (int(v) for v in conn.source.shape)
        d.cout, d.dout, d.hout, d.wout = (int(v) for v in conn.target.shape)
        (d.kd, d.kh, d.kw), (d.sd, d.sh, d.sw), (d.pd, d.ph, d.pw) = conn.kernel_size, conn.stride, conn.padding
        d.dh = d.dw = 1
        d.has_norm = int(conn.norm is not None)                                           # topology.py:1004-1018
        d.norm, d.norm_abs = (_f(conn.norm) if conn.norm is not None else 0.0), 0
        rule = conn.update_rule
        name = type(rule).__name__
        if name in ("NoOp", "PostPre", "WeightDependentPostPre"):
            d.rule = {"NoOp": _abi.SNN_RULE_NOOP, "PostPre": _abi.SNN_RULE_POSTPRE, "WeightDependentPostPre": _abi.SNN_RULE_WDEP_POSTPRE}[name]
            d.nu0, d.nu1 = _f(rule.nu[0]), _f(rule.nu[1])
            d.weight_decay = _f(rule.weight_decay)                                        # learning.py:85
            d.wmin, d.wmax = _f(conn.wmin), _f(conn.wmax)
            d.has_clamp = int((math.isfinite(d.wmin) or math.isfinite(d.wmax)) and name != "NoOp")   # learning.py:97-104
        for t in (conn.w, conn.b):
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise TypeError("weights and bias must be contiguous float32")
        d.w, d.b = conn.w.data_ptr(), conn.b.data_ptr()
        return
    if type(conn).__name__ == "Conv1dConnection":
        # topology.py:540-683: w [out, in, k], b [out]; the geometry of F.conv1d (dilation 1: the constructor refuses any
        # other) with the height axis set to 1
        if len(conn.source.shape) != 2 or len(conn.target.shape) != 2:
            raise NotImplementedError("Conv1dConnection between populations other than [C, L]")
        d.kind = _abi.SNN_CONN_CONV1D
        d.cin, d.win = (int(v) for v in conn.source.shape)
        d.cout, d.wout = (int(v) for v in conn.target.shape)
        d.kw, d.sw, d.pw = int(conn.kernel_size), int(conn.stride), int(conn.padding)
        d.hin = d.hout = d.kh = d.sh = 1
        d.dh = d.dw = 1
        d.has_norm = int(conn.norm is not None)                                           # topology.py:665-676
        d.norm, d.norm_abs = (_f(conn.norm) if conn.norm is not None else 0.0), 0
        rule = conn.update_rule
        name = type(rule).__name__
        d.rule = {"NoOp": _abi.SNN_RULE_NOOP, "PostPre": _abi.SNN_RULE_POSTPRE, "Hebbian": _abi.SNN_RULE_HEBBIAN,
                  "WeightDependentPostPre": _abi.SNN_RULE_WDEP_POSTPRE}.get(name, -1)
        if d.rule < 0:
            raise NotImplementedError(f"learning rule {name} on a Conv1dConnection")
        d.nu0, d.nu1 = _f(rule.nu[0]), _f(rule.nu[1])
        d.reduction = _reduction_code(rule.reduction)
        d.weight_decay = _f(rule.weight_decay)                                            # learning.py:85
        d.wmin, d.wmax = _f(conn.wmin), _f(conn.wmax)
        d.has_clamp = int((math.isfinite(d.wmin) or math.isfinite(d.wmax)) and name != "NoOp")   # learning.py:97-104
        for t in (conn.w, conn.b):
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise TypeError("weights and bias must be contiguous float32")
        d.w, d.b = conn.w.data_ptr(), conn.b.data_ptr()
        return
    if hasattr(conn, "pipeline"):
        # MulticompartmentConnection (topology.py:402-537) with one Weight feature (topology_features.py:575-671) and at most
        # one Probability (:365-464), Mask (:467-549) and Intensity (:724-769) feature each, in any order
        kinds = [type(f).__name__ for f in conn.pipeline]
        if kinds.count("Weight") != 1 or any(k not in ("Weight", "Probability", "Mask", "Intensity") or kinds.count(k) > 1 for k in kinds):
            raise NotImplementedError("only MulticompartmentConnection pipelines of one Weight feature and at most one Probability, "
                                      "Mask and Intensity feature each")
        by = {type(f).__name__: f for f in conn.pipeline}
        feat = by["Weight"]
        shape = (conn.source.n, conn.target.n)
        if "Probability" in by:                               # the window's draw: snn_synapse_draw(opts.seed, step, c, i, j)
            p = by["Probability"].value.detach().to(torch.float32).contiguous()
            keep.append(p)
            d.f_prob = p.data_ptr()
        if "Mask" in by:
            m = _u8(torch.broadcast_to(by["Mask"].value.detach(), shape)).contiguous()
            keep.append(m)
            d.f_mask = m.data_ptr()
        if "Intensity" in by:                                 # an int64 value (the default draw, :761-767) is -1 / 0 / 1
            i = torch.broadcast_to(by["Intensity"].value.detach().to(torch.float32), shape).contiguous()
            keep.append(i)
            d.f_int = i.data_ptr()
        rule = feat.learning_rule                                                         # an MCC_learning instance after priming
        d.kind = _abi.SNN_CONN_MCC
        w = feat.value
        d.has_norm = int(feat.norm is not None)                                           # topology_features.py:250-266: plain sum
        d.norm, d.norm_abs = (_f(feat.norm) if feat.norm is not None and not isinstance(feat.norm, torch.Tensor) else 0.0), 0
        norm, step = feat.norm, feat.norm_frequency == "time step"                         # :633-645, :663-671
        name = type(rule).__name__
        if name == "NoOp" or conn.manual_update:                                          # MCC_learning.py:120-146; topology.py:509-518
            d.rule = _abi.SNN_RULE_NONE
        elif name == "PostPre":
            d.rule = _abi.SNN_RULE_MCC_POSTPRE                                            # MCC_learning.py:224-302
            d.nu0, d.nu1 = _f(rule.nu[0]), _f(rule.nu[1])
            d.reduction = _reduction_code(rule.reduction)
            d.weight_decay = _f(rule.decay)                                               # MCC_learning.py:84: 1 - decay (1.0 = off)
            d.dt_scale = _f(conn.dt if getattr(conn, "dt", None) is not None else dt)     # MCC_learning.py:262,298
            lo, hi = rule.min, rule.max
            d.wmin = _f(lo) if lo is not None else -math.inf
            d.wmax = _f(hi) if hi is not None else math.inf
            d.has_clamp = int(lo is not None or hi is not None)                           # MCC_learning.py:101-110
            if getattr(rule, "average_update", 0) > 0:                                    # MCC_learning.py:210-220
                _fill_average(d, rule, keep)
        else:
            raise NotImplementedError(f"MCC learning rule {name}")
    else:
        # Connection (topology.py:265-399) + learning.LearningRule (learning.py:31-104)
        if type(conn).__name__ not in ("Connection", "LocalConnection", "SparseConnection"):
            raise NotImplementedError(f"{type(conn).__name__} is outside the accelerated path")
        rule = conn.update_rule
        d.kind = _abi.SNN_CONN_DENSE
        if not conn.w.is_sparse and not conn.w.is_contiguous():
            # ann_to_snn hands nn.Linear weights over as weight.t() (conversion.py:177-180): stored contiguous in place,
            # with the same values, since the core updates w in its own row-major storage
            with torch.no_grad():
                conn.w.data = conn.w.data.contiguous()
        w = conn.w
        d.has_norm = int(conn.norm is not None)                                           # topology.py:383-392: sum of |w|
        norm, step = conn.norm, False
        if isinstance(norm, torch.Tensor) and (type(conn).__name__ != "Connection" or tuple(norm.shape) in ((), (1,))):
            norm = _f(norm)                                                               # one value: the scalar division
        d.norm, d.norm_abs = (_f(norm) if norm is not None and not isinstance(norm, torch.Tensor) else 0.0), 1
        if type(conn).__name__ == "LocalConnection":
            # a dense matrix confined to its receptive fields by the connection's own mask (topology.py:1431, 1457-1469),
            # plain column sums in normalize (:1471-1479; norm is already scaled by the kernel size, :1437-1438)
            d.norm_abs = 0
            m = _u8(conn.mask.to(w.device)).contiguous()
            keep.append(m)
            d.mask = m.data_ptr()
        # wmin / wmax: scalars or tensors broadcasting to w (topology.py:74-81); the rule's nu: a pair of scalars or of
        # tensors (learning.py:58-67)
        tensors = conn.wmin.numel() != 1 or conn.wmax.numel() != 1 or rule.nu.dim() > 1
        if tensors and type(conn).__name__ != "Connection":
            raise NotImplementedError(f"per-synapse wmin / wmax or learning-rate tensors on a {type(conn).__name__}")
        d.wmin = _f(conn.wmin) if conn.wmin.numel() == 1 else -math.inf
        d.wmax = _f(conn.wmax) if conn.wmax.numel() == 1 else math.inf
        name = type(rule).__name__
        d.rule = {"NoOp": _abi.SNN_RULE_NOOP, "PostPre": _abi.SNN_RULE_POSTPRE, "Hebbian": _abi.SNN_RULE_HEBBIAN,
                  "WeightDependentPostPre": _abi.SNN_RULE_WDEP_POSTPRE}.get(name, -1)
        if d.rule < 0:
            raise NotImplementedError(f"learning rule {name}")
        if rule.nu.dim() == 1:
            d.nu0, d.nu1 = _f(rule.nu[0]), _f(rule.nu[1])
        d.reduction = _reduction_code(rule.reduction)
        d.weight_decay = _f(rule.weight_decay)                                            # learning.py:85
        from .network.topology import bounds_clamp, fill_synapse_tensors

        d.has_clamp = int(bounds_clamp(conn.wmin, conn.wmax) and name != "NoOp")          # learning.py:97-104
        if tensors:
            # the tensors the plan points at are kept alive with the plan (a copy only for a non-contiguous full layout)
            owner = type("_Keep", (), {})()
            fill_synapse_tensors(d, int(conn.source.n), int(conn.target.n), conn.w.device, conn.wmin.detach(), conn.wmax.detach(),
                                 rule.nu if rule.nu.dim() > 1 else None, owner=owner)
            keep.append(owner)
        if conn.b is not None:
            d.b = conn.b.data_ptr()
        if w.is_sparse:
            # SparseConnection (topology.py:2009-2017): the torch.sparse_coo w as CSR.  NoOp's decay leaves it
            # uncoalesced (learning.py:93-94); it is coalesced in place, and the values are the tensor's own
            _fill_sparse(d, conn, keep)
            return
    if w.dtype != torch.float32 or not w.is_contiguous():
        raise TypeError("weights must be contiguous float32")
    d.w = w.data_ptr()
    # plan-time structure hints for static square matrices (DiehlAndCook2015's exc / inh, models.py:204,217-220)
    static = d.rule == _abi.SNN_RULE_NONE or (d.rule == _abi.SNN_RULE_NOOP and d.weight_decay in (0.0, 1.0))
    if static and not d.has_norm and w.dim() == 2 and w.shape[0] == w.shape[1] and w.shape[0] > 1:
        with torch.no_grad():
            diag, eye = torch.diagonal(w), torch.eye(w.shape[0], dtype=torch.bool, device=w.device)
            if bool(((w == 0) | eye).all() & (diag == diag[0]).all()):
                d.structure, d.structure_val = _abi.SNN_W_DIAG, _f(diag[0])
            elif bool(((w == w[0, 1]) | eye).all() & (diag == 0).all()):
                d.structure, d.structure_val = _abi.SNN_W_OFFDIAG, _f(w[0, 1])
    if d.has_norm and (isinstance(norm, torch.Tensor) or step):
        _fill_norm(d, norm, step, int(conn.target.n), w.device, keep)


def _fill_norm(d: "_abi.SnnConn", norm, step: bool, n: int, device, keep: List[torch.Tensor]) -> None:
    """A per-target norm tensor (float32 [n] or [1, n]) and / or a Weight's per-step normalisation (snn_b200.h
    SNN_CONN_WNORM)."""
    d.kind |= _abi.SNN_CONN_WNORM
    d.norm_step = int(step)
    if isinstance(norm, torch.Tensor):
        v = norm.detach()
        if v.dim() == 2 and v.shape[0] == 1:
            v = v[0]
        if v.dtype != torch.float32 or tuple(v.shape) != (n,):
            raise NotImplementedError(f"a norm of shape {list(norm.shape)} and dtype {norm.dtype}: the CUDA core scales by a "
                                      f"float32 norm per target neuron ([{n}]) only")
        v = v.to(device).contiguous()
        keep.append(v)
        d.norm_t = v.data_ptr()


def _fill_sparse(d: "_abi.SnnConn", conn, keep: List[torch.Tensor]) -> None:
    d.kind = _abi.SNN_CONN_SPARSE
    if d.rule not in (_abi.SNN_RULE_NOOP, _abi.SNN_RULE_NONE):
        raise NotImplementedError("SparseConnection with a learning rule other than NoOp (the pattern would grow)")
    if not conn.w.is_coalesced():
        with torch.no_grad():
            conn.w.data = conn.w.data.coalesce()
    w = conn.w
    if w.dtype != torch.float32:
        raise TypeError("weights must be float32")
    idx, vals = w._indices(), w._values()
    if idx.shape[1] >= 2**31:
        raise NotImplementedError("more than 2**31 - 1 stored synapses")
    rowptr = torch.zeros(int(conn.source.n) + 1, dtype=torch.int32, device=idx.device)
    rowptr[1:] = torch.cumsum(torch.bincount(idx[0], minlength=int(conn.source.n)), 0).to(torch.int32)
    col = idx[1].to(torch.int32).contiguous()
    keep += [rowptr, col]
    d.nnz = int(idx.shape[1])
    d.sp_rowptr, d.sp_col = rowptr.data_ptr(), col.data_ptr() if d.nnz else None
    d.w = vals.data_ptr() if d.nnz else None


def build_net(network, inputs: Dict[str, torch.Tensor], T: int, B: int):
    """The window plan of a live reference ``Network`` (insertion orders: network.py:225, 386)."""
    from .network._plan import check_passthrough

    net = _abi.SnnNet()
    net.abi_version = _abi.SNN_ABI_VERSION
    net.n_layers, net.n_conns = len(network.layers), len(network.connections)
    net.learning = int(bool(network.learning))
    keep: List[torch.Tensor] = []
    names = list(network.layers)
    for i, name in enumerate(names):
        layer = network.layers[name]
        fill_layer(net.layers[i], layer, B, keep)
        if name in inputs:                                                                # network.py:388-392
            x = inputs[name][:T]
            if x.dtype not in (torch.bool, torch.uint8, torch.float32):
                x = x.float()
            x = _u8(x.to(layer.s.device).reshape(T, B, layer.n).contiguous())
            net.layers[i].ext = x.data_ptr()
            net.layers[i].ext_dtype = _abi.SNN_EXT_F32 if x.dtype == torch.float32 else _abi.SNN_EXT_U8
            keep.append(x)
    dev = next(iter(network.layers.values())).s.device
    layers = list(network.layers.values())
    for i, ((s, t), conn) in enumerate(network.connections.items()):
        if network.learning and type(conn).__name__ in ("MaxPool2dConnection", "MaxPoo3dConnection"):
            # the reference fails in the first step's update: learning.NoOp.update scales connection.w (learning.py:87-94)
            name = type(conn).__name__
            raise AttributeError(f"'{name}' object has no attribute 'w' (run {name} networks with learning off)")
        if network.learning and type(conn).__name__ == "Conv3dConnection":
            rule = conn.update_rule
            name = type(rule).__name__
            stdp = name in ("PostPre", "WeightDependentPostPre")
            if (name != "NoOp" and not stdp) or (stdp and bool(rule.nu[0] != 0)):
                # learning.py:499-559, 978-1050, 1382-1438, 2017-2121, 2739-2855: the bool unfolded source meets torch.bmm
                raise RuntimeError("expected m1 and m2 to have the same dtype, but got: float != bool")
            if stdp and bool(rule.nu[1] != 0):
                raise NotImplementedError(f"{name} with only a post-synaptic rate on a Conv3dConnection")
        # the source is connection.source (network.py:226-248): ann_to_snn's keys need not name it
        src = next((k for k, layer in enumerate(layers) if layer is conn.source), None)
        fill_connection(net.conns[i], conn, names.index(s) if src is None else src, names.index(t), float(network.dt), keep, B=B,
                        device=dev)
        check_passthrough(net, i, type(conn).__name__)
    return net, keep


def _fill_average(d: "_abi.SnnConn", rule, keep: List[torch.Tensor]) -> None:
    """PostPre's averaging state (include/snn_b200.h SNN_RULE_AVG): the reference's buffers and indices in place, and the
    slot bitmaps the core keeps beside them, built from the buffers (a row / column of a slot is marked when it holds a
    non-zero value; the other slots' values are zeros)."""
    k = int(rule.average_update)
    pre, post = rule.average_buffer_pre, rule.average_buffer_post
    for t in (pre, post):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise TypeError("the averaging buffers must be contiguous float32")

    def words(nz: torch.Tensor) -> torch.Tensor:   # [k, n] bool -> [k, ceil(n / 32)] int32 bit words
        n = nz.shape[1]
        pad = torch.zeros(k, (n + 31) // 32 * 32, dtype=torch.int64, device=nz.device)
        pad[:, :n] = nz.to(torch.int64)
        w = (pad.view(k, -1, 32) << torch.arange(32, device=nz.device)).sum(2)
        return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32).contiguous()

    rows, cols = words((pre != 0).any(2)), words((post != 0).any(1))
    keep += [rows, cols]
    d.rule |= _abi.SNN_RULE_AVG
    d.avg_k, d.avg_continues = k, int(bool(rule.continues_update))
    d.avg_idx_pre, d.avg_idx_post = int(rule.average_buffer_index_pre), int(rule.average_buffer_index_post)
    d.avg_pre, d.avg_post, d.avg_rows, d.avg_cols = pre.data_ptr(), post.data_ptr(), rows.data_ptr(), cols.data_ptr()


def _advance_averages(network, T: int) -> None:
    """After a window: each averaged PostPre's indices move by the window's updates on the sides whose rate is non-zero
    (MCC_learning.py:252-254, :286-288)."""
    if not network.learning:
        return
    for conn in network.connections.values():
        for f in getattr(conn, "pipeline", ()):
            rule = getattr(f, "learning_rule", None)
            if type(rule).__name__ == "PostPre" and getattr(rule, "average_update", 0) > 0 and not conn.manual_update:
                k = int(rule.average_update)
                if rule.nu[0]:
                    rule.average_buffer_index_pre = (rule.average_buffer_index_pre + T) % k
                if rule.nu[1]:
                    rule.average_buffer_index_post = (rule.average_buffer_index_post + T) % k


def run_window(network, inputs: Dict[str, torch.Tensor], time: int, seed: Optional[int] = None, library: Optional[C.CDLL] = None) -> int:
    """Drop-in for ``network.run(inputs, time)`` of a reference ``Network`` (the body of network.py:329-465).
    ``library``: a CDLL exporting ``snn_oracle_run_window`` (CPU tensors) — default: the CUDA core on CUDA tensors."""
    inputs = dict(inputs)
    for k in inputs:                                                                       # network.py:329-340
        if inputs[k].dim() == 1:
            inputs[k] = inputs[k].unsqueeze(0).unsqueeze(0)
        elif inputs[k].dim() == 2:
            inputs[k] = inputs[k].unsqueeze(1)
    for k in inputs:                                                                       # network.py:342-353
        if inputs[k].size(1) != network.batch_size:
            network.batch_size = inputs[k].size(1)
            for layer in network.layers.values():
                layer.set_batch_size(network.batch_size)
        break
    T, B = int(time / network.dt), int(network.batch_size)
    net, keep = build_net(network, inputs, T, B)
    opts = _abi.SnnRunOpts()
    opts.T, opts.B, opts.normalize = T, B, 1
    opts.seed = (int(torch.randint(0, 2**31 - 1, (1,)).item()) if seed is None else seed) & 0xFFFFFFFF
    if library is not None:
        err = C.c_int32(0)
        opts.err_flag = C.cast(C.pointer(err), C.c_void_p).value
        library.snn_oracle_run_window.restype = C.c_int
        library.snn_oracle_run_window.argtypes = [C.POINTER(_abi.SnnNet), C.POINTER(_abi.SnnRunOpts), C.c_int, C.c_int]
        rc = library.snn_oracle_run_window(C.byref(net), C.byref(opts), 0, 0)
        del keep
        if rc == 0:
            _advance_averages(network, T)
        return rc | int(err.value)
    from . import _backend

    dev = next(iter(network.layers.values())).s.device
    _backend.run_window(net, opts, dev)
    del keep
    _advance_averages(network, T)
    return 0
