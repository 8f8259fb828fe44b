"""``Network`` — host-side mirror of ``bindsnet/network/network.py``.

Same registry API (``add_layer`` / ``add_connection`` / ``add_monitor``, network.py:119-161),
same ``run(inputs, time, **kwargs)`` contract (network.py:252-465), same
``reset_state_variables`` / ``train`` / ``save`` / ``load`` / ``clone``.  The difference is
inside ``run``: instead of a Python loop over timesteps that dispatches ~80 ATen ops and
three host syncs per step, the whole window is described once (``_plan.build_net``) and
executed by one persistent CUDA kernel behind ``snn_b200_run_window``.
"""
from __future__ import annotations

import tempfile
from typing import Dict, Optional, Tuple

import torch

from .. import _abi, _backend
from . import _plan
from .monitors import AbstractMonitor, Monitor, SpikeCounter
from .nodes import Nodes


def load(file_name: str, map_location: str = "cpu", learning: bool = None) -> "Network":
    """Reference: network.py:12-28."""
    network = torch.load(open(file_name, "rb"), map_location=map_location, weights_only=False)
    if learning is not None and "learning" in vars(network):
        network.learning = learning
    return network


class Network(torch.nn.Module):
    """Registry of layers, connections and monitors plus the simulation entry point
    (reference: network.py:31-491)."""

    def __init__(self, dt: float = 1.0, batch_size: int = 1, learning: bool = True, reward_fn=None) -> None:
        super().__init__()
        self.dt = dt
        self.batch_size = batch_size
        self.layers = {}
        self.connections = {}
        self.monitors = {}
        self.train(learning)
        # network.py:114-117: the class is instantiated here; run() asks it for each window's reward
        self.reward_fn = reward_fn() if reward_fn is not None else None
        #: seed of the last window's draws: the one_spike tie-break (snn_one_spike_key) and the Probability features'
        #: synapse draws (snn_synapse_draw)
        self.last_one_spike_seed: Optional[int] = None

    # -- registry (network.py:119-161) ----------------------------------------------------
    def add_layer(self, layer: Nodes, name: str) -> None:
        self.layers[name] = layer
        self.add_module(name, layer)
        layer.train(self.learning)
        layer.compute_decays(self.dt)
        layer.set_batch_size(self.batch_size)

    def add_connection(self, connection, source: str, target: str) -> None:
        self.connections[(source, target)] = connection
        self.add_module(source + "_to_" + target, connection)
        connection.dt = self.dt
        connection.train(self.learning)

    def add_monitor(self, monitor: AbstractMonitor, name: str) -> None:
        self.monitors[name] = monitor
        monitor.network = self
        monitor.dt = self.dt

    # -- persistence (network.py:163-209) -------------------------------------------------
    def save(self, file_name: str) -> None:
        torch.save(self, open(file_name, "wb"))

    def clone(self) -> "Network":
        virtual_file = tempfile.SpooledTemporaryFile()
        torch.save(self, virtual_file)
        virtual_file.seek(0)
        return torch.load(virtual_file, weights_only=False)

    # -- simulation -----------------------------------------------------------------------
    def run(self, inputs: Dict[str, torch.Tensor], time: int, one_step=False, **kwargs) -> None:
        """Simulate ``int(time / dt)`` steps (reference: network.py:252-465).

        ``inputs[l]`` has shape ``[time, batch, *layer.shape]`` (or the shorter forms the
        reference accepts, network.py:329-340).  Keyword arguments: ``clamp``, ``unclamp``,
        ``injects_v`` as in the reference (network.py:268-281).  Extensions: ``one_spike_seed``
        fixes the window's draws — the tie-break of ``DiehlAndCookNodes(one_spike=True)`` and the synapse draws of
        ``Probability`` features (without it, a seed is drawn from torch's CPU generator);
        ``b200_normalize=False`` skips the end-of-run normalize (used by the multi-GPU combine,
        ``bindsnet_b200.distributed``).
        """
        assert type(inputs) == dict, (
            "'inputs' must be a dict of names of layers (str) and relevant input tensors. "
            f"Got {type(inputs).__name__} instead."
        )
        # network.py:325-326: a reward_fn replaces the run's reward by its own (e.g. a prediction error)
        if self.reward_fn is not None:
            kwargs["reward"] = self.reward_fn.compute(**kwargs)
        # reward-modulated rules (learning.MSTDP) read these from the run's kwargs (network.py:319-377,
        # learning.py:1540-1556)
        self._rule_kwargs = {k: kwargs.get(k, None) for k in ("reward", "a_plus", "a_minus")}

        # network.py:329-353: canonical [T, B, ...] shape, batch-size inference, state reset
        inputs = dict(inputs)
        for key in inputs:
            if inputs[key].dim() == 1:
                inputs[key] = inputs[key].unsqueeze(0).unsqueeze(0)
            elif inputs[key].dim() == 2:
                inputs[key] = inputs[key].unsqueeze(1)
        for key in inputs:
            if inputs[key].size(1) != self.batch_size:
                self.batch_size = inputs[key].size(1)
                for l in self.layers:
                    self.layers[l].set_batch_size(self.batch_size)
                for m in self.monitors:
                    self.monitors[m].reset_state_variables()
            break

        timesteps = int(time / self.dt)  # network.py:356
        self._run_window(
            inputs, timesteps, normalize=bool(kwargs.get("b200_normalize", True)), delta=kwargs.get("b200_delta", None),
            clamp=kwargs.get("clamp", {}), unclamp=kwargs.get("unclamp", {}),
            injects_v=kwargs.get("injects_v", {}), seed=kwargs.get("one_spike_seed", None), one_step=bool(one_step),
            masks=kwargs.get("masks", {}) or {},
        )

    def _rule_kwargs_of(self, key) -> dict:
        """The reward-modulation kwargs one connection's rule sees (network.py:359-377, 440-461): ``a_plus`` /
        ``a_minus`` may be dicts keyed by connection; a connection without an entry falls back to the rule's default."""
        out = dict(getattr(self, "_rule_kwargs", None) or {})
        for k in ("a_plus", "a_minus"):
            if isinstance(out.get(k, None), dict):
                out[k] = out[k].get(key, None)
        return out

    def _get_inputs(self, layers=None) -> Dict[str, torch.Tensor]:
        """What every layer (or the named ones) receives from the connections ending in it, given the sources'
        current spikes: the sum of ``compute`` over those connections in insertion order (network.py:211-250).
        Inside a window the kernels do this themselves (the gather phase); this host form — one single-operator
        launch per connection — serves the scripted tier and callers that step a network by hand."""
        from .topology import MeanFieldConnection, MulticompartmentConnection

        B = self.batch_size
        cur = {}
        draw = getattr(self, "_draw", None)   # (seed, step) of the scripted tier's current step
        for k, ((src, tgt), conn) in enumerate(self.connections.items()):
            if layers is not None and tgt not in layers:
                continue
            if draw is not None and type(conn) is MulticompartmentConnection:
                out = _plan.compute_single_connection(conn, conn.source.s, draw=(draw[0], draw[1], k))
            else:
                out = conn.compute(conn.source.s)
            if isinstance(conn, MeanFieldConnection):   # shaped like w: broadcast into the input as network.py:248 adds it
                out = out.broadcast_to((B, *self.layers[tgt].shape))
            out = out.view(B, *self.layers[tgt].shape).float()
            cur[tgt] = cur[tgt] + out if tgt in cur else out
        return cur

    def _device(self) -> torch.device:
        return _plan.network_device(self)

    def _stage_input(self, name: str, x: torch.Tensor, T: int, dev: torch.device) -> torch.Tensor:
        layer = self.layers[name]
        if x.size(0) < T:
            raise ValueError(f"inputs['{name}'] has {x.size(0)} time steps, {T} required")
        x = x[:T]
        if x.dtype in (torch.bool, torch.uint8, torch.float32):
            pass
        elif x.dtype.is_floating_point:
            x = x.float()
        else:
            x = x.to(torch.uint8) if layer.kind == _abi.SNN_NODE_INPUT else x.float()
        x = x.to(dev, non_blocking=True)
        return x.reshape(T, self.batch_size, layer.n).contiguous()

    def _stage_mask(self, name: str, m, T: int, dev: torch.device, as_float: bool) -> torch.Tensor:
        layer = self.layers[name]
        m = torch.as_tensor(m)
        is_index = not as_float and m.dtype not in (torch.bool, torch.uint8)
        per_step = (m.dim() != 1) and not is_index  # network.py:418-421: 1-D = static, else [T, ...]
        if as_float:
            out = m.to(dev, torch.float32)
        elif not is_index:
            out = m.to(dev, torch.uint8)
        else:  # index tensor, as accepted by ``s[:, clamp] = 1`` (network.py:419)
            idx = m.to(dev).long()
            if m.dim() == 1:
                out = torch.zeros(layer.n, dtype=torch.uint8, device=dev)
                out[idx] = 1
            else:  # [T, k]: the neurons ``clamp[t]`` names at step t (network.py:421); negative indices wrap like indexing
                per_step = True
                idx = idx[:T].reshape(T, -1)
                out = torch.zeros(T, layer.n, dtype=torch.uint8, device=dev)
                out.scatter_(1, torch.where(idx < 0, idx + layer.n, idx), 1)
        out = out.reshape(T, layer.n) if per_step else out.reshape(layer.n)
        return out.contiguous()

    def _fusable_monitor(self, mon) -> Optional[str]:
        if isinstance(mon, SpikeCounter):
            for name, layer in self.layers.items():
                if mon.obj is layer:
                    return name
            return None
        if not isinstance(mon, Monitor):
            return None
        for name, layer in self.layers.items():
            if mon.obj is layer:
                ok = all(v in Monitor.FUSED_VARS for v in mon.state_vars)
                ok = ok and not ("v" in mon.state_vars and layer.kind in (_abi.SNN_NODE_INPUT, _abi.SNN_NODE_PASSTHROUGH))
                return name if ok else None
        return None

    def _stage_conn_masks(self, masks, dev: torch.device):
        """``masks={(source, target): bool tensor}`` (network.py:279-280,321): weights to clamp to zero after every
        step's update (AbstractConnection.update, topology.py:127-131)."""
        from .topology import Connection, SparseConnection, _MaxPoolConnection

        out = {}
        for key, m in (masks or {}).items():
            if m is None:
                continue
            if key not in self.connections:
                continue                                  # network.py:449 looks masks up per connection: unknown keys are ignored
            conn = self.connections[key]
            if isinstance(conn, SparseConnection):
                raise NotImplementedError("Mask isn't supported for SparseConnection")   # topology.py:129-131
            if isinstance(conn, _MaxPoolConnection):
                raise AttributeError(conn._no_w_message())                              # self.w.masked_fill_, topology.py:127-131
            if hasattr(conn, "pipeline"):
                continue                                  # MulticompartmentConnection.update ignores the kwarg (topology.py:509-518)
            if not isinstance(conn, Connection):
                raise NotImplementedError(f"masks for {type(conn).__name__} are outside the implemented path (dense Connection only)")
            m = torch.as_tensor(m)
            if tuple(m.shape) != tuple(conn.w.shape):
                raise ValueError(f"mask for {key} has shape {tuple(m.shape)}, weights {tuple(conn.w.shape)}")
            out[key] = (m != 0).to(dev, torch.uint8).contiguous()
        # a connection with a structural mask of its own (LocalConnection.update, topology.py:1457-1469) uses it
        # whenever the caller passes none for it
        for key, conn in self.connections.items():
            own = getattr(conn, "mask", None)
            if key not in out and isinstance(conn, Connection) and isinstance(own, torch.Tensor):
                cache = getattr(conn, "_b200_mask_u8", None)
                if cache is None or cache.device != dev or cache.shape != own.shape:
                    cache = (own != 0).to(dev, torch.uint8).contiguous()
                    conn._b200_mask_u8 = cache
                out[key] = cache
        return out

    def _run_window(self, inputs, T: int, normalize: bool, clamp=None, unclamp=None, injects_v=None,
                    seed: Optional[int] = None, step_offset: int = 0, one_step: bool = False, masks=None, delta=None) -> None:
        self._one_step = bool(one_step)
        dev = self._device()
        self._conn_masks = self._stage_conn_masks(masks, dev)
        B = self.batch_size
        if T <= 0:
            if normalize:
                for c in self.connections.values():
                    c.normalize()
            return
        for conn in self.connections.values():   # errors the reference raises inside the window, before anything runs
            if hasattr(conn, "_check_window"):
                conn._check_window(bool(self.learning))
        ext = {k: self._stage_input(k, v, T, dev) for k, v in inputs.items() if k in self.layers}
        clamps = {k: self._stage_mask(k, v, T, dev, False) for k, v in (clamp or {}).items() if v is not None}
        unclamps = {k: self._stage_mask(k, v, T, dev, False) for k, v in (unclamp or {}).items() if v is not None}
        injects = {k: self._stage_mask(k, v, T, dev, True) for k, v in (injects_v or {}).items() if v is not None}
        if seed is None:
            # only a one_spike population and a Probability feature consume the window's draws; a network without either
            # leaves torch's generator alone (as the reference does: its only draws on the path are DiehlAndCookNodes'
            # multinomial, nodes.py:1097-1105, and Probability's bernoulli, topology_features.py:425-429)
            if any(getattr(l, "one_spike", False) for l in self.layers.values()) or any(
                    _plan.has_probability(c) for c in self.connections.values()):
                seed = int(torch.randint(0, 2**31 - 1, (1,)).item())  # CPU generator: torch.manual_seed governs it
            else:
                seed = 0
        self.last_one_spike_seed = seed

        if delta is not None and (self._scripted_required() or T <= 0):
            raise _backend.BackendError("b200_delta windows run on the fused DiehlAndCook2015 kernel only")
        if self._scripted_required():
            return self._run_scripted(ext, T, normalize, clamps, unclamps, injects, self._conn_masks, bool(one_step), seed, step_offset)

        fused = {name: self._fusable_monitor(m) for name, m in self.monitors.items()}
        if any(layer is None for layer in fused.values()):
            if delta is not None:
                raise _backend.BackendError("b200_delta windows run on the fused DiehlAndCook2015 kernel only")
            return self._run_stepwise(ext, T, normalize, clamps, unclamps, injects, seed, step_offset)

        rec: Dict[str, Tuple[Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor]]] = {}
        for mname, lname in fused.items():
            mon, layer = self.monitors[mname], self.layers[lname]
            rs, rv, rc = rec.get(lname, (None, None, None))
            if isinstance(mon, SpikeCounter):
                rec[lname] = (rs, rv, mon._begin_window(B, dev))
                continue
            if "s" in mon.state_vars and rs is None:
                rs = torch.empty(T, B, layer.n, dtype=torch.uint8, device=dev)
            if "v" in mon.state_vars and rv is None:
                rv = torch.empty(T, B, layer.n, dtype=torch.float32, device=dev)
            rec[lname] = (rs, rv, rc)

        net, keep = _plan.build_net(self, B, ext, clamps, unclamps, injects, rec)
        opts = _abi.SnnRunOpts()
        opts.T, opts.B, opts.normalize = T, B, int(normalize)
        opts.tier = int(getattr(self, "force_tier", 0))
        opts.seed, opts.step_offset = seed & 0xFFFFFFFF, step_offset
        opts.one_step = int(self._one_step)
        if delta is not None:   # multi-GPU window: weight / theta changes go to the caller's all-reduce buffer (include/snn_b200.h)
            opts.delta_w, opts.delta_theta = delta[0].data_ptr(), delta[1].data_ptr()
        self._launch(net, opts, dev)
        self._advance_rules(T)
        del keep

        for mname, lname in fused.items():
            mon, layer = self.monitors[mname], self.layers[lname]
            if isinstance(mon, SpikeCounter):
                continue
            rs, rv, _ = rec[lname]
            if "s" in mon.state_vars:   # (a PassThroughNodes layer's s is float32)
                rs = rs.float() if layer.kind == _abi.SNN_NODE_PASSTHROUGH else rs.view(torch.bool)
                mon._push_window("s", rs.view(T, B, *layer.shape))
            if "v" in mon.state_vars:
                mon._push_window("v", rv.view(T, B, *layer.shape))

    def _launch(self, net, opts, dev) -> None:
        for layer in self.layers.values():
            _backend.require_cuda(layer.s, "layer state")
        from .topology import _MaxPoolConnection

        for conn in self.connections.values():
            if isinstance(conn, _MaxPoolConnection):
                _backend.require_cuda(conn.firing_rates, f"{type(conn).__name__}.firing_rates")
            else:
                _backend.require_cuda(conn.w, "connection weights")
        try:
            _backend.run_window(net, opts, dev)
        except _backend.BackendError:
            self._forget_structure()
            raise

    def _advance_rules(self, T: int) -> None:
        """After a window of T steps: an averaged MCC PostPre's slot indices move by the window's updates
        (MCC_learning.py:252-288); a window with learning off leaves them."""
        if self.learning:
            for conn in self.connections.values():
                if hasattr(conn, "pipeline") and not conn.manual_update:
                    advance = getattr(conn._weight().learning_rule, "_advance", None)
                    if advance is not None:
                        advance(T)

    def _forget_structure(self) -> None:
        """Drop the cached structure hints of the static weight matrices (``_plan.weight_structure``): after a
        device-side error they are re-verified on the next window."""
        for conn in self.connections.values():
            conn.__dict__.pop("_b200_structure", None)

    def _run_stepwise(self, ext, T, normalize, clamps, unclamps, injects, seed, step_offset) -> None:
        """Fallback for per-step observers the kernels cannot serve (monitors on ``x``,
        ``theta``, ``w`` ...): T one-step windows with ``Monitor.record`` after each, like
        network.py:380-461.  Still CUDA-only; just launch-bound."""
        B = self.batch_size
        for t in range(T):
            e = {k: v[t:t + 1] for k, v in ext.items()}
            c = {k: (v[t] if v.dim() == 2 else v) for k, v in clamps.items()}
            u = {k: (v[t] if v.dim() == 2 else v) for k, v in unclamps.items()}
            i = {k: (v[t] if v.dim() == 2 else v) for k, v in injects.items()}
            net, keep = _plan.build_net(self, B, e, c, u, i, {})
            opts = _abi.SnnRunOpts()
            opts.T, opts.B, opts.normalize = 1, B, 0     # the end-of-run normalize follows the last record (below)
            opts.tier = int(getattr(self, "force_tier", 0))
            opts.seed, opts.step_offset = seed & 0xFFFFFFFF, step_offset + t
            opts.one_step = int(getattr(self, "_one_step", False))
            self._launch(net, opts, self._device())
            self._advance_rules(1)
            for m in self.monitors.values():
                if isinstance(m, SpikeCounter) and t == 0:
                    m._begin_window(B, self._device())
                m.record()
        if normalize:                                     # network.py:463-465: after the last step's monitors
            for c in self.connections.values():
                c.normalize()

    # -- scripted tier: user-defined populations / rules / connections -------------------------------
    def _scripted_required(self) -> bool:
        """True when the network holds an object the window kernels cannot execute: a ``Nodes`` subclass with its
        own ``forward``, a ``LearningRule`` subclass with its own ``update``, a connection class of the user's.
        Such networks run step by step like the reference's loop (network.py:380-461), every built-in piece still on
        its CUDA single-operator kernel, the user's pieces as the torch code they are."""
        from ..learning import learning as L
        from ..learning import MCC_learning as ML
        from . import nodes as N, topology as Tp
        from ..conversion import nodes as CN

        builtin_nodes = (N.Input, N.LIFNodes, N.DiehlAndCookNodes, N.IFNodes, N.CurrentLIFNodes, N.AdaptiveLIFNodes, N.BoostedLIFNodes,
                         N.McCullochPitts, CN.SubtractiveResetIFNodes, CN.PassThroughNodes)
        for layer in self.layers.values():
            if type(layer) not in builtin_nodes and (layer.kind is None or type(layer).forward is not N.Nodes.forward):
                return True
        builtin_conns = (Tp.Connection, Tp.MulticompartmentConnection, Tp.Conv2dConnection, Tp.LocalConnection, Tp.SparseConnection,
                         Tp.MaxPool2dConnection, Tp.LocalConnection2D, Tp.Conv3dConnection, Tp.Conv1dConnection,
                         Tp.LocalConnection3D, Tp.MaxPoo3dConnection, Tp.MeanFieldConnection)
        for conn in self.connections.values():
            if type(conn) not in builtin_conns:
                return True
            rule = getattr(conn, "update_rule", None)
            if rule is not None and (rule.rule_code is None or type(rule).update is not L.LearningRule.update
                                     and type(rule) not in (L.NoOp, L.PostPre, L.WeightDependentPostPre, L.MSTDP, L.MSTDPET)):
                return True
        return False

    def _run_scripted(self, ext, T, normalize, clamps, unclamps, injects, masks, one_step, seed=0, step_offset=0) -> None:
        """Per-timestep executor with the reference's own control flow (network.py:380-465): inputs from the
        previous step's spikes in connection insertion order, layers in insertion order, clamp / unclamp /
        injects_v, connection updates, monitors, end-of-run normalize.  Probability features draw what the window
        kernel draws for the same seed and step."""
        try:
            self._scripted_steps(ext, T, normalize, clamps, unclamps, injects, masks, one_step, seed, step_offset)
        finally:
            self._draw = None

    def _scripted_steps(self, ext, T, normalize, clamps, unclamps, injects, masks, one_step, seed, step_offset) -> None:
        B = self.batch_size
        dev = self._device()
        get_inputs = self._get_inputs

        for t in range(T):
            self._draw = (seed, step_offset + t)
            current = {} if one_step else get_inputs()
            for lname, layer in self.layers.items():                          # network.py:386-413
                if one_step:
                    current.update(get_inputs([lname]))
                e = ext.get(lname)
                if e is not None:
                    x_ext = e[t].view(B, *layer.shape)
                    if lname in current and not one_step:
                        x = current[lname] + x_ext.float()
                    elif lname in current:
                        x = current[lname]                                    # one-step mode drops the external input (network.py:393-396)
                    else:
                        x = x_ext
                else:
                    x = current.get(lname)
                    if x is None:
                        x = torch.zeros(B, *layer.shape, device=dev)
                inj = injects.get(lname)
                if inj is not None:                                           # network.py:398-404
                    layer.v += (inj[t] if inj.dim() == 2 else inj).view(1, *layer.shape)
                layer.forward(x=x)
                c = clamps.get(lname)
                if c is not None:                                             # network.py:415-421
                    m = (c[t] if c.dim() == 2 else c).bool().view(1, *layer.shape).expand(B, *layer.shape)
                    layer.s = layer.s | m if layer.s.dtype == torch.bool else layer.s.masked_fill(m, 1)
                u = unclamps.get(lname)
                if u is not None:                                             # network.py:423-429
                    m = (u[t] if u.dim() == 2 else u).bool().view(1, *layer.shape).expand(B, *layer.shape)
                    layer.s = layer.s & ~m if layer.s.dtype == torch.bool else layer.s.masked_fill(m, 0)
            for key, conn in self.connections.items():                        # network.py:431-454
                rule_kwargs = {k: v for k, v in self._rule_kwargs_of(key).items() if v is not None}
                conn.update(mask=masks.get(key), learning=self.learning, **rule_kwargs)
            for m in self.monitors.values():                                  # network.py:460-461
                if isinstance(m, SpikeCounter) and t == 0:
                    m._begin_window(B, dev)
                m.record()
        if normalize:
            for conn in self.connections.values():                            # network.py:464-465
                conn.normalize()

    def check_errors(self) -> None:
        """Synchronise and raise if the device reported an error (non-binary input spikes,
        barrier time-out).  Errors otherwise surface on the next ``run``."""
        dev = self._device()
        if dev.type == "cuda":
            try:
                _backend.poll_errors(dev, sync=True)
            except _backend.BackendError:
                self._forget_structure()
                raise

    def reset_state_variables(self) -> None:
        """network.py:467-479.  Layers whose reset is the stock one (it is for every population this
        package implements) are cleared together: one multi-tensor zero plus one fill per voltage,
        instead of three to four launches per layer."""
        from .nodes import Nodes, LIFNodes, DiehlAndCookNodes

        from .nodes import CurrentLIFNodes, IFNodes

        from .nodes import BoostedLIFNodes

        stock = {Nodes.reset_state_variables, LIFNodes.reset_state_variables, DiehlAndCookNodes.reset_state_variables,
                 CurrentLIFNodes.reset_state_variables, BoostedLIFNodes.reset_state_variables}
        zeros, fills = [], []
        for layer in self.layers.values():
            if type(layer).reset_state_variables in stock and hasattr(layer, "_reset_plan"):
                z, f = layer._reset_plan()
                zeros += z
                fills += f
            else:
                layer.reset_state_variables()
        if zeros:
            torch._foreach_zero_(zeros)
        for t, value in fills:
            t.fill_(value)
        for connection in self.connections.values():
            connection.reset_state_variables()
        for monitor in self.monitors.values():
            monitor.reset_state_variables()

    def train(self, mode: bool = True) -> "torch.nn.Module":
        """network.py:481-491."""
        self.learning = mode
        return super().train(mode)
