"""Multi-GPU windows: batch shards with ONE exchange per window (SURVEY.md §8e).

The reference has no multi-device path at all.  The north_star defines one: every rank holds
a full replica of the weights and adaptive thresholds and a shard of the input batch, runs the
ordinary window locally (per-step STDP / clamp / theta on its shard), and at the window
boundary the accumulated changes are summed over ranks —

    dW_r = W_r - W0,  dtheta_r = theta_r - theta0          (snn_b200_delta_prepare)
    all_reduce(sum) of one fused fp32 buffer over NCCL      (no per-timestep collective)
    W = clamp(W0 + sum_r dW_r, wmin, wmax); theta = theta0 + sum_r dtheta_r
    normalize()                                             (snn_b200_delta_apply)

On the fused DiehlAndCook2015 kernel the first line costs nothing: the window's epilogue writes dW_r and dtheta_r
straight into the all-reduce buffer and leaves W0 / theta0 in place (``snn_run_opts_t.delta_w / delta_theta``), and
the last two lines are one launch (``snn_b200_delta_apply_fused``) — window kernel, all-reduce, apply.

This is "replicas + one exchange", NOT a single-process run at the global batch size: that
would need the batch-summed dW and dtheta exchanged every timestep.  tests/test_distributed.py
checks it against the combination of independent oracle replicas.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from . import _abi, _backend


class ShardedWindowRunner:
    """Wraps a ``Network`` replica; ``run`` has ``Network.run``'s signature."""

    def __init__(self, network, process_group: Optional["dist.ProcessGroup"] = None):
        self.network = network
        self.group = process_group
        self._flat: Optional[torch.Tensor] = None
        self._snap: Optional[torch.Tensor] = None
        self._delta_windows: Optional[bool] = None   # None: not tried yet; False: this graph / tier has no delta window

    def _learned(self) -> List[Tuple[object, "_abi.SnnConn"]]:
        """Connections whose weights change inside a window (a learning rule, or the end-of-run normalize),
        with the constants the combine needs.  Built from the objects' attributes — not from the per-window
        plan, which reward-modulated rules can only fill during a run."""
        from .network.topology import Conv1dConnection, Conv2dConnection, Conv3dConnection, LocalConnection3D

        out = []
        for conn in self.network.connections.values():
            if hasattr(conn, "pipeline"):  # MulticompartmentConnection[Weight]: plain-sum normalize, dt-scaled rule
                d = _abi.SnnConn()
                conn._fill_desc(d, float(self.network.dt))
                if d.rule & _abi.SNN_RULE_AVG:
                    raise NotImplementedError("PostPre(average_update>0) is not supported by ShardedWindowRunner: each rank "
                                              "would average its own shard's updates, and the buffers would diverge")
                w = conn._weight()
                if w.norm is not None and (w.norm_frequency == "time step" or isinstance(w.norm, torch.Tensor)):
                    raise NotImplementedError("a Weight normalised every time step or by a norm tensor is not supported by "
                                              "ShardedWindowRunner: each rank would normalise its own replica, and the "
                                              "combine normalises with a scalar norm at the end")
            else:
                if getattr(conn, "_norm_tensor", lambda: None)() is not None:
                    raise NotImplementedError("a per-target norm tensor is not supported by ShardedWindowRunner: the combine "
                                              "normalises with a scalar norm")
                rule = getattr(conn, "update_rule", None)
                code = getattr(rule, "rule_code", None)
                code = int(code) if code is not None else _abi.SNN_RULE_NONE
                d = _abi.SnnConn()
                d.rule = code
                d.has_norm = int(conn.norm is not None)
                d.norm = float(conn.norm) if conn.norm is not None else 0.0
                d.norm_abs = 1
                import math
                if (conn.wmin.numel() != 1 or conn.wmax.numel() != 1) and code >= _abi.SNN_RULE_POSTPRE:
                    raise NotImplementedError("the multi-GPU combine clamps with scalar bounds: a learned connection with "
                                              "per-synapse wmin / wmax tensors is not supported by ShardedWindowRunner")
                d.wmin, d.wmax = (float(conn.wmin), float(conn.wmax)) if conn.wmin.numel() == 1 and conn.wmax.numel() == 1 else (-math.inf, math.inf)
                d.has_clamp = int(code >= _abi.SNN_RULE_POSTPRE and (math.isfinite(d.wmin) or math.isfinite(d.wmax)))
            if d.rule >= _abi.SNN_RULE_POSTPRE or d.has_norm:
                # [Cout,Cin,kh,kw] / [Cout,Cin,kd,kh,kw] / [Cout,Cin,k] weights normalise per filter (topology.py:824-837,
                # 1004-1018, 665-676), a LocalConnection3D's [Cin,n,K] per contiguous row (:1898-1909), the combine kernel
                # per column of an [n_src,n_tgt] matrix: for them it applies sum + clamp only, the connection's own
                # normalize follows
                d._conv = isinstance(conn, (Conv1dConnection, Conv2dConnection, Conv3dConnection, LocalConnection3D))
                out.append((conn, d))
        return out

    def _thetas(self) -> List[torch.Tensor]:
        return [l.theta for l in self.network.layers.values() if getattr(l, "kind", None) == _abi.SNN_NODE_DC]

    def run(self, inputs: Dict[str, torch.Tensor], time: int, **kwargs) -> None:
        net = self.network
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        learned = self._learned() if net.learning else []
        thetas = self._thetas() if net.learning else []
        if world == 1 or not net.learning:
            net.run(inputs, time, **kwargs)
            return
        total = sum(c.w.numel() for c, _ in learned) + sum(t.numel() for t in thetas)
        dev = net._device()
        if self._flat is None or self._flat.numel() != total or self._flat.device != dev:
            self._flat = torch.empty(total, dtype=torch.float32, device=dev)
            self._snap = torch.empty(total, dtype=torch.float32, device=dev)
        # (`_emulated`: set by tests/test_distributed.py, whose ranks run the CUDA sources on tests/emu's CPU emulation)
        if ((dev.type == "cuda" or getattr(self, "_emulated", False)) and self._delta_windows is not False and len(learned) == 1 and len(thetas) == 1
                and int(time / net.dt) > 0 and learned[0][0].w.dim() == 2):
            # fused path: the window writes dW / dtheta into the all-reduce buffer, W0 / theta0 stay where they are
            conn, d = learned[0]
            w, th = conn.w.detach(), thetas[0]
            dw, dth = self._flat[:w.numel()].view_as(w), self._flat[w.numel():]
            try:
                net.run(inputs, time, b200_normalize=False, b200_delta=(dw, dth), **kwargs)
                self._delta_windows = True
            except _backend.BackendError:
                if self._delta_windows:   # it worked before: a real error
                    raise
                self._delta_windows = False   # not the fused DiehlAndCook2015 graph / tier: the general path below
            else:
                dist.all_reduce(self._flat, op=dist.ReduceOp.SUM, group=self.group)
                _backend.delta_apply_fused(w, dw, d.has_clamp, d.wmin, d.wmax, d.has_norm, d.norm_abs, d.norm, theta=th, dtheta_sum=dth)
                return
        # snapshot W0 / theta0
        off = 0
        views = []
        for t in [c.w for c, _ in learned] + thetas:
            v = self._snap[off:off + t.numel()].view_as(t)
            v.copy_(t.detach())
            views.append((t, v, off))
            off += t.numel()

        net.run(inputs, time, b200_normalize=False, **kwargs)

        for t, v0, o in views:
            _backend.delta_prepare(t.detach(), v0, self._flat[o:o + t.numel()].view_as(t))
        dist.all_reduce(self._flat, op=dist.ReduceOp.SUM, group=self.group)
        k = 0
        for conn, d in learned:
            t, v0, o = views[k]; k += 1
            if getattr(d, "_conv", False):
                rows = conn.w.shape[0]
                _backend.delta_apply(conn.w.detach().view(rows, -1), v0.view(rows, -1), self._flat[o:o + t.numel()].view(rows, -1),
                                     d.has_clamp, d.wmin, d.wmax, 0, 1, 0.0)
                if d.has_norm:
                    conn.normalize()
                continue
            _backend.delta_apply(conn.w.detach(), v0, self._flat[o:o + t.numel()].view_as(t), d.has_clamp, d.wmin,
                                 d.wmax, d.has_norm, d.norm_abs, d.norm)
        for th in thetas:
            t, v0, o = views[k]; k += 1
            th.copy_(v0 + self._flat[o:o + t.numel()].view_as(t))
