"""Learning rules for ``Connection`` — host-side mirror of ``bindsnet/learning/learning.py``
(``LearningRule`` :25-104, ``NoOp`` :107-146, ``PostPre`` :149-420 / :457-497 (conv2d),
``WeightDependentPostPre`` :562-653 / :920-975, ``Hebbian`` :1052-1136 / :1348-1380, ``MSTDP``; the three unsupervised
rules also on ``LocalConnection2D``, :258-320 / :717-791 / :1186-1250, on ``LocalConnection3D``, :322-388 / :793-871 /
:1249-1314, and on ``Conv1dConnection``, :422-455 / :873-918 / :1316-1346; on ``Conv3dConnection`` only what the reference can run, see ``Conv3dConnection``).  The rule objects hold hyper-parameters; the update
itself is fused into the CUDA window kernels (``Network.run``) or submitted for one step by
``rule.update()``."""
from __future__ import annotations

import warnings
from abc import ABC
from typing import Optional, Sequence, Union

import numpy as np
import torch

from .. import _abi
from .MCC_learning import _EligibilityTrace, _RewardModulated, _reduction_code


class LearningRule(ABC):
    """Reference: learning.py:25-104."""

    rule_code = None

    def __init__(
        self,
        connection,
        nu: Optional[Union[float, Sequence[float], Sequence[torch.Tensor]]] = None,
        reduction: Optional[callable] = None,
        weight_decay: float = 0.0,
        **kwargs,
    ) -> None:
        self.connection = connection
        self.source = connection.source
        self.target = connection.target
        self.wmin = connection.wmin
        self.wmax = connection.wmax
        # learning.py:58-66
        if nu is None:
            self.nu = torch.tensor([0.0, 0.0], dtype=torch.float)
        elif isinstance(nu, (float, int)):
            self.nu = torch.tensor([nu, nu], dtype=torch.float)
        elif all(isinstance(e, (float, int)) for e in nu):
            self.nu = torch.tensor(nu, dtype=torch.float)
        else:
            # a pair of tensors (learning.py:66): per-neuron or per-synapse rates, on a dense Connection only
            from ..network.topology import Connection

            if not isinstance(connection, Connection) or not connection._synapse_tensors:
                raise NotImplementedError(f"per-synapse learning-rate tensors are not supported by the CUDA core on a "
                                          f"{type(connection).__name__} (dense Connection only)")
            self.nu = torch.stack(tuple(nu), dim=0).to(dtype=torch.float)
        # rates the kernels read from the tensor (0-d rates are scalars, read once per version of the tensor)
        self._nu_tensors = self.nu.dim() > 1
        if not self.nu.any() and not isinstance(self, NoOp):
            warnings.warn(
                f"nu is set to zeros for {type(self).__name__} learning rule. "
                "It will disable the learning process."
            )
        self.reduction = reduction if reduction is not None else (
            torch.squeeze if self.source.batch_size == 1 else torch.sum
        )
        self._squeeze = self.reduction is torch.squeeze
        from ..network.topology import MeanFieldConnection

        # a MeanFieldConnection passes its weight_decay in the reduction slot (reference topology.py:1957); NoOp, the only
        # rule it runs, never reduces
        self._reduction_code = (_abi.SNN_REDUCE_SUM if isinstance(connection, MeanFieldConnection)
                                else _reduction_code(reduction, self.source.batch_size))
        self.weight_decay = 1.0 - weight_decay if weight_decay else 1.0

    def update(self, **kwargs) -> None:
        """Apply this rule once to the connection from the layers' current ``s``/``x``
        (reference: the rule-specific ``_connection_update`` + learning.py:87-104).

        A USER-DEFINED rule (a subclass that changes ``self.connection.w`` itself with torch ops and then calls
        ``super().update()``, learning.py:31-104) gets the reference's base behaviour here: weight decay and the
        clamp to ``[wmin, wmax]``; ``Network.run`` drives networks with such rules step by step (the scripted tier)."""
        if self.rule_code is None:
            w = self.connection.w
            if self.weight_decay:                                         # learning.py:93-94
                w *= self.weight_decay
            wmin, wmax = self.connection.wmin, self.connection.wmax       # learning.py:97-104
            if bool((wmin != -np.inf).any()) or bool((wmax != np.inf).any()):
                w.clamp_(wmin, wmax)
            return
        from ..network import _plan

        _plan.update_single_connection(self.connection)

    def _fill_desc(self, d: "_abi.SnnConn") -> None:
        if self.rule_code is None:
            raise NotImplementedError(
                f"user-defined learning rule {type(self).__name__} cannot be fused into the CUDA window; "
                "supported: NoOp, PostPre, WeightDependentPostPre, Hebbian, MSTDP"
            )
        d.rule = self.rule_code
        d.reduction = self._reduction_code
        if self._nu_tensors:   # Connection._fill_desc points the kernels at the tensors and sets the gates
            d.nu0 = d.nu1 = 0.0
        else:
            d.nu0 = float(self.nu[0])
            d.nu1 = float(self.nu[1])
        d.weight_decay = float(self.weight_decay)
        # learning.py:97-104: clamp iff some element of wmin is not -inf or some element of wmax is not +inf, and the
        # rule is not NoOp
        from ..network.topology import bounds_clamp

        d.has_clamp = int(bounds_clamp(self.connection.wmin, self.connection.wmax) and not isinstance(self, NoOp))


def _check_connection(rule, connection) -> None:
    """The STDP-family rules exist for ``Connection`` (``_connection_update``), ``Conv2dConnection``
    (``_conv2d_connection_update``) and ``LocalConnection2D`` (``_local_connection2d_update``); the reference's im2col
    ignores dilation, so a dilated filter is refused.  On ``Conv3dConnection`` (``_conv3d_connection_update``) the
    post-synaptic-only form of PostPre / WeightDependentPostPre pairs the kernel axes transposed against ``w``
    (learning.py:517-530, 996-1010); it is not built, so such a rule is refused here.  ``Conv1dConnection``
    (``_conv1d_connection_update``) and ``LocalConnection3D`` (``_local_connection3d_update``) run all three."""
    from ..network.topology import (Connection, Conv1dConnection, Conv2dConnection, Conv3dConnection, LocalConnection2D,
                                    LocalConnection3D)

    if not isinstance(connection, (Connection, Conv2dConnection, LocalConnection2D, Conv3dConnection, Conv1dConnection,
                                   LocalConnection3D)):
        raise NotImplementedError("This learning rule is not supported for this Connection type.")
    if isinstance(connection, Conv3dConnection) and isinstance(rule, (PostPre, WeightDependentPostPre)) and \
            float(rule.nu[0]) == 0.0 and float(rule.nu[1]) != 0.0:
        raise NotImplementedError(f"{type(rule).__name__} with only a post-synaptic rate on a Conv3dConnection: the reference "
                                  "pairs its kernel axes transposed against w, which is not implemented (DESIGN.md section 8)")
    if isinstance(connection, Conv2dConnection) and connection._geometry[3] != (1, 1):
        raise NotImplementedError(f"{type(rule).__name__} on a dilated Conv2dConnection is undefined in the reference (im2col ignores dilation)")


class NoOp(LearningRule):
    """Reference: learning.py:107-146 — weight decay only."""

    rule_code = _abi.SNN_RULE_NOOP


class PostPre(LearningRule):
    """Pair-based STDP (reference: learning.py:149-420; dense update :390-420, conv2d :457-497)."""

    rule_code = _abi.SNN_RULE_POSTPRE

    def __init__(self, connection, nu=None, reduction=None, weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(connection=connection, nu=nu, reduction=reduction, weight_decay=weight_decay, **kwargs)
        assert self.source.traces and self.target.traces, (
            "Both pre- and post-synaptic nodes must record spike traces."
        )
        _check_connection(self, connection)


class WeightDependentPostPre(LearningRule):
    """Weight-dependent STDP (reference: learning.py:562-653; dense update :626-653, conv2d :920-975)."""

    rule_code = _abi.SNN_RULE_WDEP_POSTPRE

    def __init__(self, connection, nu=None, reduction=None, weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(connection=connection, nu=nu, reduction=reduction, weight_decay=weight_decay, **kwargs)
        assert self.source.traces, "Pre-synaptic nodes must record spike traces."
        assert self.target.traces, "Post-synaptic nodes must record spike traces."
        assert (connection.wmin != -np.inf).any() and (connection.wmax != np.inf).any(), (
            "Connection must define finite wmin and wmax."
        )
        _check_connection(self, connection)


class Hebbian(LearningRule):
    """Hebbian rule: both terms positive, learning rates applied after the batch reduction
    (reference: learning.py:1052-1438; dense update :1110-1136, conv2d :1348-1380)."""

    rule_code = _abi.SNN_RULE_HEBBIAN

    def __init__(self, connection, nu=None, reduction=None, weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(connection=connection, nu=nu, reduction=reduction, weight_decay=weight_decay, **kwargs)
        assert self.source.traces and self.target.traces, (
            "Both pre- and post-synaptic nodes must record spike traces."
        )
        _check_connection(self, connection)


class MSTDP(_RewardModulated, LearningRule):
    """Reward-modulated STDP (reference: learning.py:1440-2121): dense ``Connection``
    (``_connection_update`` :1504-1574) and ``Conv2dConnection`` (``_conv2d_connection_update``
    :1942-2015).  Rule state lives here like in the reference: ``p_plus``, ``p_minus`` and — for the
    convolutional form — ``eligibility`` ``[B, *w.shape]``.  The dense form never materialises the
    ``[B, n_src, n_tgt]`` eligibility: it is ``p_plus (x) s_post + s_pre (x) p_minus`` of the previous
    step, so the spikes the rule saw last are kept instead (``eligibility`` rebuilds it on request).
    ``Network.run(..., reward=r)`` is mandatory, ``a_plus`` / ``a_minus`` optional (:1540-1556).  For
    ``Conv2dConnection`` the eligibility is per sample for any batch size (the reference's final
    ``.view(w.size())`` at :2013 only works for batch size 1; SURVEY.md §0.8)."""

    rule_code = _abi.SNN_RULE_MSTDP

    def __init__(self, connection, nu=None, reduction=None, weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(connection=connection, nu=nu, reduction=reduction, weight_decay=weight_decay, **kwargs)
        from ..network.topology import Connection, Conv1dConnection, Conv2dConnection, Conv3dConnection, LocalConnection3D

        if isinstance(connection, LocalConnection3D):
            # learning.py:1764-1866 / 2458-: the local forms of the reward-modulated rules are not built
            raise NotImplementedError(f"{type(self).__name__} on a LocalConnection3D is not implemented: its local form "
                                      "(learning.py:1764-1866) is not built on the CUDA core")
        if isinstance(connection, Conv1dConnection):
            # learning.py:1868-1940 / 2571-: at B > 1 the eligibility [B, out, in * k] is viewed into w's shape, which
            # fails; at B = 1 the rule sums the eligibility over the output channels from the second step on
            raise NotImplementedError(f"{type(self).__name__} on a Conv1dConnection is not implemented: the reference's update "
                                      "fails at batch size > 1 and sums the eligibility over output channels at batch size 1")
        if not isinstance(connection, (Connection, Conv2dConnection, Conv3dConnection)):
            raise NotImplementedError("This learning rule is not supported for this Connection type.")
        self._conv = isinstance(connection, Conv2dConnection)
        # built as in the reference; its learning windows are refused (Conv3dConnection._check_learning)
        self._conv3d = isinstance(connection, Conv3dConnection)
        if self._conv and connection._geometry[3] != (1, 1):
            raise NotImplementedError("MSTDP on a dilated Conv2dConnection is undefined in the reference (im2col ignores dilation)")
        self.tc_plus = torch.tensor(kwargs.get("tc_plus", 20.0))
        self.tc_minus = torch.tensor(kwargs.get("tc_minus", 20.0))
        self._run_kwargs = {}

    def update(self, **kwargs) -> None:
        raise NotImplementedError("MSTDP.update is fused into Network.run (it needs the run's reward); the standalone call is not exposed")

    def _prepare(self, B: int, dev: torch.device, run_kwargs: dict) -> None:
        """Allocate / validate the rule state for a window (learning.py:1519-1535, 1958-1961, 1979-1991)."""
        if self._conv3d:   # the rule never runs (Conv3dConnection._check_learning): no state
            return
        self._take_run_kwargs(run_kwargs)
        src, tgt = self.source, self.target
        if self._conv:
            self._ensure("p_plus", (B, *src.shape), dev)
            self._ensure("p_minus", (B, tgt.shape[0], tgt.shape[1] * tgt.shape[2]), dev)
            self._ensure("_elig", (B, *self.connection.w.shape), dev)
        else:
            self._prepare_traces((B, src.n), (B, tgt.n), dev)

    @property
    def eligibility(self) -> torch.Tensor:
        """``[B, *w.shape]`` eligibility that the next update will apply (learning.py:1568-1572, 2005-2010)."""
        if self._conv:
            return self._elig
        return _RewardModulated.eligibility.fget(self)

    def _fill_desc(self, d: "_abi.SnnConn") -> None:
        super()._fill_desc(d)
        self._fill_reward(d, float(self.connection.dt))
        if self._conv:
            d.elig = self._elig.data_ptr()


class MSTDPET(_EligibilityTrace, MSTDP):
    """Reward-modulated STDP with an eligibility trace on a dense ``Connection`` (reference: learning.py:2124-2249;
    ``_connection_update`` :2187-2249).  Batch size 1 only: the reference flattens the spikes of the whole batch into its
    ``[n]`` traces (:2214-2215), which only has a meaning for one sample.  Rule state like the reference's: ``p_plus [n_src]``,
    ``p_minus [n_tgt]``, ``eligibility_trace [n_src, n_tgt]``; ``eligibility`` is rebuilt on request from the traces and the
    spikes the rule saw last.  The convolutional / local forms (:2251-2855) are outside the implemented path."""

    rule_code = _abi.SNN_RULE_MSTDPET

    def __init__(self, connection, nu=None, reduction=None, weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(connection=connection, nu=nu, reduction=reduction, weight_decay=weight_decay, **kwargs)
        if self._conv:
            raise NotImplementedError("MSTDPET on a Conv2dConnection is outside the implemented path (dense Connection only)")
        self.tc_e_trace = torch.tensor(kwargs.get("tc_e_trace", 25.0))

    def _prepare(self, B: int, dev: torch.device, run_kwargs: dict) -> None:
        if self._conv3d:
            return
        self._prepare_trace(B, tuple(self.connection.w.shape), dev)
        super()._prepare(B, dev, run_kwargs)

    def _fill_desc(self, d: "_abi.SnnConn") -> None:
        super()._fill_desc(d)
        self._fill_trace(d, float(self.connection.dt))


def _unsupported(name: str, where: str):
    class _Unsupported(LearningRule):
        __doc__ = f"``{name}`` (reference: {where}) — not on the accelerated path (SURVEY.md §8f)."

        def __init__(self, *args, **kwargs):
            raise NotImplementedError(f"learning.{name} is outside the hot path bindsnet_b200 implements")

    _Unsupported.__name__ = name
    return _Unsupported


class Rmax(LearningRule):
    """Reward-maximisation rule for stochastic ``SRM0Nodes`` targets (reference: learning.py:2858-2960; update
    :2921-2960): per synapse an eligibility trace that decays by ``1 - dt / tc_e_trace`` and gains
    ``(s_post - p / (1 + tc_c / dt * p)) * x_pre`` each step (``p`` the target's spike probability of the step), and
    ``w += nu[0] * reward * eligibility``.  Its target draws from torch's generator, so — like ``SRM0Nodes`` — the rule
    has no kernel form: it is host torch code on the connection's device and the network runs on the scripted tier.
    As in the reference the flattened views make it a batch-size-1 rule."""

    rule_code = None

    def __init__(self, connection, nu=None, reduction=None, weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(connection=connection, nu=nu, reduction=reduction, weight_decay=weight_decay, **kwargs)
        from ..network.nodes import SRM0Nodes
        from ..network.topology import Connection

        assert self.source.traces and self.source.traces_additive, "Pre-synaptic nodes must use additive spike traces."
        assert isinstance(self.target, SRM0Nodes), "R-max needs stochastically firing neurons, use SRM0Nodes."
        if not isinstance(connection, Connection):        # Connection and its subclass LocalConnection (learning.py:2905-2910)
            raise NotImplementedError("This learning rule is not supported for this Connection type.")
        self.tc_c = torch.tensor(kwargs.get("tc_c", 5.0))                 # 0: naive Hebbian ... inf: policy gradient
        self.tc_e_trace = torch.tensor(kwargs.get("tc_e_trace", 25.0))

    def update(self, **kwargs) -> None:
        w, dt = self.connection.w, self.connection.dt
        if not hasattr(self, "eligibility_trace"):
            self.eligibility_trace = torch.zeros(*w.shape, device=w.device)
        fired = self.target.s.view(-1).float()
        p = self.target.s_prob.view(-1)
        self.eligibility_trace *= 1 - dt / self.tc_e_trace
        self.eligibility_trace += (fired - p / (1.0 + self.tc_c / dt * p)) * self.source.x.view(-1)[:, None]
        with torch.no_grad():
            w += self.nu[0] * kwargs["reward"] * self.eligibility_trace
        super().update()
