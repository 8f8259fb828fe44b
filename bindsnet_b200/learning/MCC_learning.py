"""Learning rules for ``MulticompartmentConnection`` features — host-side mirror of
``bindsnet/learning/MCC_learning.py`` (``MCC_LearningRule`` :16-118, ``NoOp`` :121-146,
``PostPre`` :149-302, ``MSTDP`` :392-551, ``MSTDPET`` :554-738).  The rule objects hold hyper-parameters
(and, for the reward-modulated rules, their state); the update itself is fused into the CUDA window kernels."""
from __future__ import annotations

import warnings
from abc import ABC
from typing import Optional, Sequence, Union

import torch

from .. import _abi


def _reduction_code(reduction, batch_size) -> int:
    if reduction is None:
        # learning.py:76-80 / MCC_learning.py:73-79: squeeze when batch_size == 1 at rule
        # construction, else sum.  Over a batch of one they coincide; over a larger batch
        # the reference's squeeze raises (SURVEY.md §0.9) — we check that at plan time.
        return _abi.SNN_REDUCE_SUM
    if reduction in (torch.sum,):
        return _abi.SNN_REDUCE_SUM
    if reduction in (torch.mean,):
        return _abi.SNN_REDUCE_MEAN
    if reduction is torch.squeeze:
        return _abi.SNN_REDUCE_SUM
    raise NotImplementedError(
        f"reduction {reduction!r} is not supported by the CUDA core (torch.sum, torch.mean, torch.squeeze)"
    )


class MCC_LearningRule(ABC):
    """Reference: MCC_learning.py:16-118."""

    rule_code = _abi.SNN_RULE_NONE

    def __init__(
        self,
        connection,
        feature_value: Union[float, int, torch.Tensor],
        range: Optional[Union[list, tuple]] = None,
        nu: Optional[Union[float, Sequence[float]]] = None,
        reduction: Optional[callable] = None,
        decay: float = 0.0,
        enforce_polarity: bool = False,
        **kwargs,
    ) -> None:
        self.connection = connection
        self.source = connection.source
        self.target = connection.target
        self.feature_value = feature_value
        self.enforce_polarity = enforce_polarity
        self.min, self.max = range
        if nu is None:
            nu = [0.2, 0.1]
        elif isinstance(nu, (float, int)):
            nu = [nu, nu]
        self.nu = torch.zeros(2, dtype=torch.float)
        self.nu[0] = nu[0]
        self.nu[1] = nu[1]
        if (self.nu == torch.zeros(2)).all() and not isinstance(self, NoOp):
            warnings.warn(
                f"nu is set to [0., 0.] for {type(self).__name__} learning rule. "
                "It will disable the learning process."
            )
        self._squeeze = reduction is None and self.source.batch_size == 1 or reduction is torch.squeeze
        self.reduction = reduction if reduction is not None else (
            torch.squeeze if self.source.batch_size == 1 else torch.sum
        )
        self._reduction_code = _reduction_code(reduction, self.source.batch_size)
        self.decay = 1.0 - decay if decay else 1.0

    def update(self, **kwargs) -> None:
        from ..network import _plan

        _plan.update_single_connection(self.connection)

    def reset_state_variables(self) -> None:
        pass

    def _fill_desc(self, d: "_abi.SnnConn") -> None:
        d.rule = self.rule_code
        d.reduction = self._reduction_code
        d.nu0 = float(self.nu[0])
        d.nu1 = float(self.nu[1])
        d.weight_decay = float(self.decay)
        d.wmin = float(self.min) if self.min is not None else float("-inf")
        d.wmax = float(self.max) if self.max is not None else float("inf")
        d.has_clamp = int(self.min is not None or self.max is not None)


class NoOp(MCC_LearningRule):
    """Reference: MCC_learning.py:121-146 — really does nothing (no decay, no clamp)."""

    rule_code = _abi.SNN_RULE_NONE

    def __init__(self, **args) -> None:
        pass

    def update(self, **kwargs) -> None:
        pass

    def _fill_desc(self, d) -> None:
        d.rule = _abi.SNN_RULE_NONE
        d.reduction = _abi.SNN_REDUCE_SUM
        d.weight_decay = 1.0
        d.wmin, d.wmax = float("-inf"), float("inf")
        d.has_clamp = 0


class PostPre(MCC_LearningRule):
    """Pair-based STDP on a ``Weight`` feature (reference: MCC_learning.py:149-302): both
    terms are scaled by ``connection.dt`` (:262,:298), then decay and clamp (:86-110).

    ``average_update=k > 0`` (:210-220, :244-291) keeps the last k terms of each side in ``average_buffer_pre`` /
    ``average_buffer_post`` (``[k, *w.shape]``, on the weight's device) and applies their mean times ``dt``: every update
    with ``continues_update=True``, else on every k-th update (when the side's index wraps to 0).  A side whose rate is 0
    never touches its buffer or index.  The buffers and ``average_buffer_index_pre`` / ``_post`` survive
    ``reset_state_variables`` (it does nothing, :304-305); a window advances each used index by its learning steps.
    Besides the buffers the rule keeps, per slot, the rows (pre) and columns (post) that may hold non-zero values: a slot
    outside them is zero, which lets the kernel skip it (include/snn_b200.h SNN_RULE_AVG)."""

    rule_code = _abi.SNN_RULE_MCC_POSTPRE

    def __init__(
        self,
        connection,
        feature_value: Union[torch.Tensor, float, int],
        range: Optional[Sequence[float]] = None,
        nu: Optional[Union[float, Sequence[float]]] = None,
        reduction: Optional[callable] = None,
        decay: float = 0.0,
        enforce_polarity: bool = False,
        **kwargs,
    ) -> None:
        super().__init__(
            connection=connection, feature_value=feature_value,
            range=[-1, +1] if range is None else range, nu=nu, reduction=reduction,
            decay=decay, enforce_polarity=enforce_polarity, **kwargs,
        )
        assert self.source.traces and self.target.traces, (
            "Both pre- and post-synaptic nodes must record spike traces "
            "(use traces='True' on source/target layers)"
        )
        from ..network.topology import MulticompartmentConnection

        if not isinstance(connection, MulticompartmentConnection):
            raise NotImplementedError("This learning rule is not supported for this Connection type.")
        if enforce_polarity:
            raise NotImplementedError("enforce_polarity is not implemented by the CUDA core")
        self.average_update = kwargs.get("average_update", 0)
        self.continues_update = kwargs.get("continues_update", False)
        if self.average_update > 0:
            if getattr(connection, "sparse", False) or self.feature_value.is_sparse:
                raise NotImplementedError("PostPre(average_update>0) on sparse weights is not implemented by the CUDA core")
            k, dev = int(self.average_update), self.feature_value.device
            self.average_buffer_pre = torch.zeros(k, *self.feature_value.shape, device=dev)
            self.average_buffer_post = torch.zeros_like(self.average_buffer_pre)
            self.average_buffer_index_pre = 0
            self.average_buffer_index_post = 0
            n_src, n_tgt = self.source.n, self.target.n
            self._avg_rows = torch.zeros(k, (n_src + 31) // 32, dtype=torch.int32, device=dev)
            self._avg_cols = torch.zeros(k, (n_tgt + 31) // 32, dtype=torch.int32, device=dev)

    def _prepare(self, B: int, dev: torch.device, run_kwargs: dict) -> None:
        """The averaging state on the weight's device (moved with its contents when the network moved)."""
        if self.average_update > 0:
            for name in ("average_buffer_pre", "average_buffer_post", "_avg_rows", "_avg_cols"):
                t = getattr(self, name)
                if t.device != dev or not t.is_contiguous():
                    setattr(self, name, t.to(dev).contiguous())
            shape = (int(self.average_update), *self.feature_value.shape)
            for name in ("average_buffer_pre", "average_buffer_post"):
                t = getattr(self, name)
                if tuple(t.shape) != shape or t.dtype != torch.float32:
                    raise ValueError(f"PostPre.{name} must be a float32 tensor of shape {list(shape)}, got {t.dtype} {list(t.shape)}")

    def _fill_desc(self, d: "_abi.SnnConn") -> None:
        super()._fill_desc(d)
        if self.average_update > 0:
            d.rule = self.rule_code | _abi.SNN_RULE_AVG
            d.avg_k = int(self.average_update)
            d.avg_idx_pre, d.avg_idx_post = int(self.average_buffer_index_pre), int(self.average_buffer_index_post)
            d.avg_continues = int(bool(self.continues_update))
            d.avg_pre, d.avg_post = self.average_buffer_pre.data_ptr(), self.average_buffer_post.data_ptr()
            d.avg_rows, d.avg_cols = self._avg_rows.data_ptr(), self._avg_cols.data_ptr()

    def _advance(self, steps: int) -> None:
        """After ``steps`` learning updates: each side whose rate is non-zero moves its index (MCC_learning.py:252-254,
        :286-288)."""
        if self.average_update > 0 and steps > 0:
            k = int(self.average_update)
            if float(self.nu[0]) != 0.0:
                self.average_buffer_index_pre = (self.average_buffer_index_pre + steps) % k
            if float(self.nu[1]) != 0.0:
                self.average_buffer_index_post = (self.average_buffer_index_post + steps) % k

    def update(self, **kwargs) -> None:
        super().update(**kwargs)
        self._advance(1)

    def reset_state_variables(self) -> None:
        """MCC_learning.py:304-305: nothing (the averaging buffers and indices persist)."""


class _RewardModulated:
    """Rule state and plan fields of the reward-modulated rules: ``learning.MSTDP`` / ``MSTDPET`` on a ``Connection`` and
    ``MSTDP`` / ``MSTDPET`` below on a ``MulticompartmentConnection``'s Weight, which share their arithmetic
    (snn_b200.h SNN_RULE_MSTDP / SNN_RULE_MSTDPET).  ``p_plus`` / ``p_minus`` are the rule's traces; the
    ``[B, n_src, n_tgt]`` eligibility of the previous step is ``p_plus (x) s_post + s_pre (x) p_minus`` of that step, so
    the spikes the rule saw last (``_spre`` / ``_spost``) are kept instead and ``eligibility`` rebuilds it on request.
    ``Network.run(..., reward=r)`` is mandatory, ``a_plus`` / ``a_minus`` optional, all three scalars."""

    def _take_run_kwargs(self, run_kwargs: dict) -> None:
        if run_kwargs.get("reward", None) is None:
            raise KeyError("reward")  # learning.py:1541, MCC_learning.py:507: kwargs["reward"]
        for key in ("reward", "a_plus", "a_minus"):
            v = run_kwargs.get(key, None)
            if isinstance(v, dict) or (isinstance(v, torch.Tensor) and v.numel() != 1):
                raise NotImplementedError(f"run(..., {key}=...) must be a scalar for the CUDA core")
        self._run_kwargs = run_kwargs

    def _ensure(self, name: str, shape, dev: torch.device, dtype=torch.float32) -> None:
        t = getattr(self, name, None)
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != tuple(shape) or t.device != dev or t.dtype != dtype:
            setattr(self, name, torch.zeros(*shape, dtype=dtype, device=dev))

    def _prepare_traces(self, pre_shape, post_shape, dev: torch.device) -> None:
        self._ensure("p_plus", pre_shape, dev)
        self._ensure("p_minus", post_shape, dev)
        self._ensure("_spre", pre_shape, dev, torch.uint8)
        self._ensure("_spost", post_shape, dev, torch.uint8)

    @property
    def eligibility(self) -> torch.Tensor:
        """The eligibility the next update applies: ``[B, n_src, n_tgt]`` (learning.py:1568-1572, MCC_learning.py:543-546)."""
        return torch.bmm(self.p_plus.unsqueeze(2), self._spost.float().unsqueeze(1)) + torch.bmm(
            self._spre.float().unsqueeze(2), self.p_minus.unsqueeze(1))

    def _fill_reward(self, d: "_abi.SnnConn", dt: float) -> None:
        rk = self._run_kwargs
        d.reward = float(rk["reward"])
        d.a_plus = float(rk["a_plus"]) if rk.get("a_plus", None) is not None else 1.0
        d.a_minus = float(rk["a_minus"]) if rk.get("a_minus", None) is not None else -1.0
        d.p_plus_decay = float(torch.exp(-dt / self.tc_plus))    # learning.py:1565 (fp32 tensor arithmetic)
        d.p_minus_decay = float(torch.exp(-dt / self.tc_minus))  # learning.py:1567
        d.p_plus, d.p_minus = self.p_plus.data_ptr(), self.p_minus.data_ptr()
        if getattr(self, "_spre", None) is not None:
            d.mst_spre, d.mst_spost = self._spre.data_ptr(), self._spost.data_ptr()


class _EligibilityTrace(_RewardModulated):
    """The ``MSTDPET`` form (learning.py:2187-2249, MCC_learning.py:652-733): batch size 1 only, since the reference
    flattens the spikes of the whole batch into its ``[n]`` traces.  ``eligibility_trace [n_src, n_tgt]`` is the
    materialised state; ``eligibility`` is ``[n_src, n_tgt]``."""

    @property
    def eligibility(self) -> torch.Tensor:
        """``[n_src, n_tgt]`` (learning.py:2245-2247, MCC_learning.py:729-731)."""
        return torch.outer(self.p_plus.view(-1), self._spost.float().view(-1)) + torch.outer(
            self._spre.float().view(-1), self.p_minus.view(-1))

    def _prepare_trace(self, B: int, shape, dev: torch.device) -> None:
        if B != 1:
            raise NotImplementedError("MSTDPET is defined for batch size 1 only (learning.py:2214-2215 flattens the batch)")
        t = getattr(self, "eligibility_trace", None)
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != tuple(shape) or t.device != dev:
            self.eligibility_trace = torch.zeros(*shape, device=dev)

    def _fill_trace(self, d: "_abi.SnnConn", dt: float) -> None:
        d.e_trace = self.eligibility_trace.data_ptr()
        d.e_trace_decay = float(torch.exp(-dt / self.tc_e_trace))          # learning.py:2229
        d.tc_e_trace = float(self.tc_e_trace)
        # update = nu[0] * dt * reward * eligibility_trace (learning.py:2232): the scalar product in fp32, left to right
        if getattr(self, "_nu_tensors", False):   # per-synapse rates: the kernel scales each one (snn_b200.h)
            d.et_coef = 0.0
        else:
            d.et_coef = float(self.nu[0].float() * dt * float(self._run_kwargs["reward"]))


class MSTDP(_RewardModulated, MCC_LearningRule):
    """Reward-modulated STDP on a ``Weight`` feature (reference: MCC_learning.py:392-551).  Each step
    (``_connection_update`` :468-548): ``value += nu[0] * reduction(reward * eligibility, 0)`` with the previous step's
    eligibility, then the traces decay by ``exp(-connection.dt / tc)`` and gain ``a_plus * s_pre`` / ``a_minus * s_post``,
    then the new per-sample eligibility, then decay and the clamp to ``range`` (default ``[-1, +1]``, :86-110).  That is
    the arithmetic of ``learning.MSTDP`` on a dense ``Connection``, and it runs on the same kernel phase.  Eligibility
    comes from the spikes: a masked or undrawn synapse learns like any other.  Rule state: ``p_plus [B, n_src]``,
    ``p_minus [B, n_tgt]``, allocated by the first run for its batch size."""

    rule_code = _abi.SNN_RULE_MSTDP

    def __init__(
        self,
        connection,
        feature_value: Union[torch.Tensor, float, int],
        range: Optional[Sequence[float]] = None,
        nu: Optional[Union[float, Sequence[float]]] = None,
        reduction: Optional[callable] = None,
        decay: float = 0.0,
        enforce_polarity: bool = False,
        **kwargs,
    ) -> None:
        super().__init__(
            connection=connection, feature_value=feature_value,
            range=[-1, +1] if range is None else range, nu=nu, reduction=reduction,
            decay=decay, enforce_polarity=enforce_polarity, **kwargs,
        )
        from ..network.topology import MulticompartmentConnection

        if not isinstance(connection, MulticompartmentConnection):
            raise NotImplementedError("This learning rule is not supported for this Connection type.")
        self.tc_plus = torch.tensor(kwargs.get("tc_plus", 20.0))
        self.tc_minus = torch.tensor(kwargs.get("tc_minus", 20.0))
        self.average_update = kwargs.get("average_update", 0)
        self.continues_update = kwargs.get("continues_update", False)
        if enforce_polarity:
            raise NotImplementedError("enforce_polarity is not implemented by the CUDA core")
        if self.average_update > 0 or self.continues_update:
            raise NotImplementedError(f"{type(self).__name__}(average_update>0 / continues_update) is not implemented by the CUDA core")
        self._run_kwargs = {}

    def update(self, **kwargs) -> None:
        raise NotImplementedError(f"{type(self).__name__}.update is fused into Network.run (it needs the run's reward); "
                                  "the standalone call is not exposed")

    def _prepare(self, B: int, dev: torch.device, run_kwargs: dict) -> None:
        """Allocate / validate the rule state for a window (MCC_learning.py:487-505)."""
        self._take_run_kwargs(run_kwargs)
        self._prepare_traces((B, self.source.n), (B, self.target.n), dev)

    def _fill_desc(self, d: "_abi.SnnConn") -> None:
        super()._fill_desc(d)
        if self._run_kwargs:   # a window's plan: _prepare has taken the run's kwargs
            self._fill_reward(d, float(self.connection.dt))


class MSTDPET(_EligibilityTrace, MSTDP):
    """Reward-modulated STDP with an eligibility trace on a ``Weight`` feature (reference: MCC_learning.py:554-738).  Each
    step (``_connection_update`` :652-733): ``eligibility_trace = eligibility_trace * exp(-dt / tc_e_trace) +
    eligibility / tc_e_trace``, ``value += nu[0] * dt * reward * eligibility_trace``, then the traces and the eligibility
    as in ``MSTDP``, then decay and clamp — the arithmetic of ``learning.MSTDPET``.  Batch size 1 only.  The rule state
    is allocated at construction like the reference's (:625-638): ``p_plus [n_src]``, ``p_minus [n_tgt]``,
    ``eligibility_trace [n_src, n_tgt]``.  ``reset_state_variables`` zeroes the eligibility and its trace; as in the
    reference, ``Network.reset_state_variables`` does not reach it (``Weight.reset_state_variables`` does nothing)."""

    rule_code = _abi.SNN_RULE_MSTDPET

    def __init__(self, connection, feature_value, range=None, nu=None, reduction=None, decay: float = 0.0,
                 enforce_polarity: bool = False, **kwargs) -> None:
        super().__init__(connection=connection, feature_value=feature_value, range=range, nu=nu, reduction=reduction,
                         decay=decay, enforce_polarity=enforce_polarity, **kwargs)
        self.tc_e_trace = torch.tensor(kwargs.get("tc_e_trace", 25.0))
        dev = self.feature_value.device
        self._prepare_traces((self.source.n,), (self.target.n,), dev)
        self.eligibility_trace = torch.zeros(*self.feature_value.shape, device=dev)

    def _prepare(self, B: int, dev: torch.device, run_kwargs: dict) -> None:
        self._prepare_trace(B, tuple(self.feature_value.shape), dev)
        self._take_run_kwargs(run_kwargs)
        self._prepare_traces((self.source.n,), (self.target.n,), dev)

    def _fill_desc(self, d: "_abi.SnnConn") -> None:
        super()._fill_desc(d)
        if self._run_kwargs:
            self._fill_trace(d, float(self.connection.dt))

    def reset_state_variables(self) -> None:
        """MCC_learning.py:735-738: the eligibility (the stored spikes it is rebuilt from) and its trace to zero."""
        self._spre.zero_()
        self._spost.zero_()
        self.eligibility_trace.zero_()
