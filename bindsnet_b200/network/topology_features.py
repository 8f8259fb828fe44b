"""Connection features — host-side mirror of ``bindsnet/network/topology_features.py``.

On the accelerated path are ``Weight`` (reference: topology_features.py:575-671, base class :15-362), the single
feature every ``bindsnet.models`` network puts in a ``MulticompartmentConnection`` pipeline (models.py:185-236), and
the three multiplicative features a pipeline may add to it: ``Probability`` (stochastic synapses, :365-464), ``Mask``
(:467-549) and ``Intensity`` (:724-769).  Learning and normalisation act on the ``Weight`` only.
"""
from __future__ import annotations

import warnings
from abc import ABC
from typing import Optional, Sequence, Union

import torch
from torch.nn import Parameter

from .. import _abi


class AbstractFeature(ABC):
    """Reference: topology_features.py:15-362."""

    _value_dtype = torch.float32   # the value dtype the CUDA core reads

    def __init__(
        self,
        name: str,
        value: Union[torch.Tensor, float, int] = None,
        value_dtype: torch.dtype = torch.float32,
        range: Optional[Union[list, tuple]] = None,
        clamp_frequency: Optional[int] = 1,
        norm: Optional[Union[torch.Tensor, float, int]] = None,
        learning_rule=None,
        nu: Optional[Union[list, tuple, int, float]] = None,
        reduction: Optional[callable] = None,
        enforce_polarity: Optional[bool] = False,
        decay: float = 0.0,
        parent_feature=None,
        sparse: Optional[bool] = False,
        batch_size: int = 1,
        **kwargs,
    ) -> None:
        from ..learning.MCC_learning import MSTDP, MSTDPET, NoOp, PostPre

        assert isinstance(name, str), f"Feature {name}'s name should be of type str"
        assert value is None or isinstance(value, (torch.Tensor, float, int)), (
            f"Feature {name} should be of type float, int, or torch.Tensor, not {type(value)}"
        )
        assert norm is None or isinstance(norm, (torch.Tensor, float, int)), (
            f"Feature {name}'s norm should be of type float, int, or torch.Tensor, not {type(norm)}"
        )
        assert learning_rule is None or learning_rule in (NoOp, PostPre, MSTDP, MSTDPET), (
            f"Feature {name}'s learning_rule should be an MCC learning rule, not {learning_rule}"
        )
        assert nu is None or isinstance(nu, (list, tuple)), (
            f"Feature {name}'s nu should be of type list or tuple, not {type(nu)}"
        )
        assert decay is None or isinstance(decay, float), f"Feature {name}'s decay should be of type float"
        if sparse:
            raise NotImplementedError("sparse feature values are not implemented by the CUDA core")
        if parent_feature is not None:
            raise NotImplementedError("feature linking (parent_feature) is not implemented by the CUDA core")
        if value_dtype != self._value_dtype:
            raise NotImplementedError("bindsnet_b200 computes in float32 only (SURVEY.md §8b)")

        self.name = name
        self.value = value
        self.range = [-1.0, 1.0] if range is None else range
        self.clamp_frequency = clamp_frequency
        self.norm = norm
        self.learning_rule = learning_rule
        self.nu = nu
        self.reduction = reduction
        self.decay = decay
        self.parent_feature = parent_feature
        self.sparse = sparse
        self.batch_size = batch_size
        self.kwargs = kwargs
        self.is_primed = False

        # topology_features.py:310-328
        r = self.range
        assert isinstance(r, (list, tuple)) and len(r) == 2, f"Invalid range for feature {name}"
        assert r[0] < r[1], f"Invalid range for feature {name}: the min value is larger than the max value"
        if value is None:
            return
        if isinstance(value, torch.Tensor):
            # topology_features.py:330-351
            assert (value >= r[0]).all() and (value <= r[1]).all(), (
                f"Feature out of range for {name}: Features values not in [{r[0]}, {r[1]}]"
            )
            if value.dtype != value_dtype:
                warnings.warn(f"Provided value has data type {value.dtype} but parameter w_dtype is {value_dtype}")
                self.value = value.to(dtype=value_dtype)

    def initialize_value(self):
        raise NotImplementedError

    def prime_feature(self, connection, device, **kwargs) -> None:
        """topology_features.py:173-240: wrap the value, move it to ``device`` and
        instantiate the learning rule."""
        from ..learning.MCC_learning import NoOp

        if self.is_primed:
            return
        self.is_primed = True
        if isinstance(self.value, torch.Tensor):
            assert tuple(self.value.shape) == (connection.source.n, connection.target.n)
        if self.norm is not None and isinstance(self.norm, torch.Tensor):
            assert self.norm.shape[0] == connection.target.n
        if self.value is None:
            self.value = self.initialize_value()
        if isinstance(self.value, (int, float)):
            self.value = torch.Tensor([self.value])
        self.value = Parameter(self.value.detach().clone().contiguous(), requires_grad=False).to(device)
        rule_cls = self.learning_rule or NoOp
        self.learning_rule = rule_cls(
            connection=connection, feature_value=self.value, range=self.range, nu=self.nu,
            reduction=self.reduction, decay=self.decay, **kwargs,
        )
        del self.nu, self.reduction, self.decay, self.range

    def update(self, **kwargs) -> None:
        """topology_features.py:242-248."""
        self.learning_rule.update(**kwargs)

    def normalize(self) -> None:
        """topology_features.py:250-266 (plain, not absolute, column sums)."""
        if self.norm is not None:
            from . import _plan

            _plan.normalize_feature(self)

    def reset_state_variables(self) -> None:
        pass

    def _apply(self, fn) -> None:
        if isinstance(self.value, torch.Tensor):
            moved = fn(self.value)
            if moved is not self.value:
                self.value = moved
                if getattr(self.learning_rule, "feature_value", None) is not None:
                    self.learning_rule.feature_value = moved


class Weight(AbstractFeature):
    """Per-synapse multiplicative weight (reference: topology_features.py:575-671)."""

    def __init__(
        self,
        name: str,
        value: Union[torch.Tensor, float, int] = None,
        value_dtype: torch.dtype = torch.float32,
        range: Optional[Sequence[float]] = None,
        norm: Optional[Union[torch.Tensor, float, int]] = None,
        norm_frequency: Optional[str] = "sample",
        learning_rule=None,
        nu: Optional[Union[list, tuple]] = None,
        reduction: Optional[callable] = None,
        enforce_polarity: Optional[bool] = False,
        decay: float = 0.0,
        sparse: Optional[bool] = False,
        batch_size: int = 1,
    ) -> None:
        if norm_frequency not in ("sample", "time step"):
            raise NotImplementedError(f"Weight(norm_frequency={norm_frequency!r}) is not implemented by the CUDA core "
                                      "(only 'sample' and 'time step')")
        if enforce_polarity:
            raise NotImplementedError("Weight(enforce_polarity=True) is not implemented by the CUDA core")
        self.norm_frequency = norm_frequency
        self.enforce_polarity = enforce_polarity
        super().__init__(
            name=name, value=value, value_dtype=value_dtype,
            range=[-torch.inf, +torch.inf] if range is None else range,
            norm=norm, learning_rule=learning_rule, nu=nu, reduction=reduction,
            decay=decay, sparse=sparse, batch_size=batch_size,
        )

    def prime_feature(self, connection, device, **kwargs) -> None:
        """topology_features.py:647-661."""
        if self.value is None:
            self.initialize_value = lambda: torch.rand(connection.source.n, connection.target.n)
        super().prime_feature(connection, device, enforce_polarity=self.enforce_polarity, **kwargs)

    def normalize(self, time_step_norm: bool = False) -> None:
        """topology_features.py:663-671: a 'time step' Weight normalises from its compute (``time_step_norm=True``), a
        'sample' one from ``Network.run``'s end-of-run normalize; each call does nothing for the other frequency."""
        if self.norm is None or time_step_norm != (self.norm_frequency == "time step"):
            return
        from . import _plan

        _plan.normalize_feature(self, time_step=time_step_norm)

    def _norm_tensor(self):
        """The norm as float32 ``[target.n]`` (prime_feature asserted its first dimension), or None for a number."""
        if not isinstance(self.norm, torch.Tensor):
            return None
        from . import _plan

        return _plan.norm_tensor(self, self.value.shape[1], self.value.device)

    def _fill_desc(self, d: "_abi.SnnConn", dt: float, manual_update: bool) -> None:
        if self.value.dim() != 2:
            raise NotImplementedError("scalar Weight values are not supported by the CUDA core")
        norm_t = self._norm_tensor()
        d.has_norm = int(self.norm is not None)
        d.norm_abs = 0
        d.norm = float(self.norm) if self.norm is not None and norm_t is None else 0.0
        d.dt_scale = float(dt)
        self.learning_rule._fill_desc(d)
        if d.rule & _abi.SNN_RULE_AVG and self.norm is not None and (norm_t is not None or self.norm_frequency == "time step"):
            raise NotImplementedError("PostPre(average_update>0) on a Weight normalised every time step or by a norm tensor "
                                      "is not implemented by the CUDA core")
        if manual_update:
            d.rule = _abi.SNN_RULE_NONE


def _scalar_value(cls: str, value) -> None:
    """A Python number as the value: the reference fails on it in ``cast_dtype_if_needed`` (topology_features.py:146-153)."""
    if isinstance(value, (int, float)):
        raise AttributeError(f"'{type(value).__name__}' object has no attribute 'dtype'")


def _no_learning(cls: str, learning_rule, norm) -> None:
    from ..learning.MCC_learning import NoOp

    if learning_rule is not None and learning_rule is not NoOp:
        raise NotImplementedError(f"a learning rule on a {cls} feature is not implemented by the CUDA core (only the Weight learns)")
    if norm is not None:
        raise NotImplementedError(f"norm on a {cls} feature is not implemented by the CUDA core (only the Weight is normalised)")


class Probability(AbstractFeature):
    """Stochastic synapses (reference: topology_features.py:365-464): each step, synapse (i, j) transmits with probability
    ``value[i, j]``, one draw for the whole batch (``torch.bernoulli(value)`` broadcast over the samples, :425-429).  The
    draw is the counter-based ``snn_synapse_draw`` of include/snn_b200.h, keyed by the window's seed
    (``Network.run(one_spike_seed=...)``, ``Network.last_one_spike_seed``), the step and the connection's position."""

    def __init__(
        self,
        name: str,
        value: Union[torch.Tensor, float, int] = None,
        value_dtype: torch.dtype = torch.float32,
        range: Optional[Sequence[float]] = None,
        norm: Optional[Union[torch.Tensor, float, int]] = None,
        learning_rule=None,
        nu: Optional[Union[list, tuple]] = None,
        reduction: Optional[callable] = None,
        decay: float = 0.0,
        parent_feature=None,
        sparse: Optional[bool] = False,
        batch_size: int = 1,
    ) -> None:
        r = [0, 1] if range is None else range
        super().__init__(
            name=name, value=value, value_dtype=value_dtype, range=r, norm=norm, learning_rule=learning_rule, nu=nu,
            reduction=reduction, decay=decay, parent_feature=parent_feature, sparse=sparse, batch_size=batch_size,
        )
        # topology_features.py:445-464
        if isinstance(r[0], torch.Tensor):
            assert (r[0] >= 0).all(), f"Invalid range for feature {name}: a min value is less than 0"
        elif isinstance(r[0], (float, int)):
            assert r[0] >= 0, f"Invalid range for feature {name}: the min value is less than 0"
        else:
            assert False, f"Invalid range for feature {name}: the min value must be of type torch.Tensor, float, or int"
        _scalar_value("Probability", value)
        _no_learning("Probability", learning_rule, norm)

    def prime_feature(self, connection, device, **kwargs) -> None:
        """topology_features.py:434-443."""
        if self.value is None:
            lo, hi = self.range
            self.initialize_value = lambda: torch.clamp(torch.rand(connection.source.n, connection.target.n, device=device), lo, hi)
        super().prime_feature(connection, device, **kwargs)


class Mask(AbstractFeature):
    """Boolean synapse mask (reference: topology_features.py:467-549): ``True`` lets a spike pass.  A scalar or
    broadcastable value is expanded to the ``[source.n, target.n]`` matrix on the host; an all-``True`` one is dropped."""

    _value_dtype = torch.bool

    def __init__(self, name: str, value: Union[torch.Tensor, float, int] = None, sparse: Optional[bool] = False,
                 batch_size: int = 1) -> None:
        # topology_features.py:485-505
        if isinstance(value, torch.Tensor):
            assert value.dtype == torch.bool, f"Mask must be of type bool, not {value.dtype}"
        elif value is not None:
            if not isinstance(value, bool):
                raise AttributeError(f"'{type(value).__name__}' object has no attribute 'dtype'")
            value = torch.tensor(value)
        super().__init__(name=name, value=value, value_dtype=torch.bool, sparse=sparse, batch_size=batch_size)

    def prime_feature(self, connection, device, **kwargs) -> None:
        """topology_features.py:513-549 (the learning rule is MCC_learning.NoOp: a Mask never changes)."""
        from ..learning.MCC_learning import NoOp

        if self.is_primed:
            return
        self.is_primed = True
        if self.value is None:
            self.value = (torch.rand(connection.source.n, connection.target.n) > 0.99).to(device=device)
        self.value = Parameter(self.value.detach().clone(), requires_grad=False).to(device)
        f = self.value
        if f.dim() > 1:   # topology_features.py:347-361: a matrix must be [source.n, target.n]; fewer dims broadcast
            assert tuple(f.shape) == (connection.source.n, connection.target.n), (
                f"Feature {self.name} has an incorrect shape of {f.shape}. Should be of shape "
                f"{(connection.source.n, connection.target.n)}"
            )
        self.learning_rule = NoOp(connection=connection)


class Intensity(AbstractFeature):
    """Per-synapse multiplicative factor (reference: topology_features.py:724-769), by default in [-1, 1].  With a
    ``Weight`` the term a spike carries is the single rounding of ``w * value``."""

    def __init__(
        self,
        name: str,
        value: Union[torch.Tensor, float, int] = None,
        value_dtype: torch.dtype = torch.float32,
        range: Optional[Sequence[float]] = None,
        sparse: Optional[bool] = False,
        batch_size: int = 1,
    ) -> None:
        super().__init__(name=name, value=value, value_dtype=value_dtype, range=range, sparse=sparse, batch_size=batch_size)
        _scalar_value("Intensity", value)

    def prime_feature(self, connection, device, **kwargs) -> None:
        """topology_features.py:758-769.  The reference keeps the int64 tensor its default draw makes; its values
        (-1, 0, 1) are stored as float32 here."""
        if self.value is None:
            lo, hi = self.range
            self.initialize_value = lambda: torch.clamp(
                torch.sign(torch.randint(-1, +2, (connection.source.n, connection.target.n))), lo, hi
            ).to(torch.float32)
        super().prime_feature(connection, device, **kwargs)


def _unsupported(name: str, where: str):
    class _Unsupported:
        __doc__ = f"``{name}`` (reference: {where}) — not on the accelerated path."

        def __init__(self, *args, **kwargs):
            raise NotImplementedError(
                f"the {name} feature is outside the hot path bindsnet_b200 implements (Weight, Probability, Mask, "
                "Intensity): it makes every synapse carry a signal, so the spike gather would turn dense"
            )

    _Unsupported.__name__ = name
    return _Unsupported


MeanField = _unsupported("MeanField", "topology_features.py:552-572")
Bias = _unsupported("Bias", "topology_features.py:674-721")
Degradation = _unsupported("Degradation", "topology_features.py:772-813")
