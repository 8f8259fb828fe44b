"""The two connections ``ann_to_snn`` builds for ``Permute`` and ``nn.ConstantPad2d`` (reference:
``bindsnet/conversion/topology.py``).  In the reference neither implements ``AbstractConnection.update`` nor
``reset_state_variables``, which it declares abstract, so neither can be constructed: the constructor raises
``TypeError``, and so does every ``ann_to_snn`` call that meets such a module.  They are kept that way here."""
from __future__ import annotations

from abc import abstractmethod
from typing import Iterable, Optional, Sequence, Union

from ..network.nodes import Nodes
from ..network.topology import AbstractConnection


class _Unfinished(AbstractConnection):
    """The reference's abstract methods, left abstract."""

    @abstractmethod
    def update(self, **kwargs) -> None: ...

    @abstractmethod
    def reset_state_variables(self) -> None: ...


class PermuteConnection(_Unfinished):
    """Reference: conversion/topology.py:9-55.  Constructing it raises ``TypeError``."""

    def __init__(self, source: Nodes, target: Nodes, dims: Iterable, nu: Optional[Union[float, Sequence[float]]] = None,
                 weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(source, target, nu, weight_decay=weight_decay, **kwargs)
        self.dims = dims


class ConstantPad2dConnection(_Unfinished):
    """Reference: conversion/topology.py:58-106.  Constructing it raises ``TypeError``."""

    def __init__(self, source: Nodes, target: Nodes, padding: tuple, nu: Optional[Union[float, Sequence[float]]] = None,
                 weight_decay: float = 0.0, **kwargs) -> None:
        super().__init__(source, target, nu, weight_decay=weight_decay, **kwargs)
        self.padding = padding
