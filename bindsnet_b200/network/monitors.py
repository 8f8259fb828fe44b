"""State recording — host-side mirror of ``bindsnet/network/monitors.py`` (``Monitor``
:30-124).  During a fused window the kernels write ``s``/``v`` rasters straight into a
``[T, B, n]`` device buffer (no per-step copies, no Python list churn); ``get`` serves the
reference's ``[time, batch, *shape]`` view from that buffer."""
from __future__ import annotations

from abc import ABC
from typing import Dict, Iterable, Optional

import torch


class AbstractMonitor(ABC):
    """Reference: monitors.py:23-27."""


class Monitor(AbstractMonitor):
    """Records state variables of one object over time (reference: monitors.py:30-124)."""

    #: state variables the window kernels can record in-kernel; anything else makes
    #: ``Network.run`` fall back to one-step windows with a host-side snapshot per step.
    FUSED_VARS = ("s", "v")

    def __init__(
        self,
        obj,
        state_vars: Iterable[str],
        time: Optional[int] = None,
        batch_size: int = 1,
        device: str = "cpu",
        sparse: Optional[bool] = False,
    ):
        super().__init__()
        self.obj = obj
        self.state_vars = list(state_vars)
        self.time = time
        self.batch_size = batch_size
        self.device = device
        self.sparse = sparse
        if self.time is None:
            self.device = "cpu"  # monitors.py:68-70
        self.recording = {}
        self.reset_state_variables()

    def get(self, var: str) -> torch.Tensor:
        """``[time, batch, *shape]`` recording (reference: monitors.py:75-92).  With
        ``time=None`` the log is drained by the call, as in the reference."""
        chunks = self.recording[var]
        if self.clean or not chunks:
            return torch.empty(0, device=self.device)
        out = torch.cat(chunks, 0) if len(chunks) > 1 else chunks[0]
        if self.time is None:
            self.recording[var] = []
        else:
            self.recording[var] = [out]
        if self.sparse:
            out = out.to_sparse()
        return out

    def record(self) -> None:
        """Append the object's current value (reference: monitors.py:94-111) — used by the
        one-step fallback and by user code; fused windows call ``_push_window``."""
        for v in self.state_vars:
            data = getattr(self.obj, v)
            if not isinstance(data, torch.Tensor):
                data = torch.as_tensor(data)
            self._push_window(v, data.detach().unsqueeze(0).clone())

    def _push_window(self, var: str, block: torch.Tensor) -> None:
        """Append a ``[t, B, *shape]`` block; keeps only the last ``time`` steps when a
        horizon was given (monitors.py:109-111)."""
        self.clean = False
        block = block.to(self.device)
        chunks = self.recording[var]
        chunks.append(block)
        if self.time is not None:
            total = sum(c.shape[0] for c in chunks)
            while total - chunks[0].shape[0] >= self.time:
                total -= chunks[0].shape[0]
                chunks.pop(0)
            if total > self.time:
                chunks[0] = chunks[0][total - self.time:]

    def reset_state_variables(self) -> None:
        """monitors.py:113-124."""
        self.recording = {v: [] for v in self.state_vars}
        self.clean = True


class SpikeCounter(AbstractMonitor):
    """Per-neuron spike counts of the last ``run`` window, ``[batch, *shape]`` int32 — what the
    reference's callers reduce the full raster to (``spikes.sum(time)``, e.g.
    examples/mnist/batch_eth_mnist.py:280-284; ``evaluation.assign_labels`` consumes exactly
    this, evaluation/evaluation.py:8-61).  The window kernels count in registers, so no
    ``[T, B, n]`` raster is ever written (SURVEY.md §8f row 2).  Extension: not in the reference.
    """

    def __init__(self, obj, device: str = None):
        super().__init__()
        self.obj = obj
        self.device = device
        self.counts = None

    def get(self, var: str = "s") -> torch.Tensor:
        assert var == "s", "SpikeCounter records spikes only"
        if self.counts is None:
            return torch.empty(0, dtype=torch.int32)
        out = self.counts.view(self.counts.shape[0], *self.obj.shape)
        return out if self.device is None else out.to(self.device)

    def record(self) -> None:  # step-wise fallback path
        s = self.obj.s
        if self.counts is None or self.counts.shape[0] != s.shape[0] or self.counts.device != s.device:
            self.counts = torch.zeros(s.shape[0], self.obj.n, dtype=torch.int32, device=s.device)
        self.counts += s.reshape(s.shape[0], -1).to(torch.int32)

    def _begin_window(self, B: int, device) -> torch.Tensor:
        if self.counts is None or self.counts.shape[0] != B or self.counts.device != device:
            self.counts = torch.zeros(B, self.obj.n, dtype=torch.int32, device=device)
        else:
            self.counts.zero_()
        return self.counts

    def reset_state_variables(self) -> None:
        if self.counts is not None:
            self.counts.zero_()


class NetworkMonitor(AbstractMonitor):
    """Whole-network recorder (reference: monitors.py:127-329): every step, the named state variables
    (default ``v``, ``s``, ``w``) of the chosen layers and connections.  Not one of the monitors the window
    kernels fill themselves: a network that carries one runs its windows step by step (``Network._run_stepwise``)
    and ``record`` reads the tensors between the steps, as the reference does.  ``time=None`` grows the recordings
    (:222-236), ``time=T`` keeps the last ``T`` steps (:238-254); layer variables are stored as float, connection
    variables as they are.  Recordings stay on the device of what they record."""

    def __init__(self, network, layers=None, connections=None, state_vars=None, time: Optional[int] = None):
        super().__init__()
        self.network = network
        self.layers = layers if layers is not None else list(network.layers.keys())
        self.connections = connections if connections is not None else list(network.connections.keys())
        self.state_vars = state_vars if state_vars is not None else ("v", "s", "w")
        self.time = time
        self.reset_state_variables()

    def _sources(self):
        """(key, variable, object, is_layer) of everything recorded: a variable is skipped where the object does not
        have it (:166-173); a MulticompartmentConnection has no ``w`` of its own in the reference (it lives in the
        pipeline's feature), so none is recorded for it."""
        for v in self.state_vars:
            for l in self.layers:
                if hasattr(self.network.layers[l], v):
                    yield l, v, self.network.layers[l], True
            for c in self.connections:
                obj = self.network.connections[c]
                if hasattr(obj, v) and not (v == "w" and hasattr(obj, "pipeline")):
                    if v == "w" and obj.w.is_sparse:
                        raise NotImplementedError(f"NetworkMonitor does not record the sparse w of {c} (SparseConnection)")
                    yield c, v, obj, False

    def get(self) -> Dict:
        return self.recording

    def record(self) -> None:
        for key, v, obj, is_layer in self._sources():
            data = getattr(obj, v).detach()
            data = (data.float() if is_layer else data).unsqueeze(0)
            old = self.recording[key][v]
            if self.time is not None:
                old = old[1:]                                   # rolling window of the last `time` steps
            if old.numel() == 0 and old.dim() <= 1:
                self.recording[key][v] = data.clone()
            else:
                self.recording[key][v] = torch.cat((old.to(device=data.device, dtype=data.dtype), data), 0)
        if self.time is not None:
            self.i += 1

    def save(self, path: str, fmt: str = "npz") -> None:
        """monitors.py:258-292: ``npz`` (keys ``<layer>_<var>`` / ``<source>-<target>_<var>``) or ``pickle``."""
        import os

        import numpy as np

        folder = os.path.dirname(path)
        if folder and not os.path.exists(folder):
            os.makedirs(folder)
        if fmt == "npz":
            arrays = {}
            for key, rec in self.recording.items():
                stem = "-".join(key) if isinstance(key, tuple) else key
                for v, t in rec.items():
                    arrays[f"{stem}_{v}"] = t.cpu().numpy()
            np.savez_compressed(path, **arrays)
        elif fmt == "pickle":
            with open(path, "wb") as f:
                torch.save(self.recording, f)

    def reset_state_variables(self) -> None:
        """monitors.py:294-329: empty recordings, or ``time`` rows of zeros per variable."""
        self.recording = {k: {} for k in list(self.layers) + list(self.connections)}
        if self.time is not None:
            self.i = 0
        for key, v, obj, _ in self._sources():
            t = getattr(obj, v)
            self.recording[key][v] = torch.Tensor() if self.time is None else torch.zeros(self.time, *t.size(), device=t.device)
