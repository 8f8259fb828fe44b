"""Plan building: turns the user's objects into the POD structs of ``include/snn_b200.h``.

``Network.run`` calls ``build_net`` once per window; the standalone object methods
(``Nodes.forward``, ``Connection.compute`` / ``update`` / ``normalize``) go through the
single-operator entry points.  Everything here is host bookkeeping — no arithmetic.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from .. import _abi, _backend
from .topology import LocalConnection2D, MeanFieldConnection, _MaxPoolConnection, meanfield_offsets


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _as_u8(t: torch.Tensor) -> torch.Tensor:
    """Reinterpret a bool tensor as uint8 without copying (same storage)."""
    return t.view(torch.uint8) if t.dtype == torch.bool else t


def _state(t: torch.Tensor, name: str, owner: str) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise TypeError(f"{owner}.{name} must be float32, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{owner}.{name} must be contiguous (it is updated in place by the CUDA core)")
    return t


def fill_layer(d: "_abi.SnnLayer", layer, name: str, B: int) -> None:
    layer._fill_desc(d)
    if d.kind == _abi.SNN_NODE_PASSTHROUGH:
        # PassThroughNodes.forward stores its float input as s (conversion/nodes.py:137-144): the kernel keeps it float32
        if tuple(layer.s.shape) != (B, *layer.shape):
            layer.s = torch.zeros(B, *layer.shape, dtype=torch.float32, device=layer.s.device)
        elif layer.s.dtype != torch.float32:
            layer.s = layer.s.float()
    elif layer.s.dtype not in (torch.bool, torch.uint8) or tuple(layer.s.shape) != (B, *layer.shape):
        # Input.forward aliases user input into s in the reference (nodes.py:219); we keep a
        # private bool tensor of the canonical shape instead.
        layer.s = torch.zeros(B, *layer.shape, dtype=torch.bool, device=layer.s.device)
    if not layer.s.is_contiguous():
        layer.s = layer.s.contiguous()
    d.s = _ptr(_as_u8(layer.s))
    if d.kind not in (_abi.SNN_NODE_INPUT, _abi.SNN_NODE_PASSTHROUGH):
        d.v = _ptr(_state(layer.v, "v", name))
        if d.kind != _abi.SNN_NODE_MCP:
            d.refrac_count = _ptr(_state(layer.refrac_count, "refrac_count", name))
    if d.kind & ~_abi.SNN_NODE_PN == _abi.SNN_NODE_DC:   # (with or without per-neuron parameters)
        d.theta = _ptr(_state(layer.theta, "theta", name))
    if d.kind == _abi.SNN_NODE_CURRENT_LIF:
        d.i = _ptr(_state(layer.i, "i", name))
    if layer.traces:
        d.x = _ptr(_state(layer.x, "x", name))
    if layer.sum_input:
        d.summed = _ptr(_state(layer.summed, "summed", name))


def weight_structure(conn, w: torch.Tensor):
    """Plan-time structure detection for STATIC square weight matrices (DiehlAndCook2015's
    ``exc * I`` and ``-inh * (1 - I)``, models.py:204,217-220): lets the fused kernel replace an
    n x n matrix by one constant.  Verified on the actual tensor (one small reduction + host
    read) and cached until the tensor is modified in place (``Tensor._version``) or replaced."""
    key = (w.data_ptr(), w._version, tuple(w.shape), str(w.device))
    cached = getattr(conn, "_b200_structure", None)
    if cached is not None and cached[0] == key:
        return cached[1]
    result = (_abi.SNN_W_DENSE, 0.0)
    if w.dim() == 2 and w.shape[0] == w.shape[1] and w.shape[0] > 1:
        with torch.no_grad():
            diag = torch.diagonal(w)
            d0, o0 = diag[0], w[0, 1]
            eye = torch.eye(w.shape[0], dtype=torch.bool, device=w.device)
            is_diag = bool(((w == 0) | eye).all() & (diag == d0).all())
            is_off = bool(((w == o0) | eye).all() & (diag == 0).all())
        if is_diag:
            result = (_abi.SNN_W_DIAG, float(d0))
        elif is_off:
            result = (_abi.SNN_W_OFFDIAG, float(o0))
    conn._b200_structure = (key, result)
    return result


def fill_conn(d: "_abi.SnnConn", conn, src_idx: int, tgt_idx: int, dt: float, B: int, rule_kwargs=None, rule: bool = True) -> None:
    """``rule=False``: geometry, weights and normalisation only (the single-operator compute / normalize calls
    do not involve the learning rule, whose plan entry may need a run's keyword arguments)."""
    d.src, d.tgt = src_idx, tgt_idx
    rule0 = getattr(conn, "update_rule", None)
    if rule0 is None and hasattr(conn, "pipeline") and not conn.manual_update:
        rule0 = conn._weight().learning_rule   # MulticompartmentConnection.update never reaches it with manual_update
    if rule and hasattr(rule0, "_prepare"):  # rules with state of their own (MSTDP): allocate for this batch size / device
        rule0._prepare(B, conn.w.device, rule_kwargs or {})
    if isinstance(conn, _MaxPoolConnection):   # no weights: the rates buffer and the geometry are all there is
        conn._check((B, *conn.source.shape))
        conn._fill_desc(d, dt, rule)
        return
    conn._fill_desc(d, dt, rule)
    if d.kind == _abi.SNN_CONN_MEANFIELD:   # w in its own shape, read through the per-target offset map
        w = conn.w
        if w.dtype != torch.float32 or not w.is_contiguous():
            raise TypeError("connection weights must be contiguous float32")
        off, d.mf_stride = meanfield_offsets(conn, B)
        d.w, d.mf_off = _ptr(w), _ptr(off)
        return
    if d.kind in (_abi.SNN_CONN_LOCAL2D, _abi.SNN_CONN_LOCAL3D):   # [cin, n, K] weights, no bias (compute never reads b)
        w = conn.w
        if w.dtype != torch.float32 or not w.is_contiguous():
            raise TypeError("connection weights must be contiguous float32")
        d.w = _ptr(w)
        check_squeeze(d, conn, B)
        return
    if d.kind == _abi.SNN_CONN_CONV3D:   # [cout, cin, kd, kh, kw] weights and [cout] bias (shapes checked by _fill_desc)
        w, b = conn.w, conn.b
        if w.dtype != torch.float32 or not w.is_contiguous() or b.dtype != torch.float32 or not b.is_contiguous():
            raise TypeError("connection weights and bias must be contiguous float32")
        d.w, d.b = _ptr(w), _ptr(b)
        return   # (no batch reduction runs: its rules are decay and clamp only)
    if d.kind == _abi.SNN_CONN_CONV1D:   # [cout, cin, kw] weights and [cout] bias (shapes checked by _fill_desc)
        w, b = conn.w, conn.b
        if w.dtype != torch.float32 or not w.is_contiguous() or b.dtype != torch.float32 or not b.is_contiguous():
            raise TypeError("connection weights and bias must be contiguous float32")
        d.w, d.b = _ptr(w), _ptr(b)
        check_squeeze(d, conn, B)
        return
    if d.kind == _abi.SNN_CONN_SPARSE:
        fill_sparse(d, conn)
        d.b = _ptr(target_bias(conn, B))
        return
    w = conn.w
    if w.dtype != torch.float32 or not w.is_contiguous():
        raise TypeError("connection weights must be contiguous float32")
    if d.kind != _abi.SNN_CONN_CONV2D and tuple(w.shape) != (conn.source.n, conn.target.n):
        raise ValueError(f"weight shape {tuple(w.shape)} != ({conn.source.n}, {conn.target.n})")
    if d.kind == _abi.SNN_CONN_CONV2D and tuple(conn.b.shape) != (d.cout,):
        # F.conv2d's own error in the reference's first compute (topology.py:799-815); ann_to_snn makes such a bias for
        # an nn.Conv2d without one (conversion.py:197-199)
        raise RuntimeError(f"Given weight of size {list(w.shape)}, expected bias to be 1-dimensional with {d.cout} elements, "
                           f"but got bias of size {list(conn.b.shape)} instead")
    d.w = _ptr(w)
    static = d.rule == _abi.SNN_RULE_NONE or (d.rule == _abi.SNN_RULE_NOOP and d.weight_decay in (0.0, 1.0))
    if static and not d.has_norm:
        d.structure, d.structure_val = weight_structure(conn, w)
    if d.kind == _abi.SNN_CONN_DENSE:
        d.b = _ptr(target_bias(conn, B))
    else:
        b = getattr(conn, "b", None)
        d.b = _ptr(b) if b is not None else None
    if d.kind == _abi.SNN_CONN_MCC:
        fill_features(d, conn)
    check_squeeze(d, conn, B)
    if d.kind in (_abi.SNN_CONN_DENSE, _abi.SNN_CONN_MCC):
        fill_norm(d, conn)


def fill_norm(d: "_abi.SnnConn", conn) -> None:
    """A per-target norm tensor or a per-step normalisation (snn_b200.h SNN_CONN_WNORM) of a dense ``Connection`` or an
    MCC ``Weight``; other plans keep the scalar ``norm`` ``_fill_desc`` wrote."""
    owner = conn._weight() if d.kind == _abi.SNN_CONN_MCC else conn
    norm_t = getattr(owner, "_norm_tensor", lambda: None)()
    step = d.kind == _abi.SNN_CONN_MCC and owner.norm_frequency == "time step"
    if not d.has_norm or (norm_t is None and not step):
        return
    d.kind |= _abi.SNN_CONN_WNORM
    d.norm_t = _ptr(norm_t) if norm_t is not None else None
    d.norm_step = int(step)


def norm_tensor(owner, n: int, device: torch.device) -> Optional[torch.Tensor]:
    """``owner.norm`` as the kernels read a per-target norm: float32 ``[n]``, one value per target neuron (a ``[1, n]``
    norm is viewed as ``[n]``).  Read in place when it lies contiguously on the weights' device, so that in-place edits
    take effect; otherwise through a copy cached until the norm changes (``Tensor._version``)."""
    v = owner.norm.detach()
    if v.dim() == 2 and v.shape[0] == 1:
        v = v[0]
    if v.dtype != torch.float32 or tuple(v.shape) != (n,):
        raise NotImplementedError(f"{type(owner).__name__}.norm of shape {list(owner.norm.shape)} and dtype {owner.norm.dtype}: "
                                  f"the CUDA core scales by a float32 norm per target neuron ([{n}]) only")
    if v.is_contiguous() and v.device == device:
        return v
    key = (v.data_ptr(), v._version, str(v.device), str(device))
    cached = getattr(owner, "_b200_norm", None)
    if cached is None or cached[0] != key:
        cached = (key, v.to(device).contiguous(), v)
        owner._b200_norm = cached
    return cached[1]


def target_bias(conn, B: int) -> Optional[torch.Tensor]:
    """The bias of a dense ``Connection`` or a ``SparseConnection`` as the kernels read it: ``b[j]`` for every target
    neuron j, contiguous float32.  The reference adds ``b`` to the ``[B, n_tgt]`` product (topology.py:342-345), so every
    bias that broadcasts there is valid.  One that is the same for every sample (0-d, ``[1]``, ``[n_tgt]``, ``[1, n_tgt]``,
    any strides) is read in place when it already lies contiguously, so that in-place edits take effect, and otherwise
    through a contiguous ``[n_tgt]`` copy cached on the connection until the bias changes (the cache keeps the copy alive
    as long as any plan that points at it)."""
    b = getattr(conn, "b", None)
    if b is None:
        return None
    name, n = type(conn).__name__, conn.target.n
    if b.dtype != torch.float32:
        raise TypeError(f"{name}.b must be float32, got {b.dtype}")
    shape = tuple(b.shape)
    try:
        ok = torch.broadcast_shapes(shape, (B, n))[-2:] == (B, n) and all(k == 1 for k in shape[:-2])
    except RuntimeError:
        ok = False
    if not ok:   # (the reference's sum, or the view of its result as [B, *target.shape], fails)
        raise RuntimeError(f"{name}.b of shape {list(shape)} does not broadcast to the [{B}, {n}] input of its target")
    if b.dim() >= 2 and shape[-2] != 1:
        raise NotImplementedError(f"{name}.b of shape {list(shape)}: a per-sample bias is not implemented by the CUDA core "
                                  f"(it adds one value per target neuron)")
    v = b.detach()
    while v.dim() > 2:
        v = v[0]
    v = v.broadcast_to((1, n)).reshape(n)   # (always a view of b)
    if v.is_contiguous():
        return v
    key = (b.data_ptr(), b._version, shape, tuple(b.stride()), str(b.device))
    cached = getattr(conn, "_b200_bias", None)
    if cached is None or cached[0] != key:
        cached = (key, v.contiguous(), b)   # (b stays referenced, so its address cannot be reused by another bias)
        conn._b200_bias = cached
    return cached[1]


def check_squeeze(d: "_abi.SnnConn", conn, B: int) -> None:
    rule = getattr(conn, "update_rule", None)
    if rule is None and hasattr(conn, "pipeline"):
        rule = conn._weight().learning_rule
    if d.rule >= _abi.SNN_RULE_POSTPRE and getattr(rule, "_squeeze", False) and B != 1:
        # The reference would fail inside torch with a broadcast error (SURVEY.md §0.9).
        raise RuntimeError(
            "learning rule was built with reduction=torch.squeeze (source.batch_size == 1 at construction) "
            f"but the run uses batch size {B}; pass reduction=torch.sum like the reference requires"
        )


def fill_sparse(d: "_abi.SnnConn", conn) -> None:
    """The CSR view of a ``SparseConnection``'s ``torch.sparse_coo`` weights.  An uncoalesced ``w`` (what NoOp's decay
    leaves in the reference, or what a user assigns) is coalesced in place.  The int32 ``rowptr`` / ``col`` arrays are
    built on the tensor's device and cached for as long as ``w``'s index tensor is unchanged; the values pointer is
    ``w``'s own values, so the kernel's decay shows in the user's tensor."""
    w = conn.w
    if not w.is_sparse or w.sparse_dim() != 2 or w.dense_dim() != 0:
        raise TypeError("SparseConnection.w must be a 2-D torch.sparse_coo tensor")
    if w.dtype != torch.float32:
        raise TypeError(f"SparseConnection.w must be float32, got {w.dtype}")
    n_src, n_tgt = conn.source.n, conn.target.n
    if tuple(w.shape) != (n_src, n_tgt):
        raise ValueError(f"weight shape {tuple(w.shape)} != ({n_src}, {n_tgt})")
    if not w.is_coalesced():
        with torch.no_grad():
            conn.w.data = w.coalesce()
        w = conn.w
    idx = w._indices()
    nnz = idx.shape[1]
    if nnz >= 2**31:
        raise NotImplementedError(f"SparseConnection with {nnz} stored entries: the CUDA core indexes them with int32 (< 2**31)")
    key = (idx.data_ptr(), idx._version, tuple(w.shape), str(idx.device))
    cached = getattr(conn, "_b200_csr", None)
    if cached is None or cached[0] != key:
        with torch.no_grad():
            counts = torch.bincount(idx[0], minlength=n_src)
            rowptr = torch.zeros(n_src + 1, dtype=torch.int32, device=idx.device)
            rowptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
            col = idx[1].to(torch.int32).contiguous()
        # the index tensor stays referenced by the cache, so its address cannot be reused by another pattern
        cached = (key, rowptr, col, idx)
        conn._b200_csr = cached
    vals = w._values()
    if not vals.is_contiguous():
        raise ValueError("SparseConnection.w values must be contiguous (they are updated in place by the CUDA core)")
    d.w = _ptr(vals) if nnz > 0 else None
    d.sp_rowptr = _ptr(cached[1])
    d.sp_col = _ptr(cached[2]) if nnz > 0 else None
    d.nnz = int(nnz)


def _feature_matrix(f, conn, dtype: torch.dtype) -> torch.Tensor:
    v = f.value
    shape = (conn.source.n, conn.target.n)
    if v.dtype != dtype or tuple(v.shape) != shape or not v.is_contiguous():
        raise TypeError(f"{type(f).__name__} feature {f.name!r}: value must be a contiguous {dtype} tensor of shape {shape}, "
                        f"got {v.dtype} {tuple(v.shape)}")
    if v.device != conn.w.device:
        raise ValueError(f"{type(f).__name__} feature {f.name!r} is on {v.device}, the Weight on {conn.w.device}")
    return v


def _mask_bytes(f, conn) -> Optional[torch.Tensor]:
    """A Mask's value as [n_src, n_tgt] bytes, or None when it lets every spike pass.  A [n_src, n_tgt] bool value is
    read in place; a scalar or broadcast one (topology_features.py:347-362) is expanded once and cached until the
    value changes."""
    v = f.value
    shape = (conn.source.n, conn.target.n)
    if tuple(v.shape) == shape and v.is_contiguous() and v.device == conn.w.device:
        return _as_u8(v)
    key = (v.data_ptr(), v._version, tuple(v.shape), str(v.device), str(conn.w.device))
    cached = getattr(f, "_b200_bytes", None)
    if cached is None or cached[0] != key:
        with torch.no_grad():
            full = torch.broadcast_to(v, shape)
            u8 = None if bool(full.all()) else full.to(conn.w.device, torch.uint8).contiguous()
        cached = (key, u8, v)
        f._b200_bytes = cached
    return cached[1]


def fill_features(d: "_abi.SnnConn", conn) -> None:
    """Probability / Mask / Intensity of a MulticompartmentConnection (snn_conn_t f_prob / f_mask / f_int)."""
    feats = conn._features()
    p, m, i = feats.get("Probability"), feats.get("Mask"), feats.get("Intensity")
    d.f_prob = _ptr(_feature_matrix(p, conn, torch.float32)) if p is not None else None
    d.f_mask = _ptr(_mask_bytes(m, conn)) if m is not None else None
    d.f_int = _ptr(_feature_matrix(i, conn, torch.float32)) if i is not None else None


def has_probability(conn) -> bool:
    from .topology_features import Probability

    return any(isinstance(f, Probability) for f in getattr(conn, "pipeline", ()))


def network_device(network) -> torch.device:
    for layer in network.layers.values():
        return layer.s.device
    return torch.device("cpu")


def build_net(
    network,
    B: int,
    ext: Dict[str, torch.Tensor],
    clamps: Dict[str, torch.Tensor],
    unclamps: Dict[str, torch.Tensor],
    injects: Dict[str, torch.Tensor],
    rec: Dict[str, Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]],
) -> Tuple["_abi.SnnNet", List[torch.Tensor]]:
    """Describe ``network`` for one window.  ``ext`` maps layer name to a contiguous
    ``[T, B, n]`` device tensor (uint8/bool or float32)."""
    if len(network.layers) > _abi.SNN_MAX_LAYERS or len(network.connections) > _abi.SNN_MAX_CONNS:
        raise NotImplementedError(
            f"networks with more than {_abi.SNN_MAX_LAYERS} layers / {_abi.SNN_MAX_CONNS} connections "
            "are not supported by this build"
        )
    net = _abi.SnnNet()
    net.abi_version = _abi.SNN_ABI_VERSION
    net.n_layers = len(network.layers)
    net.n_conns = len(network.connections)
    net.learning = int(bool(network.learning))
    keep: List[torch.Tensor] = []
    index = {}
    for i, (name, layer) in enumerate(network.layers.items()):
        index[name] = i
        d = net.layers[i]
        fill_layer(d, layer, name, B)
        e = ext.get(name)
        if e is not None:
            d.ext = _ptr(_as_u8(e))
            d.ext_dtype = _abi.SNN_EXT_F32 if e.dtype == torch.float32 else _abi.SNN_EXT_U8
            keep.append(e)
        for key, table, field, flag in (
            ("clamp", clamps, "clamp", "clamp_per_step"),
            ("unclamp", unclamps, "unclamp", "unclamp_per_step"),
            ("inject_v", injects, "inject_v", "inject_per_step"),
        ):
            m = table.get(name)
            if m is not None:
                setattr(d, field, _ptr(_as_u8(m)))
                setattr(d, flag, int(m.dim() == 2))
                keep.append(m)
        r = rec.get(name)
        if r is not None:
            if r[0] is not None:
                d.rec_s = _ptr(_as_u8(r[0])); keep.append(r[0])
            if r[1] is not None:
                d.rec_v = _ptr(r[1]); keep.append(r[1])
            if len(r) > 2 and r[2] is not None:
                d.rec_count = _ptr(r[2]); keep.append(r[2])
        if d.kind == _abi.SNN_NODE_PASSTHROUGH and name in injects:
            raise NotImplementedError(f"injects_v into {name!r}: a PassThroughNodes layer has no voltage of its own")
    masks = getattr(network, "_conn_masks", None) or {}
    by_id = {id(layer): i for i, layer in enumerate(network.layers.values())}
    for i, ((src, tgt), conn) in enumerate(network.connections.items()):
        if network.learning and isinstance(conn, _MaxPoolConnection):
            raise AttributeError(conn._no_w_message())   # the reference fails in the first step's update
        # the source is the connection's own source layer (network.py:226-248 reads connection.source.s): ann_to_snn's
        # keys name the previous ANN child, which need not be a layer
        s_idx = by_id.get(id(conn.source), index.get(src))
        if s_idx is None:
            raise KeyError(f"the source of connection {(src, tgt)} is not a layer of the network")
        fill_conn(net.conns[i], conn, s_idx, index[tgt], float(network.dt), B, network._rule_kwargs_of((src, tgt)))
        m = masks.get((src, tgt))
        if m is not None:
            net.conns[i].mask = _ptr(m)
            keep.append(m)
        check_passthrough(net, i, type(conn).__name__)
    conns = [net.conns[i] for i in range(net.n_conns)]
    layers = [net.layers[i] for i in range(net.n_layers)]
    if (any(d.kind in POOL_INST_KINDS for d in conns) or any(d.kind in CONVERSION_KINDS for d in layers)) and any(
            d.kind == _abi.SNN_CONN_SPARSE or d.f_prob or d.f_mask or d.f_int for d in conns):
        raise NotImplementedError("a network with a MaxPool2dConnection, MaxPoo3dConnection, LocalConnection2D, Conv3dConnection, "
                                  "Conv1dConnection, LocalConnection3D, SubtractiveResetIFNodes or PassThroughNodes and a SparseConnection or MulticompartmentConnection "
                                  "features is not implemented by the CUDA core (each has its own instantiation of the window kernel)")
    check_neuron_params(layers, conns)
    return net, keep


def check_neuron_params(layers, conns) -> None:
    """Per-neuron parameters (include/snn_b200.h SNN_NODE_PN) run on their own instantiations of the window kernel,
    alone or with per-synapse bounds and rates: refuse, before anything runs, a plan that also needs the sparse, feature
    or pooling one."""
    if not any(d.kind & _abi.SNN_NODE_PN for d in layers):
        return
    if any(d.kind == _abi.SNN_CONN_SPARSE or d.kind in POOL_INST_KINDS or (d.kind == _abi.SNN_CONN_MCC and (d.f_prob or d.f_mask or d.f_int))
           for d in conns) or any(d.kind in CONVERSION_KINDS for d in layers):
        raise NotImplementedError("per-neuron parameter tensors in a network with a SparseConnection, MulticompartmentConnection "
                                  "features, a MaxPool2dConnection, MaxPoo3dConnection, LocalConnection2D, Conv3dConnection, "
                                  "Conv1dConnection, LocalConnection3D, SubtractiveResetIFNodes or PassThroughNodes are not implemented by the CUDA core (each has its own instantiation of "
                                  "the window kernel)")


CONVERSION_KINDS = (_abi.SNN_NODE_SUBIF, _abi.SNN_NODE_PASSTHROUGH)
# the connection kinds that only the pooling instantiation of the window kernel runs (snn_common.cuh snn_pool_inst_kind)
POOL_INST_KINDS = (_abi.SNN_CONN_MAXPOOL2D, _abi.SNN_CONN_MAXPOOL3D, _abi.SNN_CONN_LOCAL2D, _abi.SNN_CONN_CONV3D, _abi.SNN_CONN_CONV1D,
                   _abi.SNN_CONN_LOCAL3D)


def check_passthrough(net: "_abi.SnnNet", i: int, what: str) -> None:
    """A PassThroughNodes layer carries 0 / 1 spikes (include/snn_b200.h): refuse, before anything runs, a connection
    into one that is not a MaxPool2dConnection (its input could take other values) and a learning rule other than NoOp
    at either end."""
    d = net.conns[i]
    into, at = net.layers[d.tgt].kind == _abi.SNN_NODE_PASSTHROUGH, _abi.SNN_NODE_PASSTHROUGH in (net.layers[d.src].kind, net.layers[d.tgt].kind)
    if into and d.kind != _abi.SNN_CONN_MAXPOOL2D:
        raise NotImplementedError(f"a {what} into a PassThroughNodes layer is not implemented by the CUDA core (only "
                                  "MaxPool2dConnection, whose output is 0 / 1 spikes)")
    if at and d.rule not in (_abi.SNN_RULE_NONE, _abi.SNN_RULE_NOOP):
        raise NotImplementedError(f"a learning rule other than NoOp on a {what} to or from a PassThroughNodes layer is not "
                                  "implemented by the CUDA core")


# ---- single-operator helpers ---------------------------------------------------------------

def _conn_desc(conn, B: int, dt: float = 1.0, rule: bool = True) -> "_abi.SnnConn":
    d = _abi.SnnConn()
    fill_conn(d, conn, 0, 1, dt, B, rule=rule)
    return d


def compute_single_connection(conn, s: torch.Tensor, draw: Optional[Tuple[int, int, int]] = None) -> torch.Tensor:
    """``conn.compute(s)``: ``[B, *target.shape]`` currents for spikes ``s``.  ``draw`` = (seed, step, connection index)
    of a Probability feature's draw; by default a fresh seed from torch's CPU generator, step 0, index 0.  A 'time step'
    Weight is normalised after the product, as its compute does (so also on the scripted tier's gather)."""
    B = s.shape[0]
    if isinstance(conn, _MaxPoolConnection):
        return _compute_pool(conn, s)
    if isinstance(conn, MeanFieldConnection):
        return _compute_meanfield(conn, s)
    _backend.require_cuda(conn.w, "connection weights")
    su8 = _as_u8(s if s.dtype in (torch.bool, torch.uint8) else (s != 0)).reshape(B, -1).contiguous()
    su8 = su8.to(conn.w.device)
    out = torch.empty(B, conn.target.n, dtype=torch.float32, device=conn.w.device)
    d = _conn_desc(conn, B, rule=False)
    if d.f_prob:
        if draw is None:
            draw = (int(torch.randint(0, 2**31 - 1, (1,)).item()), 0, 0)
        d.draw_seed, d.draw_step, d.draw_conn = draw[0] & 0xFFFFFFFF, draw[1] & 0xFFFFFFFF, draw[2]
    _backend.conn_compute(d, conn.source.n, conn.target.n, B, su8, out)
    if d.kind & _abi.SNN_CONN_WNORM and d.norm_step:   # Weight.compute normalises after the product (topology_features.py:641-643)
        conn._weight().normalize(time_step_norm=True)
    return out.view(B, *conn.target.shape)


def _compute_meanfield(conn, s: torch.Tensor) -> torch.Tensor:
    """``MeanFieldConnection.compute(s)``: ``s.float().mean() * w``, shaped like ``w`` as the reference returns it.  The
    operator reads all of ``s`` as one sample and writes every element of ``w`` once (offsets 0 .. w.numel() - 1)."""
    w = conn.w
    _backend.require_cuda(w, "connection weights")
    if w.dtype != torch.float32 or not w.is_contiguous():
        raise TypeError("connection weights must be contiguous float32")
    su8 = _as_u8(s if s.dtype in (torch.bool, torch.uint8) else (s != 0)).reshape(1, -1).contiguous().to(w.device)
    n = su8.shape[1]
    if n >= 1 << 24:
        raise NotImplementedError(f"MeanFieldConnection.compute on {n} spikes: the float32 mean is exact below 2**24 only")
    if n == 0 or w.numel() == 0:   # (the reference's mean of nothing is NaN)
        return torch.full_like(w, float("nan")) if n == 0 else torch.empty_like(w)
    d = _abi.SnnConn()
    conn._fill_desc(d, 1.0)
    off = torch.arange(w.numel(), dtype=torch.int32, device=w.device)
    d.w, d.mf_off, d.mf_stride = _ptr(w), _ptr(off), 0
    out = torch.empty(1, w.numel(), dtype=torch.float32, device=w.device)
    _backend.conn_compute(d, n, w.numel(), 1, su8, out)
    return out.view(w.shape)


def _compute_pool(conn, s: torch.Tensor) -> torch.Tensor:
    """``MaxPool2dConnection.compute(s)`` / ``MaxPoo3dConnection.compute(s)``: the rates advance in place, ``[B, C,
    Hout, Wout]`` / ``[B, C, Dout, Hout, Wout]`` pooled spikes."""
    fr = conn.firing_rates
    _backend.require_cuda(fr, "firing_rates")
    conn._check(tuple(s.shape))
    B = s.shape[0]
    su8 = _as_u8(s if s.dtype in (torch.bool, torch.uint8) else (s != 0)).reshape(B, -1).contiguous().to(fr.device)
    d = _abi.SnnConn()
    conn._fill_desc(d, 1.0)
    shape = conn._out_shape()
    out = torch.empty(B, math.prod(shape), dtype=torch.float32, device=fr.device)
    _backend.conn_compute(d, conn.source.n, out.shape[1], B, su8, out)
    return out.view(B, *shape)


def _pair_net(conn, B: int) -> "_abi.SnnNet":
    net = _abi.SnnNet()
    net.abi_version = _abi.SNN_ABI_VERSION
    net.n_layers, net.n_conns, net.learning = 2, 1, 1
    dt = getattr(conn, "dt", None) or 1.0
    for k, layer in enumerate((conn.source, conn.target)):
        if layer.dt is None:
            layer.compute_decays(dt)
        if layer.kind is None:
            _fill_endpoint(net.layers[k], layer, f"layer{k}", B)
        else:
            fill_layer(net.layers[k], layer, f"layer{k}", B)
    fill_conn(net.conns[0], conn, 0, 1, float(dt), B)
    return net


def _fill_endpoint(d: "_abi.SnnLayer", layer, name: str, B: int) -> None:
    """A USER-DEFINED population (no ``kind``: its ``forward`` is torch code, scripted tier) as the source or target of a
    built-in connection's single-operator update: the rule reads the population's current spikes and traces and nothing
    else (snn_b200_conn_update), so that is all the descriptor carries."""
    if layer.s.dtype not in (torch.bool, torch.uint8) or layer.s.numel() != B * layer.n:
        raise TypeError(f"{name}.s must be a bool / uint8 tensor of {B} x {layer.n} spikes, got {layer.s.dtype} {tuple(layer.s.shape)}")
    if not layer.s.is_contiguous():
        layer.s = layer.s.contiguous()
    d.kind, d.n = _abi.SNN_NODE_INPUT, layer.n
    d.traces = int(bool(layer.traces))
    d.traces_additive = int(bool(layer.traces_additive))
    d.learning = int(bool(getattr(layer, "learning", True)))
    d.dt = float(layer.dt) if layer.dt is not None else 1.0
    d.s = _ptr(_as_u8(layer.s))
    if layer.traces:
        d.x = _ptr(_state(layer.x, "x", name))


def update_single_connection(conn) -> None:
    """``conn.update(learning=True)`` from the layers' current ``s`` / ``x``."""
    B = conn.source.s.shape[0]
    if hasattr(conn, "_check_learning"):   # (Conv3dConnection: the rules the reference cannot run)
        conn._check_learning()
    _backend.require_cuda(conn.w, "connection weights")
    net = _pair_net(conn, B)
    _backend.conn_update(net, 0, B, conn.w.device)


def normalize_single_connection(conn) -> None:
    _backend.require_cuda(conn.w, "connection weights")
    d = _conn_desc(conn, 1, rule=False)
    _backend.conn_normalize(d, conn.source.n, conn.target.n, conn.w.device)


def normalize_feature(feature, time_step: bool = False) -> None:
    """A Weight's normalize: the window-end formula, or the per-step one when ``time_step`` (snn_b200.h SNN_CONN_WNORM)."""
    _backend.require_cuda(feature.value, "feature value")
    d = _abi.SnnConn()
    d.w = feature.value.data_ptr()
    d.has_norm, d.norm_abs = 1, 0
    norm_t = feature._norm_tensor()
    d.norm = float(feature.norm) if norm_t is None else 0.0
    if norm_t is not None or time_step:
        d.kind = _abi.SNN_CONN_MCC | _abi.SNN_CONN_WNORM
        d.norm_t = _ptr(norm_t) if norm_t is not None else None
        d.norm_step = int(time_step)
    _backend.conn_normalize(d, feature.value.shape[0], feature.value.shape[1], feature.value.device)


def step_single_layer(layer, x: torch.Tensor) -> None:
    """``layer.forward(x)``: one step of one population, submitted as a one-layer window."""
    from .network import Network

    if layer.dt is None:
        raise RuntimeError("add the layer to a Network (or call compute_decays/set_batch_size) before forward()")
    host = Network(dt=float(layer.dt), batch_size=layer.batch_size or x.shape[0], learning=layer.learning)
    host.layers["L"] = layer  # bypass add_layer: keep the layer's state and batch size
    host._run_window({"L": x.unsqueeze(0)}, 1, normalize=False)
